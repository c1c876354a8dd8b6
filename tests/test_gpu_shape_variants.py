"""GPU: the class run's store of fresh-node variants (csrc/pack_kernel.cuh, VarStoreEntry) against the oracle. Deployments
of one shape replay each other's fresh nodes (tests/shape_problems.py); the near misses must not. Every scenario is
compared on the whole result at every block size, with the store on and with KSCHED_NO_VARSTORE."""
import pytest

import shape_problems as sp

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,seed", sp.CORPUS, ids=[f"{n}-{s}" for n, s in sp.CORPUS])
def test_shape_variants_match_oracle(pkg, oracle, monkeypatch, name, seed):
    problem = pkg.Problem.from_dict(sp.build(name, seed)[0])
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    for store in ("on", "off"):
        for threads in (32, 64, 128, 256, 512):
            monkeypatch.setenv("KSCHED_PACK_THREADS", str(threads))
            if store == "off":
                monkeypatch.setenv("KSCHED_NO_VARSTORE", "1")
            else:
                monkeypatch.delenv("KSCHED_NO_VARSTORE", raising=False)
            rs.run()
            res = rs.download()
            assert (res.assign == want.assign).all(), (store, threads)
            assert res.digest() == want.digest(), (store, threads)
