"""GPU: the class run's derivation of a missing fresh-node variant (csrc/pack_kernel.cuh, run_derive) against the oracle.
Every scenario of tests/run_variant_problems.py is compared on the whole result at block sizes 32, 128 and 512 with the
derivation on and with KSCHED_NO_RUNDERIVE (the run stops and the generic step opens the node), then at 128 threads under
each mode switch, with and without the derivation. The corpora of the other run paths (runs, shared variants, round and
fill stretches) are compared the same way at 128 threads."""
import pytest

import fill_stretch_problems as fsp
import round_stretch_problems as rsp
import run_problems as rp
import run_variant_problems as vp
import shape_problems as sp
from oracle_compare import MODE_SWITCHES, set_modes

pytestmark = pytest.mark.gpu

DERIVE = ("", "KSCHED_NO_RUNDERIVE")


def _match(pkg, oracle, monkeypatch, problem, runs):
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    for specs in runs:
        monkeypatch.delenv("KSCHED_NO_RUNDERIVE", raising=False)  # (not one of MODE_SWITCHES: set_modes leaves it)
        set_modes(monkeypatch, *specs)
        rs.run()
        res = rs.download()
        assert (res.assign == want.assign).all(), specs
        assert res.digest() == want.digest(), specs


def _per_switch(threads):
    return [(derive, switch, threads) for switch in MODE_SWITCHES for derive in DERIVE]


@pytest.mark.parametrize("name,seed", vp.CORPUS, ids=[f"{n}-{s}" for n, s in vp.CORPUS])
def test_run_variants_match_oracle(pkg, oracle, monkeypatch, name, seed):
    runs = [(derive, f"KSCHED_PACK_THREADS={t}") for derive in DERIVE for t in (32, 128, 512)]
    _match(pkg, oracle, monkeypatch, pkg.Problem.from_dict(vp.build(name, seed)[0]), runs + _per_switch("KSCHED_PACK_THREADS=128"))


OTHER = [(m, n, s) for m in (rp, sp, rsp, fsp) for n, s in m.CORPUS]


@pytest.mark.parametrize("mod,name,seed", OTHER, ids=[f"{m.__name__}-{n}-{s}" for m, n, s in OTHER])
def test_run_corpora_without_derivation_match_oracle(pkg, oracle, monkeypatch, mod, name, seed):
    runs = [(derive, "KSCHED_PACK_THREADS=128") for derive in DERIVE] + _per_switch("KSCHED_PACK_THREADS=128")
    _match(pkg, oracle, monkeypatch, pkg.Problem.from_dict(mod.build(name, seed)[0]), runs)
