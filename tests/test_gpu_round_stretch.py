"""GPU: the mask run's round stretches (csrc/pack_kernel.cuh, DESIGN.md section 4) against the oracle, whole result. The
corpus (tests/round_stretch_problems.py) ends stretches by each of their rules and builds near misses that must fall back
to single rounds; every problem is solved at 32, 128 and 512 pack threads with and without KSCHED_NO_ROUNDSTRETCH, and
under each of the other KSCHED_NO_* switches."""
import pytest

import round_stretch_problems as rs
from oracle_compare import compare

pytestmark = pytest.mark.gpu

SWITCHES = ("KSCHED_NO_ROUNDSTRETCH", "KSCHED_NO_CLASSRUN", "KSCHED_NO_LEVELSTEP", "KSCHED_NO_LEVELRUN", "KSCHED_NO_MASKRUN",
            "KSCHED_NO_LEVELWARP", "KSCHED_NO_VARSTORE", "KSCHED_PACK_THREADS")


def _clear(monkeypatch):
    for v in SWITCHES:
        monkeypatch.delenv(v, raising=False)


@pytest.mark.parametrize("name,seed", rs.CORPUS, ids=[f"{n}-{s}" for n, s in rs.CORPUS])
def test_round_stretch_matches_oracle(pkg, oracle, monkeypatch, name, seed):
    _clear(monkeypatch)
    compare(pkg, oracle, pkg.Problem.from_dict(rs.build(name, seed)[0]))


@pytest.mark.parametrize("name,seed", rs.CORPUS, ids=[f"{n}-{s}" for n, s in rs.CORPUS])
def test_round_stretch_every_block_size_and_switch(pkg, oracle, monkeypatch, name, seed):
    problem = pkg.Problem.from_dict(rs.build(name, seed)[0])
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    run = pkg.ResidentSolve(problem)
    run.set_count_visited(False)
    run.load()
    envs = [[("KSCHED_PACK_THREADS", str(t))] + stretch for t in (32, 128, 512) for stretch in ([], [("KSCHED_NO_ROUNDSTRETCH", "1")])]
    envs += [[(v, "1")] for v in SWITCHES[1:-1]]
    for env in envs:
        _clear(monkeypatch)
        for k, v in env:
            monkeypatch.setenv(k, v)
        run.run()
        res = run.download()
        assert (res.assign == want.assign).all(), env
        assert res.digest() == want.digest(), env
    _clear(monkeypatch)


@pytest.mark.parametrize("config,pods,types,seed", [(4, 6000, 1000, 7), (4, 2500, 1000, 3), (3, 5000, 1000, 7), (2, 3000, 500, 7)])
def test_round_stretch_modes_agree(pkg, monkeypatch, config, pods, types, seed):
    """synthetic BASELINE-shaped batches: the same whole result with the stretches on and off, alone and next to the
    other switches of the class-run loop"""
    problem = pkg.Problem.synth(config, pods, types, seed, 0)
    run = pkg.ResidentSolve(problem)
    run.set_count_visited(False)
    run.load()
    digests = {}
    for off in ("", "KSCHED_NO_ROUNDSTRETCH", "KSCHED_NO_ROUNDSTRETCH,KSCHED_NO_VARSTORE", "KSCHED_NO_MASKRUN"):
        _clear(monkeypatch)
        for v in off.split(","):
            if v:
                monkeypatch.setenv(v, "1")
        run.run()
        res = run.download()
        digests[off or "all on"] = (int(res.digest()), int(res.num_new_nodes), int((res.assign >= 0).sum()))
    _clear(monkeypatch)
    assert len(set(digests.values())) == 1, digests
