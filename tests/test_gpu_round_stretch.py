"""GPU: the mask run's round stretches (csrc/pack_kernel.cuh, DESIGN.md section 4) against the oracle, whole result. The
corpus (tests/round_stretch_problems.py) ends stretches by each of their rules and builds near misses that must fall back
to single rounds; every problem is solved at 32, 128 and 512 pack threads with and without KSCHED_NO_ROUNDSTRETCH, and
under each of the other KSCHED_NO_* switches."""
import pytest

import round_stretch_problems as rs
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,seed", rs.CORPUS, ids=[f"{n}-{s}" for n, s in rs.CORPUS])
def test_round_stretch_matches_oracle(pkg, oracle, monkeypatch, name, seed):
    set_modes(monkeypatch)
    compare(pkg, oracle, pkg.Problem.from_dict(rs.build(name, seed)[0]))


@pytest.mark.parametrize("name,seed", rs.CORPUS, ids=[f"{n}-{s}" for n, s in rs.CORPUS])
def test_round_stretch_every_block_size_and_switch(pkg, oracle, monkeypatch, name, seed):
    problem = pkg.Problem.from_dict(rs.build(name, seed)[0])
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    run = pkg.ResidentSolve(problem)
    run.set_count_visited(False)
    run.load()
    envs = [f"KSCHED_PACK_THREADS={t}{stretch}" for t in (32, 128, 512) for stretch in ("", ",KSCHED_NO_ROUNDSTRETCH")]
    envs += [v for v in MODE_SWITCHES if v != "KSCHED_NO_ROUNDSTRETCH"]
    for env in envs:
        set_modes(monkeypatch, env)
        run.run()
        res = run.download()
        assert (res.assign == want.assign).all(), env
        assert res.digest() == want.digest(), env
    set_modes(monkeypatch)


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
        set_modes(monkeypatch, off)
        run.run()
        res = run.download()
        digests[off or "all on"] = (int(res.digest()), int(res.num_new_nodes), int((res.assign >= 0).sum()))
    set_modes(monkeypatch)
    assert len(set(digests.values())) == 1, digests
