"""GPU: the mask run's fill stretches (csrc/pack_kernel.cuh, DESIGN.md section 4) against the oracle, whole result. The
corpus (tests/fill_stretch_problems.py) ends stretches by each of their limits and builds near misses that must not take
them; every problem is solved at 32, 128 and 512 pack threads with and without KSCHED_NO_FILLSTRETCH, and under each of
the other KSCHED_NO_* switches."""
import pytest

import fill_stretch_problems as fs
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu


def _modes(monkeypatch, spec=""):
    """set_modes, with KSCHED_NO_FILLSTRETCH cleared too"""
    monkeypatch.delenv("KSCHED_NO_FILLSTRETCH", raising=False)
    set_modes(monkeypatch, spec)


@pytest.mark.parametrize("name,seed", fs.CORPUS, ids=[f"{n}-{s}" for n, s in fs.CORPUS])
def test_fill_stretch_matches_oracle(pkg, oracle, monkeypatch, name, seed):
    _modes(monkeypatch)
    compare(pkg, oracle, pkg.Problem.from_dict(fs.build(name, seed)[0]))


@pytest.mark.parametrize("name,seed", fs.CORPUS, ids=[f"{n}-{s}" for n, s in fs.CORPUS])
def test_fill_stretch_every_block_size_and_switch(pkg, oracle, monkeypatch, name, seed):
    problem = pkg.Problem.from_dict(fs.build(name, seed)[0])
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    run = pkg.ResidentSolve(problem)
    run.set_count_visited(False)
    run.load()
    envs = [f"KSCHED_PACK_THREADS={t}{fill}" for t in (32, 128, 512) for fill in ("", ",KSCHED_NO_FILLSTRETCH")]
    envs += list(MODE_SWITCHES)
    for env in envs:
        _modes(monkeypatch, env)
        run.run()
        res = run.download()
        assert (res.assign == want.assign).all(), env
        assert res.digest() == want.digest(), env
    _modes(monkeypatch)


@pytest.mark.parametrize("config,pods,types,seed", [(4, 6000, 1000, 7), (4, 2500, 1000, 3), (3, 5000, 1000, 7), (2, 3000, 500, 7)])
def test_fill_stretch_modes_agree(pkg, monkeypatch, config, pods, types, seed):
    """synthetic BASELINE-shaped batches: the same whole result with the fill stretches on and off"""
    problem = pkg.Problem.synth(config, pods, types, seed, 0)
    run = pkg.ResidentSolve(problem)
    run.set_count_visited(False)
    run.load()
    digests = {}
    for off in ("", "KSCHED_NO_FILLSTRETCH", "KSCHED_NO_ROUNDSTRETCH"):
        _modes(monkeypatch, off)
        run.run()
        res = run.download()
        digests[off or "all on"] = (int(res.digest()), int(res.num_new_nodes), int((res.assign >= 0).sum()))
    _modes(monkeypatch)
    assert len(set(digests.values())) == 1, digests
