"""GPU: the pack kernel's run paths at their capacity limits (tests/run_problems.py; test_run_reach.py shows on the
oracle that each scenario gets there). Every problem is inside the supported envelope, so a KSCHED_ERR_UNSUPPORTED
refusal fails the test. Compared with the oracle: the whole result (both nodes_visited settings), the result under every
mode switch of the class-run loop, and the result at every block size the pack kernel can be launched with."""
import pytest

import run_problems as rp
from oracle_compare import compare

pytestmark = pytest.mark.gpu

IDS = [f"{n}-{s}" for n, s in rp.CORPUS]
SWITCHES = ("KSCHED_NO_CLASSRUN", "KSCHED_NO_LEVELRUN", "KSCHED_NO_LEVELWARP", "KSCHED_NO_MASKRUN", "KSCHED_NO_LEVELSTEP", "KSCHED_WARPLOOP")
MODES = ("",) + SWITCHES + ("KSCHED_NO_LEVELRUN,KSCHED_NO_MASKRUN",)
BLOCK_SIZES = (32, 64, 128, 256, 512)  # ksched.cu picks 128 / 256 / 512 by existing-node count; KSCHED_PACK_THREADS overrides it


def _oracle(pkg, oracle, problem):
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    return want


def _check(res, want, label):
    assert (res.assign == want.assign).all(), label
    assert (res.relax_level == want.relax_level).all(), label
    assert res.digest() == want.digest(), f"{label}: same placements, different nodes (options / requests / requirements)"


def _set_env(monkeypatch, names):
    for v in SWITCHES + ("KSCHED_PACK_THREADS",):
        monkeypatch.delenv(v, raising=False)
    for kv in names:
        k, _, v = kv.partition("=")
        monkeypatch.setenv(k, v or "1")


@pytest.mark.parametrize("name,seed", rp.CORPUS, ids=IDS)
def test_run_corpus_matches_oracle(pkg, oracle, monkeypatch, name, seed):
    _set_env(monkeypatch, [])
    compare(pkg, oracle, pkg.Problem.from_dict(rp.build(name, seed)[0]))


@pytest.mark.parametrize("name,seed", rp.CORPUS, ids=IDS)
def test_every_mode_switch_matches_oracle(pkg, oracle, monkeypatch, name, seed):
    """the switches are read on every solve, so one resident problem runs under each of them in turn"""
    problem = pkg.Problem.from_dict(rp.build(name, seed)[0])
    want = _oracle(pkg, oracle, problem)
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    for mode in MODES:
        _set_env(monkeypatch, [m for m in mode.split(",") if m])
        rs.run()
        _check(rs.download(), want, mode or "default")
    _set_env(monkeypatch, [])


FIRST_SEEDS = [(n, s) for n, s in rp.CORPUS if s == rp.SEEDS.get(n, (0,))[0]]


@pytest.mark.parametrize("name,seed", FIRST_SEEDS, ids=[f"{n}-{s}" for n, s in FIRST_SEEDS])
def test_every_block_size_matches_oracle(pkg, oracle, monkeypatch, name, seed):
    """every reduction, scan and staging size of the pack kernel depends on blockDim"""
    problem = pkg.Problem.from_dict(rp.build(name, seed)[0])
    want = _oracle(pkg, oracle, problem)
    for count_visited in (False, True):
        rs = pkg.ResidentSolve(problem)
        rs.set_count_visited(count_visited)  # taken when the problem is loaded
        rs.load()
        for threads in BLOCK_SIZES:
            _set_env(monkeypatch, [f"KSCHED_PACK_THREADS={threads}"])
            rs.run()
            res = rs.download()
            _check(res, want, f"{threads} threads, count_visited={count_visited}")
            if count_visited:
                assert res.nodes_visited == want.nodes_visited, threads
    _set_env(monkeypatch, [])
