"""GPU: the pack kernel's generic step on the scenarios of tests/generic_step_problems.py (test_generic_step_reach.py shows
on the oracle that each one reaches its exclusion count, front shape, memo keys, cursor refusal or table edge). Every problem
is inside the supported envelope, so a KSCHED_ERR_UNSUPPORTED refusal fails the test. Compared with the oracle: the whole
result (both nodes_visited settings), one resident problem under every mode switch plus KSCHED_NO_CLASSRUN and
KSCHED_NO_FILLSTRETCH, every block size the pack kernel can be launched with, and the placement invariants.

Before each compared run a different problem with the same catalog and templates runs on the device, so that no state an
earlier run left behind can stand in for the one under test."""
import pytest

import generic_step_problems as gp
import placement_invariants
from oracle_compare import INSTANCE_TYPE, MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu

IDS = [n for n, _ in gp.CORPUS]
MODES = ("",) + MODE_SWITCHES + ("KSCHED_NO_FILLSTRETCH",)
BLOCK_SIZES = (32, 64, 128, 256, 512)


def _scrub(pkg, prob):
    """a different problem with the same catalog and templates: one tiny pod per scenario pod"""
    pods = [{"name": f"scrub-{i}", "uid": f"scrub-{i}", "requests": {"cpu": "10m"}, "labels": {"scrub": str(i % 7)}}
            for i in range(len(prob["pods"]))]
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(dict(prob, pods=pods, nodes=[])))
    rs.set_count_visited(False)
    rs.load()
    rs.run()


def _oracle(pkg, oracle, problem):
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    return want


def _check(res, want, label):
    """field by field as compare() does: the device reports a new node's requirements without the instance-type key (its
    options carry it), so a whole-result digest differs wherever a pod names instance types"""
    g, w = res.to_dict(), want.to_dict()
    for k in ("assign", "relax", "existing"):
        assert g[k] == w[k], f"{label}: {k}"
    assert len(g["newNodes"]) == len(w["newNodes"]), label
    for i, (a, b) in enumerate(zip(g["newNodes"], w["newNodes"])):
        b = dict(b, requirements={k: v for k, v in b["requirements"].items() if k != INSTANCE_TYPE})
        for f in ("provisioner", "pods", "options", "requests", "requirements", "launch"):
            assert a.get(f) == b.get(f), f"{label}: new node {i}, {f}"


@pytest.mark.parametrize("name", IDS)
def test_generic_step_matches_oracle(pkg, oracle, monkeypatch, name):
    set_modes(monkeypatch)
    prob = gp.build(name)[0]
    _scrub(pkg, prob)
    problem = pkg.Problem.from_dict(prob)
    got, _ = compare(pkg, oracle, problem)
    if not prob.get("daemonSetPods") and not prob.get("nodes"):  # (the invariants model neither)
        placement_invariants.check(problem, got)


@pytest.mark.parametrize("name", IDS)
def test_every_mode_switch_matches_oracle(pkg, oracle, monkeypatch, name):
    """the switches are read on every solve, so one resident problem runs under each of them in turn"""
    prob = gp.build(name)[0]
    problem = pkg.Problem.from_dict(prob)
    want = _oracle(pkg, oracle, problem)
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    for mode in MODES:
        set_modes(monkeypatch, mode)
        rs.run()
        _check(rs.download(), want, mode or "default")
    set_modes(monkeypatch)


@pytest.mark.parametrize("name", IDS)
def test_every_block_size_matches_oracle(pkg, oracle, monkeypatch, name):
    """the cooperative check's word loops, the front reduction and the fit ranks depend on blockDim"""
    prob = gp.build(name)[0]
    problem = pkg.Problem.from_dict(prob)
    want = _oracle(pkg, oracle, problem)
    for count_visited in (False, True):
        for threads in BLOCK_SIZES:
            _scrub(pkg, prob)
            set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
            rs = pkg.ResidentSolve(problem)
            rs.set_count_visited(count_visited)  # taken when the problem is loaded
            rs.load()
            rs.run()
            res = rs.download()
            _check(res, want, f"{threads} threads, count_visited={count_visited}")
            if count_visited:
                assert res.nodes_visited == want.nodes_visited, threads
    set_modes(monkeypatch)
