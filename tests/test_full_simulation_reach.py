"""CPU: every scenario of tests/full_simulation_problems.py reaches what it is there for. The oracle's Solve with each set of
the scenario removed (simulateScheduling's problem) shows the scenario's property, and the oracle's fast mode gives the
literal path's result on it."""
import pytest

import full_simulation_problems as fp

CORPUS = fp.corpus()
IDS = [c[0] for c in CORPUS]


def _initialized(node):
    return node["labels"].get("karpenter.sh/initialized") == "true"


def _check(pkg, prob, problem, res, removed, prop):
    d = res.to_dict()
    if prop == "new3":
        assert len(d["newNodes"]) >= 3
    elif prop == "relaxed":
        assert any(r > 0 for r in d["relax"])
    elif prop == "pending":
        assert prob["pods"] and all(a >= 0 for a in d["assign"][:len(prob["pods"])])
    elif prop == "deleting":
        gone = sum(len(n["pods"]) for n in prob["nodes"] if n.get("markedForDeletion"))
        assert gone and len(d["assign"]) == len(prob["pods"]) + sum(len(prob["nodes"][i]["pods"]) for i in removed) + gone
    elif prop == "uninitialized":
        stays = [e["node"] for e in d["existing"] if e["pods"]]
        assert any(not _initialized(prob["nodes"][i]) for i in stays)
    elif prop == "unschedulable":
        assert -1 in d["assign"]
    elif prop == "topology":
        pods = [p for i in removed for p in prob["nodes"][i]["pods"]]
        assert any(p.get("topologySpreadConstraints") for p in pods) and any(p.get("podAntiAffinity") for p in pods)
        assert all(a >= 0 for a in d["assign"])
    else:
        dims = pkg.ResidentSolve(problem, removed).dims
        if prop == "ext":
            assert dims["resources_ext"] > 0
        elif prop == "folded":
            keys = set()
            for p in prob["provisioners"]:
                keys |= {r["key"] for r in p.get("requirements", [])} | set(p.get("labels", {}))
            for p in prob["pods"] + [p for i in removed for p in prob["nodes"][i]["pods"]]:
                keys |= set(p.get("nodeSelector", {}))
            assert len(keys) > 16 and dims["keys"] <= 16
        elif prop == "hostname":
            assert dims["hostname_reqs"] > 0
        elif prop == "hostport":
            assert dims["hostports"] > 0
        elif prop == "volume":
            assert dims["volume_claims"] > 0
        elif prop == "limits":
            assert sum(1 for p in prob["provisioners"] if p.get("limits")) > 1
        else:
            raise AssertionError(prop)


@pytest.mark.parametrize("name,prob,sets,prop", CORPUS, ids=IDS)
def test_scenario_reaches_its_property(pkg, oracle, name, prob, sets, prop):
    problem = pkg.Problem.from_dict(prob)
    order, _ = oracle.rank_candidates(problem)
    resolved = fp.resolve_sets(prob, sets, order)
    assert resolved and all(resolved)
    for s in resolved:
        assert set(s) <= set(order), (name, s)  # every set names candidates of the consolidation pass
        _, res = oracle.solve_dict(pkg, prob, s)
        _check(pkg, prob, problem, res, s, prop)
        _, fast = oracle.solve_dict(pkg, prob, s, fast=True)
        assert fast.digest() == res.digest() and fast.to_dict() == res.to_dict(), (name, s)
