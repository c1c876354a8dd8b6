"""CPU: clusters whose owned existing nodes carry more than 64 distinct taint sets (tests/taint_problems.py) encode without
refusal, and the oracle's placements are sound: every pod it puts on an existing node tolerates that node's taints, and some
land on nodes whose taint set no template has (ids of 64 and above in the encoding)."""
import pytest

import placement_invariants
import taint_problems as tp

CORPUS = tp.corpus()
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_encoder_accepts_more_than_64_taint_sets(pkg, name, prob):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["taintsets"] == len(tp.distinct_sets(prob)) > 64
    assert rs.dims["templates"] == len(prob["provisioners"])


def test_cluster_and_after_are_accepted(pkg):
    for prob in (tp.cluster(0), tp.after(0)):
        assert len(tp.distinct_sets(prob)) > 64
        cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands[:3])
        assert rs.dims["taintsets"] > 64


def test_problems_with_at_most_64_sets_keep_their_dims(pkg):
    """without node-only sets the template sets are the whole id space"""
    prob = tp.many(24, 0)
    prob["nodes"] = [n for n in prob["nodes"] if tp.taint_set(tp.node_taints(n)) in tp.template_sets(prob)]
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["taintsets"] == 24


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_oracle_places_only_on_tolerated_nodes(pkg, oracle, name, prob):
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    d = res.to_dict()
    tmpl = tp.template_sets(prob)
    on_existing = beyond = 0
    for e in d["existing"]:
        node = prob["nodes"][e["node"]]
        taints = tp.node_taints(node)
        for p in e["pods"]:
            assert tp.tolerates(taints, prob["pods"][p].get("tolerations", []) + _relaxed(d, p, prob)), (node["name"], p)
            on_existing += 1
            beyond += tp.taint_set(taints) not in tmpl
    assert on_existing > 0 and beyond > 0, (on_existing, beyond)


def _relaxed(d, p, prob):
    """Relax adds a PreferNoSchedule toleration once the soft constraints are gone (preferences.go:36-56): give it to pods
    that were relaxed at all when some pool has a PreferNoSchedule taint; the check stays strict for every other taint"""
    any_pns = any(t["effect"] == "PreferNoSchedule" for pr in prob["provisioners"] for t in pr.get("taints", []))
    return [{"operator": "Exists", "effect": "PreferNoSchedule"}] if any_pns and d["relax"][p] > 0 else []


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_oracle_results_pass_placement_invariants(pkg, oracle, name, prob):
    # the invariants know the zones of new nodes only: zone spread over existing nodes is left to the GPU comparison
    prob = dict(prob, pods=[{k: v for k, v in p.items() if k != "topologySpreadConstraints"} for p in prob["pods"]])
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    stats = placement_invariants.check(problem, res)
    assert stats["scheduled"] > 0 and stats["anti"] > 0
