"""CPU: every scenario of tests/variant_table_problems.py reaches the edge of the variant table it was built for, from the
problem and the literal oracle's result alone: every class opens fresh nodes (so its runs need variants), and each near
miss crosses the guard it names."""
import pytest

import variant_table_problems as vt
from fixtures import ZONE
from test_run_reach import Placed


def fresh_nodes(facts, pl, cls):
    """the new nodes whose first pod belongs to class cls"""
    members = set(facts["classes"][cls])
    return [t for t, nn in enumerate(pl.res["newNodes"]) if nn["pods"][0] in members]


@pytest.mark.parametrize("name,seed", vt.CORPUS, ids=[f"{n}-{s}" for n, s in vt.CORPUS])
def test_variant_table_scenario_reaches(pkg, oracle, name, seed):
    prob, facts = vt.build(name, seed)
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    pl = Placed(prob, res.to_dict())
    assert not prob.get("nodes"), "an existing node keeps the class runs off"
    for cls in facts["classes"]:
        assert fresh_nodes(facts, pl, cls), f"{cls} opens no fresh node"
    if name == "zone_subset":
        keep = set(prob["pods"][facts["classes"]["sub"][0]]["nodeAffinity"]["required"][0][0]["values"])
        zones = {pl.value(pl.ne + t, ZONE) for t in fresh_nodes(facts, pl, "sub")}
        assert zones == keep, zones  # the third zone's entry must not be taken
    if name == "closes_at_once":
        assert all(len(nn["pods"]) == 1 for nn in pl.res["newNodes"])
    if name == "taint_first":
        assert prob["provisioners"][0]["taints"] and prob["provisioners"][0]["weight"] > prob["provisioners"][1]["weight"]
        assert all(nn["provisioner"] in (1, "default") for nn in pl.res["newNodes"]), "a node of the tainted template"
    if name == "relaxed":
        assert any(res.relax_level), "the preferred term is never relaxed"
    if name == "daemonset":
        assert prob["daemonSetPods"]
    if name == "two_masks":
        assert len(prob["pods"][0]["topologySpreadConstraints"]) == 2
    if name == "volume":
        assert prob["pods"][0]["volumes"] and not any("volumeLimits" in n for n in prob.get("nodes", []))
    if name == "beyond_capacity":
        assert len(facts["classes"]) > vt.VT_CLASSES
        shapes = {tuple(sorted(prob["pods"][ix[0]]["requests"].items())) for ix in facts["classes"].values()}
        assert len(shapes) == len(facts["classes"]), "every deployment is a class of its own"
