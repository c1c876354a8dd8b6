"""CPU: every scenario of tests/run_variant_problems.py reaches the condition it was built for, from the problem and the
literal oracle's result alone: its classes open fresh nodes in as many zones as the scenario needs (so the class run
needs a variant it does not have), the new shapes really are new, and each near miss crosses the guard it names."""
import pytest

import run_variant_problems as vp
from fixtures import ZONE
from test_run_reach import Placed

K_RUN_VARIANTS = 4    # pack_kernel.cuh kRunVariants: fresh-node variants one class keeps
K_VAR_STORE = 256     # kVarStore: variants one Solve shares between classes
K_RUN_W32 = 64        # kRunW32: option words of a variant


def fresh_nodes(facts, pl, cls):
    """the new nodes whose first pod belongs to class cls, in creation order"""
    members = set(facts["classes"][cls])
    return [t for t, nn in enumerate(pl.res["newNodes"]) if nn["pods"][0] in members]


@pytest.mark.parametrize("name,seed", vp.CORPUS, ids=[f"{n}-{s}" for n, s in vp.CORPUS])
def test_run_variant_scenario_reaches(pkg, oracle, name, seed):
    prob, facts = vp.build(name, seed)
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    pl = Placed(prob, res.to_dict())
    pairs = 0
    for cls in facts["fresh"]:
        nodes = fresh_nodes(facts, pl, cls)
        assert nodes, f"{cls} opens no fresh node"
        zones = {pl.value(pl.ne + t, ZONE) for t in nodes}
        pairs += len(zones)
        want = facts["zones"][cls]
        if want is not None:
            assert len(zones) >= want, (cls, zones)
        if "min_nodes" in facts:
            assert len(nodes) >= facts["min_nodes"], (cls, len(nodes))
            assert max(len(pl.res["newNodes"][t]["pods"]) for t in nodes) == facts["pods_cap"], cls  # whole nodes: the bulk fill
    first = {tuple(sorted(prob["pods"][facts["classes"][c][0]]["requests"].items())) for c in facts["fresh"]}
    if facts["near"] is None:
        assert len(first) == len(facts["fresh"]), "two deployments share a shape: a store hit, not a derivation"
    if "first_zone" in facts:
        cls, zone = facts["first_zone"]
        assert pl.value(pl.ne + fresh_nodes(facts, pl, cls)[0], ZONE) == zone
    if "variants" in facts:
        assert pairs >= facts["variants"] > K_VAR_STORE
        assert all(facts["zones"][c] > K_RUN_VARIANTS for c in facts["fresh"])
    if name == "unshared":
        assert all(prob["pods"][facts["classes"][c][0]]["volumes"] for c in facts["fresh"])
    near = facts["near"]
    if near == "limits":
        assert any(p.get("limits") for p in prob["provisioners"])
    elif near == "wide":
        assert (len(prob["instanceTypes"]) + 31) // 32 > K_RUN_W32
    elif near == "closed":
        assert all(len(nn["pods"]) == 1 for nn in pl.res["newNodes"])
    elif near == "templates":
        assert len(prob["provisioners"]) > 1
