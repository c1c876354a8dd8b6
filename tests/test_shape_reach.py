"""CPU: every scenario of tests/shape_problems.py reaches the variant store of the pack kernel's class run. From the
oracle's result alone: a later class of a group that shares its row opens a fresh node in a domain (its zone, for zone
spreads) in which an earlier class of the group already opened one, so the later class's fresh node can be replayed from
the earlier class's variant instead of being created by the generic step."""
import pytest

import shape_problems as sp
from fixtures import ZONE
from test_run_reach import Placed


def _zone_spread(pod):
    return any(s["topologyKey"] == ZONE for s in pod.get("topologySpreadConstraints", []))


def opened(prob, facts, pl, cls):
    """domains in which class cls opened a new node (its first pod belongs to cls)"""
    members = set(facts["classes"][cls])
    zoned = _zone_spread(prob["pods"][facts["classes"][cls][0]])
    return {pl.value(pl.ne + t, ZONE) if zoned else None for t, nn in enumerate(pl.res["newNodes"]) if nn["pods"][0] in members}


@pytest.mark.parametrize("name,seed", sp.CORPUS, ids=[f"{n}-{s}" for n, s in sp.CORPUS])
def test_shape_scenario_shares_fresh_nodes(pkg, oracle, name, seed):
    prob, facts = sp.build(name, seed)
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    pl = Placed(prob, res.to_dict())
    for group in facts["share"]:
        seen, shared = set(), []
        for cls in group:
            doms = opened(prob, facts, pl, cls)
            shared += [(cls, d) for d in doms & seen]
            seen |= doms
        assert shared, f"no class of {group} opens a fresh node in a domain an earlier one of them opened one in"
