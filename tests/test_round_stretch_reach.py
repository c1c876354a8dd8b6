"""CPU: every scenario of tests/round_stretch_problems.py really crosses the rule of the mask run's round stretches it was
built for. Each predicate is computed from the problem and the oracle's result alone."""
from collections import Counter

import pytest

import round_stretch_problems as rs
from fixtures import ZONE

K_M1_LV = 12  # pack_kernel.cuh kM1Lv: pod counts the mask run's lists represent


def _single(req):
    op, _, rest = (req or "").partition(" ")
    vals = rest.strip()[1:-1].split()
    return vals[0] if op == "In" and len(vals) == 1 else None


class Placed:
    def __init__(self, res):
        self.res = res
        self.assign = res["assign"]
        self.ne = len(res["existing"])

    def zone(self, node):
        nn = self.res["newNodes"][node - self.ne]
        return _single(nn["requirements"].get(ZONE)) or nn["launch"]["zone"]

    def nodes_of(self, pods):
        return [self.assign[i] for i in pods if self.assign[i] >= 0]

    def opened_by(self, pods):
        """the new nodes whose first pod is one of pods"""
        ps = set(pods)
        return {self.ne + k for k, nn in enumerate(self.res["newNodes"]) if nn["pods"][0] in ps}


def reach_pinned(facts, pl):
    spread, base = facts["classes"]["spread"], pl.opened_by(facts["classes"]["base"])
    on_base = Counter(n for n in pl.nodes_of(spread) if n in base)
    assert len({pl.zone(n) for n in on_base}) == facts["zones"], "the spread should use base nodes in every zone"
    assert sum(on_base.values()) >= 2 * len(base), "every base node should take at least two spread pods"
    assert max(on_base.values()) >= 2


def reach_unequal(facts, pl):
    zs = facts["zones"]
    assert all(pl.zone(n) == zs[0] for n in pl.nodes_of(facts["classes"]["lead"]))
    first = facts["classes"]["spread"][0]  # spread pods are identical: the first in creation order is placed first
    assert pl.zone(pl.assign[first]) != zs[0], "the counts should start unequal"


def reach_unpinned_between(facts, pl):
    spread = set(pl.nodes_of(facts["classes"]["spread"]))
    assert spread & pl.opened_by(facts["classes"]["p"]) and spread & pl.opened_by(facts["classes"]["u"])


def reach_room_slow(facts, pl):
    base = pl.opened_by(facts["classes"]["base"])
    assert len({pl.zone(n) for n in pl.nodes_of(facts["classes"]["spread"]) if n in base}) == 3


def reach_levels(facts, pl):
    assert max(Counter(pl.nodes_of(facts["classes"]["spread"])).values()) >= K_M1_LV


def reach_fresh_anti(facts, pl):
    nodes = pl.nodes_of(facts["classes"]["spread"])
    assert len(nodes) == len(set(nodes)) == len(facts["classes"]["spread"])
    per_zone = Counter(pl.zone(n) for n in nodes)
    assert len(per_zone) == facts["zones"] and max(per_zone.values()) - min(per_zone.values()) <= 1


def reach_fresh_room(facts, pl):
    most = max(Counter(pl.nodes_of(facts["classes"]["spread"])).values())
    assert most == (2 if facts["two"] else 1)


def reach_host_spread(facts, pl):
    nodes = pl.nodes_of(facts["classes"]["spread"])
    assert len({pl.zone(n) for n in nodes}) == 3 and len(set(nodes)) >= 6


REACH = {name: globals()["reach_" + name.rstrip("0123456789")] for name in rs.SCENARIOS}


@pytest.mark.parametrize("name,seed", rs.CORPUS, ids=[f"{n}-{s}" for n, s in rs.CORPUS])
def test_round_stretch_scenario_reaches_its_rule(pkg, oracle, name, seed):
    prob, facts = rs.build(name, seed)
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    REACH[name](facts, Placed(res.to_dict()))
