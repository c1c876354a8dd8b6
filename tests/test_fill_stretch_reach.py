"""CPU: every scenario of tests/fill_stretch_problems.py really crosses the rule of the mask run's fill stretches it was
built for. Each predicate is computed from the problem and the oracle's result alone."""
from collections import Counter

import pytest

import fill_stretch_problems as fs
from test_round_stretch_reach import K_M1_LV, Placed, reach_pinned, reach_room_slow


def _spread_on(facts, pl, cls):
    """{node opened by class cls: spread pods it took}"""
    nodes = pl.opened_by(facts["classes"][cls])
    got = Counter(n for n in pl.nodes_of(facts["classes"]["spread"]) if n in nodes)
    return {n: got[n] for n in nodes}


def _total(pl, n):
    return sum(1 for a in pl.assign if a == n)


def reach_levels(facts, pl):
    on = _spread_on(facts, pl, "anchor")
    assert len(on) == facts["zones"] and min(on.values()) >= 2
    assert max(_total(pl, n) for n in on) >= K_M1_LV, "the anchors should pass the last level the lists represent"
    assert len(facts["classes"]["spread"]) % facts["zones"], "the last round should be partial (staged end)"
    if facts["zones"] == 8:
        assert min(on.values()) * 8 > 32, "one step should be cut at 32 pods"


def reach_room(facts, pl):
    on = _spread_on(facts, pl, "anchor")
    assert len(on) == facts["zones"] and len(set(on.values())) == 1 and min(on.values()) >= 2, on
    rest = Counter(n for n in pl.nodes_of(facts["classes"]["spread"]) if n not in on)
    assert rest and max(rest.values()) >= 2, "fresh nodes should take more than one pod"


def reach_host_spread(facts, pl):
    on = _spread_on(facts, pl, "anchor")
    assert set(on.values()) == {facts["skew"]}
    assert max(Counter(pl.nodes_of(facts["classes"]["spread"])).values()) == facts["skew"]


def reach_unpinned(facts, pl):
    (plain,) = pl.opened_by(facts["classes"]["plain"])
    assert _total(pl, plain) > len(facts["classes"]["plain"]), "the unpinned node should take spread pods"
    assert min(_spread_on(facts, pl, "anchor").values()) >= 2


def reach_behind(facts, pl):
    on = _spread_on(facts, pl, "x")
    assert len(on) == 6 and min(on.values()) >= 2
    zone_counts = {}
    for n in on:
        zone_counts.setdefault(pl.zone(n), []).append(_total(pl, n) - on[n])
    assert all(sorted(v) == [1, 2] for v in zone_counts.values()), zone_counts  # per zone: a node with a pod more


def reach_unequal(facts, pl):
    zs = facts["zones"]
    assert all(pl.zone(n) == zs[0] for n in pl.nodes_of(facts["classes"]["lead"]))
    first = facts["classes"]["spread"][0]
    assert pl.zone(pl.assign[first]) != zs[0], "the counts should start unequal"
    assert min(_spread_on(facts, pl, "anchor").values()) >= 2


def reach_bucket(facts, pl):
    reach_pinned(facts, pl)


REACH = {name: globals()["reach_" + name.rstrip("0123456789")] for name in fs.SCENARIOS}
REACH["room_slow"] = reach_room_slow


@pytest.mark.parametrize("name,seed", fs.CORPUS, ids=[f"{n}-{s}" for n, s in fs.CORPUS])
def test_fill_stretch_scenario_reaches_its_rule(pkg, oracle, name, seed):
    prob, facts = fs.build(name, seed)
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    REACH[name](facts, Placed(res.to_dict()))
