"""Seeded problems for the mask run's round stretches (csrc/pack_kernel.cuh, DESIGN.md section 4).

A zone spread with max skew 1 that counts its own pods places its pods in rounds, one per least-loaded zone. When every zone
has the same count, a stretch places several rounds in one step: on pinned nodes (the next members of each zone's bucket of
equal pod count) or on fresh nodes that take no second pod. Each scenario makes stretches end by one of their rules, or
builds a near miss that must fall back to single rounds; tests/test_round_stretch_reach.py checks on the oracle's result
that it does."""
import random

import fixtures as fx
import run_problems as rp
from fixtures import CAPACITY_TYPE, HOSTNAME, ZONE

TINY = {"cpu": "50m", "memory": "32Mi"}


def _anti(app):
    return {"required": [fx.affinity_term(HOSTNAME, {"app": app})]}


def _base(r, rng, nz, app="base"):
    """a zone-spread deployment of 1-cpu pods: its nodes (4 cpu) are pinned to their zone and hold up to 3 of them, so the
    zone lists meet the next class with buckets of several nodes"""
    r.run(app, nz * rng.choice([9, 13, 24]), {"cpu": "1", "memory": "1Gi"}, **rp.zone_spread(app))


def pinned(nz):
    """a tiny-pod zone spread over the nodes of an earlier one, nz zones: stretches walk the buckets until one is exhausted
    (its nodes re-enter at count + 1), the staged entries end, or 32 pods are placed"""
    def make(seed):
        rng = random.Random(seed * 31 + nz)
        zs = rp.zone_names(nz, "eu-north")
        its = rp.zonal_types(zs, [(4, 16)])
        r = rp.Runs(f"p{nz}")
        _base(r, rng, nz)
        r.run("spread", rng.choice([129, 250, 600]), TINY, **rp.zone_spread("spread"))
        return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "zones": nz}
    return make


def unequal(seed):
    """pods with the spread's label but without the spread are placed in the first zone before the run: the counts start
    unequal, so the first rounds leave that zone out and no stretch may start until the counts are level"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-central")
    its = rp.zonal_types(zs, [(4, 16)])
    r = rp.Runs("uneq")
    r.run("lead", rng.choice([1, 2, 5]), {"cpu": "2", "memory": "2Gi"}, labels={"app": "spread"},
          nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": [zs[0]]}]]})
    _base(r, rng, 3)
    r.run("spread", rng.choice([129, 250]), TINY, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "zones": zs}


def unpinned_between(seed):
    """one-pod nodes pinned to a zone and one-pod nodes in no zone alternate in the order (two deployments alternate pod by
    pod under one anti-affinity): an unpinned key lies between the pinned heads, so a stretch stops before it"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "us-north")
    its = rp.zonal_types(zs, [(2, 4), (8, 32)])
    r = rp.Runs("ub")
    anti = _anti("solo")
    spec_p = {"labels": {"app": "solo", "tier": "p"}, "podAntiAffinity": anti,
              "topologySpreadConstraints": [fx.spread(ZONE, {"tier": "p"})]}
    spec_u = {"labels": {"app": "solo", "tier": "u"}, "podAntiAffinity": anti}
    r.interleave("p", "u", rng.choice([12, 21, 40]), {"cpu": "1", "memory": "1Gi"}, spec_p, spec_u)
    r.run("spread", rng.choice([60, 129]), TINY, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes}


def room_slow(seed):
    """the second zone spread names a node affinity that the first one's nodes satisfy: its verdict on those nodes is not
    known in closed form (kRoomSlow) until it has placed a pod there itself, so buckets mix exact and inexact nodes"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "ap-north")
    its = rp.zonal_types(zs, [(4, 16)])
    r = rp.Runs("slow")
    _base(r, rng, 3)
    r.run("spread", rng.choice([60, 129, 250]), TINY, nodeAffinity={"required": [[{"key": CAPACITY_TYPE, "operator": "In",
                                                                                     "values": ["spot", "on-demand"]}]]},
          **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes}


def levels(seed):
    """one large node per zone, then a long tiny-pod zone spread: every round adds a pod to each of them, so their pod
    counts climb past kM1Lv = 12 inside the run and the stretch stops at the last count the lists represent"""
    rng = random.Random(seed)
    nz = (2, 3, 4)[seed % 3]
    zs = rp.zone_names(nz, "sa-east")
    its = rp.zonal_types(zs, [(32, 64)])
    r = rp.Runs("lv")
    r.run("anchor", nz, {"cpu": "2", "memory": "1Gi"}, labels={"app": "anchor"}, podAntiAffinity=_anti("anchor"),
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "anchor"})])
    r.run("spread", rng.choice([60, 129]), TINY, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes}


def fresh_anti(nz):
    """zone spread with hostname anti-affinity: every pod opens a fresh node that takes no second pod (fresh stretches)"""
    def make(seed):
        rng = random.Random(seed * 17 + nz)
        zs = rp.zone_names(nz, "me-west")
        its = rp.zonal_types(zs, [(2, 4), (8, 32)])
        r = rp.Runs(f"fa{nz}")
        r.run("spread", rng.choice([33, 129, 250]), {"cpu": "500m", "memory": "512Mi"}, podAntiAffinity=_anti("spread"),
              **rp.zone_spread("spread"))
        return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "zones": nz}
    return make


def fresh_room(seed):
    """pods that fill their node by resources: seed 0 and 1 one pod per node (fresh stretches: the node has no room left);
    seed 2 two pods per node (a near miss: the fresh node re-enters its zone's list, so every round stays single)"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "af-south")
    its = rp.zonal_types(zs, [(2, 4)])
    cpu = "700m" if seed % 3 == 2 else "1500m"
    r = rp.Runs("fr")
    r.run("spread", rng.choice([64, 129]), {"cpu": cpu, "memory": "512Mi"}, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "two": seed % 3 == 2}


def host_spread(seed):
    """zone spread combined with a hostname spread (max skew 1, or 2 on odd seeds): a fresh node takes a second pod only as
    far as the hostname spread lets it"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "ca-west")
    its = rp.zonal_types(zs, [(2, 4), (8, 32)])
    r = rp.Runs("hs")
    r.run("spread", rng.choice([60, 129]), {"cpu": "250m", "memory": "256Mi"}, labels={"app": "spread"},
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"}), fx.spread(HOSTNAME, {"app": "spread"}, max_skew=1 + seed % 2)])
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes}


SCENARIOS = {"pinned2": pinned(2), "pinned3": pinned(3), "pinned8": pinned(8), "unequal": unequal,
             "unpinned_between": unpinned_between, "room_slow": room_slow, "levels": levels, "fresh_anti2": fresh_anti(2),
             "fresh_anti3": fresh_anti(3), "fresh_anti8": fresh_anti(8), "fresh_room": fresh_room, "host_spread": host_spread}
SEEDS = {"fresh_room": (0, 1, 2), "levels": (0, 1, 2)}
CORPUS = [(name, seed) for name in SCENARIOS for seed in SEEDS.get(name, (0, 1))]


def build(name, seed):
    """(problem dict, facts): facts names the classes (pod indices per class) the scenario's predicate talks about"""
    return SCENARIOS[name](seed)
