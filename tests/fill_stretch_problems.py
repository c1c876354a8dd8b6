"""Seeded problems for the mask run's fill stretches (csrc/pack_kernel.cuh, DESIGN.md section 4).

A zone spread with max skew 1 that counts its own pods places its pods in rounds, one per zone. When every zone's head is
the only node of its pod count in its zone's list, a round sends it back to the front of its list, so the next rounds take
the same node per zone and one step places them all. Each scenario makes fill stretches end by one of their limits (room,
hostname spread, kM1Lv, the unpinned head, the node behind the head, the staged entries, 32 pods), starts them after a
partial round, or builds a near miss that must not take them (an inexact room word, a second node in a bucket);
tests/test_fill_stretch_reach.py checks on the oracle's result that it does."""
import random

import fixtures as fx
import round_stretch_problems as rs
import run_problems as rp
from fixtures import HOSTNAME, ZONE

TINY = rs.TINY


def _anti(app):
    return {"required": [fx.affinity_term(HOSTNAME, {"app": app})]}


def _anchors(r, nz, cpu="2"):
    """one node per zone, pinned to it, that holds one pod of its own: the spread's zone lists start with one head each"""
    r.run("anchor", nz, {"cpu": cpu, "memory": "1Gi"}, labels={"app": "anchor"}, podAntiAffinity=_anti("anchor"),
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "anchor"})])


def levels(nz):
    """one large node per zone, then a long tiny-pod zone spread: the fill stretches run until the pod counts reach the
    last level the lists represent (kM1Lv); with 8 zones a step holds 4 rounds (32 pods), and odd pod counts end the last
    stretch at the staged entries"""
    def make(seed):
        rng = random.Random(seed * 13 + nz)
        zs = rp.zone_names(nz, "sa-east")
        its = rp.zonal_types(zs, [(32, 64)])
        r = rp.Runs(f"lv{nz}")
        _anchors(r, nz)
        r.run("spread", rng.choice([61, 97, 130]) if nz < 8 else rng.choice([83, 130]), TINY, **rp.zone_spread("spread"))
        return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "zones": nz}
    return make


def room(nz):
    """anchors on 4-cpu nodes and 500m spread pods: each anchor node's room ends its stretch after a few rounds, and the
    fresh nodes the spread opens afterwards (one per zone, each the only node of its count) fill the same way"""
    def make(seed):
        rng = random.Random(seed * 7 + nz)
        zs = rp.zone_names(nz, "af-north")
        its = rp.zonal_types(zs, [(4, 16)])
        r = rp.Runs(f"rm{nz}")
        _anchors(r, nz)
        r.run("spread", nz * rng.choice([5, 9, 14]) + seed % 2, {"cpu": "500m", "memory": "256Mi"}, **rp.zone_spread("spread"))
        return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "zones": nz}
    return make


def host_spread(skew):
    """zone spread plus a hostname spread of max skew 1, 2 or 4: an anchor node takes `skew` spread pods (the hostname
    limit ends the stretch), then fresh nodes do the same"""
    def make(seed):
        rng = random.Random(seed * 5 + skew)
        zs = rp.zone_names(3, "ca-east")
        its = rp.zonal_types(zs, [(32, 64)])
        r = rp.Runs(f"hs{skew}")
        _anchors(r, 3)
        r.run("spread", rng.choice([40, 61, 99]), TINY, labels={"app": "spread"},
              topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"}), fx.spread(HOSTNAME, {"app": "spread"}, max_skew=skew)])
        return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "skew": skew}
    return make


def unpinned(seed):
    """a node in no zone holding several pods of another deployment (kept off the anchors by anti-affinity): the anchors'
    stretches climb to its pod count, and one round later its key comes first, so the unpinned head ends the stretch"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "us-south")
    its = rp.zonal_types(zs, [(32, 64)])
    r = rp.Runs("up")
    _anchors(r, 3)
    r.run("plain", rng.choice([3, 5, 7]), {"cpu": "1", "memory": "1Gi"}, labels={"app": "plain"}, podAntiAffinity=_anti("anchor"))
    r.run("spread", rng.choice([40, 61]), TINY, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes}


def behind(seed):
    """two nodes per zone, one with a pod more than the other: the head's stretch ends where its count passes the node
    behind it, and the two then share a bucket"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-south")
    its = rp.zonal_types(zs, [(32, 64)])
    r = rp.Runs("bh")
    r.run("x", 6, {"cpu": "2", "memory": "1Gi"}, labels={"app": "x"}, podAntiAffinity=_anti("x"),
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "x"})])
    r.run("y", 3, {"cpu": "1500m", "memory": "1Gi"}, labels={"app": "y"}, podAntiAffinity=_anti("y"),
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "y"})])
    r.run("spread", rng.choice([40, 61, 99]), TINY, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes}


def unequal(seed):
    """a pod with the spread's label sits on the first zone's anchor before the run: the first round is partial (the zones
    one pod behind), then the counts are level and the stretches start"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "ap-east")
    its = rp.zonal_types(zs, [(32, 64)])
    r = rp.Runs("ue")
    _anchors(r, 3)
    r.run("lead", 1 + seed % 2, {"cpu": "1", "memory": "1Gi"}, labels={"app": "spread"},
          nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": [zs[0]]}]]})
    r.run("spread", rng.choice([40, 61]), TINY, **rp.zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "zones": zs}


SCENARIOS = {"levels2": levels(2), "levels3": levels(3), "levels8": levels(8), "room2": room(2), "room3": room(3),
             "room8": room(8), "host_spread1": host_spread(1), "host_spread2": host_spread(2), "host_spread4": host_spread(4),
             "unpinned": unpinned, "behind": behind, "unequal": unequal,
             # near misses: a second node in the head's bucket, an inexact room word
             "bucket": rs.pinned(3), "room_slow": rs.room_slow}
SEEDS = {"unpinned": (0, 1, 2), "behind": (0, 1, 2)}
CORPUS = [(name, seed) for name in SCENARIOS for seed in SEEDS.get(name, (0, 1))]


def build(name, seed):
    """(problem dict, facts): facts names the classes (pod indices per class) the scenario's predicate talks about"""
    return SCENARIOS[name](seed)
