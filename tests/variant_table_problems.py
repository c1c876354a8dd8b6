"""Seeded problems at the edges of the pack kernel's variant table (csrc/pack_kernel.cuh, vt_build_entry): the fresh-node
variants of the class runs, built per Solve before the pack kernel, one entry per (class, domain its zone spread pins).

Every scenario returns (problem dict, facts). facts["reach"] says where the runs' fresh-node variants come from:
 * "table": the table holds every variant the runs ask for (taint_first: a template the class does not tolerate,
   weighted first; daemonset: the templates carry daemonset overhead; zone_subset: a zone spread whose node affinity
   admits two of three zones - the third zone's entry is none, since the pod's own requirement excludes it, and the run
   never asks for it; volume: a claim no CSI limit tracks, so the row is a plain one);
 * "none": no entry is taken, the runs derive their variants or stop (closes_at_once: every fresh node is full after one
   pod; two_masks: a zone and a capacity-type spread; relaxed: a preferred zone that does not exist, so no template opens
   a node for the class - its pods are relaxed and placed by the generic step when the queue comes round to them);
 * "both": beyond_capacity, more classes than the table holds (kVtClasses = 1 024): the classes below the limit take
   entries, the others derive.
Every class needs fresh nodes, and no scenario has an existing node (a class run needs a problem without them)."""
import random

import fixtures as fx
import run_problems as rp
from fixtures import CAPACITY_TYPE, ZONE

SHAPE = {"cpu": "1", "memory": "1Gi"}
VT_CLASSES = 1024  # pack_kernel.cuh: kVtClasses


def _types(zones, pods_cap=5):
    return rp.zonal_types(zones, [(4, 8), (8, 32)], pods_cap=pods_cap)


def zone_subset(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-west")
    keep = sorted(rng.sample(zs, 2))
    r = rp.Runs("zsub")
    r.run("sub", rng.choice([33, 61, 129]), SHAPE, nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": keep}]]},
          **rp.zone_spread("sub"))
    r.run("full", rng.choice([31, 64]), SHAPE, **rp.zone_spread("full"))
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=[rp.unlimited()]), {"classes": r.classes, "reach": "table"}


def closes_at_once(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "us-west")
    r = rp.Runs("once")
    r.run("one", rng.choice([17, 33]), SHAPE, **rp.zone_spread("one"))
    return fx.problem(r.pods, instance_types=_types(zs, pods_cap=1), provisioners=[rp.unlimited()]), {"classes": r.classes, "reach": "none"}


def taint_first(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "ap-south")
    r = rp.Runs("taint")
    r.run("plain", rng.choice([31, 64]), SHAPE, labels={"app": "plain"})
    r.run("spread", rng.choice([33, 61]), SHAPE, **rp.zone_spread("spread"))
    provs = [rp.unlimited("tainted", weight=50, taints=[{"key": "dedicated", "value": "x", "effect": "NoSchedule"}]),
             rp.unlimited("default", weight=10)]
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=provs), {"classes": r.classes, "reach": "table"}


def relaxed(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-north")
    prefer = {"preferred": [{"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": ["no-such-zone"]}]}]}
    r = rp.Runs("rlx")
    r.run("pref", rng.choice([31, 33]), SHAPE, labels={"app": "pref"}, nodeAffinity=prefer)
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=[rp.unlimited()]), {"classes": r.classes, "reach": "none"}


def daemonset(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "sa-east")
    r = rp.Runs("ds")
    r.run("plain", rng.choice([31, 64]), SHAPE, labels={"app": "plain"})
    r.run("spread", rng.choice([33, 61]), SHAPE, **rp.zone_spread("spread"))
    daemons = [fx.pod({"cpu": "500m", "memory": "256Mi"}), fx.pod({"cpu": "250m", "memory": "1Gi"}, nodeSelector={ZONE: zs[seed % 3]})]
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=[rp.unlimited()], daemonSetPods=daemons), \
        {"classes": r.classes, "reach": "table"}


def two_masks(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "us-east")
    r = rp.Runs("two")
    r.run("zc", rng.choice([33, 61]), SHAPE, **rp.zone_spread("zc", extra=[fx.spread(CAPACITY_TYPE, {"app": "zc"})]))
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=[rp.unlimited()]), {"classes": r.classes, "reach": "none"}


def volume(seed):
    rng = random.Random(seed)
    zs = rp.zone_names(3, "ca-central")
    r = rp.Runs("vol")
    r.run("vol", rng.choice([30, 35]), SHAPE, labels={"app": "vol"}, volumes=[{"driver": "ebs", "pvc": f"default/v{seed}"}])
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=[rp.unlimited()]), {"classes": r.classes, "reach": "table"}


def beyond_capacity(seed):
    """VT_CLASSES + 40 deployments of 5 pods whose memory requests differ by 1 Mi: one class each, one full node each"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-south")
    r = rp.Runs("cap")
    order = list(range(VT_CLASSES + 40))
    rng.shuffle(order)
    for i in order:
        r.run(f"d{i}", 5, {"cpu": "1", "memory": f"{1024 + i}Mi"}, labels={"app": f"d{i}"})
    return fx.problem(r.pods, instance_types=_types(zs), provisioners=[rp.unlimited()]), {"classes": r.classes, "reach": "both"}


SCENARIOS = {
    "zone_subset": zone_subset,
    "closes_at_once": closes_at_once,
    "taint_first": taint_first,
    "relaxed": relaxed,
    "daemonset": daemonset,
    "two_masks": two_masks,
    "volume": volume,
    "beyond_capacity": beyond_capacity,
}
SEEDS = {"beyond_capacity": (0,)}
CORPUS = [(name, seed) for name in SCENARIOS for seed in SEEDS.get(name, (0, 1))]


def build(name, seed):
    return SCENARIOS[name](seed)
