"""Seeded generator of problems where several deployments of ONE shape follow each other in FFD order, for the class run's
store of fresh-node variants (csrc/pack_kernel.cuh, VarStoreEntry). Deployments of one shape with different relation
patterns (plain, anti-affinity, hostname spreads, zone spreads, zone plus capacity-type spread) replay each other's fresh
nodes; the near misses differ from their neighbour in one field of the class row NewNode + Add reads and must not.

Every scenario returns (problem dict, facts): facts["share"] lists groups of class names whose rows agree on every such
field; tests/test_shape_reach.py checks on the oracle's result that a later class of a group opens a fresh node in a
domain an earlier one of the group opened one in."""
import random

import fixtures as fx
import run_problems as rp
from fixtures import CAPACITY_TYPE, HOSTNAME, ZONE

SHAPE = {"cpu": "1", "memory": "1Gi"}


def _types(zones, pods_cap):
    return rp.zonal_types(zones, [(4, 8), (8, 32)], pods_cap=pods_cap)


def _anti(app):
    return {"labels": {"app": app}, "podAntiAffinity": {"required": [fx.affinity_term(HOSTNAME, {"app": app})]}}


def _host_spread(app, skew):
    return {"labels": {"app": app}, "topologySpreadConstraints": [fx.spread(HOSTNAME, {"app": app}, max_skew=skew)]}


def hostname_patterns(seed):
    """plain, anti-affinity and hostname spreads with skew 1, 2 and 4, two deployments of each, all of one shape: nodes
    hold 5 pods, so every deployment opens fresh nodes"""
    rng = random.Random(seed)
    its = _types(rp.zone_names(3, "eu-west"), 5)
    r = rp.Runs("host")
    specs = [("plain", {"labels": {"app": "plain"}}), ("anti", _anti("anti"))] + \
            [(f"hs{k}", _host_spread(f"hs{k}", k)) for k in (1, 2, 4)]
    for rep in range(2):
        for name, spec in specs:
            # a second deployment of a pattern counts its own pods: a fresh label value, the same row
            spec2 = {**spec, "labels": {**spec["labels"], "rev": f"r{rep}"}}
            r.run(f"{name}-{rep}", rng.choice([31, 33, 64]), SHAPE, **spec2)
    share = [[f"{n}-{rep}" for rep in range(2) for n, _ in specs]]
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "share": share}


def zone_patterns(seed):
    """zone spreads with skew 1 and 2 and zone plus capacity-type spreads over 3 zones; a spread that does not select its
    own pods comes last"""
    rng = random.Random(seed)
    its = _types(rp.zone_names(3, "us-east"), 5)
    r = rp.Runs("zone")
    for i, skew in enumerate((1, 2, 1, 2)):
        r.run(f"z{i}", rng.choice([33, 129, 250]), SHAPE, **rp.zone_spread(f"z{i}", skew=skew))
    for i in range(2):
        r.run(f"zc{i}", rng.choice([60, 129]), SHAPE, **rp.zone_spread(f"zc{i}", extra=[fx.spread(CAPACITY_TYPE, {"app": f"zc{i}"})]))
    r.run("zo", 64, SHAPE, labels={"app": "zo"}, topologySpreadConstraints=[fx.spread(ZONE, {"app": "z0"})])
    share = [["z0", "z1", "z2", "z3", "zo"], ["zc0", "zc1"]]
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), {"classes": r.classes, "share": share}


def many_zones(nz):
    """nz zones: 6 needs more variants than the kRunVariants = 4 ring inside one mask run; 10 is beyond the mask run's
    kM1Dom = 8 domains (the per-pod loop replays the variants)"""
    def make(seed):
        rng = random.Random(seed * 31 + nz)
        its = _types(rp.zone_names(nz, "ap-north"), 4)
        r = rp.Runs(f"mz{nz}")
        for i in range(4):
            r.run(f"s{i}", rng.choice([129, 250]), SHAPE, **rp.zone_spread(f"s{i}", skew=1 + (i + seed) % 2))
        return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
            {"classes": r.classes, "share": [[f"s{i}" for i in range(4)]]}
    return make


def relaxation(seed):
    """preferred node affinity relaxed away: the relaxed classes of two deployments and a plain one share a row"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-east")
    its = _types(zs, 5)
    r = rp.Runs("rlx")
    prefer = {"preferred": [{"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": ["no-such-zone"]}]}]}
    r.run("p0", rng.choice([31, 33]), SHAPE, labels={"app": "p0"}, nodeAffinity=prefer)
    r.run("p1", rng.choice([31, 33]), SHAPE, labels={"app": "p1"}, nodeAffinity=prefer)
    r.run("plain", 33, SHAPE, labels={"app": "plain"})
    r.run("anyway", 64, SHAPE, **rp.zone_spread("anyway", when="ScheduleAnyway"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "share": [["p0", "p1", "plain"]]}


def near_misses(seed):
    """neighbours that differ in one field of the row NewNode + Add reads: requests by one milli-unit, a resource key with
    request 0, a toleration, a node-selector value, a volume claim, a host port"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "sa-east")
    its = _types(zs, 5)
    k = lambda: rng.choice([30, 35])  # whole nodes of 5 pods: no deployment's pods join another one's node
    r = rp.Runs("near")
    r.run("base", k(), SHAPE, labels={"app": "base"})
    r.run("milli", k(), {"cpu": "1001m", "memory": "1Gi"}, labels={"app": "milli"})
    r.run("zero", k(), {**SHAPE, "ephemeral-storage": "0"}, labels={"app": "zero"})
    r.run("tol", k(), SHAPE, labels={"app": "tol"}, tolerations=[{"key": "dedicated", "operator": "Exists"}])
    r.run("sel", k(), SHAPE, labels={"app": "sel"}, nodeSelector={ZONE: zs[seed % 3]})
    r.run("vol", k(), SHAPE, labels={"app": "vol"}, volumes=[{"driver": "ebs", "pvc": f"default/v{seed}"}])
    r.run("base2", 65, SHAPE, labels={"app": "base2"})
    # one node per pod (the port clashes): last, so the nodes it opens do not take the others' pods
    r.run("port", k(), SHAPE, labels={"app": "port"}, ports=[{"hostPort": 8080 + seed, "protocol": "TCP"}])
    # a tainted provisioner only the tolerating deployment may use, weighted first
    provs = [rp.unlimited("tainted", weight=50, taints=[{"key": "dedicated", "value": "x", "effect": "NoSchedule"}]),
             rp.unlimited("default", weight=10)]
    return fx.problem(r.pods, instance_types=its, provisioners=provs), {"classes": r.classes, "share": [["base", "base2"]]}


SCENARIOS = {
    "hostname_patterns": hostname_patterns,
    "zone_patterns": zone_patterns,
    "zones6": many_zones(6),
    "zones10": many_zones(10),
    "relaxation": relaxation,
    "near_misses": near_misses,
}
CORPUS = [(name, seed) for name in SCENARIOS for seed in (0, 1)]


def build(name, seed):
    return SCENARIOS[name](seed)
