"""Seeded generator of problems whose class runs need a fresh node in a domain for which no variant exists yet, for the
derivation of a missing variant inside the run (csrc/pack_kernel.cuh, run_derive). Deployments of shapes no earlier
deployment had open their first node in every zone without a variant anywhere; the near misses sit just outside the
derivation's guards and keep the stop that hands the pod to the generic step.

Every scenario returns (problem dict, facts): facts["classes"] maps class names to pod indices, facts["fresh"] lists the
classes that must open fresh nodes in facts["zones"][cls] or more distinct zones (None: any number of nodes without a zone
spread), and facts["near"] names the guard a near miss crosses; tests/test_run_variant_reach.py checks them on the
oracle's result."""
import random

import fixtures as fx
import run_problems as rp
from fixtures import HOSTNAME, ZONE


def _req(i):
    """a shape no other deployment of the problem has: cpu in milli-units, memory fixed"""
    return {"cpu": f"{900 - 7 * i}m", "memory": "1Gi"}


def _anti(app):
    return {"podAntiAffinity": {"required": [fx.affinity_term(HOSTNAME, {"app": app})]}}


def _host_spread(app, skew):
    return fx.spread(HOSTNAME, {"app": app}, max_skew=skew)


def new_zone_shapes(seed):
    """zone spreads with skew 1 and 2 and a zone spread with anti-affinity, each deployment of a shape of its own: every
    first fresh node of a deployment in a zone has no variant in the ring or in the store"""
    rng = random.Random(seed)
    its = rp.zonal_types(rp.zone_names(3, "eu-west"), [(4, 8), (8, 32)], pods_cap=6)
    r = rp.Runs("newz")
    for i, skew in enumerate((1, 2)):
        r.run(f"z{i}", rng.choice([33, 64, 129]), _req(i), **rp.zone_spread(f"z{i}", skew=skew))
    spec = rp.zone_spread("za")
    spec.update(_anti("za"))
    r.run("za", rng.choice([12, 31]), _req(2), **spec)
    names = ["z0", "z1", "za"]
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": names, "zones": {n: 3 for n in names}, "near": None}


def new_host_shapes(seed):
    """anti-affinity (the derived node takes one pod: kRpDead) and hostname spreads with skew 4, 2 and 1, each of a shape
    of its own and each too large for the room the earlier ones leave on their nodes"""
    rng = random.Random(seed)
    its = rp.zonal_types(rp.zone_names(3, "eu-south"), [(4, 8), (8, 32)], pods_cap=6)
    r = rp.Runs("newh")
    r.run("anti", rng.choice([31, 33]), _req(0), labels={"app": "anti"}, **_anti("anti"))
    for j, skew in enumerate((4, 2, 1)):
        app = f"hs{skew}"
        r.run(app, 250, _req(1 + j), labels={"app": app}, topologySpreadConstraints=[_host_spread(app, skew)])
    names = ["anti", "hs4", "hs2", "hs1"]
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": names, "zones": {n: None for n in names}, "near": None}


def counts_moved(seed):
    """a deployment that selects only two zones (nodeSelector: the generic step places it) raises those zones' counts of a
    spread group; the zone-spread deployment that counts the same pods then opens its first nodes in the third zone and
    the other zones' first nodes only after the counts have levelled: derivations mid-run"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "us-east")
    its = rp.zonal_types(zs, [(4, 8), (8, 32)], pods_cap=5)
    r = rp.Runs("mv")
    r.run("pre", rng.choice([20, 31]), _req(0), labels={"app": "mv"}, nodeSelector={ZONE: zs[seed % 2]})
    r.run("pre2", rng.choice([20, 31]), _req(1), labels={"app": "mv"}, nodeSelector={ZONE: zs[1 - seed % 2]})
    spec = rp.zone_spread("mv")
    r.run("late", rng.choice([129, 250]), _req(2), **spec)
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": ["late"], "zones": {"late": 3}, "near": None, "first_zone": ("late", zs[2])}


def bulk_fill(seed):
    """plain deployments of new shapes on nodes of 4 or 7 pods: the level run's fresh step creates several nodes at once
    (F > 1) from the variant it has just derived"""
    rng = random.Random(seed)
    cap = rng.choice([4, 7])
    its = rp.zonal_types(rp.zone_names(2, "ap-south"), [(8, 32)], pods_cap=cap)
    r = rp.Runs("bulk")
    for i in range(3):
        r.run(f"p{i}", rng.choice([64, 129, 250]), _req(i), labels={"app": f"p{i}"})
    names = [f"p{i}" for i in range(3)]
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": names, "zones": {n: None for n in names}, "near": None, "min_nodes": 4, "pods_cap": cap}


def ring_and_store(seed):
    """six zones (more than the kRunVariants = 4 ring holds, so ring slots are reused while the mask run's fresh nodes
    still replay them) and 48 zone-spread deployments of distinct shapes, 288 variants: past the kVarStore = 256 store"""
    rng = random.Random(seed)
    its = rp.zonal_types(rp.zone_names(6, "sa-east"), [(4, 8)], pods_cap=3)
    r = rp.Runs("rs")
    names = []
    for i in range(48):
        r.run(f"s{i}", 18 * (1 + (i + seed) % 2), _req(i), **rp.zone_spread(f"s{i}"))  # whole nodes: no room left for the next
        names.append(f"s{i}")
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": names, "zones": {n: 6 for n in names}, "near": None, "variants": 257}


def unshared(seed):
    """classes the store refuses but a class run admits (no topology): volume claims. Only the ring serves them"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-north")
    its = rp.zonal_types(zs, [(4, 8), (8, 32)], pods_cap=5)
    r = rp.Runs("uns")
    for i in range(2):
        r.run(f"vol{i}", rng.choice([31, 64]), _req(i), labels={"app": f"vol{i}"}, volumes=[{"driver": "ebs", "pvc": f"default/v{seed}-{i}"}])
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": ["vol0", "vol1"], "zones": {"vol0": None, "vol1": None}, "near": None}


def near_limits(seed):
    """a provisioner with a cpu limit: no variant at all"""
    zs = rp.zone_names(3, "ca-west")
    its = rp.zonal_types(zs, [(4, 8), (8, 32)], pods_cap=5)
    r = rp.Runs("nlim")
    r.run("z", 64, _req(0), **rp.zone_spread("z"))
    r.run("p", 64, _req(1), labels={"app": "p"})
    return fx.problem(r.pods, instance_types=its, provisioners=[fx.provisioner(limits={"cpu": "200"})]), \
        {"classes": r.classes, "fresh": ["z", "p"], "zones": {"z": 3, "p": None}, "near": "limits"}


def near_wide(seed):
    """2 100 instance types: more option words than a variant holds (W32 > kRunW32)"""
    zs = rp.zone_names(3, "us-west")
    its = []
    for i in range(2100):
        res = {"cpu": str(1 + i % 32), "memory": f"{2 + (i * 7) % 200}Gi", "pods": "5"}
        price = fx.price_from_resources(res) + i * 1e-4
        its.append(fx.instance_type(f"t{i:04d}", res, offerings=[{"capacityType": ct, "zone": z, "price": price, "available": True}
                                                                   for z in zs for ct in ("spot", "on-demand")], oses=("linux",)))
    r = rp.Runs("nw")
    r.run("z", 64 + seed, _req(0), **rp.zone_spread("z"))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": ["z"], "zones": {"z": 3}, "near": "wide"}


def near_closed(seed):
    """every pod fills its node: a fresh node closes at once and never becomes an open slot"""
    zs = rp.zone_names(3, "af-south")
    its = rp.zonal_types(zs, [(4, 8)], pods_cap=1)
    r = rp.Runs("ncl")
    r.run("z", 12 + seed, {"cpu": "1", "memory": "1Gi"}, **rp.zone_spread("z"))
    r.run("p", 9, {"cpu": "900m", "memory": "1Gi"}, labels={"app": "p"})
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()]), \
        {"classes": r.classes, "fresh": ["z", "p"], "zones": {"z": 3, "p": None}, "near": "closed"}


def near_templates(seed):
    """two provisioners: a zone-spread class with several templates is not run-eligible"""
    zs = rp.zone_names(3, "me-central")
    its = rp.zonal_types(zs, [(4, 8), (8, 32)], pods_cap=5)
    r = rp.Runs("ntp")
    r.run("z", 64 + seed, _req(0), **rp.zone_spread("z"))
    provs = [rp.unlimited("first", weight=50), rp.unlimited("second", weight=10)]
    return fx.problem(r.pods, instance_types=its, provisioners=provs), \
        {"classes": r.classes, "fresh": ["z"], "zones": {"z": 3}, "near": "templates"}


SCENARIOS = {
    "new_zone_shapes": new_zone_shapes,
    "new_host_shapes": new_host_shapes,
    "counts_moved": counts_moved,
    "bulk_fill": bulk_fill,
    "ring_and_store": ring_and_store,
    "unshared": unshared,
    "near_limits": near_limits,
    "near_wide": near_wide,
    "near_closed": near_closed,
    "near_templates": near_templates,
}
CORPUS = [(name, seed) for name in SCENARIOS for seed in (0, 1)]


def build(name, seed):
    return SCENARIOS[name](seed)
