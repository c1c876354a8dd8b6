"""Seeded generator of deployment-shaped problems for the pack kernel's run paths (csrc/pack_kernel.cuh: class run, mask
run, fresh-node variants, existing-node run, failure memo).

A problem is a sequence of RUNS: deployments of k identical pods, k drawn from RUN_SIZES. The queue orders pods by cpu,
then memory, then creationTimestamp, then UID (queue.go:74-110), so every run gets its own timestamp and its pods get
UIDs in creation order: runs with equal requests follow each other in the order they were written, and two runs written
with `interleave` alternate pod by pod. Every scenario is built to cross one capacity of those paths (DESIGN.md section 4);
tests/test_run_reach.py checks on the oracle's result that it does."""
import copy
import random

import fixtures as fx
from fixtures import CAPACITY_TYPE, HOSTNAME, ZONE

RUN_SIZES = (1, 31, 32, 33, 127, 128, 129, 250, 600)
RACK = "example.com/rack"


def zone_names(n, region="eu-west"):
    """custom zone names that sort in creation order (the dictionary numbers values in sorted order)"""
    return [f"{region}-{i:02d}" for i in range(n)]


def zonal_types(zones, sizes, pods_cap=110, extra=None, prefix="m", racks=None):
    """one instance type per (cpu, memory GiB) size, offered spot (cheaper) and on-demand in every zone"""
    its = []
    for cpu, mem in sizes:
        for rack in racks or [None]:
            res = {"cpu": str(cpu), "memory": f"{mem}Gi", "pods": str(pods_cap), **(extra or {})}
            price = fx.price_from_resources(res)
            offers = [{"capacityType": ct, "zone": z, "price": round(price * (0.6 if ct == "spot" else 1.0), 6), "available": True}
                      for z in zones for ct in ("spot", "on-demand")]
            name = f"{prefix}{cpu}-{mem}g-p{pods_cap}" + (f"-{rack}" if rack else "")
            it = fx.instance_type(name, res, offerings=offers, oses=("linux",))
            if rack:
                it["requirements"].append({"key": RACK, "operator": "In", "values": [rack]})
            its.append(it)
    return its


def unlimited(name="default", **kw):
    """a provisioner without limits: the fresh-node variants and bulk creation of the class run are on (s.any_limits == 0)"""
    return {"name": name, **kw}


class Runs:
    """Pods written run by run. Names and UIDs are local to the problem, so the corpus does not depend on test order."""

    def __init__(self, tag):
        self.tag = tag
        self.pods = []
        self.ts = 0
        self.classes = {}  # class name -> pod indices, in creation order

    def _pod(self, cls, requests, ts, spec):
        i = len(self.pods)
        p = fx.pod(dict(requests), name=f"{self.tag}-{i:05d}", uid=f"{self.tag}-{i:05d}", creationTimestamp=ts, **copy.deepcopy(spec))
        self.pods.append(p)
        self.classes.setdefault(cls, []).append(i)

    def run(self, cls, k, requests, **spec):
        """a deployment of k identical pods (spec: labels, spreads, affinities, selectors, tolerations)"""
        self.ts += 1
        for _ in range(k):
            self._pod(cls, requests, self.ts, spec)

    def interleave(self, a, b, k, requests, spec_a, spec_b):
        """two deployments with equal requests and one timestamp, pod UIDs alternating: the queue alternates a, b, a, ..."""
        self.ts += 1
        for _ in range(k):
            self._pod(a, requests, self.ts, spec_a)
            self._pod(b, requests, self.ts, spec_b)


def zone_spread(app, skew=1, when="DoNotSchedule", extra=()):
    return {"labels": {"app": app}, "topologySpreadConstraints": [fx.spread(ZONE, {"app": app}, max_skew=skew, when=when), *extra]}


SMALL = {"cpu": "100m", "memory": "128Mi"}


# ---------------------------------------------------------------- scenarios (each: seed -> (problem dict, facts))
def zones(nz):
    """nz zones, zone-spread runs at the chunk edge and around it, a plain run between them. nz >= 9: the mask run is
    refused (registered domains >= kM1Dom); nz == 17: the zone key has more than kRunDom values, so no spread class is
    run-eligible (only 16 zones fit the offering words: the 17th is named by the provisioner and served by existing nodes
    alone, no type is offered in it)."""
    def make(seed):
        rng = random.Random(seed * 1009 + nz)
        offered = zone_names(min(nz, 16))
        zs = zone_names(nz)
        its = zonal_types(offered, [(2, 4), (4, 16), (8, 32)], pods_cap=rng.choice([20, 110]))
        r = Runs(f"z{nz}")
        k1, k2 = rng.choice([(128, 129), (127, 250), (250, 128)])
        r.run("spread-a", k1, {"cpu": "1", "memory": "1Gi"}, **zone_spread("spread-a"))
        r.run("spread-b", k2, {"cpu": "1", "memory": "1Gi"}, **zone_spread("spread-b", skew=rng.choice([1, 2])))
        r.run("plain", rng.choice([31, 33]), {"cpu": "500m", "memory": "256Mi"}, labels={"app": "plain"})
        r.run("spread-c", rng.choice([250, 600]), SMALL, **zone_spread("spread-c"))
        nodes = []
        for i, z in enumerate(zs[16:]):
            for j in range(4):
                nodes.append(fx.state_node(f"old-{i}-{j}", its[2]["name"], zone=z, capacity_type="on-demand",
                                           allocatable={"cpu": "32", "memory": "128Gi", "pods": "110"}))
        # the provisioner names every zone, so the 17th is a registered domain (served by the existing nodes alone)
        prov = unlimited(requirements=[{"key": ZONE, "operator": "In", "values": zs}]) if nz > 16 else unlimited()
        return fx.problem(r.pods, instance_types=its, provisioners=[prov], nodes=nodes), {"classes": r.classes, "zones": nz}
    return make


def pods_capacity(seed):
    """instance types holding 11, 12, 13 or 110 pods: zone-spread nodes pass kM1Lv = 12 pods inside one mask run"""
    rng = random.Random(seed)
    caps = [(11, 12, 13, 110), (11, 12, 13), (12, 13)][seed % 3]
    zs = zone_names(3, "ap-south")
    its = [t for cap in caps for t in zonal_types(zs, [(4, 8), (16, 32)], pods_cap=cap, prefix=f"c{cap}-")]
    r = Runs("cap")
    r.run("spread-a", rng.choice([250, 600]), {"cpu": "50m", "memory": "32Mi"}, **zone_spread("spread-a"))
    r.run("spread-b", 129, {"cpu": "20m", "memory": "16Mi"}, **zone_spread("spread-b", skew=2))
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def pinned_nodes(seed):
    """an earlier class opens nodes pinned to 2 of 5 zones (In [z0 z1]); the zone-spread run after it meets nodes that
    admit only some of the registered domains"""
    rng = random.Random(seed)
    zs = zone_names(5, "us-east")
    its = zonal_types(zs, [(2, 4), (8, 32)])
    r = Runs("pin")
    r.run("pinned", rng.choice([31, 33]), {"cpu": "6", "memory": "4Gi"}, labels={"app": "pinned"},
          nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": zs[:2]}]]})
    r.run("spread", 250, {"cpu": "250m", "memory": "256Mi"}, **zone_spread("spread"))
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def two_masks(seed):
    """zone spread plus capacity-type spread, and zone spread plus a custom-key spread, on one class: two mask relations,
    10 or 15 spread domain combinations, so more fresh-node variants than the kRunVariants = 4 ring holds"""
    zs = zone_names(5, "sa-east")  # an odd zone count: zone and second-key domains do not cycle together
    racks = ["r1", "r2", "r3"]
    its = zonal_types(zs, [(4, 16), (16, 64)], racks=racks)
    r = Runs("mask2")
    second = fx.spread(CAPACITY_TYPE, {"app": "zc"}) if seed % 2 == 0 else fx.spread(RACK, {"app": "zc"})
    r.run("zc", 250, {"cpu": "1", "memory": "1Gi"}, **zone_spread("zc", extra=[second]))
    r.run("zr", 128, {"cpu": "500m", "memory": "512Mi"}, **zone_spread("zr", extra=[fx.spread(RACK, {"app": "zr"}, max_skew=2)]))
    prob = fx.problem(r.pods, instance_types=its, provisioners=[unlimited()])
    prob["wellKnownLabels"] = list(prob["wellKnownLabels"]) + [RACK]
    return prob, {"classes": r.classes, "second": CAPACITY_TYPE if seed % 2 == 0 else RACK}


def hostname_relations(seed):
    """3, 4 and 5 hostname-keyed relations on one class (anti-affinity and hostname spreads with skew 1-4); kRunHost = 4"""
    zs = zone_names(3, "eu-north")
    its = zonal_types(zs, [(8, 32), (32, 128)])
    r = Runs("host")
    r.run("db", 32, {"cpu": "2", "memory": "2Gi"}, labels={"app": "db", "tier": "data"})
    base = [fx.spread(HOSTNAME, {"tier": "web"}, max_skew=4)]
    anti = {"required": [fx.affinity_term(HOSTNAME, {"app": "db"})]}
    for n_rel, k in ((3, 128), (4, 129), (5, 33)):
        app = f"h{n_rel}"
        spreads = [fx.spread(HOSTNAME, {"app": app}, max_skew=1 + (seed % 2))] + base
        spreads += [fx.spread(HOSTNAME, {"team": f"t{j}"}, max_skew=2 + j) for j in range(n_rel - 3)]
        r.run(app, k, {"cpu": "500m", "memory": "512Mi"}, labels={"app": app, "tier": "web", "team": "t0"},
              topologySpreadConstraints=spreads, podAntiAffinity=anti)
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def big_active_set(seed):
    """an anti-affinity run of 1 300 tiny pods opens more than kActCap = 1 280 nodes (hot state spills to the ov_* arrays;
    bulk creation passes kTopoCap and kActCap), then spread runs meet an active set beyond both capacities"""
    zs = zone_names(3, "me-central")
    its = zonal_types(zs, [(16, 64), (32, 128)])
    r = Runs("big")
    r.run("anti", 1300, {"cpu": "200m", "memory": "128Mi"}, labels={"app": "anti"},
          podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "anti"})]})
    r.run("zone", 250, SMALL, **zone_spread("zone"))
    r.run("host", 128, {"cpu": "50m", "memory": "64Mi"}, labels={"app": "host"},
          topologySpreadConstraints=[fx.spread(HOSTNAME, {"app": "host"}, max_skew=1 + seed % 3)])
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def limits(seed):
    """seed 0: one provisioner whose cpu limit binds in the middle of a run; seed 1: three weighted provisioners (one with a
    limit) and zone spread"""
    zs = zone_names(3, "ca-west")
    its = zonal_types(zs, [(4, 16), (8, 32)])
    r = Runs("lim")
    if seed % 2 == 0:
        r.run("big", 250, {"cpu": "1", "memory": "1Gi"}, labels={"app": "big"})
        r.run("small", 128, SMALL, **zone_spread("small"))
        provs = [fx.provisioner(limits={"cpu": "100"})]
    else:
        r.run("a", 129, {"cpu": "1", "memory": "1Gi"}, **zone_spread("a"))
        r.run("b", 250, SMALL, labels={"app": "b"})
        r.run("c", 33, SMALL, labels={"app": "c"}, nodeSelector={"team": "blue"})
        provs = [fx.provisioner("heavy", weight=50, limits={"cpu": "40"}, requirements=[{"key": ZONE, "operator": "In", "values": zs[:2]}]),
                 unlimited("light", weight=10),
                 unlimited("blue", weight=0, labels={"team": "blue"})]
    return fx.problem(r.pods, instance_types=its, provisioners=provs), {"classes": r.classes}


def many_existing(seed):
    """2 048-2 200 existing nodes (some tainted, some marked for deletion, most with room for one pod): one plain run of
    600 pods passes more than 512 of them, so the existing-node run scans twice at 512 threads"""
    rng = random.Random(seed)
    zs = zone_names(3, "af-south")
    its = zonal_types(zs, [(4, 16), (8, 32)], pods_cap=20)
    r = Runs("ex")
    r.run("plain", 600, {"cpu": "1", "memory": "1Gi"}, labels={"app": "plain"})
    r.run("spread", 128, SMALL, **zone_spread("spread"))
    nodes = []
    n = rng.choice([2048, 2100, 2200]) + 40
    for i in range(n):
        name = f"node-{i:05d}"
        u = rng.random()
        bound = [] if u < 0.03 else [fx.pod({"cpu": "2900m", "memory": "1Gi"}, name=f"bound-{i:05d}", uid=f"bound-{i:05d}", nodeName=name, labels={"app": "old"})]
        nodes.append(fx.state_node(name, its[0]["name"], zone=zs[i % 3], capacity_type="on-demand",
                                   allocatable={"cpu": "4", "memory": "16Gi", "pods": "20"}, pods_=bound,
                                   taints=[{"key": "dedicated", "value": "x", "effect": "NoSchedule"}] if rng.random() < 0.08 else [],
                                   markedForDeletion=i % (n // 40) == 7))
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()], nodes=nodes), {"classes": r.classes}


def huge_catalog(seed):
    """2 100 instance types: more option words than a fresh-node variant holds (W32 > kRunW32), so variants are off"""
    zs = zone_names(3, "us-west")
    sizes = [(1 + i % 32, 2 + (i * 7) % 200) for i in range(2100)]
    its = []
    for i, (cpu, mem) in enumerate(sizes):
        res = {"cpu": str(cpu), "memory": f"{mem}Gi", "pods": "110"}
        price = fx.price_from_resources(res) + i * 1e-4
        its.append(fx.instance_type(f"t{i:04d}", res, offerings=[{"capacityType": ct, "zone": z, "price": price, "available": True}
                                                                   for z in zs for ct in ("spot", "on-demand")], oses=("linux",)))
    r = Runs("cat")
    r.run("spread", 250, {"cpu": "1", "memory": "1Gi"}, **zone_spread("spread"))
    r.run("plain", 128, SMALL, labels={"app": "plain"})
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def extended_resources(seed):
    """pods requesting two extended resources: resources beyond the kHotRes = 4 hot ones"""
    zs = zone_names(3, "eu-south")
    its = zonal_types(zs, [(8, 32), (16, 64)], extra={"fake.com/vendor-a": "8", "fake.com/vendor-b": "4"}, prefix="gpu")
    its += zonal_types(zs, [(8, 32)])
    r = Runs("ext")
    r.run("ext", 129, {"cpu": "1", "memory": "1Gi", "fake.com/vendor-a": "1", "fake.com/vendor-b": "1"}, labels={"app": "ext"})
    r.run("ext-spread", 33, {"cpu": "500m", "memory": "1Gi", "fake.com/vendor-a": "2", "fake.com/vendor-b": "1"}, **zone_spread("ext-spread"))
    r.run("plain", 128, SMALL, labels={"app": "plain"})
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def relaxation(seed):
    """unschedulable runs interleaved pod by pod with schedulable ones (the failure memo), preferred node affinity that
    has to be relaxed, and ScheduleAnyway spreads"""
    zs = zone_names(3, "eu-east")
    its = zonal_types(zs, [(4, 16), (8, 32)])
    r = Runs("rlx")
    r.run("too-big", 31, {"cpu": "100", "memory": "1Gi"}, labels={"app": "too-big"})
    r.interleave("ok", "nowhere", 128, {"cpu": "1", "memory": "1Gi"}, {"labels": {"app": "ok"}},
                 {"labels": {"app": "nowhere"}, "nodeSelector": {"team": "none"}})
    r.run("prefer", 127, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "prefer"},
          nodeAffinity={"preferred": [{"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": ["no-such-zone"]}]},
                                      {"weight": 10, "terms": [{"key": ZONE, "operator": "In", "values": [zs[seed % 3]]}]}]})
    r.run("anyway", 250, SMALL, **zone_spread("anyway", when="ScheduleAnyway"))
    r.run("soft-anti", 32, SMALL, labels={"app": "soft-anti"},
          podAntiAffinity={"preferred": [{"weight": 10, "term": fx.affinity_term(HOSTNAME, {"app": "soft-anti"})}]})
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes}


def chunk_edges(seed):
    """class changes placed on the kRunChunk = 128 staging edge: runs of 127 / 128 / 129 of one request vector followed by
    another class with the same requests, and two such classes interleaved pod by pod"""
    zs = zone_names(3, "il-central")
    its = zonal_types(zs, [(4, 16), (16, 64)])
    r = Runs("edge")
    req = {"cpu": "250m", "memory": "256Mi"}
    k = (127, 128, 129)[seed % 3]
    r.run("a", k, req, **zone_spread("a"))
    r.run("b", 128, req, **zone_spread("b"))
    r.run("c", k, req, labels={"app": "c"})
    r.run("a2", 1, req, **zone_spread("a"))
    r.interleave("x", "y", 33, req, zone_spread("x"), zone_spread("y", skew=2))
    return fx.problem(r.pods, instance_types=its, provisioners=[unlimited()]), {"classes": r.classes, "k": k}


def cluster(seed, nz, ct_spread=False):
    """a consolidation cluster in the run shapes: 3 * nz owned candidate nodes over nz zones (spot and on-demand) holding a
    zone-spread deployment (plus capacity-type spread when ct_spread), and pending pods of the same deployment"""
    rng = random.Random(seed)
    zs = zone_names(nz, "eu-central")
    its = zonal_types(zs, [(4, 16), (8, 32), (16, 64)])
    spec = zone_spread("web", extra=[fx.spread(CAPACITY_TYPE, {"app": "web"})] if ct_spread else [])
    req = {"cpu": "500m", "memory": "512Mi"}
    nodes = []
    for i in range(3 * nz):
        it = its[rng.randrange(len(its))]
        name = f"node-{i:03d}"
        bound = [fx.pod(dict(req), name=f"{name}-{j}", uid=f"{name}-{j}", nodeName=name, **copy.deepcopy(spec)) for j in range(rng.choice([1, 2, 3]))]
        nodes.append(fx.state_node(name, it["name"], zone=zs[i % nz], capacity_type=("spot", "on-demand")[(i // nz) % 2],
                                   allocatable=dict(it["capacity"]), pods_=bound, candidate=True, disruptionCost=float(rng.choice([0, 1, 2, 3]))))
    r = Runs("pending")
    r.run("web", rng.choice([31, 33]), req, **spec)
    return fx.problem(r.pods, instance_types=its, provisioners=[fx.provisioner()], nodes=nodes)


SCENARIOS = {
    **{f"zones{z}": zones(z) for z in (3, 7, 8, 9, 12, 16, 17)},
    "pods_capacity": pods_capacity,
    "pinned_nodes": pinned_nodes,
    "two_masks": two_masks,
    "hostname_relations": hostname_relations,
    "big_active_set": big_active_set,
    "limits": limits,
    "many_existing": many_existing,
    "huge_catalog": huge_catalog,
    "extended_resources": extended_resources,
    "relaxation": relaxation,
    "chunk_edges": chunk_edges,
}
SEEDS = {"pods_capacity": (0, 1, 2), "two_masks": (0, 1), "limits": (0, 1), "chunk_edges": (0, 1, 2), "hostname_relations": (0, 1)}
CORPUS = [(name, seed) for name in SCENARIOS for seed in SEEDS.get(name, (0,))]


def build(name, seed):
    """(problem dict, facts): facts names the classes (pod indices per class) the scenario's predicate talks about"""
    return SCENARIOS[name](seed)
