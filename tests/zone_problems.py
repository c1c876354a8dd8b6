"""Seeded problems whose catalogs offer instance types in more zones or capacity types than the ct*16 + zone offering word
holds (DESIGN.md §3, offering slots): a region's availability zones plus Local Zones, capacity-type values that only a pod
names, and the boundaries of the dense slot numbering (16 zones / 4 capacity types, 17 zones, 64 and 66 pairs, 5
capacity types).

Local Zone names (us-east-1-bos-1a) sort before the AZ names (us-east-1a), and zone ids follow string order, so the AZs get
the high ids. Local Zones offer few instance types, mostly on-demand, and some of their offerings are unavailable."""
import copy
import random

import fixtures as fx
from fixtures import CAPACITY_TYPE, ZONE
from run_problems import Runs, unlimited, zonal_types, zone_names, zone_spread, SMALL

REGION = "us-east-1"
AZS = [f"{REGION}{c}" for c in "abcdef"]
LOCAL_CITIES = ["atl", "bos", "chi", "dfw", "den", "hou", "iah", "kc", "las", "lax", "mci", "mia", "msp", "nyc", "phl", "phx",
                "pdx", "sea", "slc", "sfo", "stl", "tpa", "aus", "bna", "clt", "cmh"]
SIZES = [(2, 4), (4, 16), (8, 32), (16, 64)]


def local_zones(n):
    return [f"{REGION}-{LOCAL_CITIES[i]}-1a" for i in range(n)]


def catalog(rng, n_local, cts=("on-demand", "spot")):
    """AZ types offered in every AZ and capacity type (on-demand dearest), and 2 small types also offered in the Local
    Zones: on-demand everywhere, spot in a few, and an unavailable offering here and there"""
    lzs = local_zones(n_local)
    its = []
    for cpu, mem in SIZES:
        res = {"cpu": str(cpu), "memory": f"{mem}Gi", "pods": "110"}
        price = fx.price_from_resources(res)
        offers = [{"capacityType": ct, "zone": z, "price": round(price * (1.0 if ct == "on-demand" else 0.5 + 0.1 * i), 6), "available": True}
                  for z in AZS for i, ct in enumerate(cts)]
        if (cpu, mem) in SIZES[:2]:
            for j, z in enumerate(lzs):
                offers.append({"capacityType": "on-demand", "zone": z, "price": round(price * (1.2 + 0.01 * j), 6),
                               "available": rng.random() > 0.1})
                if j % 5 == 0 and "spot" in cts:
                    offers.append({"capacityType": "spot", "zone": z, "price": round(price * 0.7, 6), "available": True})
        its.append(fx.instance_type(f"m{cpu}-{mem}g", res, offerings=offers, oses=("linux",)))
    return its, lzs


def _problem(pods, its, provisioners=None, **kw):
    return fx.problem(pods, instance_types=its, provisioners=provisioners or [unlimited()], **kw)


def _nz(seed):
    return 11 + (seed * 7) % 16  # 17-32 zones with the 6 AZs


def _cts(seed):
    return ("on-demand", "spot", "reserved") if seed % 2 else ("on-demand", "spot")


# ---------------------------------------------------------------- scenarios
def local_pinned(seed):
    """pods pinned to one Local Zone (selector and required affinity), plain pods, a daemonset"""
    rng = random.Random(seed * 31 + 1)
    its, lzs = catalog(rng, _nz(seed), _cts(seed))
    r = Runs(f"lp{seed}")
    r.run("plain", 33, {"cpu": "1", "memory": "1Gi"}, labels={"app": "plain"})
    r.run("bos", 12, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "bos"}, nodeSelector={ZONE: lzs[1]})
    r.run("lz", 9, {"cpu": "1", "memory": "2Gi"}, labels={"app": "lz"},
          nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": [lzs[-1]]}]]})
    r.run("big-lz", 3, {"cpu": "12", "memory": "40Gi"}, labels={"app": "big-lz"}, nodeSelector={ZONE: lzs[0]})  # no type fits there
    ds = [fx.pod({"cpu": "100m", "memory": "64Mi"}, name="ds-0", uid="ds-0")]
    return _problem(r.pods, its, daemonSetPods=ds)


def spread_azs(seed):
    """zone spread over the AZs a provisioner allows, and a capacity-type spread"""
    rng = random.Random(seed * 31 + 2)
    its, _ = catalog(rng, _nz(seed), _cts(seed))
    r = Runs(f"sa{seed}")
    r.run("web", 129, {"cpu": "500m", "memory": "512Mi"}, **zone_spread("web"))
    r.run("ct", 33, SMALL, labels={"app": "ct"}, topologySpreadConstraints=[fx.spread(CAPACITY_TYPE, {"app": "ct"})])
    prov = unlimited(requirements=[{"key": ZONE, "operator": "In", "values": AZS}])
    return _problem(r.pods, its, [prov])


def spread_all(seed):
    """zone spread over every zone, Local Zones included, and zone anti-affinity"""
    rng = random.Random(seed * 31 + 3)
    its, _ = catalog(rng, _nz(seed), _cts(seed))
    r = Runs(f"sz{seed}")
    r.run("web", 128, SMALL, **zone_spread("web", skew=1 + seed % 2))
    r.run("solo", 40, {"cpu": "1", "memory": "1Gi"}, labels={"app": "solo"},
          podAntiAffinity={"required": [fx.affinity_term(ZONE, {"app": "solo"})]})
    return _problem(r.pods, its)


def not_in_local(seed):
    """NotIn lists of Local Zones, and a preferred Local-Zone affinity that has to relax"""
    rng = random.Random(seed * 31 + 4)
    its, lzs = catalog(rng, _nz(seed), _cts(seed))
    r = Runs(f"ni{seed}")
    r.run("no-lz", 31, {"cpu": "1", "memory": "1Gi"}, labels={"app": "no-lz"},
          nodeAffinity={"required": [[{"key": ZONE, "operator": "NotIn", "values": lzs[: len(lzs) // 2]}]]})
    r.run("prefer", 20, {"cpu": "6", "memory": "20Gi"}, labels={"app": "prefer"},  # only AZ types fit
          nodeAffinity={"preferred": [{"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": [lzs[2]]}]}]})
    r.run("prefer-ok", 10, SMALL, labels={"app": "prefer-ok"},
          nodeAffinity={"preferred": [{"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": [lzs[3]]}]}]})
    return _problem(r.pods, its)


def existing_local(seed):
    """existing nodes in Local Zones and AZs take pods first"""
    rng = random.Random(seed * 31 + 5)
    its, lzs = catalog(rng, _nz(seed), _cts(seed))
    nodes = [fx.state_node(f"lz-{i}", its[0]["name"], zone=lzs[i % len(lzs)], capacity_type="on-demand",
                           allocatable={"cpu": "2", "memory": "4Gi", "pods": "110"}) for i in range(6)]
    nodes += [fx.state_node(f"az-{i}", its[1]["name"], zone=AZS[i], capacity_type="spot",
                            allocatable={"cpu": "4", "memory": "16Gi", "pods": "110"}) for i in range(3)]
    r = Runs(f"ex{seed}")
    r.run("any", 40, {"cpu": "700m", "memory": "1Gi"}, labels={"app": "any"})
    r.run("lz", 6, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "lz"}, nodeSelector={ZONE: lzs[1]})
    return _problem(r.pods, its, nodes=nodes)


def ct_typo(with_second=True):
    """the default fake catalog; one pod selects capacity type `Spot` (a typo) and one requires In [capacity-block,
    reserved]: spot gets dictionary id 4"""
    pods = [fx.pod({"cpu": "1", "memory": "512Mi"}, name=f"ok-{i}", uid=f"ok-{i}") for i in range(5)]
    pods.append(fx.pod({"cpu": "1"}, name="typo", uid="typo", nodeSelector={CAPACITY_TYPE: "Spot"}))
    if with_second:
        pods.append(fx.pod({"cpu": "1"}, name="other", uid="other",
                           nodeAffinity={"required": [[{"key": CAPACITY_TYPE, "operator": "In", "values": ["capacity-block", "reserved"]}]]}))
    return fx.problem(pods)


def pod_named_zone(seed):
    """16 offered zones and a zone only one pod names, sorting first: the last offered zone gets id 16"""
    zs = zone_names(16, "eu-west")
    its = zonal_types(zs, [(2, 4), (8, 32)])
    r = Runs(f"pz{seed}")
    r.run("last", 5, SMALL, labels={"app": "last"}, nodeSelector={ZONE: zs[-1]})
    r.run("nowhere", 2, SMALL, labels={"app": "nowhere"}, nodeSelector={ZONE: "aa-nowhere-1"})
    r.run("spread", 33, SMALL, **zone_spread("spread"))
    return _problem(r.pods, its)


def zonal(nz, n_pods=11, select_last=True, cts=None):
    """zonal_types offered in nz zones; pods spread and one pod selecting the last zone"""
    zs = zone_names(nz, "ap-east")
    its = zonal_types(zs, [(2, 4), (8, 32)])
    if cts:
        for it in its:
            base = [o for o in it["offerings"] if o["capacityType"] == "on-demand"]
            it["offerings"] = [dict(o, capacityType=ct, price=round(o["price"] * (1 - 0.05 * i), 6)) for o in base for i, ct in enumerate(cts)]
            for q in it["requirements"]:
                if q["key"] == CAPACITY_TYPE:
                    q["values"] = sorted(cts)
    r = Runs(f"zn{nz}")
    r.run("a", n_pods - 1, {"cpu": "1", "memory": "1Gi"}, labels={"app": "a"})
    if select_last:
        r.run("last", 1, SMALL, labels={"app": "last"}, nodeSelector={ZONE: zs[-1]})
    # a pod that names every capacity type: the key is then a mask key with one value per capacity type
    r.run("named", 1, SMALL, labels={"app": "named"},
          nodeAffinity={"required": [[{"key": CAPACITY_TYPE, "operator": "In", "values": list(cts or ("on-demand", "spot"))}]]})
    return _problem(r.pods, its)


def cluster(seed):
    """a consolidation cluster over the AZs and Local Zones: candidates in both, the cheapest replacement for the Local Zone
    pods is priced in their Local Zone"""
    rng = random.Random(seed * 31 + 6)
    its, lzs = catalog(rng, _nz(seed), _cts(seed))
    nodes = []
    for i in range(12):
        local = i % 3 == 0
        zone = lzs[i % 4] if local else AZS[i % 6]
        it = its[0] if local else its[rng.randrange(len(its))]
        name = f"node-{i:03d}"
        spec = {"labels": {"app": "lz"}, "nodeSelector": {ZONE: zone}} if local else {"labels": {"app": "web"}}
        bound = [fx.pod({"cpu": "300m", "memory": "256Mi"}, name=f"{name}-{j}", uid=f"{name}-{j}", nodeName=name, **copy.deepcopy(spec))
                 for j in range(rng.choice([1, 2]))]
        nodes.append(fx.state_node(name, it["name"], zone=zone, capacity_type="on-demand" if local else rng.choice(["spot", "on-demand"]),
                                   allocatable=dict(it["capacity"]), pods_=bound, candidate=True,
                                   disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(i)))
    return _problem([], its, [fx.provisioner()], nodes=nodes)


def after(seed):
    """cluster(seed) after the TTL: a web pod moved, and a pending pod for a Local Zone"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 99)
    web = [n for n in a["nodes"] if any(p["labels"].get("app") == "web" for p in n["pods"])]
    src, dst = rng.sample(web, 2)
    p = next(p for p in src["pods"] if p["labels"].get("app") == "web")
    src["pods"].remove(p)
    p["nodeName"] = dst["name"]
    dst["pods"].append(p)
    lz = a["nodes"][0]["labels"][ZONE]
    a["pods"] = [fx.pod({"cpu": "200m", "memory": "128Mi"}, name="late", uid="late", labels={"app": "lz"}, nodeSelector={ZONE: lz})]
    return a


# ---------------------------------------------------------------- corpus and boundaries
def corpus():
    """[(name, problem dict, expects slot tables)]; the consolidation cluster (cluster / after) is apart: its batch is the
    candidates' pods"""
    out = []
    for seed in (0, 1, 2):
        for f in (local_pinned, spread_azs, spread_all, not_in_local, existing_local):
            out.append((f"{f.__name__}-{seed}", f(seed), True))
    out += [("ct-typo", ct_typo(), True), ("ct-typo-one", ct_typo(False), False), ("pod-named-zone", pod_named_zone(0), True),
            ("zones16x4", zonal(16, cts=("capacity-block", "on-demand", "reserved", "spot")), False),
            ("zones17", zonal(17), True), ("zones20", zonal(20), True), ("pairs64", zonal(32), True),
            ("cts5", zonal(3, cts=("a-ct", "b-ct", "c-ct", "on-demand", "spot")), True)]
    return out


def near_miss():
    """33 zones x 2 capacity types = 66 pairs with an available offering"""
    return zonal(33)


# ---------------------------------------------------------------- the reference's rules, restated
def pairs(prob, zone_key=True, ct_key=True):
    """(capacity type, zone) pairs of available offerings, in ascending (capacity-type, zone) string order (= dictionary id
    order: offerings name their values, so every one is a dictionary value). A key that is no mask key of the encoding
    (nothing but the catalog names it) has one value for every offering, written ''."""
    return sorted({(o["capacityType"] if ct_key else "", o["zone"] if zone_key else "")
                   for it in prob["instanceTypes"] for o in it["offerings"] if o.get("available", True)})


def has_offering(prob, node, idx):
    """node.go hasOffering: an available offering of type idx in a zone and capacity type the node's requirements admit"""
    zr, cr = node["requirements"].get(ZONE), node["requirements"].get(CAPACITY_TYPE)
    return any(o.get("available", True) and fx._req_has(zr, o["zone"]) and fx._req_has(cr, o["capacityType"])
               for o in prob["instanceTypes"][idx]["offerings"])

