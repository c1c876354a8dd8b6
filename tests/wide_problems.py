"""Seeded corpus of problems whose label keys or resource lists are wider than the device word, but whose requirements
only name a few of their values (DESIGN.md §3, value classes): the encoder keeps the named values and one representative
per class of the others, and leaves out resource names that no request and no limit reads.

 * fake(n): fake.InstanceTypes(n)-shaped catalogs (one `integer` value per type) with integer In / NotIn / Gt / Lt / Exists /
   DoesNotExist on pods, preferred terms that relax, and a provisioner bound on the same key;
 * cloud(seed): a cloud-shaped catalog of 600-800 types with `family` (~120 values), `size`, `cpu`, `memory` (~180 integers)
   and `generation`, pods selecting a family, NotIn lists of families, bounds on memory and cpu, zone / hostname spread and
   anti-affinity alongside; optionally existing nodes labelled with values no requirement names;
 * cluster(seed): a cloud catalog with owned candidate nodes, for the consolidation session;
 * extended(seed): types listing 9-12 resource names, one extended resource requested and another under a limit;
 * NEAR_MISSES: what the word still cannot hold and must still be refused.
"""
import random

import fixtures as fx
from fixtures import CAPACITY_TYPE, HOSTNAME, INSTANCE_TYPE, ZONE, ZONES


def _pods(n, requests, **kw):
    return [fx.pod(dict(requests), **kw) for _ in range(n)]


# ---------------------------------------------------------------- fake.InstanceTypes(n)
def fake(n, seed):
    rng = random.Random(seed * 1009 + n)
    its = fx.fake_instance_types(n)
    lo, hi = rng.randrange(5, 30), rng.randrange(n // 2, n)
    pods = []
    pods += _pods(rng.choice([3, 6]), {"cpu": "1", "memory": "1Gi"}, labels={"app": "lt"},
                  nodeAffinity={"required": [[{"key": "integer", "operator": "Lt", "values": [str(lo)]}]]})
    pods += _pods(rng.choice([2, 5]), {"cpu": "2"}, labels={"app": "gt"},
                  nodeAffinity={"required": [[{"key": "integer", "operator": "Gt", "values": [str(hi)]}]]})
    pods += _pods(3, {"cpu": "500m"}, labels={"app": "in"},
                  nodeAffinity={"required": [[{"key": "integer", "operator": "In", "values": [str(rng.randrange(1, n + 1)) for _ in range(2)]}]]})
    pods += _pods(3, {"cpu": "3"}, labels={"app": "notin"},
                  nodeAffinity={"required": [[{"key": "integer", "operator": "NotIn", "values": [str(v) for v in range(3, 9)]},
                                              {"key": "integer", "operator": "Lt", "values": [str(hi)]}]]})
    pods += _pods(2, {"cpu": "1"}, labels={"app": "exists"}, nodeAffinity={"required": [[{"key": "integer", "operator": "Exists", "values": []}]]})
    pods += _pods(1, {"cpu": "1"}, labels={"app": "dne"}, nodeAffinity={"required": [[{"key": "integer", "operator": "DoesNotExist", "values": []}]]})
    # preferred terms that cannot be met relax to the required ones
    pods += _pods(4, {"cpu": "1500m"}, labels={"app": "pref"},
                  nodeAffinity={"preferred": [{"weight": 50, "terms": [{"key": "integer", "operator": "In", "values": [str(n + 7)]}]},
                                              {"weight": 10, "terms": [{"key": "integer", "operator": "Gt", "values": [str(n + 3)]}]}],
                                "required": [[{"key": "integer", "operator": "Gt", "values": ["1"]}]]})
    pods += _pods(3, {"cpu": "1"}, labels={"app": "spread"}, topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"})],
                  nodeAffinity={"required": [[{"key": "integer", "operator": "Lt", "values": [str(lo)]}]]})
    rng.shuffle(pods)
    provs = [fx.provisioner(requirements=[{"key": "integer", "operator": "Gt", "values": ["1"]}]),
             fx.provisioner("second", weight=10, requirements=[{"key": "integer", "operator": "Lt", "values": [str(hi)]}])]
    return fx.problem(pods, instance_types=its, provisioners=provs[: rng.choice([1, 2])])


# ---------------------------------------------------------------- a cloud-shaped catalog
SIZES = [("medium", 1), ("large", 2), ("xlarge", 4), ("2xlarge", 8), ("4xlarge", 16), ("8xlarge", 32), ("12xlarge", 48), ("16xlarge", 64)]
RATIOS = [1024, 1536, 2048, 3072, 3840, 4096, 5120, 6144, 7680, 8192, 10240, 12288, 15616, 16384, 24576]  # MiB per vCPU


def cloud_types(seed):
    rng = random.Random(seed)
    families = []
    for letter in "cmrtxzgpi":
        for gen in range(3, 9):
            for suffix in ("", "a", "g", "i", "n", "d"):
                families.append((f"{letter}{gen}{suffix}", gen))
    rng.shuffle(families)
    families = families[:120]
    its = []
    for fam, gen in families:
        ratio = rng.choice(RATIOS) + rng.choice([0, 0, 128, 256])
        arch = "arm64" if fam.endswith("g") else "amd64"
        for size, cpu in rng.sample(SIZES, rng.choice([5, 6, 7])):
            if len(its) >= 800:
                break
            mem = cpu * ratio  # MiB
            name = f"{fam}.{size}"
            res = {"cpu": str(cpu), "memory": f"{mem}Mi", "pods": str(min(110, 8 * cpu))}
            price = fx.price_from_resources(res) * (0.9 if fam.endswith("a") else 1.0)
            offerings = [{"capacityType": ct, "zone": z, "price": price * (0.4 if ct == "spot" else 1.0), "available": rng.random() > 0.05}
                         for z in ZONES for ct in ("spot", "on-demand")]
            avail = [o for o in offerings if o["available"]]
            reqs = [{"key": INSTANCE_TYPE, "operator": "In", "values": [name]},
                    {"key": fx.ARCH, "operator": "In", "values": [arch]},
                    {"key": fx.OS, "operator": "In", "values": ["linux"]},
                    {"key": ZONE, "operator": "In", "values": sorted({o["zone"] for o in avail})},
                    {"key": CAPACITY_TYPE, "operator": "In", "values": sorted({o["capacityType"] for o in avail})},
                    {"key": "family", "operator": "In", "values": [fam]},
                    {"key": "size", "operator": "In", "values": [size]},
                    {"key": "cpu", "operator": "In", "values": [str(cpu)]},
                    {"key": "memory", "operator": "In", "values": [str(mem)]},
                    {"key": "generation", "operator": "In", "values": [str(gen)]}]
            its.append({"name": name, "requirements": reqs, "offerings": offerings, "capacity": res,
                        "overhead": {"kubeReserved": {"cpu": "100m", "memory": "100Mi"}}})
    return its, [f for f, _ in families]


def cloud(seed, existing=0):
    rng = random.Random(seed)
    its, families = cloud_types(seed)
    pick = rng.sample(families, 14)
    pods = []
    pods += _pods(rng.choice([4, 7]), {"cpu": "1", "memory": "2Gi"}, labels={"app": "web"}, nodeSelector={"family": pick[0]},
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "web"})])
    pods += _pods(rng.choice([3, 5]), {"cpu": "2", "memory": "4Gi"}, labels={"app": "db"},
                  nodeAffinity={"required": [[{"key": "family", "operator": "NotIn", "values": pick[1:11]},
                                              {"key": "memory", "operator": "Gt", "values": ["8192"]}]]},
                  podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "db"})]})
    pods += _pods(4, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "batch"},
                  nodeAffinity={"required": [[{"key": "cpu", "operator": "Lt", "values": ["16"]}, {"key": "cpu", "operator": "Gt", "values": ["2"]}]]},
                  topologySpreadConstraints=[fx.spread(HOSTNAME, {"app": "batch"}, max_skew=2)])
    pods += _pods(3, {"cpu": "4", "memory": "16Gi"}, labels={"app": "mem"},
                  nodeAffinity={"required": [[{"key": "memory", "operator": "Gt", "values": ["16384"]},
                                              {"key": "memory", "operator": "Lt", "values": ["262144"]}]],
                                "preferred": [{"weight": 40, "terms": [{"key": "family", "operator": "In", "values": [pick[11]]}]},
                                              {"weight": 20, "terms": [{"key": "size", "operator": "In", "values": ["nonexistent"]}]}]})
    pods += _pods(3, {"cpu": "1"}, labels={"app": "gen"},
                  nodeAffinity={"required": [[{"key": "generation", "operator": "In", "values": ["6", "7"]}]]})
    pods += _pods(2, {"cpu": "250m"}, labels={"app": "size"}, nodeSelector={"size": rng.choice(["xlarge", "2xlarge"])})
    pods += _pods(2, {"cpu": "1"}, labels={"app": "either"},
                  nodeAffinity={"required": [[{"key": "family", "operator": "In", "values": pick[12:14]}],
                                             [{"key": "cpu", "operator": "Gt", "values": ["32"]}]]})
    rng.shuffle(pods)
    provs = [fx.provisioner(requirements=[{"key": "memory", "operator": "Lt", "values": ["524288"]}])]
    nodes = []
    for i in range(existing):
        it = rng.choice(its)
        lab = {r["key"]: r["values"][0] for r in it["requirements"] if r["key"] in ("family", "size", "cpu", "memory", "generation")}
        of = rng.choice([o for o in it["offerings"] if o["available"]] or it["offerings"])
        bound = [fx.pod({"cpu": "500m"}, labels={"app": rng.choice(["web", "db", "other"])}, nodeName=f"node-{i}") for _ in range(rng.choice([0, 1, 2]))]
        alloc = {"cpu": it["capacity"]["cpu"], "memory": it["capacity"]["memory"], "pods": it["capacity"]["pods"]}
        nodes.append(fx.state_node(f"node-{i}", it["name"], zone=of["zone"], capacity_type=of["capacityType"], allocatable=alloc, pods_=bound,
                                   labels=lab))
    # instance-type labels the provider declares well known (as cloud providers do for family / cpu / memory)
    return fx.problem(pods, instance_types=its, provisioners=provs, nodes=nodes, wellKnownLabels=fx.WELL_KNOWN_EXTRA + ["family", "cpu", "memory", "generation"])


def cluster(seed):
    """owned candidate nodes of the cloud catalog, labelled with families / sizes / memories no requirement names; their pods
    carry a zone spread, a memory bound or hostname anti-affinity"""
    prob = cloud(seed, existing=0)
    rng = random.Random(seed * 17 + 3)
    its = prob["instanceTypes"]
    small = sorted(its, key=lambda it: min(o["price"] for o in it["offerings"]))[:200]
    nodes = []
    for i in range(24):
        it = rng.choice(small)
        lab = {r["key"]: r["values"][0] for r in it["requirements"] if r["key"] in ("family", "size", "cpu", "memory", "generation")}
        of = rng.choice([o for o in it["offerings"] if o["available"]])
        app = rng.choice(["web", "batch", "other"])
        extra = {"web": {"topologySpreadConstraints": [fx.spread(ZONE, {"app": "web"}, max_skew=3)]},
                 "batch": {"nodeAffinity": {"required": [[{"key": "memory", "operator": "Gt", "values": ["1024"]}]]}},
                 "other": {"podAntiAffinity": {"required": [fx.affinity_term(HOSTNAME, {"app": "other"})]}}}[app]
        bound = [fx.pod({"cpu": "250m", "memory": "256Mi"}, labels={"app": app}, nodeName=f"n{i}", **extra) for _ in range(rng.choice([1, 2, 3]))]
        nodes.append(fx.state_node(f"n{i}", it["name"], zone=of["zone"], capacity_type=of["capacityType"], labels=lab, pods_=bound,
                                   allocatable={"cpu": it["capacity"]["cpu"], "memory": it["capacity"]["memory"], "pods": it["capacity"]["pods"]},
                                   candidate=True, disruptionCost=float(rng.choice([0, 1, 2, 3])), creationTimestamp=float(i)))
    prob["pods"] = []  # the candidates' pods form each simulation's batch
    prob["nodes"] = nodes
    return prob


# ---------------------------------------------------------------- resource lists wider than the device word
def extended(seed):
    rng = random.Random(seed)
    extra = [f"example.com/device-{i}" for i in range(rng.choice([6, 7, 8, 9]))]  # 9-12 names with cpu, memory, pods
    its = []
    for i in range(40):
        res = {"cpu": str(rng.choice([2, 4, 8, 16])), "memory": f"{rng.choice([4, 8, 16, 32])}Gi", "pods": "20"}
        for name in extra:
            res[name] = str(rng.choice([0, 0, 1, 2, 4]))  # providers list extended resources even at zero
        its.append(fx.instance_type(f"ext-{i}", res))
    requested, limited = extra[0], extra[1]
    pods = _pods(5, {"cpu": "1", "memory": "1Gi", requested: "1"}, labels={"app": "dev"})
    pods += _pods(6, {"cpu": "2", "memory": "2Gi"}, labels={"app": "plain"})
    rng.shuffle(pods)
    provs = [fx.provisioner(limits={"cpu": "64", limited: "6"})]
    nodes = []
    if seed % 2:
        it = its[0]
        nodes.append(fx.state_node("ext-node", it["name"], allocatable=dict(it["capacity"]), capacity=dict(it["capacity"]),
                                   pods_=[fx.pod({"cpu": "1", extra[2]: "1"}, nodeName="ext-node")]))
    return fx.problem(pods, instance_types=its, provisioners=provs, nodes=nodes)


# ---------------------------------------------------------------- the corpus
def corpus():
    """[(name, problem dict, {key: thresholds on it})]: every problem the encoder must accept"""
    out = []
    for n in (64, 70, 500, 1000):
        for seed in range(2):
            out.append((f"fake{n}-{seed}", fake(n, seed)))
    for seed in range(3):
        out.append((f"cloud-{seed}", cloud(seed)))
    for seed in range(2):
        out.append((f"cloud-nodes-{seed}", cloud(10 + seed, existing=12)))
    for seed in range(2):
        out.append((f"extended-{seed}", extended(seed)))
    return out


def _near_misses():
    its, families = cloud_types(0)
    wide = fx.pod({"cpu": "1"}, nodeAffinity={"required": [[{"key": "family", "operator": "In", "values": families[:64]}]]})
    spread = fx.pod({"cpu": "1"}, labels={"app": "s"}, topologySpreadConstraints=[fx.spread("family", {"app": "s"})])
    return [("64-named-values", fx.problem([wide], instance_types=its)),
            ("spread-over-120-families", fx.problem([spread], instance_types=its))]


NEAR_MISSES = _near_misses()
