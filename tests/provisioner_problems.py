"""Seeded corpus of clusters with many provisioners (17 to 64) whose requirements and labels name label keys that no pod names
(DESIGN.md §3, template-only keys): instance category, family, size, cpu, hypervisor, GPU name, region, team, cost center...
Together with the keys pods do name they are more than 16, or `karpenter.sh/provisioner-name` has more than 63 values; the
encoder folds the template-only keys into the templates' instance-type lists instead of refusing.

 * many(n, seed): n provisioners over a cloud catalog (wide_problems.cloud_types): tied weights, taints some pods tolerate,
   labels under their own keys, In / NotIn / Exists / DoesNotExist / Gt / Lt on template-only keys (a beta key name among
   them), instance-type requirements, limits, keys both templates and pods name (arch, generation, workload), daemonsets,
   zone spread, hostname anti-affinity, preferred terms that relax; optionally existing nodes of several provisioners;
 * names_only(seed): 64 provisioners and at most 16 keys: only the 64 values of provisioner-name force the fold;
 * cluster(seed): owned candidate nodes of many provisioners for the consolidation session, and after(seed) the same
   cluster a little later, for validation;
 * NEAR_MISSES: what must still be refused.
"""
import copy
import random

import fixtures as fx
import wide_problems as wp
from fixtures import ARCH, CAPACITY_TYPE, HOSTNAME, INSTANCE_TYPE, PROVISIONER_NAME, ZONE, ZONES

REGION = "topology.kubernetes.io/region"
GPU = "example.com/gpu-name"
HYPERVISOR = "example.com/hypervisor"
CATEGORY = "example.com/instance-category"
TEMPLATE_LABELS = ("team", "cost-center", "billing-group", "example.com/tier", "env")


def catalog(seed, n=300):
    """the first n types of a cloud catalog, with a region, a hypervisor on most types and a GPU name on GPU families"""
    its, families = wp.cloud_types(seed)
    its = its[:n]
    for it in its:
        fam = it["name"].split(".")[0]
        it["requirements"].append({"key": REGION, "operator": "In", "values": ["eu-west-1"]})
        it["requirements"].append({"key": CATEGORY, "operator": "In", "values": [fam[0]]})
        if not fam.startswith("t"):
            it["requirements"].append({"key": HYPERVISOR, "operator": "In", "values": ["nitro" if fam[1] > "4" else "xen"]})
        if fam[0] in "gp":
            it["requirements"].append({"key": GPU, "operator": "In", "values": ["a10g" if fam[0] == "g" else "a100"]})
    return its, sorted({it["name"].split(".")[0] for it in its})


def _template_reqs(i, rng, families, names):
    """a few requirements on template-only keys (and sometimes on keys pods name too); over 17 provisioners every kind occurs"""
    pool = [
        lambda: {"key": "family", "operator": "In", "values": rng.sample(families, rng.choice([4, 8, 16]))},
        lambda: {"key": "family", "operator": "NotIn", "values": rng.sample(families, 6)},
        lambda: {"key": "size", "operator": "NotIn", "values": rng.sample(["medium", "large", "16xlarge", "12xlarge"], 2)},
        lambda: {"key": "cpu", "operator": "Lt", "values": [str(rng.choice([9, 17, 33]))]},
        lambda: {"key": "cpu", "operator": "Gt", "values": [str(rng.choice([1, 2, 4]))]},
        lambda: {"key": "memory", "operator": "Gt", "values": [str(rng.choice([2048, 8192]))]},
        lambda: {"key": HYPERVISOR, "operator": rng.choice(["Exists", "DoesNotExist"]), "values": []},
        lambda: {"key": HYPERVISOR, "operator": "In", "values": ["nitro"]},
        lambda: {"key": GPU, "operator": "DoesNotExist", "values": []},
        lambda: {"key": GPU, "operator": "Exists", "values": []},
        lambda: {"key": CATEGORY, "operator": "In", "values": rng.sample(list("cmrtxzgpi"), 4)},
        lambda: {"key": "failure-domain.beta.kubernetes.io/region", "operator": rng.choice(["In", "In", "NotIn"]), "values": ["eu-west-1"]},
        lambda: {"key": INSTANCE_TYPE, "operator": "NotIn", "values": rng.sample(names, 20)},
        lambda: {"key": ARCH, "operator": "In", "values": [rng.choice(["amd64", "arm64"])]},
        lambda: {"key": "generation", "operator": "Gt", "values": [str(rng.choice([3, 4, 5]))]},
        lambda: {"key": ZONE, "operator": "In", "values": rng.sample(ZONES, 2)},
        lambda: {"key": CAPACITY_TYPE, "operator": "In", "values": [rng.choice(["spot", "on-demand"])]},
    ]
    return [pool[i % len(pool)]()] + [f() for f in rng.sample(pool, rng.choice([1, 2, 3]))]


def provisioners(n, rng, families, names, name_fmt="team-{:02d}"):
    out = []
    for i in range(n):
        own = [TEMPLATE_LABELS[i % len(TEMPLATE_LABELS)]] + rng.sample(TEMPLATE_LABELS, rng.choice([0, 1, 2]))
        labels = {k: f"{k.split('/')[-1]}-{rng.randrange(4)}" for k in own}
        if rng.random() < 0.6:
            labels["workload"] = rng.choice(["web", "batch", "ml"])
        pr = fx.provisioner(name_fmt.format(i), weight=rng.choice([0, 0, 10, 10, 50]), labels=labels,
                            requirements=_template_reqs(i, rng, families, names))
        if i % 4 == 1:
            pr["taints"] = [{"key": "dedicated", "value": f"team-{i % 3}", "effect": "NoSchedule"}]
        pr["limits"] = {"cpu": str(rng.choice([24, 64, 2000]))}
        out.append(pr)
    return out


def _pods(n, requests, **kw):
    return [fx.pod(dict(requests), **kw) for _ in range(n)]


def workload(rng):
    pods = []
    pods += _pods(rng.choice([6, 9]), {"cpu": "1", "memory": "2Gi"}, labels={"app": "web"}, nodeSelector={"workload": "web"},
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "web"})])
    pods += _pods(rng.choice([3, 5]), {"cpu": "2", "memory": "4Gi"}, labels={"app": "db"},
                  podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "db"})]},
                  tolerations=[{"key": "dedicated", "operator": "Equal", "value": "team-1", "effect": "NoSchedule"}])
    pods += _pods(8, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "batch"}, nodeSelector={ARCH: "amd64"},
                  tolerations=[{"key": "dedicated", "operator": "Exists"}])
    pods += _pods(4, {"cpu": "3", "memory": "8Gi"}, labels={"app": "gen"},
                  nodeAffinity={"required": [[{"key": "generation", "operator": "In", "values": ["6", "7", "8"]}]],
                                "preferred": [{"weight": 30, "terms": [{"key": "generation", "operator": "In", "values": ["99"]}]},
                                              {"weight": 10, "terms": [{"key": "workload", "operator": "In", "values": ["ml"]}]}]})
    pods += _pods(3, {"cpu": "1"}, labels={"app": "ml"}, nodeSelector={"workload": "ml"},
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "ml"}, when="ScheduleAnyway")])
    pods += _pods(2, {"cpu": "6", "memory": "16Gi"}, labels={"app": "big"})
    rng.shuffle(pods)
    return pods


DAEMONS = [{"name": "ds-logs", "uid": "ds-logs", "requests": {"cpu": "100m", "memory": "128Mi"}},
           {"name": "ds-gpu", "uid": "ds-gpu", "requests": {"cpu": "200m"}, "nodeSelector": {ARCH: "amd64"},
            "tolerations": [{"operator": "Exists"}]}]


def _nodes(rng, its, provs, n, candidate=False):
    nodes = []
    for i in range(n):
        it = rng.choice(its)
        pr = rng.choice(provs)
        of = rng.choice([o for o in it["offerings"] if o["available"]])
        lab = {r["key"]: r["values"][0] for r in it["requirements"] if r["key"] in ("family", "size", "cpu", "generation", REGION)}
        lab.update(pr.get("labels", {}))
        app = rng.choice(["web", "db", "batch"])
        extra = {"web": {"topologySpreadConstraints": [fx.spread(ZONE, {"app": "web"})]},
                 "db": {"podAntiAffinity": {"required": [fx.affinity_term(HOSTNAME, {"app": "db"})]}},
                 "batch": {"nodeSelector": {ARCH: "amd64"}}}[app]
        bound = [fx.pod({"cpu": "250m", "memory": "256Mi"}, labels={"app": app}, nodeName=f"n{i}", **extra) for _ in range(rng.choice([1, 2]))]
        alloc = {"cpu": it["capacity"]["cpu"], "memory": it["capacity"]["memory"], "pods": it["capacity"]["pods"]}
        kw = dict(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(i)) if candidate else {}
        nodes.append(fx.state_node(f"n{i}", it["name"], zone=of["zone"], capacity_type=of["capacityType"], provisioner_name=pr["name"],
                                   allocatable=alloc, capacity=dict(alloc), pods_=bound, labels=lab, taints=pr.get("taints", []), **kw))
    return nodes


def many(n, seed, existing=0):
    rng = random.Random(seed * 7919 + n)
    its, families = catalog(seed)
    provs = provisioners(n, rng, families, [it["name"] for it in its])
    nodes = _nodes(rng, its, provs, existing)
    return fx.problem(workload(rng), instance_types=its, provisioners=provs, nodes=nodes, daemonSetPods=copy.deepcopy(DAEMONS),
                      wellKnownLabels=fx.WELL_KNOWN_EXTRA + ["family", "cpu", "generation"])


def names_only(seed):
    """64 provisioners that name no key but provisioner-name and one label; pods name zone and arch"""
    rng = random.Random(seed)
    its, _ = catalog(seed, n=120)
    provs = [fx.provisioner(f"tenant-{i:02d}", weight=rng.choice([0, 10]), labels={"team": f"t{i % 8}"},
                            limits={"cpu": str(rng.choice([16, 2000]))}) for i in range(64)]
    pods = _pods(12, {"cpu": "1"}, labels={"app": "web"}, topologySpreadConstraints=[fx.spread(ZONE, {"app": "web"})])
    pods += _pods(6, {"cpu": "2"}, labels={"app": "arm"}, nodeSelector={ARCH: "arm64"})
    rng.shuffle(pods)
    return fx.problem(pods, instance_types=its, provisioners=provs)


def cluster(seed):
    """owned candidate nodes of 40 provisioners; their pods form each simulation's batch"""
    rng = random.Random(seed * 13 + 5)
    its, families = catalog(seed, n=200)
    its_small = sorted(its, key=lambda it: min(o["price"] for o in it["offerings"]))[:120]
    provs = provisioners(40, rng, families, [it["name"] for it in its])
    for pr in provs:  # the nodes' own types must stay on offer: instance-type lists of the templates are left whole here
        pr["requirements"] = [r for r in pr["requirements"] if r["key"] != INSTANCE_TYPE]
    nodes = _nodes(rng, its_small, provs, 20, candidate=True)
    return fx.problem([], instance_types=its, provisioners=provs, nodes=nodes, daemonSetPods=copy.deepcopy(DAEMONS),
                      wellKnownLabels=fx.WELL_KNOWN_EXTRA + ["family", "cpu", "generation"])


def after(seed):
    """cluster(seed) after the TTL: a new pending pod, one node's allocatable shrunk, one node gone"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 99)
    a["pods"] = _pods(2, {"cpu": "1", "memory": "1Gi"}, labels={"app": "late"}, nodeSelector={"workload": "web"})
    n = a["nodes"][rng.randrange(len(a["nodes"]))]
    n["allocatable"] = dict(n["allocatable"], cpu="1")
    del a["nodes"][rng.randrange(len(a["nodes"]))]
    return a


def corpus():
    """[(name, problem dict)]: every problem the encoder must accept"""
    out = []
    for n in (17, 24, 40, 64):
        for seed in range(2):
            out.append((f"p{n}-{seed}", many(n, seed)))
        out.append((f"p{n}-nodes", many(n, 10 + n, existing=10)))
    for seed in range(2):
        out.append((f"names-only-{seed}", names_only(seed)))
    return out


def _near_misses():
    its, families = catalog(0)
    names = [it["name"] for it in its]
    rng = random.Random(5)
    too_many = fx.problem(workload(rng), instance_types=its, provisioners=provisioners(65, rng, families, names))
    selected = names_only(0)
    selected["pods"].append(fx.pod({"cpu": "1"}, nodeSelector={PROVISIONER_NAME: "tenant-03"}))
    # 15 keys that pods name, zone and capacity-type named only by templates, and template-only keys besides
    pods = [fx.pod({"cpu": "100m"}, nodeSelector={f"example.com/k{i}": "x"}) for i in range(15)]
    provs = [fx.provisioner("a", labels={"team": "a", "env": "prod"}, requirements=[{"key": ZONE, "operator": "In", "values": ZONES[:2]}]),
             fx.provisioner("b", requirements=[{"key": CAPACITY_TYPE, "operator": "In", "values": ["spot"]}, {"key": "family", "operator": "In", "values": families[:3]}])]
    keys17 = fx.problem(pods, instance_types=its, provisioners=provs)
    return [("65-provisioners", too_many, "more than 64 provisioners"),
            ("pods-select-provisioner-name", selected, "more than 63 distinct values"),
            ("15-pod-keys-plus-zone-and-capacity-type", keys17, "more than 16 active label keys")]


NEAR_MISSES = _near_misses()


def pod_side_keys(prob):
    """keys that pods, daemonsets, topology terms and bound pods' anti-affinity terms name (hostname and instance-type aside),
    plus zone and capacity-type when anything names them: the mask keys of a folded encoding"""
    keys, named = set(), set()
    norm = {"failure-domain.beta.kubernetes.io/zone": ZONE, "beta.kubernetes.io/arch": ARCH,
            "failure-domain.beta.kubernetes.io/region": REGION, "beta.kubernetes.io/os": fx.OS, "beta.kubernetes.io/instance-type": INSTANCE_TYPE}

    def pod(p, bound=False):
        if bound:
            for t in p.get("podAntiAffinity", {}).get("required", []):
                keys.add(t["topologyKey"])
            return
        keys.update(norm.get(k, k) for k in p.get("nodeSelector", {}))
        na = p.get("nodeAffinity") or {}
        for term in na.get("required", []):
            keys.update(norm.get(r["key"], r["key"]) for r in term)
        for t in na.get("preferred", []):
            keys.update(norm.get(r["key"], r["key"]) for r in t["terms"])
        for kind in ("podAffinity", "podAntiAffinity"):
            for t in (p.get(kind) or {}).get("required", []):
                keys.add(t["topologyKey"])
            for t in (p.get(kind) or {}).get("preferred", []):
                keys.add(t["term"]["topologyKey"])
        for t in p.get("topologySpreadConstraints", []):
            keys.add(t["topologyKey"])

    for p in prob["pods"] + prob.get("daemonSetPods", []):
        pod(p)
    for n in prob.get("nodes", []):
        for p in n.get("pods", []):
            pod(p, bound=not n.get("candidate"))
            if n.get("candidate"):
                pod(p, bound=True)
    for pr in prob["provisioners"]:
        named.update(norm.get(r["key"], r["key"]) for r in pr.get("requirements", []))
    named |= keys
    keys |= {k for k in (ZONE, CAPACITY_TYPE) if k in named}
    return keys - {HOSTNAME, INSTANCE_TYPE}


def template_keys(prob):
    norm = {"failure-domain.beta.kubernetes.io/region": REGION}
    keys = {PROVISIONER_NAME}
    for pr in prob["provisioners"]:
        keys.update(norm.get(r["key"], r["key"]) for r in pr.get("requirements", []))
        keys.update(pr.get("labels", {}))
    return keys - {HOSTNAME, INSTANCE_TYPE}
