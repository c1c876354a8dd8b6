"""Seeded corpus of pod classes whose requirements and topology terms touch more than 8 label keys (DESIGN.md §3, touched
keys), on a cloud-shaped catalog whose instance types carry requirements on 12 keys, and two provisioners whose labels define
the custom keys (team, tier, env, cost-center) that are not well known.

 * deployments(seed): classes naming 9-14 keys through node selector + first required term + heaviest preferred term, with
   In / NotIn / Exists / DoesNotExist and Gt / Lt on cpu, memory and generation;
 * sixteen(seed): 14 pod keys plus zone and capacity type, with a zone spread, a zone anti-affinity and a capacity-type
   spread: 16 distinct keys;
 * relaxing(seed): an 11-key class whose preferred term relaxes to 7 keys, and a 5-key class that relaxes through its second
   required term to 11 keys;
 * existing(seed): existing nodes labelled on every key, and nodes without `nvme` / `cost-center`; NotIn / DoesNotExist pods
   add those keys to such a node's requirements, and later In pods on them are judged against the grown requirements;
 * inflight(seed): classes whose new nodes hold 12+ keys when later pods of the class and of a compatible class arrive, and two
   classes that differ in one key's value;
 * memo(seed): many classes with the same keys and different values, with and without a zone spread (fresh-node memos);
 * cluster(seed) / after(seed): consolidation whose bound pods name 10-13 keys, and the cluster after the TTL;
 * nine_groups(seed) / seventeen_keys(seed): near misses that stay refused.
"""
import copy
import random

import fixtures as fx
from fixtures import ARCH, CAPACITY_TYPE, HOSTNAME, OS, PROVISIONER_NAME, ZONE, ZONES
from wide_problems import cloud_types

WELL_KNOWN = fx.WELL_KNOWN_EXTRA + ["family", "cpu", "memory", "generation", "category", "nvme"]
CUSTOM = ("team", "tier", "env", "cost-center")
TYPE_KEYS = ("family", "size", "cpu", "memory", "generation", "category", "nvme")


def types(seed):
    """wide_problems.cloud_types plus `category` (the family's letter) and `nvme`: requirements on 12 keys per type"""
    its, families = cloud_types(seed)
    for it in its:
        fam = next(r["values"][0] for r in it["requirements"] if r["key"] == "family")
        it["requirements"] += [{"key": "category", "operator": "In", "values": [fam[0]]},
                               {"key": "nvme", "operator": "In", "values": ["true" if fam.endswith("d") else "false"]}]
    return its, families


def provisioners(limits=True):
    kw = {} if limits else {"limits": None}
    return [fx.provisioner("ml", labels={"team": "ml", "tier": "gold", "env": "prod", "cost-center": "cc-1"}, **kw),
            fx.provisioner("web", weight=10, labels={"team": "web", "tier": "silver", "env": "prod"}, **kw)]


def _r(key, op, *values):
    r = {"key": key, "operator": op}
    if values:
        r["values"] = [str(v) for v in values]
    return r


def _pods(n, requests, app, selector=None, required=None, preferred=None, **kw):
    na = {}
    if required:
        na["required"] = required
    if preferred:
        na["preferred"] = [{"weight": w, "terms": t} for w, t in preferred]
    extra = dict(kw)
    if selector:
        extra["nodeSelector"] = selector
    if na:
        extra["nodeAffinity"] = na
    return [fx.pod(dict(requests), labels={"app": app}, **extra) for _ in range(n)]


def _problem(pods, its, nodes=(), limits=True):
    return fx.problem(pods, instance_types=its, provisioners=provisioners(limits), nodes=list(nodes), wellKnownLabels=WELL_KNOWN)


def _x86(families, letters="cmr"):
    return [f for f in families if f[0] in letters and not f.endswith("g")]


# ---------------------------------------------------------------- batches
def deployments(seed):
    rng = random.Random(seed)
    its, families = types(seed)
    fams = rng.sample(_x86(families), 12)
    pods = []
    # the Karpenter pod of 9 keys: arch, os, team; zone, capacity type, category, generation; family, size
    pods += _pods(rng.randint(4, 8), {"cpu": "1", "memory": "2Gi"}, "nine", selector={ARCH: "amd64", OS: "linux", "team": "ml"},
                  required=[[_r(ZONE, "In", *ZONES[:2]), _r(CAPACITY_TYPE, "In", "on-demand", "spot"), _r("category", "In", "c", "m", "r"),
                             _r("generation", "Gt", 4)]],
                  preferred=[(50, [_r("family", "In", *fams[:6]), _r("size", "In", "xlarge", "2xlarge", "4xlarge")]),
                             (10, [_r("nvme", "In", "true")])])
    # 13 keys: NotIn / Exists / DoesNotExist, Gt / Lt on cpu and memory
    pods += _pods(rng.randint(3, 6), {"cpu": "2", "memory": "4Gi"}, "thirteen", selector={OS: "linux", "tier": "silver"},
                  required=[[_r(ARCH, "In", "amd64"), _r(ZONE, "NotIn", ZONES[2]), _r(CAPACITY_TYPE, "Exists"), _r("cpu", "Gt", 1),
                             _r("cpu", "Lt", 33), _r("memory", "Gt", 4096), _r("cost-center", "DoesNotExist"), _r("env", "In", "prod")]],
                  preferred=[(70, [_r("family", "NotIn", *fams[6:12]), _r("generation", "Lt", 8), _r("size", "NotIn", "medium"),
                                   _r("category", "Exists")])])
    # 14 keys
    pods += _pods(rng.randint(4, 9), {"cpu": "500m", "memory": "1Gi"}, "fourteen",
                  selector={"team": "ml", "env": "prod", "tier": "gold", "cost-center": "cc-1"},
                  required=[[_r(ZONE, "In", *ZONES), _r(CAPACITY_TYPE, "In", "spot"), _r(ARCH, "In", "amd64"), _r(OS, "In", "linux"),
                             _r("category", "In", "c", "m"), _r("nvme", "In", "false"), _r("generation", "Gt", 3)]],
                  preferred=[(30, [_r("cpu", "Gt", 2), _r("memory", "Lt", 131072), _r("size", "Exists")])])
    # 9 keys and a zone spread (10 by the old count), with hostname anti-affinity that takes no key
    pods += _pods(rng.randint(4, 7), {"cpu": "1", "memory": "1Gi"}, "spread", selector={ARCH: "amd64", OS: "linux", "env": "prod"},
                  required=[[_r("family", "In", *fams[:8]), _r("size", "NotIn", "medium", "large"), _r("memory", "Gt", 2048),
                             _r("cpu", "Lt", 17)]],
                  preferred=[(20, [_r("generation", "Gt", 5), _r("nvme", "Exists")])],
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"})],
                  podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "spread"})]})
    pods += _pods(4, {"cpu": "250m"}, "plain")
    rng.shuffle(pods)
    return _problem(pods, its)


def _sixteen_pods(n, app, fams, requests=None):
    return _pods(n, requests or {"cpu": "1", "memory": "1Gi"}, app,
                 selector={"team": "ml", "tier": "gold", "cost-center": "cc-1", PROVISIONER_NAME: "ml"},
                 required=[[_r(ARCH, "In", "amd64"), _r(OS, "In", "linux"), _r("family", "NotIn", *fams), _r("size", "NotIn", "medium"),
                            _r("cpu", "Gt", 1), _r("memory", "Lt", 262144), _r("generation", "Gt", 3), _r("category", "In", "c", "m", "r"),
                            _r("nvme", "In", "true", "false"), _r("env", "Exists"), _r(ZONE, "In", *ZONES),
                            _r(CAPACITY_TYPE, "In", "spot", "on-demand")]],
                 topologySpreadConstraints=[fx.spread(ZONE, {"app": app}), fx.spread(CAPACITY_TYPE, {"app": app})],
                 podAntiAffinity={"required": [fx.affinity_term(ZONE, {"app": "noisy"})]})


def sixteen(seed):
    rng = random.Random(seed + 101)
    its, families = types(seed)
    fams = rng.sample(families, 5)
    noisy = [fx.pod({"cpu": "100m"}, labels={"app": "noisy"}, nodeName="noisy-0") for _ in range(2)]
    nodes = [fx.state_node("noisy-0", its[0]["name"], zone=ZONES[0], pods_=noisy, provisioner_name="ml",
                           allocatable={"cpu": "16", "memory": "64Gi", "pods": "110"})]
    pods = _sixteen_pods(rng.randint(6, 12), "sixteen", fams)
    pods += _pods(3, {"cpu": "500m"}, "noisy", selector={"team": "web"})
    rng.shuffle(pods)
    return _problem(pods, its, nodes)


def relaxing(seed):
    rng = random.Random(seed + 202)
    its, families = types(seed)
    pods = []
    # 11 keys; the preferred term names a category no type has, so the class relaxes to its 7 required keys
    pods += _pods(rng.randint(4, 8), {"cpu": "1", "memory": "2Gi"}, "down", selector={"team": "web", "tier": "silver"},
                  required=[[_r(ARCH, "In", "amd64"), _r(OS, "In", "linux"), _r(ZONE, "In", *ZONES), _r(CAPACITY_TYPE, "In", "on-demand"),
                             _r("generation", "Gt", 3)]],
                  preferred=[(80, [_r("family", "In", *rng.sample(_x86(families), 3)), _r("size", "In", "large", "xlarge"),
                                   _r("nvme", "In", "true"), _r("category", "In", "q")])],
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "down"})])
    # 5 keys; the first required term names a team no provisioner has, the second 8 more keys
    pods += _pods(rng.randint(3, 6), {"cpu": "2", "memory": "2Gi"}, "up", selector={ARCH: "amd64", OS: "linux", "env": "prod"},
                  required=[[_r("team", "In", "nobody"), _r(ZONE, "In", *ZONES)],
                            [_r("team", "In", "ml"), _r("tier", "In", "gold"), _r("cost-center", "In", "cc-1"), _r("category", "In", "m", "r"),
                             _r("generation", "Gt", 4), _r("cpu", "Gt", 1), _r("memory", "Lt", 262144), _r(CAPACITY_TYPE, "In", "spot")]],
                  topologySpreadConstraints=[fx.spread(CAPACITY_TYPE, {"app": "up"}, max_skew=2)])
    rng.shuffle(pods)
    return _problem(pods, its)


def _labels_of(it, prov_labels):
    lab = {r["key"]: r["values"][0] for r in it["requirements"] if r["key"] in TYPE_KEYS}
    lab.update(prov_labels)
    return lab


def _node(name, it, rng, prov="ml", drop=(), pods=None, **kw):
    p = next(x for x in provisioners() if x["name"] == prov)
    lab = {k: v for k, v in _labels_of(it, p["labels"]).items() if k not in drop}
    of = rng.choice([o for o in it["offerings"] if o["available"]])
    alloc = {"cpu": it["capacity"]["cpu"], "memory": it["capacity"]["memory"], "pods": it["capacity"]["pods"]}
    return fx.state_node(name, it["name"], zone=of["zone"], capacity_type=of["capacityType"], allocatable=alloc, labels=lab,
                         provisioner_name=prov, pods_=pods or [], **kw)


def _mid(its, lo=4, hi=16):
    return [it for it in its if lo <= int(it["capacity"]["cpu"]) <= hi and next(
        r["values"][0] for r in it["requirements"] if r["key"] == "category") in "cmr" and not it["name"].split(".")[0].endswith("g")]


def existing(seed):
    rng = random.Random(seed + 303)
    its, families = types(seed)
    mid = _mid(its)
    # caller order: the nodes without nvme / cost-center come first, so an In pod would take them if their grown
    # requirements were not read
    nodes = [_node(f"bare-{i}", rng.choice(mid), rng, drop=("nvme", "cost-center")) for i in range(3)]
    nodes += [_node(f"full-{i}", rng.choice(mid), rng) for i in range(5)]
    common = {ARCH: "amd64", OS: "linux", "team": "ml"}
    base = [_r(ZONE, "Exists"), _r(CAPACITY_TYPE, "Exists"), _r("category", "Exists"), _r("generation", "Gt", 2), _r("tier", "Exists"),
            _r("env", "In", "prod"), _r("cpu", "Gt", 1)]
    # larger first in the queue: they add nvme NotIn [true] and cost-center DoesNotExist to the bare nodes
    pods = _pods(rng.randint(3, 5), {"cpu": "2", "memory": "2Gi"}, "avoid", selector=common,
                 required=[base + [_r("nvme", "NotIn", "true"), _r("cost-center", "DoesNotExist")]])
    pods += _pods(rng.randint(4, 8), {"cpu": "1", "memory": "1Gi"}, "want-nvme", selector=common,
                  required=[base + [_r("nvme", "In", "true"), _r("memory", "Gt", 2048)]])
    pods += _pods(rng.randint(4, 8), {"cpu": "500m", "memory": "512Mi"}, "want-cc", selector=dict(common, **{"cost-center": "cc-1"}),
                  required=[base + [_r("nvme", "Exists"), _r("size", "Exists")]])
    pods += _pods(rng.randint(2, 4), {"cpu": "250m", "memory": "256Mi"}, "spread", selector=common,
                  required=[base + [_r("nvme", "NotIn", "true")]], topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"})])
    rng.shuffle(pods)
    return _problem(pods, its, nodes)


def inflight(seed):
    rng = random.Random(seed + 404)
    its, families = types(seed)
    sel = {ARCH: "amd64", OS: "linux", "team": "ml", "tier": "gold", "env": "prod", "cost-center": "cc-1"}
    req = [_r(ZONE, "In", *ZONES[:2]), _r(CAPACITY_TYPE, "In", "on-demand"), _r("generation", "Gt", 4), _r("cpu", "Gt", 2),
           _r("memory", "Lt", 131072), _r("nvme", "In", "false")]
    pods = []
    for cat in ("c", "m"):  # the same 13 keys, one value apart: never on one node
        pods += _pods(rng.randint(10, 20), {"cpu": "1", "memory": "1Gi"}, f"cat-{cat}", selector=sel, required=[req + [_r("category", "In", cat)]])
    # a compatible class with another request: joins the category-c nodes
    pods += _pods(rng.randint(6, 12), {"cpu": "250m", "memory": "256Mi"}, "cat-c-small", selector=sel, required=[req + [_r("category", "In", "c")]])
    # zone spread over in-flight nodes that already hold 13 keys
    pods += _pods(rng.randint(6, 12), {"cpu": "500m", "memory": "512Mi"}, "cat-c-spread", selector=sel,
                  required=[req + [_r("category", "In", "c")]], topologySpreadConstraints=[fx.spread(ZONE, {"app": "cat-c-spread"})])
    rng.shuffle(pods)
    return _problem(pods, its, limits=bool(seed % 2))


def memo(seed):
    rng = random.Random(seed + 505)
    its, families = types(seed)
    fams = rng.sample(_x86(families), 12)
    sel = {ARCH: "amd64", OS: "linux", "team": "web", "tier": "silver", "env": "prod"}
    pods = []
    for i, fam in enumerate(fams):
        size = rng.choice(["large", "xlarge", "2xlarge", "4xlarge"])
        req = [_r("family", "In", fam), _r("size", "NotIn", size), _r("generation", "Gt", 2), _r("cpu", "Lt", 65), _r("memory", "Gt", 1024),
               _r(CAPACITY_TYPE, "In", rng.choice(["spot", "on-demand"]))]
        kw = {"topologySpreadConstraints": [fx.spread(ZONE, {"app": f"m{i}"})]} if i % 2 else {}
        pods += _pods(rng.randint(2, 5), {"cpu": rng.choice(["250m", "500m", "1"]), "memory": "512Mi"}, f"m{i}", selector=sel,
                      required=[req], **kw)
    rng.shuffle(pods)
    return _problem(pods, its, limits=False)


# ---------------------------------------------------------------- consolidation
def _bound_reqs(labels, rng, n_keys):
    """a requirement list of n_keys keys that admits a node with these labels"""
    keys = rng.sample(sorted(k for k in labels if k in TYPE_KEYS + CUSTOM + (ARCH, OS, ZONE, CAPACITY_TYPE)), n_keys)
    out = []
    for k in keys:
        v = labels[k]
        op = rng.choice(["In", "NotIn", "Exists", "Gt"] if k in ("cpu", "memory", "generation") else ["In", "NotIn", "Exists"])
        if op == "In":
            out.append(_r(k, "In", v))
        elif op == "NotIn":
            out.append(_r(k, "NotIn", "none-" + k))
        elif op == "Exists":
            out.append(_r(k, "Exists"))
        else:
            out.append(_r(k, "Gt", {"cpu": 1, "memory": 1024, "generation": 2}[k]))
    return out


def cluster(seed, n_nodes=16, candidates=8):
    rng = random.Random(seed * 23 + 7)
    its, families = types(seed)
    mid = _mid(its, 2, 8)
    nodes = []
    for i in range(n_nodes):
        prov = "ml" if i % 3 else "web"
        x = f"c-{i:02d}"
        it = rng.choice(mid)
        p = next(q for q in provisioners() if q["name"] == prov)
        lab = _labels_of(it, p["labels"])
        lab.update({ARCH: "amd64", OS: "linux"})
        bound = []
        for j in range(rng.randint(1, 3)):
            app = rng.choice(["web", "spread", "batch"])
            reqs = _bound_reqs(dict(lab, **{ZONE: "z", CAPACITY_TYPE: "c"}), rng, rng.randint(10, 13))
            kw = {"topologySpreadConstraints": [fx.spread(ZONE, {"app": "spread"}, max_skew=2)]} if app == "spread" else {}
            bound.append(fx.pod({"cpu": "300m", "memory": "256Mi"}, nodeName=x, labels={"app": app}, **kw))
            bound[-1]["_reqs"] = reqs
        node = _node(x, it, rng, prov=prov, pods=bound)
        for b in bound:  # zone and capacity type are the node's own
            reqs = [r if r["key"] not in (ZONE, CAPACITY_TYPE) or r["operator"] != "In" else _r(r["key"], "In", node["labels"][r["key"]])
                    for r in b.pop("_reqs")]
            b["nodeAffinity"] = {"required": [reqs]}
        nodes.append(node)
    for k in range(candidates):
        nodes[k].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return _problem([], its, nodes)


def after(seed):
    """cluster(seed) after the TTL: a few web pods moved, and a pending many-key pod"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 99)
    for _ in range(5):
        src, dst = rng.sample(a["nodes"], 2)
        movable = [p for p in src["pods"] if p["labels"].get("app") == "web"]
        if movable:
            p = rng.choice(movable)
            src["pods"].remove(p)
            p["nodeName"] = dst["name"]
            p.pop("nodeAffinity", None)
            dst["pods"].append(p)
    a["pods"] = _pods(1, {"cpu": "200m", "memory": "128Mi"}, "spread", selector={ARCH: "amd64", OS: "linux", "team": "ml", "env": "prod"},
                      required=[[_r("tier", "Exists"), _r("cost-center", "In", "cc-1"), _r("generation", "Gt", 2), _r("cpu", "Gt", 1),
                                 _r("category", "In", "c", "m", "r"), _r("nvme", "Exists"), _r(CAPACITY_TYPE, "Exists")]],
                      topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"}, max_skew=2)])
    return a


# ---------------------------------------------------------------- near misses
def nine_groups(seed):
    """one class constrained by 9 topology groups (spreads over zone, capacity type and hostname with 9 selectors)"""
    its, _ = types(seed)
    lab = {f"k{j}": "v" for j in range(9)}
    keys = (ZONE, CAPACITY_TYPE, HOSTNAME)
    pods = [fx.pod({"cpu": "100m"}, labels=lab, nodeSelector={"team": "ml"},
                   topologySpreadConstraints=[fx.spread(keys[j % 3], {f"k{j}": "v"}) for j in range(9)]) for _ in range(3)]
    return _problem(pods, its)


def seventeen_keys(seed):
    """a pod that names the 16 keys of sixteen() and one more"""
    rng = random.Random(seed)
    its, families = types(seed)
    pods = _sixteen_pods(2, "seventeen", rng.sample(families, 3))
    for p in pods:
        p["nodeSelector"]["workload-class"] = "batch"
    return _problem(pods, its)


def corpus():
    """[(name, problem dict)]: every problem the encoder and the device must take"""
    out = []
    for seed in range(2):
        out += [(f"deployments-{seed}", deployments(seed)), (f"sixteen-{seed}", sixteen(seed)), (f"relaxing-{seed}", relaxing(seed)),
                (f"existing-{seed}", existing(seed)), (f"inflight-{seed}", inflight(seed)), (f"memo-{seed}", memo(seed))]
    out += [("cluster-0", cluster(0)), ("after-0", after(0))]
    return out
