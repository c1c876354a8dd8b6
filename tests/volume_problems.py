"""Seeded corpus of clusters and batches whose pods mount more than 64 volume claims that the present sharing rule would track
(DESIGN.md §3, volume claims beyond the word). Two drivers have node limits: EBS and a GCE PD driver; a third (EFS) has none.

 * statefulsets(n_nodes, per_node, seed): every node runs StatefulSet pods that each mount claims of their own (EBS limit 25,
   PD limit 39 on some nodes); some nodes are consolidation candidates. Nothing is shared, so no claim is tracked;
 * shared(n_nodes, per_node, n_deploy, seed): the same, plus deployments whose two replicas on different nodes share one
   claim: more than 64 claims that a candidate's pod mounts are tracked;
 * after(prob, seed): a cluster after the TTL: pods moved between nodes, a claim re-attached to a new pod on another node,
   and a new pending pod that mounts a claim a bound pod holds;
 * replicas(n_claims, seed): a Solve batch of deployments whose replicas share one RWO claim each, next to bound pods;
 * rwx(seed): PD claims mounted by batch pods and by bound pods on several nodes;
 * bound_only(seed): claims that only bound pods share, and a batch of StatefulSet-style pods: nothing is tracked;
 * traps(seed): a pod that mounts one claim twice, claims of an unlimited driver and with no driver, a class whose tracked
   claims all have ids from 64 on, two deployments that differ in one claim beyond 64, a node already over its limit,
   limit 0, and a node without a limit for a driver another node limits;
 * boundary(kind): 64 tracked ("fit64"), 65 ("one65"), 128 ("edge128"), 129 ("edge129"), and 65 by the present rule but
   64 after the rule ("narrow65");
 * tracked_claims / volume_violations: the encoder's rule and VolumeUsage's limit check restated on the problem's strings.
"""
import copy
import random

import fixtures as fx
from fixtures import ZONES

EBS, PD, EFS = "ebs.csi.aws.com", "pd.csi.storage.gke.io", "efs.csi.aws.com"


def vol(driver, claim):
    return {"driver": driver, "pvc": claim}


def _node(name, rng, pods, limits, **kw):
    it = rng.choice(["fake-it-7", "fake-it-11", "fake-it-15"])
    cpu = int(it.split("-")[-1]) + 1
    alloc = {"cpu": f"{cpu * 1000 - 100}m", "memory": f"{cpu * 2 - 1}Gi", "pods": str(cpu * 10)}
    zone = rng.choice(ZONES)
    ct = "on-demand" if zone == ZONES[2] else rng.choice(["on-demand", "spot"])  # the fake types offer no spot in zone 3
    return fx.state_node(name, it, zone=zone, capacity_type=ct, allocatable=alloc,
                         capacity=dict(alloc, cpu=f"{cpu}"), pods_=pods, volumeLimits=limits, **kw)


def _bound(node, app, volumes, cpu="250m", **kw):
    return fx.pod({"cpu": cpu, "memory": "256Mi"}, nodeName=node, labels={"app": app}, volumes=list(volumes), **kw)


def _pods(n, volumes_of, cpu="250m", **kw):
    return [fx.pod({"cpu": cpu, "memory": "256Mi"}, volumes=list(volumes_of(i)), **kw) for i in range(n)]


def _problem(pods, nodes):
    return fx.problem(pods, instance_types=fx.fake_instance_types(16), nodes=nodes)


def _limits(i):
    return {EBS: 25, PD: 39} if i % 3 == 0 else {EBS: 25}


def _mark(nodes, rng, k):
    for i in range(k):
        nodes[i].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(i))


# ---------------------------------------------------------------- consolidation clusters
def statefulsets(n_nodes, per_node, seed, candidates=None):
    """StatefulSet pods with one or two claims of their own on every node; `candidates` (default: every node) are marked"""
    rng = random.Random(seed * 13 + n_nodes)
    nodes = []
    for i in range(n_nodes):
        name = f"s-{i:03d}"
        bound = []
        for k in range(per_node):
            vs = [vol(EBS, f"db/data-{i}-{k}")]
            if k % 2 == 1 and i % 3 == 0:
                vs.append(vol(PD, f"db/wal-{i}-{k}"))
            bound.append(_bound(name, "db", vs, cpu=rng.choice(["250m", "500m"])))
        nodes.append(_node(name, rng, bound, _limits(i)))
    _mark(nodes, rng, n_nodes if candidates is None else candidates)
    return _problem([], nodes)


def shared(n_nodes, per_node, n_deploy, seed, candidates=None):
    """statefulsets() plus n_deploy deployments of two replicas on different nodes that share one EBS claim"""
    prob = statefulsets(n_nodes, per_node, seed, candidates)
    rng = random.Random(seed * 29 + n_deploy)
    nodes = prob["nodes"]
    for d in range(n_deploy):
        for n in rng.sample(nodes, 2):
            n["pods"].append(_bound(n["name"], f"web-{d}", [vol(EBS, f"web/cache-{d:03d}")], cpu="100m"))
    return prob


def after(prob, seed):
    """the cluster after the TTL: pods moved, a claim re-attached to a new pod elsewhere, and a new pending pod that mounts a
    claim a bound pod holds"""
    a = copy.deepcopy(prob)
    rng = random.Random(seed + 77)
    nodes = a["nodes"]
    for _ in range(8):
        src, dst = rng.sample(nodes, 2)
        if not src["pods"]:
            continue
        p = rng.choice(src["pods"])
        src["pods"].remove(p)
        p["nodeName"] = dst["name"]
        dst["pods"].append(p)
    src, dst = rng.sample([n for n in nodes if n["pods"]], 2)
    old = src["pods"].pop()
    dst["pods"].append(_bound(dst["name"], "db", old.get("volumes", []), cpu="250m"))
    holder = rng.choice([p for n in nodes for p in n["pods"] if p.get("volumes")])
    a["pods"] = [fx.pod({"cpu": "100m", "memory": "128Mi"}, labels={"app": "late"}, volumes=[dict(holder["volumes"][0])])]
    return a


# ---------------------------------------------------------------- Solve batches on existing nodes
def _plain_nodes(n_nodes, rng, bound_of=lambda name, i: []):
    nodes = []
    for i in range(n_nodes):
        name = f"e-{i:02d}"
        limits = {EBS: rng.choice([4, 8, 25])}
        if i % 4 == 0:
            limits[PD] = rng.choice([3, 39])
        nodes.append(_node(name, rng, bound_of(name, i), limits))
    return nodes


def replicas(n_claims, seed, n_nodes=40):
    """n_claims deployments of 2-4 replicas that share one RWO claim, some with a private claim too; bound pods hold a few
    of the claims and some private ones"""
    rng = random.Random(seed * 7 + n_claims)
    held = rng.sample(range(n_claims), n_claims // 6)
    nodes = _plain_nodes(n_nodes, rng, lambda name, i: [_bound(name, "old", [vol(EBS, f"app/claim-{c:03d}")]) for c in held[i::n_nodes]] +
                         [_bound(name, "sts", [vol(EBS, f"sts/own-{i}-{k}")]) for k in range(rng.choice([0, 3, 6]))])
    pods = []
    for d in range(n_claims):
        extra = (lambda i, d=d: [vol(EBS, f"app/scratch-{d}-{i}")]) if d % 5 == 0 else (lambda i: [])
        pods += _pods(rng.randint(2, 4), lambda i, d=d, extra=extra: [vol(EBS, f"app/claim-{d:03d}")] + extra(i),
                      cpu=rng.choice(["100m", "250m"]), labels={"app": f"dep-{d}"})
    pods += _pods(20, lambda i: [], labels={"app": "plain"})
    rng.shuffle(pods)
    return _problem(pods, nodes)


def rwx(seed, n_claims=90, n_nodes=30):
    """PD RWX claims that batch pods and bound pods on several nodes mount"""
    rng = random.Random(seed + 500)
    nodes = _plain_nodes(n_nodes, rng, lambda name, i: [_bound(name, "reader", [vol(PD, f"shared/rwx-{c:03d}")])
                                                         for c in rng.sample(range(n_claims), 3)])
    for n in nodes:
        n["volumeLimits"][PD] = rng.choice([2, 5, 39])
    pods = _pods(n_claims, lambda i: [vol(PD, f"shared/rwx-{i:03d}")], labels={"app": "writer"})
    pods += _pods(n_claims // 3, lambda i: [vol(PD, f"shared/rwx-{i:03d}"), vol(EBS, f"own/x-{i}")], labels={"app": "both"})
    rng.shuffle(pods)
    return _problem(pods, nodes)


def bound_only(seed, n_claims=80, n_nodes=30):
    """claims that only bound pods share (two bound pods each), and a batch of pods with claims of their own"""
    rng = random.Random(seed + 900)

    def bound_of(name, i):
        return [_bound(name, "pair", [vol(EBS, f"pair/c-{c:03d}")]) for c in range(n_claims) if c % n_nodes == i or (c * 7) % n_nodes == i]
    nodes = _plain_nodes(n_nodes, rng, bound_of)
    pods = _pods(60, lambda i: [vol(EBS, f"sts/new-{i}")], labels={"app": "sts"})
    pods += _pods(10, lambda i: [], labels={"app": "plain"})
    return _problem(pods, nodes)


# ---------------------------------------------------------------- traps
def traps(seed):
    rng = random.Random(seed + 4242)
    nodes = [_node("over", rng, [_bound("over", "full", [vol(EBS, f"full/o-{k}") for k in range(30)])], {EBS: 25}),
             _node("zero", rng, [], {EBS: 0, PD: 39}),
             _node("pd-only", rng, [], {PD: 2})]                       # no EBS limit, while the others have one
    nodes += _plain_nodes(12, rng)
    pods = []
    for d in range(64):  # ids 0-63: claims "a/..." sort before "z/..."
        pods += _pods(2, lambda i, d=d: [vol(EBS, f"a/c-{d:02d}")], cpu="100m", labels={"app": f"a-{d}"})
    pods += _pods(3, lambda i: [vol(EBS, "z/high-only")], cpu="100m", labels={"app": "high"})    # tracked id >= 64, nothing private
    pods += _pods(2, lambda i: [vol(EBS, "a/c-00"), vol(EBS, "z/twin-1")], cpu="100m", labels={"app": "twin"})
    pods += _pods(2, lambda i: [vol(EBS, "a/c-00"), vol(EBS, "z/twin-2")], cpu="100m", labels={"app": "twin"})
    pods += _pods(2, lambda i: [vol(EBS, f"dup/d-{i}"), vol(EBS, f"dup/d-{i}")], labels={"app": "twice"})  # one claim twice
    pods += _pods(3, lambda i: [vol(EFS, "efs/home"), vol("", f"nfs/n-{i}")], labels={"app": "unlimited"})
    pods += _pods(4, lambda i: [vol(PD, f"pd/p-{i}"), vol(PD, "pd/common")], labels={"app": "pd"})
    pods += _pods(6, lambda i: [], labels={"app": "plain"})
    return _problem(pods, nodes)


# ---------------------------------------------------------------- boundaries
def boundary(kind):
    """n deployments of two replicas that share one claim each; "narrow65" adds one claim that two bound pods share"""
    n = {"fit64": 64, "one65": 65, "edge128": 128, "edge129": 129, "narrow65": 64}[kind]
    rng = random.Random(n * 3 + len(kind))
    bound = (lambda name, i: [_bound(name, "pair", [vol(EBS, "pair/only-bound")])] if i < 2 else []) if kind == "narrow65" else (lambda name, i: [])
    nodes = _plain_nodes(20, rng, bound)
    pods = []
    for d in range(n):
        pods += _pods(2, lambda i, d=d: [vol(EBS, f"b/claim-{d:03d}")], cpu="100m", labels={"app": f"b-{d}"})
    return _problem(pods, nodes)


def corpus():
    """Solve problems: [(name, problem dict, expects a table)]"""
    return [("replicas-65", replicas(65, 0), True), ("replicas-150", replicas(150, 1), True), ("replicas-300", replicas(300, 2), True),
            ("rwx", rwx(0), True), ("bound-only", bound_only(0), False), ("traps", traps(0), True),
            ("fit64", boundary("fit64"), False), ("one65", boundary("one65"), True), ("edge128", boundary("edge128"), True),
            ("edge129", boundary("edge129"), True), ("narrow65", boundary("narrow65"), False)]


def clusters():
    """consolidation clusters: [(name, problem dict, expects a table in the superset encoding)]"""
    return [("sts-60x3", statefulsets(60, 3, 0), False), ("sts-100x1", statefulsets(100, 1, 1), False),
            ("sts-200x1", statefulsets(200, 1, 2, candidates=120), False),
            ("shared-60x3", shared(60, 3, 120, 0), True), ("shared-100x1", shared(100, 1, 160, 1), True)]


# ---------------------------------------------------------------- the reference's rules, restated
def _claims(p, limited):
    return {(v["driver"], v["pvc"]) for v in p.get("volumes", []) if v["driver"] and v["driver"] in limited}


def _reschedulable(p):
    return not p.get("isDaemonSet") and not p.get("terminal") and not p.get("terminating")


def _mounts(prob, candidates, superset):
    """per limited (driver, claim): how often the batch and the pods bound to the nodes that stay mount it (a candidate's pod
    twice in the superset form), which pods (by object) mount it, and whether a pod of the batch does"""
    cand = set(candidates)
    nodes = prob["nodes"]
    state = [n for i, n in enumerate(nodes) if (superset or i not in cand) and not n.get("markedForDeletion")]
    limited = {d for n in state for d in (n.get("volumeLimits") or {})}
    batch = list(prob["pods"]) + [p for i in candidates for p in nodes[i]["pods"] if _reschedulable(p)]
    batch += [p for i, n in enumerate(nodes) if i not in cand and n.get("markedForDeletion") for p in n["pods"] if _reschedulable(p)]
    refs, holders, in_batch = {}, {}, set()
    for p, is_batch in [(p, True) for p in batch] + [(p, False) for n in state for p in n["pods"]]:
        for c in _claims(p, limited):
            refs[c] = refs.get(c, 0) + 1
            holders.setdefault(c, set()).add(id(p))
            if is_batch:
                in_batch.add(c)
    return refs, holders, in_batch


def shared_count(prob, candidates=(), superset=False):
    """claims the sharing rule alone would track (mounted more than once)"""
    return sum(r > 1 for r in _mounts(prob, candidates, superset)[0].values())


def tracked_claims(prob, candidates=(), superset=False):
    """the tracked (driver, claim) pairs in id order: claims mounted more than once; with more than 64 such claims, only those
    two different pods mount, one of them a pod of the batch"""
    refs, holders, in_batch = _mounts(prob, candidates, superset)
    if sum(r > 1 for r in refs.values()) <= 64:
        return sorted(c for c, r in refs.items() if r > 1)
    return sorted(c for c in refs if len(holders[c]) > 1 and c in in_batch)


def volume_violations(prob, res):
    """existing nodes of a Solve result that received a pod while some limited driver's distinct claims of their bound and
    placed pods pass the node's limit (a node that was already over a limit receives no pod)"""
    bad = []
    for e in res["existing"]:
        node = prob["nodes"][e["node"]]
        mounted = node["pods"] + [prob["pods"][i] for i in e["pods"]]
        for d, lim in (node.get("volumeLimits") or {}).items():
            claims = {v["pvc"] for p in mounted for v in p.get("volumes", []) if v["driver"] == d}
            if e["pods"] and len(claims) > lim:
                bad.append((node["name"], d, len(claims), lim))
    return bad
