"""Seeded corpus of clusters whose owned existing nodes carry more than 64 distinct taint sets (DESIGN.md §3, taint sets
beyond the word). Every pool (provisioner) has a `dedicated` taint of its own, so the templates alone hold up to 64 sets;
existing nodes add sets no template has: cordoned nodes, nodes launched before their pool's taint changed, device taints,
PreferNoSchedule maintenance taints, nodes of retired pools. Those sets get ids of 64 and above.

 * many(n, seed): n pools (17 to 64), NoSchedule / PreferNoSchedule / NoExecute effects, pods with Equal tolerations for
   their own team, key-only Exists tolerations, one empty-key Exists toleration, none at all; deployments of identical
   plain pods that fill existing nodes on both sides of id 64, a zone spread and a hostname anti-affinity;
 * cluster(seed): owned candidate nodes of 64 pools for the consolidation session, and after(seed) the same cluster a
   little later (nodes cordoned and uncordoned, a new pending pod), for validation;
 * tolerates / node_taints / template_sets: the reference's rules restated, for checking placements.
"""
import copy
import random

import fixtures as fx
from fixtures import HOSTNAME, ZONE, ZONES

CORDON = {"key": "node.kubernetes.io/unschedulable", "effect": "NoSchedule"}
NOT_READY = {"key": "node.kubernetes.io/not-ready", "effect": "NoSchedule"}
MAINTENANCE = {"key": "example.com/maintenance", "value": "soon", "effect": "PreferNoSchedule"}
AGENT = {"key": "example.com/agent-not-ready", "effect": "NoSchedule"}
DEVICES = ("nvidia.com/gpu", "example.com/fpga")


def _effect(i):
    return "PreferNoSchedule" if i % 7 == 3 else "NoExecute" if i % 7 == 5 else "NoSchedule"


def pool_taint(i):
    return {"key": "dedicated", "value": f"team-{i:02d}", "effect": _effect(i)}


def pools(n, rng):
    out = []
    for i in range(n):
        pr = fx.provisioner(f"pool-{i:02d}", weight=rng.choice([0, 10, 10, 50]), taints=[pool_taint(i)])
        if i % 9 == 4:
            pr["startupTaints"] = [AGENT]
        out.append(pr)
    return out


def _variants(i):
    """state taints of the nodes of pool i (the first is the pool's own set), then the raw Spec.Taints to give the node"""
    own = pool_taint(i)
    stale = dict(own, value=f"team-{i:02d}-old")
    dev = {"key": DEVICES[i % 2], "value": "present", "effect": "NoSchedule"}
    return [
        [own],
        [own, CORDON],
        [stale],
        [own, dev],
        [own, MAINTENANCE],
        [own, dev, CORDON],
        [stale, CORDON],
        [own, dict(dev, value="absent")],
        [own, MAINTENANCE, CORDON],
    ]


def _bound(name, rng, n):
    tol = rng.choice([[{"operator": "Exists"}], [{"key": "dedicated", "operator": "Exists"}]])
    return [fx.pod({"cpu": "500m", "memory": "512Mi"}, labels={"app": "bound"}, nodeName=name, tolerations=tol) for _ in range(n)]


def _node(name, i, taints, rng, pool=None, initialized=True):
    it = rng.choice(["fake-it-7", "fake-it-11", "fake-it-15"])
    cpu = int(it.split("-")[-1]) + 1
    alloc = {"cpu": f"{cpu * 1000 - 100}m", "memory": f"{cpu * 2 - 1}Gi", "pods": str(cpu * 10)}
    of = rng.choice([("on-demand", ZONES[0]), ("on-demand", ZONES[1]), ("on-demand", ZONES[2]), ("spot", ZONES[0]), ("spot", ZONES[1])])
    return fx.state_node(name, it, zone=of[1], capacity_type=of[0], provisioner_name=pool or f"pool-{i:02d}", allocatable=alloc,
                         capacity=dict(alloc), pods_=_bound(name, rng, rng.choice([0, 1, 2])), taints=copy.deepcopy(taints),
                         initialized=initialized)


def nodes(n_pools, rng, per_pool, candidates=0):
    """per_pool nodes of every pool, each a different variant; a few uninitialised nodes whose startup taints and a not-ready
    node whose ephemeral taint state.Node.Taints() drops; nodes of three retired pools. Shuffled, so that node slots of
    template sets and of node-only sets alternate in slice order."""
    out = []
    for i in range(n_pools):
        vs = _variants(i)
        for k in range(per_pool):
            out.append(_node(f"n-{i:02d}-{k}", i, vs[(k + i) % len(vs)], rng))
        if i % 9 == 4:  # uninitialised: the pool's startup taint is still on the node and is ignored (state/node.go:61-78)
            out.append(_node(f"n-{i:02d}-init", i, [pool_taint(i), AGENT], rng, initialized=False))
            out[-1]["startupTaints"] = [AGENT]
        if i % 11 == 2:
            out.append(_node(f"n-{i:02d}-nr", i, [pool_taint(i), NOT_READY], rng))
    for r in range(3):
        out.append(_node(f"n-retired-{r}", 0, [{"key": "dedicated", "value": f"retired-{r}", "effect": "NoSchedule"}] if r else [], rng,
                         pool=f"retired-{r}"))
    rng.shuffle(out)
    for k in range(candidates):
        n = out[k]
        n.update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return out


def _pods(n, requests, **kw):
    return [fx.pod(dict(requests), **kw) for _ in range(n)]


def workload(n_pools, rng, scale=1):
    pods = []
    # plain deployments: existing_run over every node, then over the dedicated-only ones
    pods += _pods(60 * scale, {"cpu": "1", "memory": "1Gi"}, labels={"app": "all"}, tolerations=[{"operator": "Exists"}])
    pods += _pods(40 * scale, {"cpu": "500m", "memory": "256Mi"}, labels={"app": "ded"}, tolerations=[{"key": "dedicated", "operator": "Exists"}])
    for t in rng.sample(range(n_pools), min(n_pools, 8)):
        eff = rng.choice([_effect(t), ""])
        tol = {"key": "dedicated", "operator": "Equal", "value": f"team-{t:02d}"}
        if eff:
            tol["effect"] = eff
        pods += _pods(rng.choice([3, 6, 12]), {"cpu": rng.choice(["1", "2"]), "memory": "2Gi"}, labels={"app": f"team-{t}"}, tolerations=[tol])
    pods += _pods(6, {"cpu": "1", "memory": "1Gi"}, labels={"app": "none"})  # no toleration: PreferNoSchedule pools after Relax
    pods += _pods(4, {"cpu": "2", "memory": "1Gi"}, labels={"app": "pref"},
                  nodeAffinity={"preferred": [{"weight": 10, "terms": [{"key": ZONE, "operator": "In", "values": ["nowhere"]}]}]})
    pods += _pods(9, {"cpu": "1", "memory": "512Mi"}, labels={"app": "web"}, tolerations=[{"key": "dedicated", "operator": "Exists"}],
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "web"})])
    pods += _pods(4, {"cpu": "1", "memory": "512Mi"}, labels={"app": "db"}, tolerations=[{"operator": "Exists"}],
                  podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "db"})]})
    pods += _pods(5, {"cpu": "1"}, labels={"app": "maint"},
                  tolerations=[{"key": "dedicated", "operator": "Exists"}, {"key": "example.com/maintenance", "operator": "Exists"}])
    rng.shuffle(pods)
    return pods


def many(n, seed, per_pool=None):
    rng = random.Random(seed * 7919 + n)
    provs = pools(n, rng)
    per_pool = per_pool or max(2, -(-150 // n))
    return fx.problem(workload(n, rng), instance_types=fx.fake_instance_types(16), provisioners=provs, nodes=nodes(n, rng, per_pool))


def cluster(seed):
    """64 pools, three nodes each; 24 of them are consolidation candidates whose pods form the simulations' batches"""
    rng = random.Random(seed * 13 + 5)
    return fx.problem([], instance_types=fx.fake_instance_types(16), provisioners=pools(64, rng), nodes=nodes(64, rng, 3, candidates=24))


def after(seed):
    """cluster(seed) after the TTL: some nodes cordoned, some uncordoned, a new pending pod"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 99)
    a["pods"] = _pods(2, {"cpu": "1", "memory": "1Gi"}, labels={"app": "late"}, tolerations=[{"key": "dedicated", "operator": "Exists"}])
    for n in rng.sample(a["nodes"], 12):
        if CORDON in n["taints"]:
            n["taints"] = [t for t in n["taints"] if t != CORDON]
        else:
            n["taints"] = n["taints"] + [CORDON]
    return a


def corpus():
    """[(name, problem dict)]: every problem has more than 64 distinct taint sets"""
    out = []
    for n in (17, 40, 64):
        out.append((f"t{n}-0", many(n, 0)))
    out.append(("t64-1", many(64, 1, per_pool=2)))
    out.append(("t24-0", many(24, 0)))
    return out


# ---------------------------------------------------------------- the reference's rules, restated
def _tolerates_taint(t, taint):  # k8s.io/api core/v1 Toleration.ToleratesTaint
    if t.get("effect") and t["effect"] != taint.get("effect", ""):
        return False
    if t.get("key") and t["key"] != taint.get("key", ""):
        return False
    op = t.get("operator", "")
    if op in ("", "Equal"):
        return t.get("value", "") == taint.get("value", "")
    return op == "Exists"


def tolerates(taints, tolerations):
    """Taints.Tolerates (taints.go:28-40): every taint is tolerated by some toleration"""
    return all(any(_tolerates_taint(t, taint) for t in tolerations) for taint in taints)


def _key(t):
    return (t.get("key", ""), t.get("value", ""), t.get("effect", ""))


def node_taints(node):
    """state.Node.Taints() (state/node.go:61-78): Spec.Taints without the ephemeral ones, and without the startup taints of an
    owned node that is not initialised yet"""
    labels = node.get("labels", {})
    eph = [NOT_READY, {"key": "node.kubernetes.io/unreachable", "effect": "NoSchedule"}]
    if labels.get(fx.INITIALIZED) != "true" and labels.get(fx.PROVISIONER_NAME):
        eph = eph + node.get("startupTaints", [])
    drop = {_key(t) for t in eph}
    return [t for t in node.get("taints", []) if _key(t) not in drop]


def taint_set(taints):
    return tuple(_key(t) for t in taints)


def template_sets(prob):
    return {taint_set(pr.get("taints", [])) for pr in prob["provisioners"]}


def distinct_sets(prob):
    """taint sets of the templates and of the owned existing nodes (the encoder's id space)"""
    sets = template_sets(prob)
    sets |= {taint_set(node_taints(n)) for n in prob.get("nodes", []) if n["labels"].get(fx.PROVISIONER_NAME)}
    return sets
