"""Seeded corpus of pods whose kubernetes.io/hostname requirements go beyond one In / NotIn value (DESIGN.md §3, hostname
requirements). Local persistent volumes pin a pod to its node on every required term, data-locality jobs prefer a list of
hosts, and operators keep deployments off a few named nodes.

 * in_list(k, seed): 70 existing nodes, a deployment required onto k of them (among them slots 64-69, beyond the first word);
   the listed nodes fill and the rest of the pods stay unscheduled, since no new node is ever on the list;
 * not_in(n, k, seed): a deployment of n pods kept off the k nodes with the most room;
 * selector_and_affinity(seed): a node selector `a` plus affinity In [a, b] (one node), and `a` plus NotIn [a] (nothing);
 * forms(seed): Exists, DoesNotExist, Gt / Lt on a cluster whose node names are partly integers;
 * preferred(seed): Spark-like executors that prefer one of 50 host lists, with weights, and relax to unconstrained;
 * two_terms(seed): two required terms; when the first list is full, relaxation drops it and the second list applies;
 * local_pv(seed): a StatefulSet on local volumes, two hostname requirements per pod, zone spread whose node filter names the
   hostname, and hostname anti-affinity;
 * spread_lists(seed): hostname spread and hostname anti-affinity next to NotIn / In lists;
 * affinity_lists(seed): hostname pod affinity next to In / NotIn lists and the single-value form, with matching pods on
   excluded nodes, on admitted nodes, on a node no provisioner owns, and nowhere;
 * unlabelled(seed): nodes without a hostname label (their hostname is the node name), with a zone spread filtered by hostname;
 * cluster(seed) / after(seed): consolidation with local-PV pods pinned to their nodes, and the cluster after the TTL;
 * near_misses(): problems that must be refused; old_forms(seed): the single-value forms, which get no table;
 * admits(req, hostname): the reference's Requirement.Has on strings, for the tests' restatement.
"""
import copy
import random
import re

import fixtures as fx
from fixtures import HOSTNAME, ZONE, ZONES

PLACEHOLDER = "hostname-placeholder-"


def _node(name, rng, cpu=4, pods=None, labels=None, hostname_label=True, **kw):
    alloc = {"cpu": f"{cpu * 1000 - 100}m", "memory": f"{cpu * 4}Gi", "pods": str(cpu * 10)}
    n = fx.state_node(name, "fake-it-15", zone=rng.choice(ZONES), allocatable=alloc, capacity=dict(alloc, cpu=str(cpu)),
                      pods_=pods or [], labels=labels, **kw)
    if not hostname_label:
        del n["labels"][HOSTNAME]
    return n


def _req(op, values=()):
    r = {"key": HOSTNAME, "operator": op}
    if values:
        r["values"] = list(values)
    return r


def _pods(n, cpu="1", **kw):
    return [fx.pod({"cpu": cpu, "memory": "256Mi"}, **kw) for _ in range(n)]


def _problem(pods, nodes, **kw):
    return fx.problem(pods, instance_types=fx.fake_instance_types(16), nodes=nodes, **kw)


def _names(n, prefix="n"):
    return [f"{prefix}-{i:03d}" for i in range(n)]


# ---------------------------------------------------------------- lists
def in_list(k, seed):
    rng = random.Random(seed * 13 + k)
    names = _names(70)
    nodes = [_node(n, rng) for n in names]
    listed = names[64:64 + min(k, 6)] + rng.sample(names[:64], k - min(k, 6))
    pods = _pods(3 * k + 5, labels={"app": "pinned"}, nodeAffinity={"required": [[_req("In", listed)]]})
    pods += _pods(6, cpu="500m", labels={"app": "free"})
    return _problem(pods, nodes)


def not_in(n, k, seed):
    rng = random.Random(seed * 7 + n + k)
    names = _names(40)
    big = set(rng.sample(names, k))
    nodes = [_node(x, rng, cpu=16 if x in big else 2) for x in names]
    pods = _pods(n, cpu="250m", labels={"app": "web"}, nodeAffinity={"required": [[_req("NotIn", sorted(big))]]})
    pods += _pods(20, cpu="250m", labels={"app": "other"})
    return _problem(pods, nodes)


def selector_and_affinity(seed):
    rng = random.Random(seed + 101)
    names = _names(12)
    nodes = [_node(x, rng) for x in names]
    a, b = names[3], names[7]
    pods = _pods(5, nodeSelector={HOSTNAME: a}, nodeAffinity={"required": [[_req("In", [a, b])]]}, labels={"app": "one"})
    pods += _pods(3, nodeSelector={HOSTNAME: a}, nodeAffinity={"required": [[_req("NotIn", [a])]]}, labels={"app": "none"})
    pods += _pods(4, labels={"app": "free"})
    return _problem(pods, nodes)


def forms(seed):
    rng = random.Random(seed + 202)
    names = [str(100 + i) for i in range(12)] + _names(6, "host")
    nodes = [_node(x, rng, cpu=2) for x in names]
    pods = _pods(6, labels={"app": "exists"}, nodeAffinity={"required": [[_req("Exists")]]})
    pods += _pods(3, labels={"app": "dne"}, nodeAffinity={"required": [[_req("DoesNotExist")]]})
    pods += _pods(8, labels={"app": "gt"}, nodeAffinity={"required": [[_req("Gt", ["105"])]]})
    pods += _pods(4, labels={"app": "lt"}, nodeAffinity={"required": [[_req("Lt", ["103"])]]})
    pods += _pods(5, labels={"app": "band"}, nodeAffinity={"required": [[_req("Gt", ["101"]), _req("Lt", ["110"]), _req("NotIn", ["104", "host-001"])]]})
    return _problem(pods, nodes)


def preferred(seed):
    rng = random.Random(seed + 303)
    names = _names(60)
    nodes = [_node(x, rng, cpu=2) for x in names]
    pods = []
    for j in range(50):
        hosts = rng.sample(names, 8)
        prefs = [{"weight": rng.randint(1, 100), "terms": [_req("In", hosts)]},
                 {"weight": rng.randint(1, 100), "terms": [{"key": ZONE, "operator": "In", "values": [rng.choice(ZONES)]}]}]
        pods += _pods(rng.randint(2, 6), cpu=rng.choice(["500m", "1"]), labels={"app": f"exec-{j}"}, nodeAffinity={"preferred": prefs})
    rng.shuffle(pods)
    return _problem(pods, nodes)


def two_terms(seed):
    rng = random.Random(seed + 404)
    names = _names(10)
    nodes = [_node(x, rng, cpu=2) for x in names]
    terms = [[_req("In", names[0:2])], [_req("In", names[5:8])]]
    pods = _pods(14, labels={"app": "two"}, nodeAffinity={"required": terms})
    return _problem(pods, nodes)


def local_pv(seed):
    rng = random.Random(seed + 505)
    names = _names(24)
    nodes = [_node(x, rng) for x in names]
    pods = []
    lab = {"app": "db"}
    for i in range(18):
        own = names[i]
        pv = [own, names[(i + 1) % 24]] if i % 3 else [own]
        term = [_req("In", pv), _req("In", [own, names[(i + 5) % 24]])]
        pods.append(fx.pod({"cpu": "1", "memory": "1Gi"}, labels=lab, nodeAffinity={"required": [term]},
                           topologySpreadConstraints=[fx.spread(ZONE, lab, max_skew=2)],
                           podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, lab)]}))
    pods += _pods(6, labels={"app": "web"})
    return _problem(pods, nodes)


def spread_lists(seed):
    rng = random.Random(seed + 606)
    names = _names(16)
    nodes = [_node(x, rng, cpu=8) for x in names]
    lab1, lab2 = {"app": "spread"}, {"app": "anti"}
    pods = _pods(30, cpu="500m", labels=lab1, topologySpreadConstraints=[fx.spread(HOSTNAME, lab1, max_skew=1)],
                 nodeAffinity={"required": [[_req("NotIn", names[:5])]]})
    pods += _pods(10, cpu="500m", labels=lab2, podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, lab2)]},
                  nodeAffinity={"required": [[_req("In", names[4:12])]]})
    return _problem(pods, nodes)


def affinity_lists(seed):
    """hostname pod affinity (bootstrap) next to hostname requirements: the group's options are the hostnames the pod admits
    that have a matching pod, so a matching pod on a node the pod excludes still leaves them empty (bootstrap)"""
    rng = random.Random(seed + 909)
    names = _names(16)
    bound = {x: [] for x in names}
    for app, x in (("a1", "n-000"), ("a2", "n-006"), ("a3", "n-001")):
        bound[x].append(fx.pod({"cpu": "100m"}, nodeName=x, labels={"app": app}))
    nodes = [_node(x, rng, cpu=4, pods=bound[x]) for x in names]
    # a node no provisioner owns (no existing slot) holds a matching pod: a domain only the encoder sees
    nodes.append(_node("u-000", rng, pods=[fx.pod({"cpu": "100m"}, nodeName="u-000", labels={"app": "a4"})], provisioner_name=""))
    pods = []
    for app, req in (("a1", _req("In", ["n-004", "n-005", "n-012"])),  # matching pod only outside the list: bootstrap
                     ("a2", _req("In", ["n-006", "n-007"])),            # matching pod on a listed node
                     ("a3", _req("In", ["n-010"])),                     # the single-value pair form, matching pod elsewhere
                     ("a4", _req("NotIn", ["n-002", "n-003"])),         # the only matching pod is on the unowned node
                     ("a5", _req("NotIn", ["n-000"]))):                 # no matching pod anywhere
        lab = {"app": app}
        pods += _pods(4, cpu="500m", labels=lab, podAffinity={"required": [fx.affinity_term(HOSTNAME, lab)]},
                      nodeAffinity={"required": [[req]]})
    return _problem(pods, nodes)


def unlabelled(seed):
    rng = random.Random(seed + 707)
    names = _names(14)
    lab = {"app": "z"}
    nodes = []
    for i, x in enumerate(names):
        bound = [fx.pod({"cpu": "100m"}, nodeName=x, labels=lab)] if i % 2 else []
        nodes.append(_node(x, rng, pods=bound, hostname_label=i % 3 != 0))
    pods = _pods(6, labels={"app": "pin"}, nodeAffinity={"required": [[_req("In", [names[0], names[3], names[4]])]]})
    pods += _pods(12, cpu="500m", labels=lab, topologySpreadConstraints=[fx.spread(ZONE, lab)],
                  nodeAffinity={"required": [[_req("NotIn", [names[1], names[6]])]]})
    return _problem(pods, nodes)


# ---------------------------------------------------------------- consolidation
def cluster(seed, n_nodes=20, candidates=10):
    """local-PV pods pinned to their own node (In [own]) on some nodes, plain pods elsewhere; the first `candidates` nodes are
    consolidation candidates. A removed node admits nobody, so a candidate holding a pinned pod can never go"""
    rng = random.Random(seed * 17 + 9)
    names = _names(n_nodes, "c")
    nodes = []
    for i, x in enumerate(names):
        bound = [fx.pod({"cpu": "300m", "memory": "256Mi"}, nodeName=x, labels={"app": "web"}) for _ in range(rng.randint(0, 3))]
        if i % 3 == 0:
            bound.append(fx.pod({"cpu": "200m", "memory": "256Mi"}, nodeName=x, labels={"app": "db"},
                                nodeAffinity={"required": [[_req("In", [x]), _req("In", [x, names[(i + 1) % n_nodes]])]]}))
        nodes.append(_node(x, rng, pods=bound))
    for k in range(candidates):
        nodes[k].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return _problem([], nodes)


def after(seed):
    """cluster(seed) after the TTL: a few web pods moved, and a pending pod kept off two nodes"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 77)
    for _ in range(6):
        src, dst = rng.sample(a["nodes"], 2)
        movable = [p for p in src["pods"] if p["labels"].get("app") == "web"]
        if movable:
            p = rng.choice(movable)
            src["pods"].remove(p)
            p["nodeName"] = dst["name"]
            dst["pods"].append(p)
    a["pods"] = _pods(1, cpu="200m", labels={"app": "late"}, nodeAffinity={"required": [[_req("NotIn", ["c-000", "c-001"])]]})
    return a


# ---------------------------------------------------------------- refused and old forms
def near_misses():
    rng = random.Random(9)
    nodes = [_node(x, rng) for x in _names(4)]
    placeholder = _problem(_pods(2, nodeAffinity={"required": [[_req("In", ["n-000", PLACEHOLDER + "0001"])]]}), nodes)
    prov = _problem(_pods(2), nodes, provisioners=[fx.provisioner(requirements=[_req("NotIn", ["n-001", "n-002"])])])
    ds = _problem(_pods(2), nodes, daemonSetPods=[fx.pod({"cpu": "100m"}, nodeAffinity={"required": [[_req("In", ["n-000", "n-001"])]]})])
    return [("placeholder-value", placeholder), ("provisioner", prov), ("daemonset", ds)]


def old_forms(seed):
    rng = random.Random(seed + 808)
    names = _names(8)
    nodes = [_node(x, rng, cpu=2) for x in names]
    pods = _pods(4, labels={"app": "in"}, nodeAffinity={"required": [[_req("In", [names[2]])]]})
    pods += _pods(4, labels={"app": "notin"}, nodeAffinity={"required": [[_req("NotIn", [names[0]])]]})
    pods += _pods(3, labels={"app": "exists"}, nodeAffinity={"required": [[_req("Exists")]]})
    pods += _pods(3, labels={"app": "sel"}, nodeSelector={HOSTNAME: names[5]})
    return _problem(pods, nodes)


def corpus():
    """[(name, problem dict, expects a table)]"""
    return [("in-2", in_list(2, 0), True), ("in-5", in_list(5, 1), True), ("in-40", in_list(40, 2), True),
            ("notin-2000", not_in(2000, 3, 0), True), ("notin-6000", not_in(6000, 5, 1), True),
            ("selector-and-affinity", selector_and_affinity(0), True), ("forms", forms(0), True),
            ("preferred", preferred(0), True), ("two-terms", two_terms(0), True), ("local-pv", local_pv(0), True),
            ("spread-lists", spread_lists(0), True), ("affinity-lists", affinity_lists(0), True), ("unlabelled", unlabelled(0), True),
            ("old-forms", old_forms(0), False)]


# ---------------------------------------------------------------- the reference's rules, restated
def _int(s):
    """strconv.Atoi: an optional sign and decimal digits"""
    return int(s) if re.fullmatch(r"[+-]?[0-9]+", s) else None


def admits(req, host):
    """Requirement.Has (requirement.go:171-176) of one NodeSelectorRequirement on a hostname"""
    op, vals = req["operator"], req.get("values", [])
    if op == "In":
        return host in vals
    if op == "NotIn":
        return host not in vals
    if op == "Exists":
        return True
    if op == "DoesNotExist":
        return False
    v = _int(host)
    if v is None:
        return False
    return v > int(vals[0]) if op == "Gt" else v < int(vals[0])


def hostname_reqs(pod, term=0):
    """the pod's hostname requirements with required term `term` in force and its heaviest preferred term (unrelaxed)"""
    out = [_req("In", [v]) for k, v in pod.get("nodeSelector", {}).items() if k == HOSTNAME]
    na = pod.get("nodeAffinity") or {}
    prefs = sorted(na.get("preferred", []), key=lambda t: -t["weight"])
    if prefs:
        out += [r for r in prefs[0]["terms"] if r["key"] == HOSTNAME]
    req = na.get("required") or []
    if len(req) > term:
        out += [r for r in req[term] if r["key"] == HOSTNAME]
    return out


def node_hostname(node):
    return node["labels"].get(HOSTNAME) or node["name"]
