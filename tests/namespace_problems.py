"""Problems whose pod affinity and anti-affinity terms carry a namespaceSelector. buildNamespaceList
(topology.go:326-347) resolves the selector against the cluster's Namespace objects (the document's top-level
`namespaces`), so a group counts pods of every namespace the selector matches plus those the term names.

corpus() is seeded and builds its own terms: the restated topology_test.go:2131-2168 case, matchLabels whose target namespace
does and does not carry the label, matchExpressions with each operator, a selector together with a namespace list, a
selector that matches nothing, deployments of three namespaces under `{}` with hostname and zone anti-affinity, preferred
cross-namespace terms that are relaxed, and bound pods whose required anti-affinity spans namespaces (inverse groups).
cluster() / after() are a consolidation cluster and the same cluster after the TTL with one namespace relabelled.
near_misses() are documents the loader must refuse. resolve() / explicit() / check() restate the semantics in Python, so
the tests can judge a result without the oracle."""
import copy
import random

import consolidation_answers as ca
import fixtures as fx
from fixtures import HOSTNAME, ZONE

EVERY = {"matchLabels": {}}   # `namespaceSelector: {}` selects every namespace


def ns(name, **labels):
    return {"name": name, "labels": labels}


def term(key, labels, selector=None, namespaces=None):
    t = {"topologyKey": key, "labelSelector": {"matchLabels": labels}}
    if selector is not None:
        t["namespaceSelector"] = selector
    if namespaces:
        t["namespaces"] = namespaces
    return t


def _req(cpu="1"):
    return {"cpu": cpu}


def _problem(pods_, namespaces, **kw):
    return fx.problem(pods_, namespaces=namespaces, **kw)


# ---------------------------------------------------------------- scenarios (rng -> problem dict)
def restated_empty_selector(rng=None):
    """topology_test.go:2131-2168: the target lives in another namespace; `{}` selects it, so both share a node"""
    labels, aff = {"test": "test"}, {"security": "s2"}
    noise = fx.pods(10, labels=labels, topologySpreadConstraints=[fx.spread(HOSTNAME, labels)])
    target = fx.pod(labels=aff, namespace="empty-ns-selector")
    follower = fx.pod(podAffinity={"required": [term(HOSTNAME, aff, EVERY)]})
    return _problem(noise + [target, follower], [ns("default"), ns("empty-ns-selector", foo="bar")])


def match_labels(rng, target_labelled):
    aff = {"app": "cache"}
    n = rng.randint(2, 4)
    target = fx.pod(_req("500m"), labels=aff, namespace="data")
    followers = fx.pods(n, requests=_req("500m"), namespace="web",
                        podAffinity={"required": [term(HOSTNAME, aff, {"matchLabels": {"team": "storage"}})]})
    spaces = [ns("web", team="frontend"), ns("data", **({"team": "storage"} if target_labelled else {"team": "other"}))]
    return _problem([target] + followers, spaces)


def match_expression(rng, op):
    """anti-affinity to app=web pods of the namespaces a single expression selects: prod (env=prod), dev (env=dev), bare
    (no env label)"""
    values = {"In": ["prod"], "NotIn": ["prod"], "Exists": None, "DoesNotExist": None}[op]
    expr = {"key": "env", "operator": op}
    if values:
        expr["values"] = values
    web = {"app": "web"}
    pods_ = []
    for space in ("prod", "dev", "bare"):
        pods_ += fx.pods(rng.randint(1, 3), requests=_req("300m"), labels=web, namespace=space)
    pods_ += fx.pods(rng.randint(2, 4), requests=_req("300m"), labels={"app": "guard"}, namespace="default",
                     podAntiAffinity={"required": [term(HOSTNAME, web, {"matchExpressions": [expr]})]})
    rng.shuffle(pods_)
    return _problem(pods_, [ns("default"), ns("prod", env="prod"), ns("dev", env="dev"), ns("bare")])


def selector_and_list(rng):
    """the selector matches `a`, the term names `b`: the group counts both, not `c`"""
    web = {"app": "web"}
    pods_ = []
    for space in ("a", "b", "c"):
        pods_ += fx.pods(rng.randint(1, 2), requests=_req("300m"), labels=web, namespace=space)
    pods_ += fx.pods(2, requests=_req("300m"), namespace="default",
                     podAntiAffinity={"required": [term(HOSTNAME, web, {"matchLabels": {"pick": "yes"}}, namespaces=["b"])]})
    return _problem(pods_, [ns("default"), ns("a", pick="yes"), ns("b"), ns("c", pick="no")])


def selector_matches_nothing(rng, self_affinity):
    """an empty resolved set: anti-affinity selects nobody; self-affinity cannot bootstrap (the pod does not select itself)"""
    web = {"app": "web"}
    nothing = {"matchLabels": {"absent": "label"}}
    if self_affinity:
        pods_ = fx.pods(rng.randint(2, 4), requests=_req("300m"), labels=web, namespace="a",
                        podAffinity={"required": [term(HOSTNAME, web, nothing)]})
    else:
        pods_ = fx.pods(rng.randint(2, 4), requests=_req("300m"), labels=web, namespace="a",
                        podAntiAffinity={"required": [term(HOSTNAME, web, nothing)]})
    return _problem(pods_, [ns("default"), ns("a", team="x")])


def three_namespace_deployments(rng, key):
    """one deployment per namespace, each anti-affine to app=db in every namespace: hostname spreads all of them on their own
    nodes, zone admits one pod per zone across the three deployments"""
    db = {"app": "db"}
    pods_ = []
    for space in ("east", "west", "north"):
        pods_ += fx.pods(rng.randint(2, 4), requests=_req(rng.choice(["300m", "1"])), labels=db, namespace=space,
                         podAntiAffinity={"required": [term(key, db, EVERY)]})
    return _problem(pods_, [ns("default"), ns("east", region="e"), ns("west", region="w"), ns("north", region="n")])


def preferred_relaxed(rng):
    """preferred zone anti-affinity across namespaces for more pods than zones, and a preferred affinity to a pod of a namespace
    no selector reaches: both are relaxed"""
    db = {"app": "db"}
    pods_ = []
    for space in ("east", "west"):
        pods_ += fx.pods(rng.randint(2, 3), requests=_req("300m"), labels=db, namespace=space,
                         podAntiAffinity={"preferred": [{"weight": 10, "term": term(ZONE, db, EVERY)}]})
    pods_ += fx.pods(2, requests=_req("300m"), namespace="east",
                     podAffinity={"preferred": [{"weight": 5, "term": term(HOSTNAME, {"app": "ghost"}, {"matchLabels": {"region": "w"}})}]})
    pods_.append(fx.pod(_req("300m"), labels={"app": "ghost"}, namespace="east"))
    return _problem(pods_, [ns("default"), ns("east", region="e"), ns("west", region="w")])


def bound_inverse(rng):
    """existing nodes host pods of namespace `ops` whose required anti-affinity selects app=web in every namespace: pending
    web pods of other namespaces must stay off those nodes (inverse anti-affinity groups)"""
    web = {"app": "web"}
    nodes = []
    for i in range(3):
        bound = [fx.pod(_req("100m"), nodeName=f"node-{i}", namespace="ops", labels={"app": "agent"},
                        podAntiAffinity={"required": [term(HOSTNAME, web, EVERY)]})]
        nodes.append(fx.state_node(f"node-{i}", zone=fx.ZONES[i], pods_=bound))
    nodes.append(fx.state_node("node-free", zone=fx.ZONES[0]))
    pods_ = []
    for space in ("shop", "blog"):
        pods_ += fx.pods(rng.randint(1, 3), requests=_req("200m"), labels=web, namespace=space)
    pods_ += fx.pods(rng.randint(1, 2), requests=_req("200m"), labels={"app": "other"}, namespace="shop")
    return _problem(pods_, [ns("default"), ns("ops"), ns("shop", tier="front"), ns("blog", tier="front")], nodes=nodes)


def corpus(seeds=(1, 2)):
    out = [("restated_2131", restated_empty_selector())]
    for seed in seeds:
        rng = random.Random(seed)
        out += [(f"match_labels_target_labelled_s{seed}", match_labels(rng, True)),
                (f"match_labels_target_unlabelled_s{seed}", match_labels(rng, False))]
        out += [(f"match_expression_{op}_s{seed}", match_expression(rng, op)) for op in ("In", "NotIn", "Exists", "DoesNotExist")]
        out += [(f"selector_and_list_s{seed}", selector_and_list(rng)),
                (f"selects_nothing_anti_s{seed}", selector_matches_nothing(rng, False)),
                (f"selects_nothing_self_affinity_s{seed}", selector_matches_nothing(rng, True)),
                (f"three_namespaces_hostname_s{seed}", three_namespace_deployments(rng, HOSTNAME)),
                (f"three_namespaces_zone_s{seed}", three_namespace_deployments(rng, ZONE)),
                (f"preferred_relaxed_s{seed}", preferred_relaxed(rng)),
                (f"bound_inverse_s{seed}", bound_inverse(rng))]
    return out


# ---------------------------------------------------------------- consolidation: a cluster and its state after the TTL
def cluster(seed=0):
    """candidate nodes of the most expensive type, one app=web pod each, in namespaces shop (tier=front), blog (tier=front)
    and tools; every web pod is anti-affine on the hostname to app=web in the tier=front namespaces"""
    rng = random.Random(seed)
    its = ca.assorted()
    big = ca.on_demand_by_price(its)[-1]
    web = {"app": "web"}
    anti = {"required": [term(HOSTNAME, web, {"matchLabels": {"tier": "front"}})]}
    nodes = []
    for i, space in enumerate(("shop", "shop", "blog", "blog", "tools", "shop")):
        name = f"node{i}"
        pods_ = [fx.pod(_req(rng.choice(["1", "2"])), nodeName=name, namespace=space, labels=web, podAntiAffinity=anti)]
        nodes.append(ca.node_of_type(name, big, pods_, 1.0))
    return fx.problem([], instance_types=its, provisioners=[fx.provisioner(consolidationEnabled=True)], nodes=nodes,
                      deriveCandidates=True, namespaces=[ns("shop", tier="front"), ns("blog", tier="front"), ns("tools")])


def after(seed=0):
    """the cluster when the TTL ends: shop was relabelled tier=back, so its web pods no longer repel each other"""
    d = cluster(seed)
    d["namespaces"][0]["labels"] = {"tier": "back"}
    return d


# ---------------------------------------------------------------- documents the loader refuses
def near_misses():
    web = {"app": "web"}
    pod = lambda sel: fx.pod(_req(), podAntiAffinity={"required": [term(HOSTNAME, web, sel)]})
    no_list = fx.problem([pod(EVERY)])
    bound_no_list = fx.problem([], nodes=[fx.state_node("n0", pods_=[fx.pod(_req(), nodeName="n0", podAffinity={
        "preferred": [{"weight": 1, "term": term(HOSTNAME, web, EVERY)}]})])])
    bad_op = _problem([pod({"matchExpressions": [{"key": "env", "operator": "Gt", "values": ["1"]}]})], [ns("default")])
    no_values = _problem([pod({"matchExpressions": [{"key": "env", "operator": "In", "values": []}]})], [ns("default")])
    bad_key = _problem([pod({"matchLabels": {"bad key": "x"}})], [ns("default")])
    duplicate = _problem([pod(EVERY)], [ns("default"), ns("default", team="x")])
    reserved = _problem([fx.pod(_req(), namespace="<no namespace>")], [ns("default")])   # the name of an empty resolved set
    return [("selector_without_namespace_list", no_list), ("bound_pod_selector_without_namespace_list", bound_no_list),
            ("invalid_operator", bad_op), ("in_without_values", no_values), ("invalid_label_key", bad_key),
            ("duplicate_namespace", duplicate), ("pod_in_the_empty_set_namespace", reserved)]


# ---------------------------------------------------------------- the semantics restated
def selector_matches(sel, labels):
    """metav1.LabelSelector (matchLabels, matchExpressions In / NotIn / Exists / DoesNotExist) against a label map"""
    for k, v in sel.get("matchLabels", {}).items():
        if labels.get(k) != v:
            return False
    for e in sel.get("matchExpressions", []):
        has, val = e["key"] in labels, labels.get(e["key"])
        op, values = e["operator"], e.get("values", [])
        if (op == "In" and (not has or val not in values)) or (op == "NotIn" and has and val in values) or \
                (op == "Exists" and not has) or (op == "DoesNotExist" and has):
            return False
    return True


def resolve(doc, pod, t):
    """buildNamespaceList: the namespaces a term's group counts"""
    if "namespaceSelector" not in t:
        return set(t.get("namespaces") or [pod.get("namespace", "default")])
    picked = {n["name"] for n in doc["namespaces"] if selector_matches(t["namespaceSelector"], n.get("labels", {}))}
    return picked | set(t.get("namespaces") or [])


def _terms(pod):
    for kind in ("podAffinity", "podAntiAffinity"):
        a = pod.get(kind) or {}
        for t in a.get("required", []):
            yield kind, True, t
        for w in a.get("preferred", []):
            yield kind, False, w["term"]


def _all_pods(doc):
    yield from doc.get("pods", [])
    yield from doc.get("daemonSetPods", [])
    for n in doc.get("nodes", []):
        yield from n.get("pods", [])


def explicit(doc):
    """the same document with every namespaceSelector replaced by the namespace list it resolves to; None when some selector
    resolves to nothing (an empty list means the pod's own namespace)"""
    out = copy.deepcopy(doc)
    for pod in _all_pods(out):
        for _, _, t in _terms(pod):
            if "namespaceSelector" in t:
                names = sorted(resolve(doc, pod, t))
                if not names:
                    return None
                del t["namespaceSelector"]
                t["namespaces"] = names
    out.pop("namespaces", None)
    return out


def _domains(doc, result, a, key):
    """the domains a placed pod may occupy: one hostname per node, the node's zone or its new node's zone requirement"""
    n_existing = len(result["existing"])
    if a < n_existing:
        node = doc["nodes"][result["existing"][a]["node"]]
        return {node["name"]} if key == HOSTNAME else {node["labels"].get(key)}
    if key == HOSTNAME:
        return {("new", a)}
    req = result["newNodes"][a - n_existing]["requirements"].get(key, "")
    op, _, rest = req.partition(" ")
    vals = set(rest.strip()[1:-1].split())
    return vals if op == "In" else {("any", a)}


def check(doc, result):
    """independent check of a Solve result: no two pods a required anti-affinity term separates share a domain, and a pod
    with a required affinity term shares its domain with a pod the term selects (itself, when it is the only one)"""
    placed = []   # (pod, namespace, labels, node index of the result's numbering)
    for i, p in enumerate(doc["pods"]):
        if result["assign"][i] >= 0:
            placed.append((p, result["assign"][i]))
    for e, ex in enumerate(result["existing"]):
        for p in doc["nodes"][ex["node"]].get("pods", []):
            placed.append((p, e))
    for p, a in placed:
        for kind, required, t in _terms(p):
            if not required:
                continue
            spaces, key = resolve(doc, p, t), t["topologyKey"]
            mine = _domains(doc, result, a, key)
            others = [(q, b) for q, b in placed if q is not p and q.get("namespace", "default") in spaces and
                      selector_matches(t["labelSelector"], q.get("labels", {}))]
            if kind == "podAntiAffinity":
                for q, b in others:
                    assert not (mine & _domains(doc, result, b, key)), (p["name"], q["name"], key)
            elif others:
                assert any(mine & _domains(doc, result, b, key) for _, b in others), (p["name"], key)
            else:
                assert p.get("namespace", "default") in spaces and selector_matches(t["labelSelector"], p.get("labels", {})), p["name"]
