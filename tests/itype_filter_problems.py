"""Seeded corpus of topology spread constraints whose owner names node.kubernetes.io/instance-type in its node selector or a
required node-affinity term, so that the spread's node filter (TopologyNodeFilter) has an instance-type part (DESIGN.md §3,
instance-type node filters). GPU jobs pinned to a few types and spread over zones, deployments kept off a bad type, and
pods that select one exact type all have one.

 * listed_unlisted(seed): the instance-type form of topology_test.go:661-695: existing nodes of a listed and an unlisted type
   hold matching pods, and only the first are counted;
 * cloud_lists(seed): In lists over a catalog of 720 types, naming columns beyond the first word, with zone spread;
 * operators(seed): NotIn, Exists and DoesNotExist parts, with zone, hostname and capacity-type spread;
 * two_terms(seed): two required terms, only the first names the type (OR of terms), on a cluster with nodes of both kinds;
 * provisioners(seed): a provisioner with an instance-type requirement, and two provisioners whose type lists do and do not
   meet the term;
 * narrowed(seed): pods that select a spread group but carry no instance-type requirement are recorded on in-flight nodes that
   earlier pods narrowed to other types, and spread pods are recorded on nodes whose earlier pods never named the key;
 * relaxed(seed): pods with three required terms that name instance types; Relax drops them one at a time and each relaxed
   level gets a dormant group with another filter;
 * unlabelled(seed): existing nodes without an instance-type label and nodes whose label names a type outside the catalog;
 * cluster(seed) / after(seed): consolidation with filtered zone spreads, and the cluster after the TTL;
 * near_misses(): problems that must be refused; old_forms(seed): problems without such a term, which get no table;
 * term_matches(term, labels): TopologyNodeFilter.Matches on a node's labels, on strings, for the tests' restatement.
"""
import copy
import random

import fixtures as fx
from fixtures import CAPACITY_TYPE, HOSTNAME, INSTANCE_TYPE, ZONE, ZONES

TYPES = fx.fake_instance_types(16)


def _it(op, values=()):
    r = {"key": INSTANCE_TYPE, "operator": op}
    if values:
        r["values"] = list(values)
    return r


def _zone(op, values):
    return {"key": ZONE, "operator": op, "values": list(values)}


def _node(name, itype, rng, cpu=8, pods=None, **kw):
    alloc = {"cpu": f"{cpu * 1000 - 100}m", "memory": f"{cpu * 4}Gi", "pods": str(cpu * 10)}
    return fx.state_node(name, itype, zone=rng.choice(ZONES), allocatable=alloc, capacity=dict(alloc, cpu=str(cpu)), pods_=pods or [], **kw)


def _pods(n, cpu="1", **kw):
    return [fx.pod({"cpu": cpu, "memory": "256Mi"}, **kw) for _ in range(n)]


def _bound(node, n, lab, **kw):
    return [fx.pod({"cpu": "200m", "memory": "128Mi"}, nodeName=node, labels=lab, **kw) for _ in range(n)]


def _problem(pods, nodes=(), types=None, **kw):
    return fx.problem(pods, instance_types=types or TYPES, nodes=list(nodes), **kw)


# ---------------------------------------------------------------- counting and recording
def listed_unlisted(seed):
    rng = random.Random(seed + 11)
    lab = {"app": "spread"}
    nodes = [_node("listed-a", "fake-it-7", rng, pods=_bound("listed-a", 2, lab)),
             _node("listed-b", "fake-it-7", rng, pods=_bound("listed-b", 1, lab)),
             _node("unlisted-a", "fake-it-9", rng, pods=_bound("unlisted-a", 3, lab)),
             _node("unlisted-b", "fake-it-11", rng, pods=_bound("unlisted-b", 2, lab))]
    pods = _pods(9, cpu="500m", labels=lab, nodeSelector={INSTANCE_TYPE: "fake-it-7"},
                 topologySpreadConstraints=[fx.spread(ZONE, lab)])
    pods += _pods(6, cpu="250m", labels=lab)  # selected by the group, no requirement of their own
    return _problem(pods, nodes)


def cloud_lists(seed):
    rng = random.Random(seed + 22)
    types = fx.fake_instance_types(720)
    names = [t["name"] for t in types]
    pods = []
    for j in range(6):
        lab = {"app": f"train-{j}"}
        listed = rng.sample(names[64:], 5) + ([rng.choice(names[:64])] if j % 2 else [])
        pods += _pods(rng.randint(4, 10), cpu=rng.choice(["2", "4"]), labels=lab, nodeAffinity={"required": [[_it("In", listed)]]},
                      topologySpreadConstraints=[fx.spread(ZONE, lab, max_skew=1)])
    lab = {"app": "avoid"}
    pods += _pods(8, cpu="1", labels=lab, nodeAffinity={"required": [[_it("NotIn", rng.sample(names, 40))]]},
                  topologySpreadConstraints=[fx.spread(ZONE, lab)])
    nodes = [_node(f"e-{i}", names[rng.randrange(720)], rng, cpu=16,
                   pods=_bound(f"e-{i}", 1, {"app": f"train-{i % 6}"})) for i in range(8)]
    return _problem(pods, nodes, types=types)


def operators(seed):
    rng = random.Random(seed + 33)
    labs = [{"app": a} for a in ("notin", "exists", "dne", "ct")]
    nodes = [_node(f"o-{i}", f"fake-it-{i % 4 + 8}", rng, pods=_bound(f"o-{i}", 1, labs[i % 4])) for i in range(8)]
    pods = _pods(10, labels=labs[0], nodeAffinity={"required": [[_it("NotIn", ["fake-it-8", "fake-it-9"])]]},
                 topologySpreadConstraints=[fx.spread(ZONE, labs[0]), fx.spread(HOSTNAME, labs[0], max_skew=2)])
    pods += _pods(8, labels=labs[1], nodeAffinity={"required": [[_it("Exists")]]},
                  topologySpreadConstraints=[fx.spread(HOSTNAME, labs[1])])
    # first term In, second DoesNotExist: the filter is the OR of both; relaxation drops the first
    pods += _pods(6, labels=labs[2], nodeAffinity={"required": [[_it("In", ["fake-it-10", "fake-it-12"])], [_it("DoesNotExist")]]},
                  topologySpreadConstraints=[fx.spread(ZONE, labs[2])])
    pods += _pods(8, cpu="500m", labels=labs[3], nodeSelector={INSTANCE_TYPE: "fake-it-11"},
                  topologySpreadConstraints=[fx.spread(CAPACITY_TYPE, labs[3])])
    pods += _pods(6, cpu="250m", labels=labs[0])
    return _problem(pods, nodes)


def two_terms(seed):
    rng = random.Random(seed + 44)
    lab = {"app": "or"}
    nodes = [_node(f"t-{i}", f"fake-it-{6 + i % 3}", rng, pods=_bound(f"t-{i}", 1 + i % 2, lab)) for i in range(6)]
    terms = [[_it("In", ["fake-it-6", "fake-it-13"])], [_zone("In", ZONES[:2])]]
    pods = _pods(12, cpu="500m", labels=lab, nodeAffinity={"required": terms}, topologySpreadConstraints=[fx.spread(ZONE, lab)])
    pods += _pods(5, cpu="250m", labels=lab, nodeSelector={INSTANCE_TYPE: "fake-it-8"})
    return _problem(pods, nodes)


def provisioners(seed):
    rng = random.Random(seed + 55)
    lab1, lab2 = {"app": "p1"}, {"app": "p2"}
    prov = [fx.provisioner("gpu", requirements=[_it("In", ["fake-it-12", "fake-it-13", "fake-it-14"])]),
            fx.provisioner("general", requirements=[_it("NotIn", ["fake-it-12", "fake-it-13"])])]
    pods = _pods(10, labels=lab1, nodeAffinity={"required": [[_it("In", ["fake-it-13", "fake-it-5"])]]},
                 topologySpreadConstraints=[fx.spread(ZONE, lab1)])
    pods += _pods(6, cpu="250m", labels=lab1)
    pods += _pods(8, labels=lab2, nodeAffinity={"required": [[_it("In", ["fake-it-2", "fake-it-3"])]]},
                  topologySpreadConstraints=[fx.spread(HOSTNAME, lab2)])
    pods += _pods(4, cpu="250m", labels=lab2)
    nodes = [_node("g-0", "fake-it-13", rng, provisioner_name="gpu", pods=_bound("g-0", 1, lab1))]
    return _problem(pods, nodes, provisioners=prov)


def narrowed(seed):
    rng = random.Random(seed + 66)
    lab = {"app": "s"}
    # big pods first (queue order): they open nodes narrowed away from the listed types; then the spread pods; then small
    # pods of the spread's selector without requirements join the open nodes and are recorded only where the filter matches
    pods = _pods(6, cpu="3", labels={"app": "big"}, nodeAffinity={"required": [[_it("NotIn", ["fake-it-10", "fake-it-11"])]]})
    pods += _pods(4, cpu="3", labels={"app": "big-in"}, nodeAffinity={"required": [[_it("In", ["fake-it-10", "fake-it-14"])]]})
    pods += _pods(4, cpu="2500m", labels={"app": "plain"})
    pods += _pods(10, cpu="1", labels=lab, nodeAffinity={"required": [[_it("In", ["fake-it-10", "fake-it-11"])]]},
                  topologySpreadConstraints=[fx.spread(ZONE, lab)])
    pods += _pods(16, cpu="250m", labels=lab)
    rng.shuffle(pods)
    return _problem(pods)


def relaxed(seed):
    rng = random.Random(seed + 77)
    lab = {"app": "relax"}
    nodes = [_node(f"r-{i}", f"fake-it-{i + 3}", rng, cpu=2, pods=_bound(f"r-{i}", 1, lab)) for i in range(5)]
    terms = [[_it("In", ["fake-it-0"])], [_it("In", ["fake-it-1", "fake-it-4"])], [_it("NotIn", ["fake-it-0", "fake-it-1"])]]
    pods = _pods(8, cpu="1", labels=lab, nodeAffinity={"required": terms}, topologySpreadConstraints=[fx.spread(ZONE, lab)])
    pods += _pods(4, cpu="250m", labels=lab)
    return _problem(pods, nodes, provisioners=[fx.provisioner(requirements=[_it("NotIn", ["fake-it-0"])])])


def unlabelled(seed):
    rng = random.Random(seed + 88)
    lab = {"app": "u"}
    nodes = []
    for i in range(8):
        n = _node(f"u-{i}", "retired-type" if i % 4 == 1 else f"fake-it-{i + 4}", rng, pods=_bound(f"u-{i}", 1 + i % 2, lab))
        if i % 4 == 0:
            del n["labels"][INSTANCE_TYPE]
        nodes.append(n)
    # complement requirements only: an In requirement never admits an unlabelled node or a type outside the catalog here
    pods = _pods(10, labels=lab, nodeAffinity={"required": [[_it("NotIn", ["fake-it-6"])]]},
                 topologySpreadConstraints=[fx.spread(ZONE, lab)])
    pods += _pods(6, cpu="250m", labels=lab, nodeAffinity={"required": [[_it("Exists")]]},
                  topologySpreadConstraints=[fx.spread(HOSTNAME, lab, max_skew=2)])
    pods += _pods(6, cpu="250m", labels=lab)
    return _problem(pods, nodes)


# ---------------------------------------------------------------- consolidation
def cluster(seed, n_nodes=16, candidates=8):
    """nodes of four types; pods pinned to two of them spread over zones with the type in their node filter"""
    rng = random.Random(seed * 19 + 3)
    lab = {"app": "pinned"}
    nodes = []
    for i in range(n_nodes):
        x, t = f"c-{i:02d}", f"fake-it-{4 + i % 4}"
        bound = [fx.pod({"cpu": "300m", "memory": "256Mi"}, nodeName=x, labels={"app": "web"}) for _ in range(rng.randint(0, 2))]
        if t in ("fake-it-4", "fake-it-5"):
            bound += _bound(x, rng.randint(1, 2), lab, nodeAffinity={"required": [[_it("In", ["fake-it-4", "fake-it-5"])]]},
                            topologySpreadConstraints=[fx.spread(ZONE, lab, max_skew=2)])
        nodes.append(_node(x, t, rng, cpu=4, pods=bound))
    for k in range(candidates):
        nodes[k].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return _problem([], nodes)


def after(seed):
    """cluster(seed) after the TTL: a few web pods moved, and a pending filtered spread pod"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 99)
    for _ in range(5):
        src, dst = rng.sample(a["nodes"], 2)
        movable = [p for p in src["pods"] if p["labels"].get("app") == "web"]
        if movable:
            p = rng.choice(movable)
            src["pods"].remove(p)
            p["nodeName"] = dst["name"]
            dst["pods"].append(p)
    lab = {"app": "pinned"}
    a["pods"] = _pods(1, cpu="200m", labels=lab, nodeAffinity={"required": [[_it("In", ["fake-it-5"])]]},
                      topologySpreadConstraints=[fx.spread(ZONE, lab, max_skew=2)])
    return a


# ---------------------------------------------------------------- refused and old forms
def near_misses():
    rng = random.Random(5)
    lab = {"app": "x"}
    nodes = [_node(f"m-{i}", "fake-it-3", rng) for i in range(3)]
    spread = [fx.spread(ZONE, lab)]
    gt = _problem(_pods(2, labels=lab, nodeAffinity={"required": [[_it("Gt", ["3"])]]}, topologySpreadConstraints=spread), nodes)
    term_unlisted = _problem(_pods(2, labels=lab, nodeAffinity={"required": [[_it("In", ["fake-it-3", "p5.48xlarge"])]]},
                                   topologySpreadConstraints=spread), nodes)
    notin_unlisted = _problem(_pods(2, labels=lab, nodeAffinity={"required": [[_it("NotIn", ["m5.large"])]]},
                                    topologySpreadConstraints=spread), nodes)
    pod_unlisted = _problem(_pods(2, labels=lab, nodeSelector={INSTANCE_TYPE: "fake-it-3"}, topologySpreadConstraints=spread) +
                            _pods(2, nodeAffinity={"required": [[_it("In", ["fake-it-2", "c5.xlarge"])]]}), nodes)
    prov_unlisted = _problem(_pods(2, labels=lab, nodeSelector={INSTANCE_TYPE: "fake-it-3"}, topologySpreadConstraints=spread), nodes,
                             provisioners=[fx.provisioner(requirements=[_it("In", ["fake-it-3", "r6i.large"])])])
    return [("gt", gt), ("term-unlisted", term_unlisted), ("notin-unlisted", notin_unlisted), ("pod-unlisted", pod_unlisted),
            ("provisioner-unlisted", prov_unlisted)]


def old_forms(seed):
    rng = random.Random(seed + 111)
    lab = {"app": "old"}
    nodes = [_node(f"f-{i}", f"fake-it-{i + 5}", rng, pods=_bound(f"f-{i}", 1, lab)) for i in range(4)]
    pods = _pods(6, labels=lab, topologySpreadConstraints=[fx.spread(ZONE, lab)], nodeSelector={"size": "large"})
    pods += _pods(6, nodeAffinity={"required": [[_it("In", ["fake-it-8", "fake-it-9"])]]})
    pods += _pods(4, nodeAffinity={"required": [[_it("NotIn", ["fake-it-8", "unlisted-type"])]]})
    return _problem(pods, nodes)


def corpus():
    """[(name, problem dict, expects the instance-type filter tables)]"""
    return [("listed-unlisted", listed_unlisted(0), True), ("cloud-lists", cloud_lists(0), True), ("operators", operators(0), True),
            ("two-terms", two_terms(0), True), ("provisioners", provisioners(0), True), ("narrowed", narrowed(0), True),
            ("narrowed-1", narrowed(1), True), ("relaxed", relaxed(0), True), ("unlabelled", unlabelled(0), True),
            ("cluster-after", after(0), True), ("old-forms", old_forms(0), False)]


# ---------------------------------------------------------------- the reference's rules, restated
def _itype_set(reqs):
    """Requirements.Add of instance-type requirements (requirement.go:117-150) as (complement, names)"""
    comp, names = True, set()
    for r in reqs:
        op, vals = r["operator"], set(r.get("values", []))
        rc = op not in ("In", "DoesNotExist")
        rv = vals if op in ("In", "NotIn") else set()
        if comp and rc:
            names = names | rv
        elif comp:
            names = rv - names
        elif rc:
            names = names - rv
        else:
            names = names & rv
        comp = comp and rc
    return comp, names


def _intersects(a, b):
    """Requirements.Intersects on one key (requirements.go:189-206)"""
    (ac, an), (bc, bn) = a, b
    if ac and bc:
        nonempty = True
    elif ac:
        nonempty = bool(bn - an)
    elif bc:
        nonempty = bool(an - bn)
    else:
        nonempty = bool(an & bn)
    negative = lambda c, n: bool(n) if c else not n  # NotIn / DoesNotExist
    return nonempty or (negative(*a) and negative(*b))


def term_matches(term_reqs, labels):
    """the instance-type part of one filter term against a node's labels: a node without the label passes"""
    its = [r for r in term_reqs if r["key"] == INSTANCE_TYPE]
    if not its or INSTANCE_TYPE not in labels:
        return True
    return _intersects(_itype_set([{"operator": "In", "values": [labels[INSTANCE_TYPE]]}]), _itype_set(its))
