"""Consolidation clusters and candidate sets for simulateScheduling's whole result (ClusterSession.simulate, DESIGN.md §5).
Each scenario is (name, problem dict, sets, property): sets are lists of node names, or an int k for "the k cheapest
candidates to disrupt, listed in reverse, and the cheapest alone" (Expiration and Drift list candidates in their own
order); property names what the oracle's Solve with a set removed must show (tests/test_full_simulation_reach.py):

 * new3: three or more new nodes, past the consolidation simulator's stop after the second;
 * relaxed / pending / deleting / uninitialized / unschedulable: a relaxed pod, pending pods, the pods of a node marked for
   deletion, a pod on an existing node that is not initialised, an unschedulable pod;
 * topology: zone-spread and hostname anti-affinity pods among the removed ones;
 * ext / folded / hostname / hostport / volume / limits: clusters of the feature corpora - resources past the row's 8,
   more than 16 label keys with template-only ones folded, hostname tables, host ports, volume claims, several provisioners
   with limits.
"""
import consolidation_answers as ca
import extended_resource_problems
import fixtures as fx
import hostname_problems
import hostport_problems
import provisioner_problems
import volume_problems

ZONE, HOSTNAME = fx.ZONE, fx.HOSTNAME


def _node(name, it, pods_, cost=1.0, cpu="32", **kw):
    n = ca.node_of_type(name, it, pods_, cost)
    n["allocatable"] = {"cpu": cpu, "memory": "64Gi", "pods": "100"}
    n.update(kw)
    return n


def _bound(node, n, cpu, **kw):
    return [fx.pod({"cpu": cpu, "memory": "1Gi"}, nodeName=node, **kw) for _ in range(n)]


def _cluster(nodes, pods_=()):
    return fx.problem(list(pods_), instance_types=ca.assorted(), provisioners=[fx.provisioner(consolidationEnabled=True)], nodes=nodes,
                      deriveCandidates=True)


def _types():
    its = ca.assorted()
    od = ca.on_demand_by_price(its)
    return od[-1], od


def new3():
    big, _ = _types()
    nodes = [_node(f"c{i}", big, _bound(f"c{i}", 2, "20"), cost=float(i)) for i in range(3)]
    nodes.append(_node("full", big, _bound("full", 1, "31"), cost=9.0))
    return _cluster(nodes)


def relaxed():
    big, _ = _types()
    pref = {"preferred": [{"weight": 5, "terms": [{"key": ZONE, "operator": "In", "values": ["nowhere"]}]}]}
    nodes = [_node("c0", big, _bound("c0", 3, "5", nodeAffinity=pref)), _node("c1", big, _bound("c1", 2, "3"), cost=2.0),
             _node("full", big, _bound("full", 1, "31"), cost=9.0)]
    return _cluster(nodes)


def pending():
    big, _ = _types()
    nodes = [_node("c0", big, _bound("c0", 2, "6")), _node("c1", big, _bound("c1", 2, "2"), cost=2.0),
             _node("roomy", big, _bound("roomy", 1, "4"), cost=9.0)]
    return _cluster(nodes, [fx.pod({"cpu": "3", "memory": "1Gi"}) for _ in range(3)])


def deleting():
    big, _ = _types()
    nodes = [_node("gone", big, _bound("gone", 3, "4"), markedForDeletion=True), _node("c0", big, _bound("c0", 2, "6")),
             _node("c1", big, _bound("c1", 1, "1"), cost=2.0), _node("full", big, _bound("full", 1, "31"), cost=9.0)]
    return _cluster(nodes, [fx.pod({"cpu": "2", "memory": "1Gi"})])


def uninitialized():
    big, _ = _types()
    cold = fx.state_node("cold", big["name"], zone=big["offerings"][0]["zone"], allocatable={"cpu": "32", "memory": "64Gi", "pods": "100"},
                         initialized=False)
    nodes = [_node("full", big, _bound("full", 1, "31"), cost=9.0), cold, _node("c0", big, _bound("c0", 2, "2")),
             _node("c1", big, _bound("c1", 1, "30"), cost=2.0)]
    return _cluster(nodes)


def unschedulable():
    big, _ = _types()
    nodes = [_node("c0", big, _bound("c0", 1, "100") + _bound("c0", 2, "1")), _node("c1", big, _bound("c1", 2, "4"), cost=2.0),
             _node("full", big, _bound("full", 1, "31"), cost=9.0)]
    return _cluster(nodes)


def topology():
    big, _ = _types()
    web = {"app": "web"}
    spread = dict(labels=web, topologySpreadConstraints=[fx.spread(ZONE, web)])
    anti = dict(labels={"app": "solo"}, podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "solo"})]})
    nodes = [_node("c0", big, _bound("c0", 3, "2", **spread) + _bound("c0", 1, "1", **anti)),
             _node("c1", big, _bound("c1", 2, "2", **spread) + _bound("c1", 1, "1", **anti), cost=2.0),
             _node("stay", big, _bound("stay", 2, "2", **spread) + _bound("stay", 1, "1", **anti), cost=9.0)]
    return _cluster(nodes)


def corpus():
    named = [("new3", new3(), [["c2", "c0", "c1"], ["c1", "c0"]], "new3"),
             ("relaxed", relaxed(), [["c0"], ["c1", "c0"]], "relaxed"),
             ("pending", pending(), [["c1", "c0"], ["c0"]], "pending"),
             ("deleting", deleting(), [["c0"], ["c1", "c0"]], "deleting"),
             ("uninitialized", uninitialized(), [["c0"], ["c0", "c1"]], "uninitialized"),
             ("unschedulable", unschedulable(), [["c0"], ["c1", "c0"]], "unschedulable"),
             ("topology", topology(), [["c1", "c0"], ["c0"]], "topology")]
    vol = dict((n, p) for n, p, _ in volume_problems.clusters())
    features = [("ext", extended_resource_problems.cluster(0), 3, "ext"),
                ("folded", provisioner_problems.cluster(1), 3, "folded"),
                ("hostname", hostname_problems.cluster(0), 3, "hostname"),
                ("hostport", hostport_problems.cluster(0), 3, "hostport"),
                ("volume", vol["shared-60x3"], 3, "volume"),
                ("limits", provisioner_problems.cluster(0), 3, "limits")]
    return named + features


def resolve_sets(prob, sets, order):
    """the scenario's sets as node indices: names looked up, an int k taken from the disruption order `order`"""
    if isinstance(sets, int):
        return [order[:sets][::-1], order[:1]]
    index = {n["name"]: i for i, n in enumerate(prob["nodes"])}
    return [[index[name] for name in s] for s in sets]
