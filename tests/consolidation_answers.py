"""Known answers for the consolidation simulator + price guards (SURVEY 8a-19), restated from
pkg/controllers/deprovisioning/suite_test.go. Each case is (problem dict, checks on one computeConsolidation probe and/or
on the multi-node search). The CPU suite pins the oracle with them; the GPU suite requires the product's probe / search
to return exactly what the oracle returns."""
import fixtures as fx
from fixtures import CAPACITY_TYPE, INSTANCE_TYPE, ZONE

ZONES = ("test-zone-1", "test-zone-2", "test-zone-3")


def assorted():
    """fake.InstanceTypesAssorted in miniature: one offering per type, price a function of the resources"""
    its = []
    for cpu in (1, 2, 4, 8, 16, 32):
        for mem in (2, 8, 32):
            for zone in ZONES:
                for ct in ("spot", "on-demand"):
                    res = {"cpu": str(cpu), "memory": f"{mem}Gi", "pods": "100"}
                    its.append(fx.instance_type(f"{cpu}c-{mem}g-{zone}-{ct}", res,
                                                offerings=[{"capacityType": ct, "zone": zone, "price": fx.price_from_resources(res), "available": True}],
                                                oses=("linux",)))
    return its


def on_demand_by_price(its):
    od = [it for it in its if it["offerings"][0]["capacityType"] == "on-demand"]
    return sorted(od, key=lambda it: it["offerings"][0]["price"])


def node_of_type(name, it, pods_, cost):
    of = it["offerings"][0]
    n = fx.state_node(name, it["name"], zone=of["zone"], capacity_type=of["capacityType"], allocatable={"cpu": "32", "memory": "64Gi", "pods": "100"}, pods_=pods_)
    n["candidate"] = True
    n["disruptionCost"] = cost
    return n


def price_of(its, idx):
    return its[idx]["offerings"][0]["price"]


CASES = []


def case(ref):
    def deco(fn):
        CASES.append((fn.__name__, ref, fn))
        return fn
    return deco


@case("deprovisioning/suite_test.go:874-929")
def can_replace_an_expensive_node():
    its = assorted()
    worst = on_demand_by_price(its)[-1]
    node = node_of_type("node-a", worst, [fx.pod(nodeName="node-a", labels={"app": "test"})], 1.0)
    prob = fx.problem([], instance_types=its, nodes=[node])

    def check(probe, search):
        action, options = probe(1)
        assert action == 2 and options
        assert all(price_of(its, i) < worst["offerings"][0]["price"] for i in options)  # filterByPrice, helpers.go:148-157
        assert all(its[i]["name"] != worst["name"] for i in options)
        assert search()["action"] == 0  # the multi-node search needs at least two candidates (multinodeconsolidation.go:44-48)
    return prob, check


@case("deprovisioning/suite_test.go:1155-1241")
def no_replacement_when_a_spot_offering_could_cost_more():
    current = fx.instance_type("current-on-demand", offerings=[{"capacityType": "on-demand", "zone": "test-zone-1a", "price": 0.5, "available": False}])
    repl = fx.instance_type("potential-spot-replacement", offerings=[
        {"capacityType": "spot", "zone": "test-zone-1a", "price": 1.0, "available": True},
        {"capacityType": "spot", "zone": "test-zone-1b", "price": 0.2, "available": True},
        {"capacityType": "spot", "zone": "test-zone-1c", "price": 0.4, "available": True}])
    its = [current, repl]
    node = fx.state_node("node-a", "current-on-demand", zone="test-zone-1a", capacity_type="on-demand", allocatable={"cpu": "32", "memory": "64Gi", "pods": "100"},
                         pods_=[fx.pod(nodeName="node-a", labels={"app": "test"})])
    node["candidate"] = True
    node["disruptionCost"] = 1.0
    prob = fx.problem([], instance_types=its, nodes=[node])

    def check(probe, search):
        action, options = probe(1)
        assert action == 0 and options == []  # worst-case spot price 1.0 is not below the current 0.5 (helpers.go:292-315)
    return prob, check


@case("deprovisioning/suite_test.go:1243-1345")
def no_replacement_when_on_demand_costs_more():
    current = fx.instance_type("current-on-demand", offerings=[{"capacityType": "on-demand", "zone": "test-zone-1a", "price": 0.5, "available": False}])
    repl = fx.instance_type("on-demand-replacement", offerings=[
        {"capacityType": "on-demand", "zone": "test-zone-1a", "price": 0.6, "available": True},
        {"capacityType": "on-demand", "zone": "test-zone-1b", "price": 0.6, "available": False},
        {"capacityType": "spot", "zone": "test-zone-1b", "price": 0.2, "available": True},
        {"capacityType": "spot", "zone": "test-zone-1c", "price": 0.3, "available": True}])
    its = [current, repl]
    node = fx.state_node("node-a", "current-on-demand", zone="test-zone-1a", capacity_type="on-demand", allocatable={"cpu": "32", "memory": "64Gi", "pods": "100"},
                         pods_=[fx.pod(nodeName="node-a", labels={"app": "test"})])
    node["candidate"] = True
    node["disruptionCost"] = 1.0
    # the provisioner only allows on-demand, so the replacement would be the 0.6 on-demand offering
    pr = fx.provisioner(requirements=[{"key": CAPACITY_TYPE, "operator": "In", "values": ["on-demand"]}])
    prob = fx.problem([], instance_types=its, provisioners=[pr], nodes=[node])

    def check(probe, search):
        action, options = probe(1)
        assert action == 0 and options == []
    return prob, check


@case("deprovisioning/suite_test.go:1423-1496")
def can_delete_a_node_whose_pods_fit_elsewhere():
    its = assorted()
    cheap = on_demand_by_price(its)[0]
    n1 = node_of_type("node-1", cheap, [fx.pod(nodeName="node-1", labels={"app": "test"})], 1.0)
    n2 = node_of_type("node-2", cheap, [fx.pod(nodeName="node-2", labels={"app": "test"}), fx.pod(nodeName="node-2", labels={"app": "test"})], 2.0)
    n2["candidate"] = False
    prob = fx.problem([], instance_types=its, nodes=[n1, n2])

    def check(probe, search):
        action, options = probe(1)
        assert action == 1 and options == []  # delete: the pod fits on node-2 (consolidation.go:230-236)
    return prob, check


@case("deprovisioning/suite_test.go:2555-2643")
def can_merge_three_nodes_into_one():
    its = assorted()
    worst = on_demand_by_price(its)[-1]
    nodes = [node_of_type(f"node-{i}", worst, [fx.pod(nodeName=f"node-{i}", labels={"app": "test"})], 1.0 + i) for i in range(3)]
    prob = fx.problem([], instance_types=its, nodes=nodes)

    def check(probe, search):
        out = search()
        assert out["action"] == 2 and out["nodes_removed"] == 3 and out["options"]
        total = 3 * worst["offerings"][0]["price"]
        assert all(price_of(its, i) < total for i in out["options"])
        assert out["probes"] == [2, 3]  # binary search over [1, 2]: first two candidates, then all three
    return prob, check


@case("deprovisioning/suite_test.go:2644-2719")
def will_not_merge_two_nodes_into_one_of_the_same_type():
    its = assorted()
    cheap = on_demand_by_price(its)[0]
    n1 = node_of_type("node-1", cheap, [fx.pod(nodeName="node-1", labels={"app": "test"})], 1.0)
    n2 = node_of_type("node-2", cheap, [fx.pod(nodeName="node-2", labels={"app": "test"}), fx.pod(nodeName="node-2", labels={"app": "test"})], 2.0)
    prob = fx.problem([], instance_types=its, nodes=[n1, n2])

    def check(probe, search):
        out = search()
        # [delete cheap, delete cheap, launch the same cheap type] is filtered out (filterOutSameType, multinodeconsolidation.go:132-165)
        assert out["action"] == 0 and out["nodes_removed"] == 0
        assert probe(1) == (1, [])  # deleting the node with the fewest pods alone is the valid single-node action
    return prob, check


# ---- cases added after the round's GPU budget was spent: pinned on the oracle (CPU); the GPU parametrisation of
# tests/test_gpu_parity.py takes CASES only, these join it once they have been run on the GPU.
CPU_ONLY_CASES = []


def cpu_case(ref):
    def deco(fn):
        CPU_ONLY_CASES.append((fn.__name__, ref, fn))
        return fn
    return deco


def _in_zone(its, zone, cheapest=True):
    od = [it for it in on_demand_by_price(its) if it["offerings"][0]["zone"] == zone]
    return od[0] if cheapest else od[-1]


def _small_node(name, it, zone, pods_, cost):
    of = it["offerings"][0]
    n = fx.state_node(name, it["name"], zone=zone, capacity_type=of["capacityType"], allocatable={"cpu": "1", "memory": "64Gi", "pods": "100"}, pods_=pods_)
    n["candidate"] = True
    n["disruptionCost"] = cost
    return n


@cpu_case("deprovisioning/suite_test.go:1828-1934")
def replacement_keeps_the_zonal_spread():
    """three one-pod nodes in three zones, the zone-2 node is the most expensive: its replacement must stay in zone 2"""
    its = assorted()
    labels = {"app": "test-zonal-spread"}
    spread = [fx.spread(ZONE, labels)]
    types = [_in_zone(its, "test-zone-1"), _in_zone(its, "test-zone-2", cheapest=False), _in_zone(its, "test-zone-3")]
    nodes = []
    for i, (it, zone) in enumerate(zip(types, ZONES)):
        bound = [fx.pod({"cpu": "1"}, labels=labels, topologySpreadConstraints=spread, nodeName=f"node-{i}")]
        nodes.append(_small_node(f"node-{i}", it, zone, bound, 1.0 if i == 1 else 5.0 + i))  # the zone-2 node is the cheapest to disrupt
    prob = fx.problem([], instance_types=its, nodes=nodes)

    def check(probe, search):
        action, options = probe(1)
        assert action == 2 and options
        assert all(its[i]["offerings"][0]["zone"] == "test-zone-2" for i in options)
        assert all(price_of(its, i) < types[1]["offerings"][0]["price"] for i in options)
        assert probe(2)[0] == 0  # two pods of the spread would need two new nodes in two zones: not a consolidation
    return prob, check


@cpu_case("deprovisioning/suite_test.go:1936-2029")
def nothing_to_do_when_deletion_would_violate_anti_affinity():
    its = assorted()
    labels = {"app": "test"}
    anti = {"required": [fx.affinity_term(fx.HOSTNAME, labels)]}
    nodes = []
    for i, zone in enumerate(ZONES):
        bound = [fx.pod({"cpu": "1"}, labels=labels, podAntiAffinity=anti, nodeName=f"node-{i}")]
        nodes.append(_small_node(f"node-{i}", _in_zone(its, zone), zone, bound, 1.0 + i))
    prob = fx.problem([], instance_types=its, nodes=nodes)

    def check(probe, search):
        for count in (1, 2, 3):
            assert probe(count)[0] == 0  # already the cheapest types; moving a pod onto a sibling's node violates the anti-affinity
        assert search()["action"] == 0
    return prob, check


@cpu_case("deprovisioning/suite_test.go:2142-2191")
def pending_pods_take_part_in_the_simulation():
    """a pending 125-cpu pod only fits the big expensive node: removing that node would strand it, so nothing is consolidated"""
    its = assorted()
    worst = on_demand_by_price(its)[-1]
    of = worst["offerings"][0]

    def cluster():
        n = fx.state_node("node-a", worst["name"], zone=of["zone"], capacity_type=of["capacityType"],
                          allocatable={"cpu": "128", "memory": "512Gi", "pods": "100"}, pods_=[fx.pod({"cpu": "1"}, nodeName="node-a")])
        n["candidate"] = True
        n["disruptionCost"] = 1.0
        return n
    with_pending = fx.problem([fx.pod({"cpu": "125"})], instance_types=its, nodes=[cluster()])

    def check(probe, search):
        assert probe(1)[0] == 0
    # the same cluster without the pending pod is consolidatable: checked through a second problem below
    return with_pending, check


@cpu_case("deprovisioning/suite_test.go:2142-2191 (control)")
def without_the_pending_pod_the_node_is_replaced():
    its = assorted()
    worst = on_demand_by_price(its)[-1]
    of = worst["offerings"][0]
    n = fx.state_node("node-a", worst["name"], zone=of["zone"], capacity_type=of["capacityType"],
                      allocatable={"cpu": "128", "memory": "512Gi", "pods": "100"}, pods_=[fx.pod({"cpu": "1"}, nodeName="node-a")])
    n["candidate"] = True
    n["disruptionCost"] = 1.0
    prob = fx.problem([], instance_types=its, nodes=[n])

    def check(probe, search):
        action, options = probe(1)
        assert action == 2 and options
    return prob, check


@cpu_case("deprovisioning/helpers.go:106-113 (simulateScheduling walks every ExistingNode Solve returns)")
def an_idle_uninitialised_node_blocks_every_command():
    """The expensive node could be replaced (control case above), but another owned node of the cluster is not initialised yet:
    simulateScheduling reports allPodsScheduled == false even though no pod would land on that node."""
    its = assorted()
    worst = on_demand_by_price(its)[-1]
    of = worst["offerings"][0]
    n = fx.state_node("node-a", worst["name"], zone=of["zone"], capacity_type=of["capacityType"],
                      allocatable={"cpu": "128", "memory": "512Gi", "pods": "100"}, pods_=[fx.pod({"cpu": "1"}, nodeName="node-a")])
    n["candidate"] = True
    n["disruptionCost"] = 1.0
    # too small for the pod (cpu 500m) and not a candidate: it only matters through its missing karpenter.sh/initialized label
    idle = fx.state_node("node-b", its[0]["name"], zone=its[0]["offerings"][0]["zone"], capacity_type=its[0]["offerings"][0]["capacityType"],
                         allocatable={"cpu": "500m", "memory": "1Gi", "pods": "100"}, initialized=False)
    prob = fx.problem([], instance_types=its, nodes=[n, idle])

    def check(probe, search):
        assert probe(1) == (0, [])
    return prob, check
