"""Known-answer scheduling cases restated from the reference's own test suites (SURVEY.md 8c). Each case builds a
problem with the reference's fixtures (tests/fixtures.py) and checks the ORDER-FREE invariant the Go test asserts
(node count, chosen instance type, skew multiset, scheduled / not scheduled, same / different node).

Used twice: on CPU against the oracle (pins the oracle), and on the GPU where the CUDA path must reproduce the
oracle bit-for-bit AND satisfy the same invariant."""
import fixtures as fx
from fixtures import ARCH, CAPACITY_TYPE, HOSTNAME, INSTANCE_TYPE, ZONE, ZONES, pod, pods, problem, provisioner

CASES = []


def case(ref):
    def deco(fn):
        CASES.append((fn.__name__, ref, fn))
        return fn
    return deco


def scheduled(res, i):
    return res["assign"][i] >= 0


def each_alone(pod_list, expect, **kw):
    """the Go tests provision these pods in separate specs: one Solve per pod"""
    prob = {"multi": [problem([p], **kw) for p in pod_list]}

    def check(results):
        got = [r["assign"][0] >= 0 for r in results]
        assert got == expect, (got, expect)
    return prob, check


def new_nodes_used(res):
    ne = len(res["existing"])
    return sorted({a - ne for a in res["assign"] if a >= ne})


def launched_type(prob, res, pod_index):
    ne = len(res["existing"])
    return fx.launch(prob, res["newNodes"][res["assign"][pod_index] - ne])[1]


# ------------------------------------------------------------------ bin packing (scheduling/suite_test.go:1079-1340)
@case("suite_test.go:1079-1089")
def small_pod_smallest_instance():
    prob = problem([pod({"memory": "100M"})])

    def check(res):
        assert scheduled(res, 0)
        assert launched_type(prob, res, 0) == "small-instance-type"
    return prob, check


@case("suite_test.go:1101-1118")
def five_small_pods_one_node():
    prob = problem(pods(5, requests={"memory": "10M"}))

    def check(res):
        assert all(scheduled(res, i) for i in range(5))
        assert len(set(res["assign"])) == 1
        assert launched_type(prob, res, 0) == "small-instance-type"
    return prob, check


@case("suite_test.go:1119-1137")
def forty_large_pods_twenty_nodes():
    prob = problem(pods(40, requests={"memory": "1.8G"}, nodeSelector={ARCH: "amd64"}))

    def check(res):
        assert all(a >= 0 for a in res["assign"])
        assert len(set(res["assign"])) == 20
        assert {launched_type(prob, res, i) for i in range(40)} == {"default-instance-type"}
    return prob, check


@case("suite_test.go:1138-1169")
def small_and_large_pods_pack_together():
    prob = problem(pods(40, requests={"memory": "1.8G"}, nodeSelector={ARCH: "amd64"}) +
                   pods(20, requests={"memory": "400M"}, nodeSelector={ARCH: "amd64"}))

    def check(res):
        assert all(a >= 0 for a in res["assign"])
        assert len(set(res["assign"])) == 20
        assert {launched_type(prob, res, i) for i in range(60)} == {"default-instance-type"}
    return prob, check


@case("suite_test.go:1170-1192")
def pack_new_nodes_tightly():
    prob = problem([pod({"cpu": "4.5"}), pod({"cpu": "1"})], instance_types=fx.fake_instance_types(5))

    def check(res):
        assert scheduled(res, 0) and scheduled(res, 1)
        assert res["assign"][0] != res["assign"][1]
        assert launched_type(prob, res, 0) != launched_type(prob, res, 1)
    return prob, check


@case("suite_test.go:1193-1204")
def zero_quantity_unknown_resource():
    prob = problem([{"name": "p", "uid": "p", "containers": [{"requests": {"foo.com/weird-resources": "0"}, "limits": {"foo.com/weird-resources": "0"}}]}])
    return prob, lambda res: scheduled(res, 0) or (_ for _ in ()).throw(AssertionError("not scheduled"))


@case("suite_test.go:1205-1214")
def exceeds_every_instance_type():
    prob = problem([pod({"memory": "2Ti"})])

    def check(res):
        assert not scheduled(res, 0)
        assert res["newNodes"] == []
    return prob, check


@case("suite_test.go:1215-1235")
def pod_count_limit_per_node():
    prob = problem(pods(25, requests={"memory": "1m", "cpu": "1m"}, nodeSelector={ARCH: "amd64"}))

    def check(res):
        assert all(a >= 0 for a in res["assign"])
        assert len(set(res["assign"])) == 5
        assert {launched_type(prob, res, i) for i in range(25)} == {"small-instance-type"}
    return prob, check


@case("suite_test.go:1236-1274")
def init_container_max_counts():
    fits = {"name": "a", "uid": "a", "containers": [{"requests": {"memory": "1Gi", "cpu": "1"}}], "initContainers": [{"requests": {"memory": "2Gi", "cpu": "2"}}]}
    too_big = {"name": "b", "uid": "b", "containers": [{"requests": {"memory": "1Gi"}}], "initContainers": [{"requests": {"memory": "1Ti"}}]}
    prob = problem([fits, too_big])

    def check(res):
        assert scheduled(res, 0) and not scheduled(res, 1)
        assert res["newNodes"][0]["requests"]["memory"] == 2 * 1024 ** 3 * 1000 + 0  # ceiling of init container
    return prob, check


# ------------------------------------------------------------------ custom labels (suite_test.go:401-551)
def _req(key, op, *values):
    return {"nodeAffinity": {"required": [[{"key": key, "operator": op, "values": list(values)}]]}}


@case("suite_test.go:401-434")
def undefined_custom_key_operators():
    return each_alone([pod(**_req("test-key", "In", "test-value")), pod(**_req("test-key", "NotIn", "test-value")),
                       pod(**_req("test-key", "Exists")), pod(**_req("test-key", "DoesNotExist"))], [False, True, False, True])


@case("suite_test.go:443-506")
def defined_custom_key_operators():
    pr = provisioner(labels={"test-key": "test-value"})
    return each_alone([pod(**_req("test-key", "In", "test-value")), pod(**_req("test-key", "NotIn", "test-value")),
                       pod(**_req("test-key", "Exists")), pod(**_req("test-key", "DoesNotExist")),
                       pod(**_req("test-key", "In", "another-value")), pod(**_req("test-key", "NotIn", "another-value"))],
                      [True, False, True, False, False, True], provisioners=[pr])


@case("suite_test.go:507-540")
def compatible_pods_share_incompatible_split():
    pr = provisioner(requirements=[{"key": "test-key", "operator": "In", "values": ["test-value", "another-value"]}])
    same = problem([pod(**_req("test-key", "In", "test-value")), pod(**_req("test-key", "NotIn", "another-value"))], provisioners=[pr])
    diff = problem([pod(**_req("test-key", "In", "test-value")), pod(**_req("test-key", "In", "another-value"))], provisioners=[pr])
    prob = {"multi": [same, diff]}

    def check(results):
        a, b = results
        assert a["assign"][0] == a["assign"][1] and a["assign"][0] >= 0
        assert b["assign"][0] != b["assign"][1] and min(b["assign"]) >= 0
    return prob, check


@case("suite_test.go:115-202")
def node_selectors_and_provisioner_constraints():
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1"]}])
    return each_alone([pod(), pod(nodeSelector={ZONE: "unknown"}), pod(nodeSelector={ZONE: "test-zone-2"}), pod(nodeSelector={ZONE: "test-zone-1"}),
                       pod(nodeSelector={HOSTNAME: "red-node"})], [True, False, False, True, False], provisioners=[pr])


# ------------------------------------------------------------------ preferential fallback (suite_test.go:555-675)
@case("suite_test.go:557-572")
def final_required_term_is_not_relaxed():
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1"]},
                                   {"key": INSTANCE_TYPE, "operator": "In", "values": ["default-instance-type"]}])
    prob = problem([pod(nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["invalid"]}]]})], provisioners=[pr])
    return prob, lambda res: (not scheduled(res, 0)) or (_ for _ in ()).throw(AssertionError("scheduled"))


@case("suite_test.go:573-595")
def relax_multiple_required_terms():
    terms = [[{"key": ZONE, "operator": "In", "values": [z]}] for z in ("invalid", "invalid", "test-zone-1", "test-zone-2")]
    prob = problem([pod(nodeAffinity={"required": terms})])

    def check(res):
        assert scheduled(res, 0)
        assert res["relax"][0] == 2
        assert res["newNodes"][0]["requirements"][ZONE] == "In [test-zone-1]"
    return prob, check


@case("suite_test.go:616-642")
def relax_to_lighter_preferences():
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-2"]}])
    pref = [{"weight": 100, "terms": [{"key": INSTANCE_TYPE, "operator": "In", "values": ["test-zone-3"]}]},
            {"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": ["test-zone-2"]}]},
            {"weight": 1, "terms": [{"key": ZONE, "operator": "In", "values": ["test-zone-1"]}]}]
    prob = problem([pod(nodeAffinity={"preferred": pref})], provisioners=[pr])

    def check(res):
        assert scheduled(res, 0)
        assert res["relax"][0] == 1
        assert res["newNodes"][0]["requirements"][ZONE] == "In [test-zone-2]"
    return prob, check


# ------------------------------------------------------------------ instance selection (suite_test.go:676-862)
@case("suite_test.go:688-707")
def different_archs_different_instances():
    prob = problem([pod(nodeSelector={ARCH: "amd64"}), pod(nodeSelector={ARCH: "arm64"})])

    def check(res):
        assert res["assign"][0] != res["assign"][1] and min(res["assign"]) >= 0
        assert launched_type(prob, res, 1) == "arm-instance-type"
    return prob, check


@case("suite_test.go:708-726")
def instance_type_node_affinity_excludes_types():
    prob = problem([pod(nodeAffinity={"required": [[{"key": INSTANCE_TYPE, "operator": "In", "values": ["arm-instance-type"]}]]}),
                    pod(nodeSelector={INSTANCE_TYPE: "small-instance-type"})])

    def check(res):
        assert min(res["assign"]) >= 0 and res["assign"][0] != res["assign"][1]
        its = prob["instanceTypes"]
        assert [its[i]["name"] for i in res["newNodes"][res["assign"][0]]["options"]] == ["arm-instance-type"]
        assert [its[i]["name"] for i in res["newNodes"][res["assign"][1]]["options"]] == ["small-instance-type"]
    return prob, check


@case("suite_test.go:820-861")
def resources_not_on_a_single_type():
    prob = problem([pod({"fake.com/vendor-a": "1"}), pod({"fake.com/vendor-b": "1"}), pod({"fake.com/vendor-a": "1", "fake.com/vendor-b": "1"})])

    def check(res):
        assert scheduled(res, 0) and scheduled(res, 1) and not scheduled(res, 2)
        assert res["assign"][0] != res["assign"][1]
    return prob, check


# ------------------------------------------------------------------ taints (topology_test.go:2209-2257, provisioning/suite_test.go:583-622)
@case("topology_test.go:2209-2257")
def taints_and_tolerations():
    pr = provisioner(taints=[{"key": "test-key", "value": "test-value", "effect": "NoSchedule"}])
    tol = lambda **kw: {"tolerations": [kw]}
    return each_alone([pod(), pod(**tol(key="test-key", operator="Equal", value="test-value", effect="NoSchedule")),
                       pod(**tol(key="test-key", operator="Exists")), pod(**tol(operator="Exists")),
                       pod(**tol(key="test-key", operator="Equal", value="other", effect="NoSchedule")),
                       pod(**tol(key="test-key", operator="Exists", effect="NoExecute"))], [False, True, True, True, False, False], provisioners=[pr])


# ------------------------------------------------------------------ host ports (suite_test.go:923-1078)
@case("suite_test.go:923-1078")
def host_ports():
    hp = lambda port, ip="", proto="TCP": {"ports": [{"hostPort": port, "hostIP": ip, "protocol": proto}], "requests": {"cpu": "10m"}}
    same = problem([pod(**hp(80)), pod(**hp(80))])
    wildcard = problem([pod(**hp(80, "1.2.3.4")), pod(**hp(80, "0.0.0.0"))])
    proto = problem([pod(**hp(80, proto="TCP")), pod(**hp(80, proto="UDP"))])
    ips = problem([pod(**hp(80, "1.2.3.4")), pod(**hp(80, "1.2.3.5"))])
    prob = {"multi": [same, wildcard, proto, ips]}

    def check(results):
        a, b, c, d = results
        assert a["assign"][0] != a["assign"][1]
        assert b["assign"][0] != b["assign"][1]
        assert c["assign"][0] == c["assign"][1]
        assert d["assign"][0] == d["assign"][1]
    return prob, check


# ------------------------------------------------------------------ limits (provisioning/suite_test.go:237-358)
@case("provisioning/suite_test.go:237-358")
def provisioner_cpu_limits():
    pr = provisioner(limits={"cpu": "20"})
    # default-instance-type has 4 cpu: five nodes exhaust the limit pessimistically (subtractMax uses the largest option)
    prob = problem(pods(12, requests={"cpu": "3"}, nodeSelector={ARCH: "amd64", INSTANCE_TYPE: "default-instance-type"}), provisioners=[pr])

    def check(res):
        assert sum(1 for a in res["assign"] if a >= 0) == 5
        assert len(res["newNodes"]) == 5
    return prob, check


# ------------------------------------------------------------------ node affinity: requirements x preferences (suite_test.go:231-346, 643-676)
def _r(key, op, *values):
    return {"key": key, "operator": op, "values": list(values)}


def _node_aff(required=None, preferred=None, **kw):
    na = {}
    if required is not None:
        na["required"] = [required]
    if preferred is not None:
        na["preferred"] = [{"weight": 1, "terms": preferred}]
    return pod(nodeAffinity=na, **kw)


def _zone_of(prob, res):
    return fx.launch(prob, res["newNodes"][res["assign"][0] - len(res["existing"])])[2]


@case("suite_test.go:231-308")
def node_affinity_requirements_and_preferences_on_zone():
    all3u = list(ZONES) + ["unknown"]
    cases = [
        (_node_aff([_r(ZONE, "In", "unknown")]), None),                                                     # :231 not scheduled
        (_node_aff([_r(ZONE, "NotIn", "test-zone-1", "test-zone-2", "unknown")]), "test-zone-3"),             # :240
        (_node_aff([_r(ZONE, "NotIn", *all3u)]), None),                                                      # :250 not scheduled
        (_node_aff([_r(ZONE, "In", *all3u)], [_r(ZONE, "In", "test-zone-2", "unknown")]), "test-zone-2"),    # :260
        (_node_aff([_r(ZONE, "In", *all3u)], [_r(ZONE, "In", "unknown")]), "any"),                          # :273 preference relaxed
        (_node_aff([_r(ZONE, "In", *all3u)], [_r(ZONE, "NotIn", "test-zone-1", "test-zone-3")]), "test-zone-2"),  # :285
        (_node_aff([_r(ZONE, "In", *all3u)], [_r(ZONE, "NotIn", *ZONES)]), "any"),                          # :298 preference relaxed
    ]
    probs = [problem([p]) for p, _ in cases]

    def check(results):
        for (p, want), prob, res in zip(cases, probs, results):
            if want is None:
                assert res["assign"] == [-1], want
            else:
                assert res["assign"][0] >= 0
                if want != "any":
                    assert _zone_of(prob, res) == want
    return {"multi": probs}, check


@case("suite_test.go:310-346")
def node_selectors_preferences_and_requirements_combine():
    p1 = _node_aff([_r(ZONE, "In", *ZONES)], [_r(ZONE, "In", *ZONES)], nodeSelector={ZONE: "test-zone-3"})
    p2 = _node_aff([_r(ZONE, "In", "test-zone-1", "test-zone-3"), _r(INSTANCE_TYPE, "In", "default-instance-type", "arm-instance-type")],
                   [_r(ZONE, "NotIn", "unknown"), _r(INSTANCE_TYPE, "NotIn", "unknown")],
                   nodeSelector={ZONE: "test-zone-3", INSTANCE_TYPE: "arm-instance-type"})
    probs = [problem([p1]), problem([p2])]

    def check(results):
        assert _zone_of(probs[0], results[0]) == "test-zone-3"
        assert _zone_of(probs[1], results[1]) == "test-zone-3"
        node = results[1]["newNodes"][results[1]["assign"][0]]
        assert fx.launch(probs[1], node)[1] == "arm-instance-type"
    return {"multi": probs}, check


@case("suite_test.go:643-676")
def conflicting_preferences_do_not_block_scheduling():
    p1 = _node_aff([_r(ZONE, "In", "test-zone-3")], [_r(ZONE, "NotIn", "test-zone-3")])
    p2 = _node_aff(None, [_r(ZONE, "In", "invalid"), _r(ZONE, "NotIn", "invalid")])
    probs = [problem([p1]), problem([p2])]

    def check(results):
        assert _zone_of(probs[0], results[0]) == "test-zone-3"
        assert results[1]["assign"][0] >= 0
    return {"multi": probs}, check


# ------------------------------------------------------------------ instance type compatibility (suite_test.go:727-819)
@case("suite_test.go:727-759")
def provisioner_arch_excludes_the_only_fitting_types():
    pr = provisioner(requirements=[{"key": ARCH, "operator": "In", "values": ["amd64"]}])
    ios = _node_aff([_r("kubernetes.io/os", "In", "ios")])          # only the arm type runs ios
    big = pod({"cpu": "14"})                                           # only the arm type has 14 cpus
    return each_alone([ios, big], [False, False], provisioners=[pr])


@case("suite_test.go:760-819")
def different_selectors_different_instances():
    pr = provisioner(requirements=[{"key": ARCH, "operator": "In", "values": ["arm64", "amd64"]}])
    by_os = problem([pod(nodeSelector={"kubernetes.io/os": "linux"}), pod(nodeSelector={"kubernetes.io/os": "windows"})], provisioners=[pr])
    by_type = problem([pod(nodeSelector={"beta.kubernetes.io/instance-type": "small-instance-type"}),
                       pod(nodeSelector={INSTANCE_TYPE: "default-instance-type"})], provisioners=[pr])
    by_zone = problem([pod(nodeSelector={ZONE: "test-zone-1"}), pod(nodeSelector={ZONE: "test-zone-2"})], provisioners=[pr])

    def check(results):
        for res in results:
            assert min(res["assign"]) >= 0 and len(set(res["assign"])) == 2
    return {"multi": [by_os, by_type, by_zone]}, check


# ------------------------------------------------------------------ topology spread (topology_test.go:65-490)
@case("topology_test.go:66-80")
def zonal_spread_four_pods():
    labels = {"test": "test"}
    prob = problem(pods(4, labels=labels, topologySpreadConstraints=[fx.spread(ZONE, labels)]))
    return prob, lambda res: _eq(fx.skew(prob, res, ZONE), [1, 1, 2])


@case("topology_test.go:124-160")
def zonal_spread_with_existing_pod_in_excluded_zone():
    """provisioner limited to zone-1/2, one matching pod already runs in zone-3: at most two per zone fit max skew 1"""
    labels = {"test": "test"}
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-2"]}])
    existing = fx.state_node("node-z3", "small-instance-type", zone="test-zone-3", allocatable={"cpu": "1900m", "memory": "2038Mi", "pods": "5"},
                             pods_=[pod({"cpu": "1.1"}, labels=labels, nodeName="node-z3")])
    prob = problem(pods(6, requests={"cpu": "1.1"}, labels=labels, topologySpreadConstraints=[fx.spread(ZONE, labels)]), provisioners=[pr],
                   nodes=[existing])

    def check(res):
        assert sum(1 for a in res["assign"] if a >= 0) == 4
        assert fx.skew(prob, res, ZONE) == [2, 2]  # plus the existing pod in zone-3 -> (1, 2, 2)
    return prob, check


@case("topology_test.go:381-394")
def hostname_spread_max_skew_one():
    labels = {"test": "test"}
    prob = problem(pods(4, labels=labels, topologySpreadConstraints=[fx.spread(HOSTNAME, labels)]))
    return prob, lambda res: _eq(fx.skew(prob, res, HOSTNAME), [1, 1, 1, 1])


@case("topology_test.go:396-410")
def hostname_spread_max_skew_four():
    labels = {"test": "test"}
    prob = problem(pods(4, labels=labels, topologySpreadConstraints=[fx.spread(HOSTNAME, labels, max_skew=4)]))
    return prob, lambda res: _eq(fx.skew(prob, res, HOSTNAME), [4])


@case("topology_test.go:412-445")
def two_deployments_hostname_spread_two_nodes():
    a, b = {"app": "a"}, {"app": "b"}
    prob = problem(pods(2, labels=a, topologySpreadConstraints=[fx.spread(HOSTNAME, a)]) +
                   pods(2, labels=b, topologySpreadConstraints=[fx.spread(HOSTNAME, b)]))

    def check(res):
        assert min(res["assign"]) >= 0
        assert len(set(res["assign"])) == 2
    return prob, check


@case("topology_test.go:341-352")
def nil_selector_spread_schedules():
    cons = [{"maxSkew": 1, "topologyKey": ZONE, "whenUnsatisfiable": "DoNotSchedule", "labelSelector": None}]
    prob = problem(pods(2, labels={"test": "test"}, topologySpreadConstraints=cons))
    return prob, lambda res: _eq([a >= 0 for a in res["assign"]], [True, True])


@case("topology_test.go:ScheduleAnyway relaxation")
def schedule_anyway_spread_is_relaxed():
    labels = {"test": "test"}
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1"]}])
    prob = problem(pods(3, labels=labels, topologySpreadConstraints=[fx.spread(ZONE, labels, when="ScheduleAnyway")]), provisioners=[pr])

    def check(res):
        assert all(a >= 0 for a in res["assign"])
    return prob, check


@case("topology_test.go:82-104")
def zonal_spread_match_expressions():
    sel = {"matchExpressions": [{"key": "test", "operator": "In", "values": ["test"]}]}
    cons = [{"maxSkew": 1, "topologyKey": ZONE, "whenUnsatisfiable": "DoNotSchedule", "labelSelector": sel}]
    prob = problem(pods(4, labels={"test": "test"}, topologySpreadConstraints=cons))
    return prob, lambda res: _eq(fx.skew(prob, res, ZONE), [1, 1, 2])


@case("topology_test.go:106-122")
def zonal_spread_respects_provisioner_zones():
    labels = {"test": "test"}
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": list(ZONES)}])
    prob = problem(pods(4, labels=labels, topologySpreadConstraints=[fx.spread(ZONE, labels)]), provisioners=[pr])
    return prob, lambda res: _eq(fx.skew(prob, res, ZONE), [1, 1, 2])


@case("topology_test.go:492-506")
def capacity_type_spread():
    labels = {"test": "test"}
    prob = problem(pods(4, labels=labels, topologySpreadConstraints=[fx.spread(CAPACITY_TYPE, labels)]))
    return prob, lambda res: _eq(fx.skew(prob, res, CAPACITY_TYPE), [2, 2])


@case("topology_test.go:508-524")
def capacity_type_spread_respects_provisioner():
    labels = {"test": "test"}
    pr = provisioner(requirements=[{"key": CAPACITY_TYPE, "operator": "In", "values": ["spot", "on-demand"]}])
    prob = problem(pods(4, labels=labels, topologySpreadConstraints=[fx.spread(CAPACITY_TYPE, labels)]), provisioners=[pr])
    return prob, lambda res: _eq(fx.skew(prob, res, CAPACITY_TYPE), [2, 2])


@case("topology_test.go:785-802")
def zone_and_hostname_spread_first_batch():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels), fx.spread(HOSTNAME, labels, max_skew=3)]
    prob = problem(pods(2, labels=labels, topologySpreadConstraints=cons))

    def check(res):
        assert fx.skew(prob, res, ZONE) == [1, 1]
        assert max(fx.skew(prob, res, HOSTNAME)) <= 3
    return prob, check


@case("topology_test.go:785-823 (eleven pods in one batch)")
def zone_and_hostname_spread_eleven_pods():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels), fx.spread(HOSTNAME, labels, max_skew=3)]
    prob = problem(pods(11, labels=labels, topologySpreadConstraints=cons))

    def check(res):
        assert all(a >= 0 for a in res["assign"])
        assert fx.skew(prob, res, ZONE) == [3, 4, 4]
        assert max(fx.skew(prob, res, HOSTNAME)) <= 3
    return prob, check


@case("topology_test.go:1031-1055")
def spread_options_limited_by_node_selector():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels)]
    prob = problem(pods(5, labels=labels, topologySpreadConstraints=cons, nodeSelector={ZONE: "test-zone-1"}) +
                   pods(10, labels=labels, topologySpreadConstraints=cons, nodeSelector={ZONE: "test-zone-2"}))
    return prob, lambda res: _eq(fx.skew(prob, res, ZONE), [5, 10])


# ------------------------------------------------------------------ pod affinity / anti-affinity (topology_test.go:1195-2207)
@case("topology_test.go:1503-1530")
def hostname_anti_affinity_splits_nodes():
    labels = {"security": "s2"}
    prob = problem(pods(3, labels=labels, podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, labels)]}))

    def check(res):
        assert min(res["assign"]) >= 0 and len(set(res["assign"])) == 3
    return prob, check


@case("topology_test.go:1713-1744")
def schroedinger_zonal_anti_affinity():
    """A zone-unconstrained pod with required zonal anti-affinity blocks every zone it might land in."""
    labels = {"security": "s2"}
    anti = pod(labels=labels, podAntiAffinity={"required": [fx.affinity_term(ZONE, labels)]})
    target = pod(labels=labels)
    prob = problem([anti, target])

    def check(res):
        assert scheduled(res, 0)
        assert not scheduled(res, 1)
    return prob, check


@case("topology_test.go:1195-1250")
def self_affinity_hostname_same_node():
    labels = {"security": "s2"}
    prob = problem(pods(3, labels=labels, podAffinity={"required": [fx.affinity_term(HOSTNAME, labels)]}))

    def check(res):
        assert min(res["assign"]) >= 0 and len(set(res["assign"])) == 1
    return prob, check


@case("topology_test.go:1300-1340")
def zonal_affinity_follows_target():
    target_labels = {"security": "s2"}
    target = pod(labels=target_labels, nodeSelector={ZONE: "test-zone-2"})
    followers = pods(3, podAffinity={"required": [fx.affinity_term(ZONE, target_labels)]})
    prob = problem([target] + followers)

    def check(res):
        assert min(res["assign"]) >= 0
        ne = len(res["existing"])
        for i in range(4):
            assert res["newNodes"][res["assign"][i] - ne]["requirements"][ZONE] == "In [test-zone-2]"
    return prob, check


# ------------------------------------------------------------------ existing / in-flight nodes (suite_test.go:1343-1893)
@case("topology_test.go:1205-1237")
def pod_affinity_hostname_with_spread_noise():
    labels, aff = {"test": "test"}, {"security": "s2"}
    noise = pods(10, labels=labels, topologySpreadConstraints=[fx.spread(HOSTNAME, labels)])
    target = pod(labels=aff)
    follower = pod(podAffinity={"required": [fx.affinity_term(HOSTNAME, aff)]})
    prob = problem(noise + [target, follower])

    def check(res):
        assert scheduled(res, 10) and scheduled(res, 11)
        assert res["assign"][10] == res["assign"][11]
    return prob, check


@case("topology_test.go:1445-1476")
def preferred_pod_affinity_may_be_violated():
    labels = {"test": "test"}
    noise = pods(10, labels=labels, topologySpreadConstraints=[fx.spread(HOSTNAME, labels)])
    follower = pod(podAffinity={"preferred": [{"weight": 50, "term": fx.affinity_term(HOSTNAME, {"security": "s2"})}]})
    prob = problem(noise + [follower])
    return prob, lambda res: _eq(scheduled(res, 10), True)


@case("topology_test.go:1478-1509")
def preferred_pod_anti_affinity_may_be_violated():
    labels = {"test": "test"}
    spreaders = pods(3, labels=labels, topologySpreadConstraints=[fx.spread(ZONE, labels)])
    avoiders = pods(10, podAntiAffinity={"preferred": [{"weight": 50, "term": fx.affinity_term(ZONE, labels)}]})
    prob = problem(spreaders + avoiders)
    return prob, lambda res: _eq([scheduled(res, i) for i in range(3, 13)], [True] * 10)


@case("topology_test.go:1533-1570")
def zonal_anti_affinity_with_every_zone_taken():
    aff = {"security": "s2"}
    zoned = [pod({"cpu": "2"}, labels=aff, nodeSelector={ZONE: z}) for z in ZONES]
    avoider = pod(podAntiAffinity={"required": [fx.affinity_term(ZONE, aff)]})
    prob = problem(zoned + [avoider])

    def check(res):
        assert all(scheduled(res, i) for i in range(3))
        assert not scheduled(res, 3)
    return prob, check


@case("topology_test.go:1879-1902")
def zonal_self_anti_affinity_first_batch_schedules_one():
    """late committal: the first pod's zone is undetermined, so it blocks all three zones for its siblings"""
    aff = {"security": "s2"}
    prob = problem(pods(3, labels=aff, podAntiAffinity={"required": [fx.affinity_term(ZONE, aff)]}))
    return prob, lambda res: _eq(sum(1 for a in res["assign"] if a >= 0), 1)


@case("topology_test.go:1924-1939")
def affinity_to_a_non_existent_pod():
    prob = problem(pods(10, podAffinity={"required": [fx.affinity_term(ZONE, {"security": "s2"})]}))
    return prob, lambda res: _eq([a >= 0 for a in res["assign"]], [False] * 10)


@case("topology_test.go:1941-1962")
def zonal_affinity_unconstrained_target_first_batch():
    aff = {"security": "s2"}
    followers = pods(10, podAffinity={"required": [fx.affinity_term(ZONE, aff)]})
    target = pod(labels=aff)
    prob = problem(followers + [target])

    def check(res):
        assert scheduled(res, 10)
        assert not any(scheduled(res, i) for i in range(10))
    return prob, check


@case("topology_test.go:2003-2035")
def multiple_dependent_affinities():
    db, web = {"type": "db", "spread": "spread"}, {"type": "web", "spread": "spread"}
    cache, ui = {"type": "cache", "spread": "spread"}, {"type": "ui", "spread": "spread"}
    prob = problem([pod(labels=db),
                    pod(labels=web, podAffinity={"required": [fx.affinity_term(HOSTNAME, db)]}),
                    pod(labels=cache, podAffinity={"required": [fx.affinity_term(HOSTNAME, web)]}),
                    pod(labels=ui, podAffinity={"required": [fx.affinity_term(HOSTNAME, cache)]})])
    return prob, lambda res: _eq([a >= 0 for a in res["assign"]], [True] * 4)


@case("topology_test.go:2037-2052")
def unsatisfiable_affinity_dependency_terminates():
    db, web = {"type": "db", "spread": "spread"}, {"type": "web", "spread": "spread"}
    prob = problem([pod(labels=db, podAffinity={"required": [fx.affinity_term(HOSTNAME, web)]})])
    return prob, lambda res: _eq(scheduled(res, 0), False)


@case("suite_test.go:1344-1358")
def reuse_existing_node():
    node = fx.state_node("node-a")
    prob = problem([pod({"cpu": "10m"})], nodes=[node])

    def check(res):
        assert res["assign"][0] == 0 and res["newNodes"] == []
    return prob, check


@case("suite_test.go:1405-1421")
def second_node_when_existing_is_full():
    node = fx.state_node("node-a", pods_=[pod({"cpu": "3"}, nodeName="node-a")])
    prob = problem([pod({"cpu": "2"})], nodes=[node])

    def check(res):
        assert res["assign"][0] == 1 and len(res["newNodes"]) == 1
    return prob, check


@case("suite_test.go:1554-1578")
def tainted_existing_node_is_skipped():
    node = fx.state_node("node-a", taints=[{"key": "foo.com/taint", "value": "tainted", "effect": "NoSchedule"}])
    prob = problem([pod({"cpu": "10m"})], nodes=[node])
    return prob, lambda res: _eq(res["assign"], [1])


@case("suite_test.go:1579-1609")
def startup_taint_ignored_until_initialized():
    taint = {"key": "foo.com/taint", "value": "tainted", "effect": "NoSchedule"}
    node = fx.state_node("node-a", taints=[taint], startupTaints=[taint], initialized=False)
    prob = problem([pod({"cpu": "10m"})], nodes=[node])
    return prob, lambda res: _eq(res["assign"], [0])


@case("suite_test.go:1460-1497")
def zonal_spread_continues_on_in_flight_nodes():
    """second round of the Go test: three nodes already hold (1, 1, 2) matching pods; five more pods fill them to (3, 3, 3)"""
    labels = {"foo": "bar"}
    spread = [fx.spread(ZONE, labels)]

    def bound(node, n):
        return [pod(labels=labels, topologySpreadConstraints=spread, nodeName=node) for _ in range(n)]
    nodes = [fx.state_node("node-1", zone="test-zone-1", pods_=bound("node-1", 1)),
             fx.state_node("node-2", zone="test-zone-2", pods_=bound("node-2", 1)),
             fx.state_node("node-3", zone="test-zone-3", pods_=bound("node-3", 2))]
    prob = problem(pods(5, labels=labels, topologySpreadConstraints=spread), nodes=nodes)

    def check(res):
        assert res["newNodes"] == []  # the in-flight nodes can hold all five
        counts = [1, 1, 2]
        for a in res["assign"]:
            assert 0 <= a < 3
            counts[a] += 1
        assert counts == [3, 3, 3]
    return prob, check


@case("suite_test.go:1498-1532")
def hostname_spread_prefers_new_nodes_over_in_flight():
    labels = {"foo": "bar"}
    spread = [fx.spread(HOSTNAME, labels)]
    nodes = [fx.state_node(f"node-{i}", pods_=[pod(labels=labels, topologySpreadConstraints=spread, nodeName=f"node-{i}")]) for i in range(4)]
    prob = problem(pods(5, labels=labels, topologySpreadConstraints=spread), nodes=nodes)

    def check(res):
        assert min(res["assign"]) >= 4 and len(set(res["assign"])) == 5  # (1 x 9): every new pod on its own new node
    return prob, check


@case("suite_test.go:1660-1731")
def bound_daemonset_pod_leaves_no_overhead_to_reserve():
    """16-cpu node (15.9 allocatable) with the daemonset's pod already bound (1 cpu): a 14.9-cpu pod still fits on it"""
    ds = pod({"cpu": "1", "memory": "1Gi"})
    ds_bound = pod({"cpu": "1", "memory": "2Gi"}, nodeName="node-a", isDaemonSet=True)
    node = fx.state_node("node-a", "arm-instance-type", allocatable={"cpu": "15900m", "memory": "131062Mi", "pods": "5"}, pods_=[ds_bound],
                         labels={ARCH: "arm64"})
    prob = problem([pod({"cpu": "14.9"})], nodes=[node], daemonSetPods=[ds])

    def check(res):
        assert res["assign"] == [0] and res["newNodes"] == []
    return prob, check


@case("suite_test.go:1824-1863")
def in_flight_nodes_are_packed_before_new_ones():
    medium = fx.instance_type("medium", {"cpu": "4.25", "pods": "4"})
    node = fx.state_node("node-a", "medium", allocatable={"cpu": "4150m", "memory": "4086Mi", "pods": "4"}, pods_=[pod({"cpu": "1"}, nodeName="node-a")])
    prob = problem(pods(5, requests={"cpu": "1"}), instance_types=[medium], nodes=[node])

    def check(res):
        assert sorted(res["assign"]).count(0) == 3  # three more fit next to the bound pod
        assert len(res["newNodes"]) == 1 and len(res["newNodes"][0]["pods"]) == 2
    return prob, check


def _eq(a, b):
    assert a == b, (a, b)


# ================================================================== cases added after the round's GPU budget was spent
# Pinned on the oracle (tests/test_oracle_known_answers.py runs CASES + CPU_ONLY_CASES); tests/test_gpu_known_answers.py takes
# CASES only - these move up once they have been run on the GPU.
CPU_ONLY_CASES = []


def cpu_case(ref):
    def deco(fn):
        CPU_ONLY_CASES.append((fn.__name__, ref, fn))
        return fn
    return deco


def _launched_capacity(prob, res):
    name = launched_type(prob, res, 0)
    it = next(i for i in prob["instanceTypes"] if i["name"] == name)
    return it["capacity"]["cpu"], it["capacity"]["memory"]


# ------------------------------------------------------------------ daemonset overhead (provisioning/suite_test.go:360-530)
@cpu_case("provisioning/suite_test.go:360-397")
def daemonset_overhead_pushes_to_the_larger_type():
    ds = pod({"cpu": "1", "memory": "1Gi"})
    plain = problem([pod({"cpu": "1", "memory": "1Gi"})], daemonSetPods=[ds])
    startup = problem([pod({"cpu": "1", "memory": "1Gi"})], daemonSetPods=[ds],
                      provisioners=[provisioner(startupTaints=[{"key": "foo.com/taint", "effect": "NoSchedule"}])])

    def check(results):
        for prob, res in zip((plain, startup), results):
            assert res["assign"] == [0]
            assert _launched_capacity(prob, res) == ("4", "4Gi")  # 2 cpu would not hold pod + daemonset + kube-reserved
    return {"multi": [plain, startup]}, check


@cpu_case("provisioning/suite_test.go:398-418")
def daemonset_overhead_too_large():
    huge = pod({"cpu": "10000", "memory": "10000Gi"})
    by_limits = pod(containers=[{"requests": {"cpu": "1"}, "limits": {"cpu": "10000", "memory": "10000Gi"}}])  # limits stand in for missing requests
    probs = [problem([pod()], daemonSetPods=[huge]), problem([pod()], daemonSetPods=[by_limits])]
    return {"multi": probs}, lambda results: _eq([r["assign"] for r in results], [[-1], [-1]])


@cpu_case("provisioning/suite_test.go:475-530")
def daemonsets_that_cannot_run_on_the_node_are_not_counted():
    req = {"cpu": "1", "memory": "1Gi"}
    tainted = provisioner(taints=[{"key": "foo", "value": "bar", "effect": "NoSchedule"}])
    p_intolerant = problem([pod(req, tolerations=[{"operator": "Exists"}])], daemonSetPods=[pod(req)], provisioners=[tainted])
    p_selector = problem([pod(req)], daemonSetPods=[pod(req, nodeSelector={"node": "invalid"})])
    p_notin = problem([pod(req, nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-2"]}]]})],
                      daemonSetPods=[pod(req, nodeAffinity={"required": [[{"key": "foo", "operator": "NotIn", "values": ["bar"]}]]})])

    def check(results):
        assert [r["assign"] for r in results] == [[0], [0], [0]]
        assert _launched_capacity(p_intolerant, results[0]) == ("2", "2Gi")  # daemonset does not tolerate the provisioner's taint
        assert _launched_capacity(p_selector, results[1]) == ("2", "2Gi")    # daemonset selects a label the node never has
        assert _launched_capacity(p_notin, results[2]) == ("4", "4Gi")       # NotIn on an undefined key is compatible: counted
    return {"multi": [p_intolerant, p_selector, p_notin]}, check


# ------------------------------------------------------------------ relaxation order, provisioner selection (provisioning/suite_test.go:1105-1183)
@cpu_case("provisioning/suite_test.go:1105-1124")
def prefer_no_schedule_is_tolerated_after_the_preferences_are_relaxed():
    prefs = [{"weight": 1, "terms": [{"key": ZONE, "operator": "In", "values": ["invalid"]}]},
             {"weight": 1, "terms": [{"key": INSTANCE_TYPE, "operator": "In", "values": ["invalid"]}]}]
    pr = provisioner(taints=[{"key": "foo", "value": "bar", "effect": "PreferNoSchedule"}])
    prob = problem([pod(nodeAffinity={"preferred": prefs})], provisioners=[pr])

    def check(res):
        assert res["assign"] == [0]
        assert res["relax"] == [3]  # two preferred terms dropped, then the PreferNoSchedule toleration (preferences.go:36-55)
    return prob, check


@cpu_case("provisioning/suite_test.go:1129-1183")
def provisioner_selection_by_name_label_taint_and_weight():
    pn = fx.PROVISIONER_NAME
    by_name = problem([pod(nodeSelector={pn: "target"})], provisioners=[provisioner("target"), provisioner("other")])
    by_label = problem([pod(nodeSelector={"foo": "bar"})], provisioners=[provisioner("labelled", labels={"foo": "bar"}), provisioner("other")])
    avoid_pns = problem([pod()], provisioners=[provisioner("tainted", taints=[{"key": "foo", "value": "bar", "effect": "PreferNoSchedule"}]),
                                               provisioner("clean")])
    weights = [provisioner("w0"), provisioner("w20", weight=20), provisioner("w100", weight=100)]
    heaviest = problem(pods(3), provisioners=weights)
    explicit = problem([pod(nodeSelector={pn: "w0"})], provisioners=weights)

    def name_of(res, i=0):
        node = res["newNodes"][res["assign"][i] - len(res["existing"])]
        return node["requirements"][pn]

    def check(results):
        assert name_of(results[0]) == "In [target]"
        assert name_of(results[1]) == "In [labelled]"
        assert name_of(results[2]) == "In [clean]"
        assert [name_of(results[3], i) for i in range(3)] == ["In [w100]"] * 3
        assert name_of(results[4]) == "In [w0]"
    return {"multi": [by_name, by_label, avoid_pns, heaviest, explicit]}, check


# ------------------------------------------------------------------ zonal spread against pods that already run (topology_test.go:163-339)
def _small_node_with(name, zone, bound):
    """a 2-cpu node (1.9 allocatable) already holding `bound` pods: a further 1.1-cpu pod does not fit, as in the Go tests"""
    return fx.state_node(name, "small-instance-type", zone=zone, allocatable={"cpu": "1900m", "memory": "2038Mi", "pods": "5"}, pods_=bound)


def _zone_counts(prob, res, base):
    counts = dict(base)
    ne = len(res["existing"])
    for a in res["assign"]:
        if a < 0:
            continue
        assert a >= ne  # the existing nodes are full
        z = res["newNodes"][a - ne]["requirements"][ZONE]
        assert z.startswith("In [") and " " not in z[4:-1], z
        counts[z[4:-1]] = counts.get(z[4:-1], 0) + 1
    return sorted(counts.values())


@cpu_case("topology_test.go:163-204")
def non_minimum_domain_when_nothing_else_is_available():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels, max_skew=5)]
    nodes = [_small_node_with("n1", "test-zone-1", [pod({"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons, nodeName="n1")]),
             _small_node_with("n2", "test-zone-2", [pod({"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons, nodeName="n2")])]
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-3"]}])
    prob = problem(pods(10, requests={"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons), provisioners=[pr], nodes=nodes)
    return prob, lambda res: _eq(_zone_counts(prob, res, {"test-zone-1": 1, "test-zone-2": 1}), [1, 1, 6])


@cpu_case("topology_test.go:205-242")
def only_minimum_domains_while_the_skew_is_violated():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels)]
    nodes = [_small_node_with(f"n{i}", "test-zone-1", [pod({"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons, nodeName=f"n{i}")])
             for i in range(3)]
    prob = problem(pods(3, requests={"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons), nodes=nodes)
    return prob, lambda res: _eq(_zone_counts(prob, res, {"test-zone-1": 3}), [1, 2, 3])


@cpu_case("topology_test.go:243-306")
def max_skew_is_not_violated_do_not_schedule():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels)]
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-2", "test-zone-3"]}])
    owning = _small_node_with("n1", "test-zone-1", [pod({"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons, nodeName="n1")])
    discovered = _small_node_with("n1", "test-zone-1", [pod({"cpu": "1.1"}, labels=labels, nodeName="n1")])  # matching labels only (:276-306)
    probs = [problem(pods(10, requests={"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons), provisioners=[pr], nodes=[n])
             for n in (owning, discovered)]

    def check(results):
        for prob, res in zip(probs, results):
            assert _zone_counts(prob, res, {"test-zone-1": 1}) == [1, 2, 2]
            assert sum(1 for a in res["assign"] if a < 0) == 6
    return {"multi": probs}, check


@cpu_case("topology_test.go:308-339")
def only_running_pods_with_matching_labels_and_a_domain_count():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels)]
    first = fx.state_node("first", zone="test-zone-1", allocatable={"cpu": "0", "memory": "0", "pods": "0"}, pods_=[
        pod(nodeName="first"),                                           # ignored: no labels
        pod(labels=labels, namespace="other", nodeName="first"),        # ignored: wrong namespace
        pod(labels=labels, nodeName="first", terminal=True),            # ignored: phase Failed / Succeeded
        pod(labels=labels, nodeName="first", terminating=True),         # ignored: terminating
        pod(labels=labels, nodeName="first"), pod(labels=labels, nodeName="first")])
    second = fx.state_node("second", zone="test-zone-2", allocatable={"cpu": "0", "memory": "0", "pods": "0"}, pods_=[pod(labels=labels, nodeName="second")])
    third = fx.state_node("third", allocatable={"cpu": "0", "memory": "0", "pods": "0"}, pods_=[pod(labels=labels, nodeName="third")])
    del third["labels"][ZONE]                                            # ignored: the node has no zone
    prob = problem(pods(2, labels=labels, topologySpreadConstraints=cons), nodes=[first, second, third])

    return prob, lambda res: _eq(_zone_counts(prob, res, {"test-zone-1": 2, "test-zone-2": 1}), [1, 2, 2])  # ConsistOf(2, 2, 1)


# ------------------------------------------------------------------ more spread / affinity (topology_test.go:353-590, 1239-1281)
@cpu_case("topology_test.go:353-378")
def spread_whose_selector_matches_no_pod_does_not_spread():
    """the selector counts pods, the owner is what the spread applies to: nothing matches, so nothing has to be spread"""
    cons = [fx.spread(HOSTNAME, {"test": "test"})]
    prob = problem(pods(5, topologySpreadConstraints=cons))
    return prob, lambda res: _eq(len(set(res["assign"])), 1)


@cpu_case("topology_test.go:447-489")
def hostname_spread_of_two_deployments_on_two_archs_needs_four_nodes():
    def app(name, arch, n):
        lab = {"app": name}
        return pods(n, labels=lab, topologySpreadConstraints=[fx.spread(HOSTNAME, lab)],
                    nodeAffinity={"required": [[{"key": ARCH, "operator": "In", "values": [arch]}]]})
    prob = problem(app("app1", "amd64", 2) + app("app2", "arm64", 2))

    def check(res):
        assert min(res["assign"]) >= 0 and len(set(res["assign"])) == 4
    return prob, check


def _ct_counts(res, base):
    counts = dict(base)
    ne = len(res["existing"])
    for a in res["assign"]:
        if a >= ne:
            ct = res["newNodes"][a - ne]["requirements"][CAPACITY_TYPE]
            counts[ct] = counts.get(ct, 0) + 1
    return sorted(counts.values())


@cpu_case("topology_test.go:526-590")
def capacity_type_skew_do_not_schedule_versus_schedule_anyway():
    labels = {"test": "test"}
    od = provisioner(requirements=[{"key": CAPACITY_TYPE, "operator": "In", "values": ["on-demand"]}])
    probs = []
    for when in ("DoNotSchedule", "ScheduleAnyway"):
        cons = [fx.spread(CAPACITY_TYPE, labels, when=when)]
        spot_node = fx.state_node("n-spot", "small-instance-type", capacity_type="spot", allocatable={"cpu": "1900m", "memory": "2038Mi", "pods": "5"},
                                  pods_=[pod({"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons, nodeName="n-spot")])
        probs.append(problem(pods(5, requests={"cpu": "1.1"}, labels=labels, topologySpreadConstraints=cons), provisioners=[od], nodes=[spot_node]))

    def check(results):
        assert _ct_counts(results[0], {"spot": 1}) == [1, 2]   # on-demand may only get one ahead of spot
        assert sum(1 for a in results[0]["assign"] if a < 0) == 3
        assert _ct_counts(results[1], {"spot": 1}) == [1, 5]   # ScheduleAnyway is relaxed away
    return {"multi": probs}, check


@cpu_case("topology_test.go:1239-1281")
def pod_affinity_on_arch_with_hostname_spread():
    aff = {"security": "s2"}
    tsc = [fx.spread(HOSTNAME, aff)]
    first = pod({"cpu": "2"}, labels=aff, topologySpreadConstraints=tsc, nodeSelector={ARCH: "arm64"})
    second = pod({"cpu": "1"}, labels=aff, topologySpreadConstraints=tsc, podAffinity={"required": [fx.affinity_term(ARCH, aff)]})
    prob = problem([first, second])

    def check(res):
        assert min(res["assign"]) >= 0 and res["assign"][0] != res["assign"][1]  # same arch, but the spread keeps them apart
        ne = len(res["existing"])
        archs = [res["newNodes"][a - ne]["requirements"][ARCH] for a in res["assign"]]
        assert archs == ["In [arm64]", "In [arm64]"]
    return prob, check


# ------------------------------------------------------------------ self pod affinity (topology_test.go:1306-1444)
@cpu_case("topology_test.go:1306-1344")
def self_affinity_on_hostname_fills_exactly_one_node():
    aff = {"security": "s2"}
    mk = lambda n: pods(n, labels=aff, podAffinity={"required": [fx.affinity_term(HOSTNAME, aff)]})
    first = problem(mk(10))
    # second batch of the Go test: the first node exists (in flight, full: 5 pods) - nobody of the next batch may open a second domain
    full = fx.state_node("node-a", pods_=[pod(labels=aff, podAffinity={"required": [fx.affinity_term(HOSTNAME, aff)]}, nodeName="node-a") for _ in range(5)])
    second = problem(mk(10), nodes=[full])

    def check(results):
        a = results[0]["assign"]
        assert sum(1 for x in a if x >= 0) == 5 and len({x for x in a if x >= 0}) == 1  # the default types hold 5 pods
        assert all(x < 0 for x in results[1]["assign"])
    return {"multi": [first, second]}, check


@cpu_case("topology_test.go:1346-1389")
def self_affinity_is_not_limited_by_the_followers_node_selectors():
    """a matching pod already runs in zone-1; followers restricted to zone-2/3 cannot bootstrap a second hostname domain"""
    aff = {"security": "s2"}
    term = {"required": [fx.affinity_term(HOSTNAME, aff)]}
    # 3 of 5 pod slots and most of the cpu are taken by unrelated pods: the node is in flight but cannot take a follower
    holder = fx.state_node("node-z1", zone="test-zone-1", allocatable={"cpu": "3900m", "memory": "4086Mi", "pods": "1"},
                           pods_=[pod(labels=aff, podAffinity=term, nodeName="node-z1")])
    followers = pods(10, labels=aff, podAffinity=term,
                     nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-2", "test-zone-3"]}]]})
    prob = problem(followers, nodes=[holder])
    return prob, lambda res: _eq([x >= 0 for x in res["assign"]], [False] * 10)


@cpu_case("topology_test.go:1390-1444")
def self_affinity_on_zone():
    aff = {"security": "s2"}
    term = {"required": [fx.affinity_term(ZONE, aff)]}
    free = problem(pods(3, labels=aff, podAffinity=term))
    pinned = problem(pods(3, labels=aff, podAffinity=term, nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-3"]}]]}))

    def check(results):
        for res in results:
            assert min(res["assign"]) >= 0 and len(set(res["assign"])) == 1
        node = results[1]["newNodes"][results[1]["assign"][0] - len(results[1]["existing"])]
        assert node["requirements"][ZONE] == "In [test-zone-3]"
    return {"multi": [free, pinned]}, check


# ------------------------------------------------------------------ pod anti-affinity variants (topology_test.go:1572-1843)
@cpu_case("topology_test.go:1572-1593")
def zonal_anti_affinity_against_a_pod_of_unknown_zone():
    aff = {"security": "s2"}
    target = pod({"cpu": "2"}, labels=aff)                                   # schedules first (larger), zone undetermined
    avoider = pod(podAntiAffinity={"required": [fx.affinity_term(ZONE, aff)]})
    prob = problem([target, avoider])
    return prob, lambda res: _eq([a >= 0 for a in res["assign"]], [True, False])


@cpu_case("topology_test.go:1594-1635")
def anti_affinity_on_arch():
    aff = {"security": "s2"}
    tsc = [fx.spread(HOSTNAME, aff)]
    first = pod({"cpu": "2"}, labels=aff, topologySpreadConstraints=tsc, nodeSelector={ARCH: "arm64"})
    second = pod({"cpu": "1"}, labels=aff, topologySpreadConstraints=tsc, podAntiAffinity={"required": [fx.affinity_term(ARCH, aff)]})
    prob = problem([first, second])

    def check(res):
        assert min(res["assign"]) >= 0
        ne = len(res["existing"])
        archs = [res["newNodes"][a - ne]["requirements"][ARCH] for a in res["assign"]]
        assert archs == ["In [arm64]", "In [amd64]"]
    return prob, check


def _zoned_avoiders(term_key, aff):
    return [pod({"cpu": "2"}, nodeSelector={ZONE: z}, podAntiAffinity={term_key: [term]})
            for z in ZONES
            for term in ([fx.affinity_term(ZONE, aff)] if term_key == "required" else [{"weight": 10, "term": fx.affinity_term(ZONE, aff)}])]


@cpu_case("topology_test.go:1637-1711")
def inverse_zonal_anti_affinity_required_versus_preferred():
    aff = {"security": "s2"}
    required = problem(_zoned_avoiders("required", aff) + [pod(labels=aff)])
    preferred = problem(_zoned_avoiders("preferred", aff) + [pod(labels=aff)])

    def check(results):
        assert [a >= 0 for a in results[0]["assign"]] == [True, True, True, False]  # every zone holds a pod that repels it
        assert [a >= 0 for a in results[1]["assign"]] == [True, True, True, True]   # a preference only
    return {"multi": [required, preferred]}, check


@cpu_case("topology_test.go:1745-1843")
def inverse_zonal_anti_affinity_from_pods_that_already_run():
    aff = {"security": "s2"}

    def cluster(term_key):
        nodes = []
        for i, z in enumerate(ZONES):
            term = fx.affinity_term(ZONE, aff)
            anti = {"required": [term]} if term_key == "required" else {"preferred": [{"weight": 10, "term": term}]}
            nodes.append(fx.state_node(f"n{i}", "small-instance-type", zone=z, allocatable={"cpu": "1900m", "memory": "2038Mi", "pods": "5"},
                                       pods_=[pod({"cpu": "1.5"}, podAntiAffinity=anti, nodeName=f"n{i}")]))
        return nodes
    required = problem([pod(labels=aff)], nodes=cluster("required"))
    preferred = problem([pod(labels=aff)], nodes=cluster("preferred"))

    def check(results):
        assert results[0]["assign"] == [-1]
        assert results[1]["assign"][0] >= 0
    return {"multi": [required, preferred]}, check


# ------------------------------------------------------------------ zonal affinity, namespaces, several provisioners (topology_test.go:1974-2207)
@cpu_case("topology_test.go:1974-2001")
def zonal_affinity_to_a_zone_constrained_target():
    aff = {"security": "s2"}
    followers = pods(10, podAffinity={"required": [fx.affinity_term(ZONE, aff)]})
    target = pod(labels=aff, nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-1"]}]]})
    prob = problem(followers + [target])

    def check(res):
        assert min(res["assign"]) >= 0
        ne = len(res["existing"])
        assert {res["newNodes"][a - ne]["requirements"][ZONE] for a in res["assign"]} == {"In [test-zone-1]"}  # ConsistOf(11)
    return prob, check


@cpu_case("topology_test.go:2054-2130")
def affinity_terms_select_by_namespace():
    labels, aff = {"test": "test"}, {"security": "s2"}
    noise = lambda: pods(10, labels=labels, topologySpreadConstraints=[fx.spread(HOSTNAME, labels)])
    elsewhere = problem(noise() + [pod(labels=aff, namespace="other-ns-no-match"),
                                   pod(podAffinity={"required": [fx.affinity_term(HOSTNAME, aff)]})])
    listed = problem(noise() + [pod(labels=aff, namespace="other-ns-list"),
                                pod(podAffinity={"required": [fx.affinity_term(HOSTNAME, aff, namespaces=["other-ns-list"])]})])

    def check(results):
        a = results[0]["assign"]
        assert a[10] >= 0 and a[11] < 0          # the target lives in another namespace: not selected
        b = results[1]["assign"]
        assert b[10] >= 0 and b[11] == b[10]     # the term lists that namespace: same node
    return {"multi": [elsewhere, listed]}, check


@cpu_case("topology_test.go:2174-2207")
def spread_counts_across_provisioners():
    labels = {"foo": "bar"}
    prs = [provisioner("zone-1-only", requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1"]}]),
           provisioner("zones-2-3", requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-2", "test-zone-3"]}])]
    prob = problem(pods(10, labels=labels, topologySpreadConstraints=[fx.spread(ZONE, labels)]), provisioners=prs)
    return prob, lambda res: _eq(fx.skew(prob, res, ZONE), [3, 3, 4])


# ------------------------------------------------------------------ TopologyNodeFilter: which nodes count for a spread (topology_test.go:661-782)
@cpu_case("topology_test.go:661-695")
def node_affinity_of_the_owner_filters_the_counted_nodes():
    """the spread owners are restricted to (zone-2, spot): the on-demand pod in zone-1 is not counted, all five fit one spot node"""
    labels = {"test": "test"}
    existing = fx.state_node("n-od", zone="test-zone-1", capacity_type="on-demand", allocatable={"cpu": "0", "memory": "0", "pods": "0"},
                             pods_=[pod(labels=labels, nodeName="n-od")])
    aff = {"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-2"]}, {"key": CAPACITY_TYPE, "operator": "In", "values": ["spot"]}]]}
    prob = problem(pods(5, labels=labels, nodeAffinity=aff, topologySpreadConstraints=[fx.spread(CAPACITY_TYPE, labels)]), nodes=[existing])

    def check(res):
        assert min(res["assign"]) >= 1 and len(set(res["assign"])) == 1
        assert _ct_counts(res, {"on-demand": 1}) == [1, 5]
    return prob, check


@cpu_case("topology_test.go:697-782")
def unconstrained_owners_see_the_existing_domain():
    labels = {"test": "test"}
    probs = []
    for key, have, only in ((CAPACITY_TYPE, "on-demand", "spot"), (ARCH, "amd64", "arm64")):
        lab = {CAPACITY_TYPE: "on-demand"} if key == CAPACITY_TYPE else {ARCH: "amd64"}
        existing = fx.state_node("n-old", "single-pod-instance-type", allocatable={"cpu": "3900m", "memory": "4086Mi", "pods": "1"},
                                 pods_=[pod(labels=labels, nodeName="n-old")], labels=lab)
        pr = provisioner(requirements=[{"key": key, "operator": "In", "values": [only]}])
        probs.append(problem(pods(5, requests={"cpu": "2"}, labels=labels, topologySpreadConstraints=[fx.spread(key, labels)]), provisioners=[pr],
                             nodes=[existing]))

    def check(results):
        for res in results:
            assert sum(1 for a in res["assign"] if a >= 0) == 2  # ConsistOf(1, 2): two more, then the skew would be violated
    return {"multi": probs}, check


# ------------------------------------------------------------------ custom spread key defined by provisioner requirements (topology_test.go:825-880)
@cpu_case("topology_test.go:825-880")
def spread_over_a_key_the_provisioners_define():
    """`capacity.spread.4-1` has values 2..5 on the spot provisioner and 1 on the on-demand one: 20 pods end up 16 : 4"""
    labels = {"test": "test"}
    key = "capacity.spread.4-1"
    spot = provisioner("spot", requirements=[{"key": CAPACITY_TYPE, "operator": "In", "values": ["spot"]},
                                             {"key": key, "operator": "In", "values": ["2", "3", "4", "5"]}])
    od = provisioner("on-demand", requirements=[{"key": CAPACITY_TYPE, "operator": "In", "values": ["on-demand"]},
                                                {"key": key, "operator": "In", "values": ["1"]}])
    prob = problem(pods(20, labels=labels, topologySpreadConstraints=[fx.spread(key, labels)]), provisioners=[spot, od])

    def check(res):
        assert min(res["assign"]) >= 0
        assert fx.skew(prob, res, key) == [4, 4, 4, 4, 4]
        assert _ct_counts(res, {}) == [4, 16]
    return prob, check


# ------------------------------------------------------------------ spread options limited by the owner's node affinity (topology_test.go:1057-1193)
@cpu_case("topology_test.go:1057-1078")
def spread_over_the_two_zones_the_node_affinity_allows():
    labels = {"test": "test"}
    aff = {"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-2"]}]]}
    prob = problem(pods(10, labels=labels, nodeAffinity=aff, topologySpreadConstraints=[fx.spread(ZONE, labels)]))
    return prob, lambda res: _eq(fx.skew(prob, res, ZONE), [5, 5])


@cpu_case("topology_test.go:1079-1125")
def a_new_zone_may_be_entered_when_that_improves_the_skew():
    """(3, 3, 0) already run in zones 1/2; a pod allowed in zones 2/3 takes the empty zone-3; five unconstrained ones end at (4, 4, 4)"""
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels)]
    z12 = {"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-2"]}]]}

    def cluster():
        nodes = []
        for i, z in enumerate(("test-zone-1", "test-zone-2")):
            bound = [pod(labels=labels, nodeAffinity=z12, topologySpreadConstraints=cons, nodeName=f"n{i}") for _ in range(3)]
            nodes.append(fx.state_node(f"n{i}", zone=z, allocatable={"cpu": "3900m", "memory": "4086Mi", "pods": "3"}, pods_=bound))
        return nodes
    one = problem([pod(labels=labels, topologySpreadConstraints=cons,
                       nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-2", "test-zone-3"]}]]})], nodes=cluster())
    third = fx.state_node("n2", zone="test-zone-3", allocatable={"cpu": "3900m", "memory": "4086Mi", "pods": "1"},
                          pods_=[pod(labels=labels, topologySpreadConstraints=cons, nodeName="n2")])
    five = problem(pods(5, labels=labels, topologySpreadConstraints=cons), nodes=cluster() + [third])

    def check(results):
        assert _zone_counts(one, results[0], {"test-zone-1": 3, "test-zone-2": 3}) == [1, 3, 3]
        assert _zone_counts(five, results[1], {"test-zone-1": 3, "test-zone-2": 3, "test-zone-3": 1}) == [4, 4, 4]
    return {"multi": [one, five]}, check


@cpu_case("topology_test.go:1127-1150")
def schedule_anyway_capacity_type_spread_with_node_selectors():
    labels = {"test": "test"}
    cons = [fx.spread(CAPACITY_TYPE, labels, when="ScheduleAnyway")]
    prob = problem(pods(5, labels=labels, topologySpreadConstraints=cons, nodeSelector={CAPACITY_TYPE: "spot"}) +
                   pods(5, labels=labels, topologySpreadConstraints=cons, nodeSelector={CAPACITY_TYPE: "on-demand"}))

    def check(res):
        assert min(res["assign"]) >= 0
        assert _ct_counts(res, {}) == [5, 5]
    return prob, check


# ------------------------------------------------------------------ instance selection and in-flight nodes (suite_test.go:1275-1404)
@cpu_case("suite_test.go:1275-1342")
def every_valid_type_is_offered_and_the_cheapest_one_launches():
    mk = lambda name, cpu, mem, price: fx.instance_type(name, {"cpu": cpu, "memory": mem},
                                                        offerings=[{"capacityType": "on-demand", "zone": "test-zone-1a", "price": price, "available": True}])
    its = [mk("medium", "2", "2Gi", 3.0), mk("small", "1", "1Gi", 2.0), mk("large", "4", "4Gi", 1.0)]  # sizes and prices do not correlate
    prob = problem([pod({"cpu": "1m", "memory": "1Mi"})], instance_types=its)

    def check(res):
        node = res["newNodes"][res["assign"][0]]
        assert sorted(its[i]["name"] for i in node["options"]) == ["large", "medium", "small"]
        assert its[node["launch"]["type"]]["name"] == "large" and node["launch"]["price"] == 1.0
    return prob, check


@cpu_case("suite_test.go:1359-1404")
def in_flight_node_is_reused_when_the_selectors_intersect():
    node = fx.state_node("node-z2", zone="test-zone-2", pods_=[pod({"cpu": "10m"}, nodeName="node-z2")])
    fits = pod({"cpu": "10m"}, nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-2"]}]]})
    other = pod({"cpu": "10m"}, nodeAffinity={"required": [[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-3"]}]]})
    probs = [problem([fits], nodes=[node]), problem([other], nodes=[node])]

    def check(results):
        assert results[0]["assign"] == [0] and results[0]["newNodes"] == []
        assert results[1]["assign"] == [1] and len(results[1]["newNodes"]) == 1
    return {"multi": probs}, check


# ------------------------------------------------------------------ in-flight nodes: deletion and taints (suite_test.go:1438-1659)
@cpu_case("suite_test.go:1438-1458")
def node_being_deleted_is_not_a_target():
    going = fx.state_node("node-a", pods_=[pod({"cpu": "10m"}, nodeName="node-a")], markedForDeletion=True)
    prob = problem([pod({"cpu": "10m"})], nodes=[going])

    def check(res):
        assert len(res["newNodes"]) == 1 and res["assign"][0] == len(res["existing"])
    return prob, check


@cpu_case("suite_test.go:1610-1658")
def startup_taint_after_initialization_blocks_ephemeral_taints_do_not():
    startup = {"key": "ignore-me", "value": "nothing-to-see-here", "effect": "NoSchedule"}
    pr = provisioner(startupTaints=[startup])
    came_back = fx.state_node("node-a", taints=[startup])  # initialized: the startup taint is a real taint now
    p1 = problem([pod()], provisioners=[pr], nodes=[came_back])
    not_ready = fx.state_node("node-b", taints=[{"key": "node.kubernetes.io/not-ready", "effect": "NoSchedule"},
                                                {"key": "node.kubernetes.io/unreachable", "effect": "NoSchedule"}],
                              pods_=[pod({"cpu": "10m"}, nodeName="node-b")])
    p2 = problem([pod({"cpu": "10m"})], nodes=[not_ready])

    def check(results):
        assert len(results[0]["newNodes"]) == 1           # a new node: the startup taint was gone once and is back
        assert results[1]["assign"] == [0] and results[1]["newNodes"] == []  # NotReady / Unreachable are ephemeral (state/node.go:93-110)
    return {"multi": [p1, p2]}, check


# ------------------------------------------------------------------ several constraints at once (topology_test.go:882-1028)
def _max_skew(counts, domains):
    cs = sorted(counts) + [0] * (domains - len(counts))
    return max(cs) - min(cs) if cs else 0


@cpu_case("topology_test.go:882-904")
def zonal_do_not_schedule_with_hostname_schedule_anyway():
    labels = {"test": "test"}
    cons = [fx.spread(ZONE, labels), fx.spread(HOSTNAME, labels, when="ScheduleAnyway")]
    pr = provisioner(requirements=[{"key": ZONE, "operator": "In", "values": ["test-zone-1", "test-zone-2"]}])
    prob = problem(pods(10, labels=labels, topologySpreadConstraints=cons), provisioners=[pr])

    def check(res):
        # zone-3 exists in the universe but the provisioner cannot reach it: one pod per reachable zone, the rest stays pending
        assert fx.skew(prob, res, ZONE) == [1, 1]
        assert fx.skew(prob, res, HOSTNAME) == [1, 1]
    return prob, check


@cpu_case("topology_test.go:906-950")
def capacity_type_and_hostname_spread_first_and_large_batches():
    labels = {"test": "test"}
    cons = [fx.spread(CAPACITY_TYPE, labels), fx.spread(HOSTNAME, labels, max_skew=3)]
    two = problem(pods(2, labels=labels, topologySpreadConstraints=cons))
    many = problem(pods(21, labels=labels, topologySpreadConstraints=cons))

    def check(results):
        assert _ct_counts(results[0], {}) == [1, 1]
        assert max(fx.skew(two, results[0], HOSTNAME)) <= 3
        assert min(results[1]["assign"]) >= 0
        assert _ct_counts(results[1], {}) == [10, 11]
        assert max(fx.skew(many, results[1], HOSTNAME)) <= 3
    return {"multi": [two, many]}, check


@cpu_case("topology_test.go:993-1028")
def capacity_type_zone_and_hostname_spread_together():
    labels = {"test": "test"}
    cons = [fx.spread(CAPACITY_TYPE, labels), fx.spread(ZONE, labels, max_skew=2), fx.spread(HOSTNAME, labels, max_skew=3)]
    its = []
    for cpu in (2, 4, 8):
        for zone in ZONES:
            for ct in ("spot", "on-demand"):
                res = {"cpu": str(cpu), "memory": f"{cpu * 2}Gi", "pods": "10"}
                its.append(fx.instance_type(f"{cpu}c-{zone}-{ct}", res, offerings=[{"capacityType": ct, "zone": zone, "price": fx.price_from_resources(res),
                                                                                 "available": True}]))
    probs = [problem(pods(n, labels=labels, topologySpreadConstraints=cons), instance_types=its) for n in (1, 2, 3, 7, 14)]

    def check(results):
        for prob, res in zip(probs, results):
            assert min(res["assign"]) >= 0
            assert _max_skew(_ct_counts(res, {}), 2) <= 1
            assert _max_skew(fx.skew(prob, res, ZONE), 3) <= 2
            assert max(fx.skew(prob, res, HOSTNAME)) <= 3
    return {"multi": probs}, check


# ------------------------------------------------------------------ daemonset bookkeeping on existing nodes (suite_test.go:1732-1821)
@cpu_case("suite_test.go:1732-1821")
def unexpected_daemonset_pod_does_not_free_capacity():
    """a label Karpenter did not put there makes a second daemonset land on the node; its pod is bound (1 cpu of 15.9):
    a 15.5-cpu pod must NOT be placed there, whatever the remaining-daemonset arithmetic says (clamped at zero)"""
    ds1 = pod({"cpu": "1", "memory": "1Gi"}, nodeSelector={"my-node-label": "value"})
    ds2 = pod({"cpu": "1m"})
    bound = pod({"cpu": "1", "memory": "2Gi"}, nodeSelector={"my-node-label": "value"}, nodeName="node-a", isDaemonSet=True)
    node = fx.state_node("node-a", "arm-instance-type", allocatable={"cpu": "15900m", "memory": "131062Mi", "pods": "5"}, pods_=[bound],
                         labels={ARCH: "arm64", "my-node-label": "value"})
    prob = problem([pod({"cpu": "15.5"})], nodes=[node], daemonSetPods=[ds1, ds2])

    def check(res):
        assert res["assign"] == [1] and len(res["newNodes"]) == 1
        assert launched_type(prob, res, 0) == "arm-instance-type"
    return prob, check


@cpu_case("suite_test.go:1963-1993")
def self_zone_affinity_prefers_the_in_flight_nodes_domain():
    """Issue #1975: nothing matches yet (the first pod is not bound), the bootstrap domain must be the in-flight node's zone"""
    aff = {"security": "s2"}
    term = {"required": [fx.affinity_term(ZONE, aff)]}
    for_zone = {}
    for z in ZONES:
        node = fx.state_node("node-a", zone=z, initialized=False)
        for_zone[z] = problem([pod(labels=aff, podAffinity=term)], nodes=[node])

    def check(results):
        for res in results:
            assert res["assign"] == [0] and res["newNodes"] == []
    return {"multi": [for_zone[z] for z in ZONES]}, check


# ------------------------------------------------------------------ Gt / Lt requirements (scheduling/suite_test.go:213-230) and complement
# requirements on instance types: carried on the device in region form (include/ksched.h: ksched_key_regions)
def _launched_integer(prob, res, pod_index=0):
    it = next(i for i in prob["instanceTypes"] if i["name"] == launched_type(prob, res, pod_index))
    return next(r["values"][0] for r in it["requirements"] if r["key"] == "integer")


@cpu_case("suite_test.go:213-221")
def provisioner_requirement_gt():
    prob = problem([pod()], provisioners=[provisioner(requirements=[{"key": "integer", "operator": "Gt", "values": ["8"]}])])

    def check(res):
        assert scheduled(res, 0)
        assert _launched_integer(prob, res) == "16"
    return prob, check


@cpu_case("suite_test.go:222-230")
def provisioner_requirement_lt():
    prob = problem([pod()], provisioners=[provisioner(requirements=[{"key": "integer", "operator": "Lt", "values": ["8"]}])])

    def check(res):
        assert scheduled(res, 0)
        assert _launched_integer(prob, res) == "2"
    return prob, check


@cpu_case("requirement.go:117-150 (Gt on the provisioner, Lt on the pod: the bounds meet on the node)")
def pod_and_provisioner_bounds_intersect():
    its = fx.fake_instance_types(12)
    pr = provisioner(requirements=[{"key": "integer", "operator": "Gt", "values": ["3"]}])
    lt = pod({"cpu": "1"}, nodeAffinity={"required": [[{"key": "integer", "operator": "Lt", "values": ["6"]}]]})
    crossing = pod({"cpu": "1"}, nodeAffinity={"required": [[{"key": "integer", "operator": "Lt", "values": ["3"]}]]})
    notin = pod({"cpu": "1"}, nodeAffinity={"required": [[{"key": "integer", "operator": "Lt", "values": ["6"]},
                                                            {"key": "integer", "operator": "NotIn", "values": ["4"]}]]})
    prob = {"multi": [problem([p], instance_types=its, provisioners=[pr]) for p in (lt, crossing, notin)]}

    def check(results):
        a, b, c = results
        assert a["assign"][0] >= 0 and b["assign"][0] < 0 and c["assign"][0] >= 0
        opts = lambda r: sorted(its[i]["name"] for i in r["newNodes"][0]["options"])
        assert opts(a) == ["fake-it-3", "fake-it-4"]     # integer in (3, 6) = cpu 4, 5
        assert opts(c) == ["fake-it-4"]                  # ... without 4
        assert a["newNodes"][0]["requirements"]["integer"] == "Exists [] >3 <6"
        assert c["newNodes"][0]["requirements"]["integer"] == "NotIn [4] >3 <6"
    return prob, check


@cpu_case("requirements.go:123-133 (a Gt requirement is Exists with bounds: not a negative operator)")
def gt_on_an_undefined_custom_key_is_incompatible():
    # "custom" is not well known and the provisioner does not define it: In / Exists / Gt / Lt are refused, NotIn / DoesNotExist pass
    mk = lambda op, vals: pod({"cpu": "1"}, nodeAffinity={"required": [[{"key": "custom", "operator": op, "values": vals}]]})
    return each_alone([mk("Gt", ["1"]), mk("Lt", ["9"]), mk("NotIn", ["x"]), mk("DoesNotExist", []), mk("Exists", [])],
                      [False, False, True, True, False])


@cpu_case("requirements.go:189-206 with cloudprovider/types.go:72-85 (instance types may carry NotIn / Exists / Gt / Lt requirements)")
def instance_types_with_complement_requirements():
    its = fx.fake_instance_types(6)
    its[0]["requirements"].append({"key": "tier", "operator": "NotIn", "values": ["gold"]})
    its[1]["requirements"].append({"key": "tier", "operator": "Exists", "values": []})
    its[2]["requirements"].append({"key": "tier", "operator": "In", "values": ["gold"]})
    its[3]["requirements"].append({"key": "tier", "operator": "DoesNotExist", "values": []})
    its[4]["requirements"].append({"key": "tier", "operator": "Gt", "values": ["5"]})
    # its[5]: no requirement on the key
    mk = lambda op, vals: pod({"cpu": "100m"}, nodeAffinity={"required": [[{"key": "tier", "operator": op, "values": vals}]]})
    cases = [("In", ["gold"]), ("In", ["silver"]), ("NotIn", ["gold"]), ("Exists", []), ("DoesNotExist", []), ("In", ["7"]), ("Lt", ["3"])]
    prob = {"multi": [problem([mk(op, v)], instance_types=its, wellKnownLabels=fx.WELL_KNOWN_EXTRA + ["tier"]) for op, v in cases]}
    want = [["fake-it-1", "fake-it-2", "fake-it-5"],                         # In gold: Exists, In gold, no requirement
            ["fake-it-0", "fake-it-1", "fake-it-5"],                         # In silver: NotIn gold, Exists, none
            ["fake-it-0", "fake-it-1", "fake-it-3", "fake-it-4", "fake-it-5"],  # NotIn gold: every complement, DoesNotExist (both negative), none
            ["fake-it-0", "fake-it-1", "fake-it-2", "fake-it-4", "fake-it-5"],  # Exists
            ["fake-it-0", "fake-it-3", "fake-it-5"],                         # DoesNotExist: NotIn (negative) and DoesNotExist, none
            ["fake-it-0", "fake-it-1", "fake-it-4", "fake-it-5"],            # In 7: NotIn gold, Exists, Gt 5, none
            ["fake-it-0", "fake-it-1", "fake-it-5"]]                         # Lt 3: complement types whose bounds do not cross (Gt 5 does)

    def check(results):
        for r, w in zip(results, want):
            assert r["assign"][0] >= 0
            assert sorted(its[i]["name"] for i in r["newNodes"][0]["options"]) == w
    return prob, check


# ------------------------------------------------------------------ CSI volume limits of existing nodes (suite_test.go:1995-2240)
def _volume_setup(claims_of, n_pods, limit=10):
    big = fx.instance_type("instance-type", {"cpu": "1024", "pods": "1024"})
    node = fx.state_node("node-0", "instance-type", allocatable={"cpu": "1000", "pods": "1000"},
                         pods_=[pod({"cpu": "1"}, nodeName="node-0")], volumeLimits={"fake.csi.provider": limit})
    ps = [pod({"cpu": "1"}, volumes=claims_of(i)) for i in range(n_pods)]
    return problem(ps, instance_types=[big], provisioners=[provisioner(limits=None)], nodes=[node])


@cpu_case("suite_test.go:1995-2057")
def volume_limits_force_a_second_node():
    prob = _volume_setup(lambda i: [{"driver": "fake.csi.provider", "pvc": f"default/my-claim-a-{i}"},
                                    {"driver": "fake.csi.provider", "pvc": f"default/my-claim-b-{i}"}], 6)

    def check(res):
        assert all(a >= 0 for a in res["assign"])
        assert sorted(res["assign"]).count(0) == 5      # the in-flight node takes 5 pods = 10 volumes
        assert len(res["newNodes"]) == 1
    return prob, check


@cpu_case("suite_test.go:2058-2123")
def one_shared_claim_fits_a_single_node():
    prob = _volume_setup(lambda i: [{"driver": "fake.csi.provider", "pvc": "default/my-claim"}, {"driver": "fake.csi.provider", "pvc": "default/my-claim"}], 100)

    def check(res):
        assert res["assign"] == [0] * 100 and res["newNodes"] == []
    return prob, check


@cpu_case("suite_test.go:2124-2240 (claims without a CSI driver are not counted)")
def non_csi_claims_are_not_counted():
    prob = _volume_setup(lambda i: [{"driver": "", "pvc": f"default/nfs-{i}"}, {"driver": "", "pvc": f"default/static-{i}"}], 12)

    def check(res):
        assert res["assign"] == [0] * 12 and res["newNodes"] == []
    return prob, check


@cpu_case("volumeusage.go:101-131 (shared and private claims on one node; a node over its limit takes nobody)")
def shared_and_private_claims_mix():
    big = fx.instance_type("instance-type", {"cpu": "1024", "pods": "1024"})
    bound = [pod({"cpu": "1"}, nodeName="node-0", volumes=[{"driver": "ebs", "pvc": "default/shared"}, {"driver": "ebs", "pvc": "default/b0"}])]
    over = [pod({"cpu": "1"}, nodeName="node-1", volumes=[{"driver": "ebs", "pvc": f"default/o{i}"} for i in range(3)])]
    nodes = [fx.state_node("node-0", "instance-type", allocatable={"cpu": "1000", "pods": "1000"}, pods_=bound, volumeLimits={"ebs": 4}),
             fx.state_node("node-1", "instance-type", allocatable={"cpu": "1000", "pods": "1000"}, pods_=over, volumeLimits={"ebs": 2}),
             fx.state_node("node-2", "instance-type", allocatable={"cpu": "1000", "pods": "1000"}, volumeLimits={"efs": 1})]
    ps = [pod({"cpu": "3"}, volumes=[{"driver": "ebs", "pvc": "default/shared"}, {"driver": "ebs", "pvc": "default/p0"}]),   # node-0: 2 + 1 new = 3
          pod({"cpu": "2"}, volumes=[{"driver": "ebs", "pvc": "default/shared"}, {"driver": "ebs", "pvc": "default/p1"}]),   # node-0: 4
          pod({"cpu": "1"}, volumes=[{"driver": "ebs", "pvc": "default/shared"}, {"driver": "ebs", "pvc": "default/p2"}]),   # node-0 full, node-1 over its limit -> node-2 (no ebs limit)
          pod({"cpu": "500m"}),                                                                                          # no volumes: node-0
          pod({"cpu": "250m"}, volumes=[{"driver": "efs", "pvc": "default/e0"}, {"driver": "efs", "pvc": "default/e1"}])]     # efs limit 1 on node-2 -> node-0
    prob = problem(ps, instance_types=[big], provisioners=[provisioner(limits=None)], nodes=nodes)

    def check(res):
        assert res["assign"] == [0, 0, 2, 0, 0]
    return prob, check
