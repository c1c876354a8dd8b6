"""CPU: daemonsets whose requirements name node.kubernetes.io/instance-type (tests/daemonset_itype_problems.py) encode, in
plain and superset form, and their overhead is the reference's: each template's daemon_requests and each existing node's
remaining requests equal getDaemonOverhead / calculateExistingMachines restated on strings, read through ctypes from the
encoding the device receives. The former rule's miscount on existing nodes is gone, daemons with a hostname requirement that
a template admits stay refused, and the oracle's results hold every node to its overhead, keep the placement invariants,
give the same answer in fast mode and give the reference's answer on the restated known answers."""
import ctypes as C

import pytest

import daemonset_itype_problems as dp
import exact_arith as ea
import placement_invariants as pi
from known_answers import launched_type

CORPUS = dp.corpus() + [("cluster", dp.cluster(0))]
IDS = [n for n, _ in CORPUS]
MAX_RES = 8


class _Catalog(C.Structure):  # the leading fields of ksched_catalog, include/ksched.h
    _fields_ = [("n_keys", C.c_int32), ("n_res", C.c_int32), ("n_types", C.c_int32), ("n_templates", C.c_int32),
                ("keys", C.c_void_p), ("key_regions", C.c_void_p), ("key_int_values", C.c_void_p), ("types", C.c_void_p),
                ("type_bounds", C.c_void_p), ("type_capacity", C.c_void_p), ("templates", C.c_void_p)]


class _Template(C.Structure):  # ksched_template
    _fields_ = [("values", C.c_uint64 * 16), ("meta", C.c_uint64), ("daemon_requests", C.c_int64 * MAX_RES),
                ("daemon_res_present", C.c_uint32), ("taintset", C.c_uint32), ("has_limits", C.c_int32), ("limit_present", C.c_uint32),
                ("remaining", C.c_int64 * MAX_RES)]


class _Problem(C.Structure):  # the leading fields of ksched_problem
    _fields_ = [("n_pods", C.c_int32), ("n_classes", C.c_int32), ("n_existing", C.c_int32), ("n_groups", C.c_int32),
                ("classes", C.c_void_p), ("class_bounds", C.c_void_p), ("pod_class", C.c_void_p), ("pod_timestamp", C.c_void_p),
                ("pod_uid_rank", C.c_void_p), ("existing", C.c_void_p)]


class _Existing(C.Structure):  # ksched_existing_node
    _fields_ = [("values", C.c_uint64 * 16), ("meta", C.c_uint64), ("available", C.c_int64 * MAX_RES), ("requests", C.c_int64 * MAX_RES),
                ("available_present", C.c_uint32), ("requests_present", C.c_uint32), ("taintset", C.c_uint32), ("itype", C.c_uint32),
                ("hostport_entries", C.c_uint64), ("label_keys_other", C.c_uint64)]


assert C.sizeof(_Template) == 280 and C.sizeof(_Existing) == 296


def _candidates(prob):
    return [i for i, n in enumerate(prob.get("nodes", [])) if n.get("candidate")] if not prob["pods"] else []


def _encode(pkg, prob, cands, superset):
    """([(daemon_requests, daemon_res_present)] per template, [(requests, requests_present)] per existing node, resource ids)
    of kh_encode / kh_encode_cluster; raises KschedError on a refusal"""
    L = pkg.lib()
    L.kh_encoded_catalog.restype = L.kh_encoded_problem.restype = C.c_void_p
    L.kh_encoded_catalog.argtypes = L.kh_encoded_problem.argtypes = [C.c_void_p]
    problem = pkg.Problem.from_dict(prob)
    arr = (C.c_int * max(1, len(cands)))(*cands)
    enc = (L.kh_encode_cluster if superset else L.kh_encode)(problem.ptr, arr, len(cands))
    if not enc:
        msg = L.kh_scheduler_error().decode()
        raise pkg.KschedError(pkg.KSCHED_ERR_UNSUPPORTED if msg.startswith("unsupported:") else pkg.KSCHED_ERR_INVALID, msg)
    try:
        cat = _Catalog.from_address(L.kh_encoded_catalog(enc))
        pb = _Problem.from_address(L.kh_encoded_problem(enc))
        tmpl = [(list(t.daemon_requests), t.daemon_res_present) for t in (_Template * cat.n_templates).from_address(cat.templates)]
        ex = [(list(e.requests), e.requests_present) for e in (_Existing * pb.n_existing).from_address(pb.existing)] if pb.n_existing else []
        names = set(ea.pod_requests({}))
        for p in prob.get("daemonSetPods", []):
            names |= set(ea.pod_requests(p))
        ids = {r: L.kh_encoded_resource_id(enc, r.encode()) for r in names}
        return tmpl, ex, ids
    finally:
        L.kh_encoded_free(enc)


def _row(resources, ids):
    """a resource list as the device row the encoder fills: values and present bits of the slots below 8"""
    vals, present = [0] * MAX_RES, 0
    for k, v in resources.items():
        i = ids.get(k, -1)
        if 0 <= i < MAX_RES:
            assert int(v) == v
            vals[i] = int(v)
            present |= 1 << i
    return vals, present


def _check(pkg, prob, superset):
    cands = _candidates(prob)
    tmpl, ex, ids = _encode(pkg, prob, cands, superset)
    want_t = [_row(o, ids) for o in dp.template_overhead(prob)]
    assert tmpl == want_t
    restated = dp.existing_overhead(prob, cands, superset)
    assert ex == [_row(o, ids) for _, o in restated]
    return restated


@pytest.mark.parametrize("superset", [False, True], ids=["plain", "superset"])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_overhead_equals_the_string_restatement(pkg, name, prob, superset):
    _check(pkg, prob, superset)


def test_scenarios_reach_what_they_were_built_for():
    """templates that charge a daemon with an instance-type requirement and templates that do not, and existing nodes of
    every kind the corpus lists"""
    by = dict(CORPUS)
    pods = lambda overheads: [o["pods"] // 1000 for o in overheads]
    assert pods(dp.template_overhead(by["neuron"])) == [2, 2]  # plugin and proxy on the neuron and the general template
    assert pods(dp.template_overhead(by["efa"])) == [1, 0, 0, 1]  # gpu and not-small meet the plugin's list, cpu and not-efa do not
    assert pods(dp.template_overhead(by["operators"])) == [2, 7, 4, 7]
    assert [o["cpu"] for o in dp.template_overhead(by["terms"])] == [200 + 400, 200 + 300 + 400 + 450]
    ex = {by["existing"]["nodes"][i]["name"]: o["cpu"] for i, o in dp.existing_overhead(by["existing"])}
    assert ex == {"e-00": 600,          # selected type
                  "e-01": 700,          # unselected type, selected by the hostname daemonset
                  "e-02": 600,          # tainted, tolerated by the plugin only
                  "e-03": 600,          # a type outside the catalog that the plugin lists
                  "e-04": 1600,         # no instance-type label: every instance-type requirement is compatible
                  "e-05": 0,            # the plugin's pod is already bound there
                  "e-06": 300,          # a type outside the catalog named "16": Gt 4 admits it
                  "e-07": 700,          # unselected type, selected by the hostname daemonset
                  "e-08": 600}          # neuron-tainted: only the plugin tolerates it


def test_former_rule_miscounted_an_existing_node(pkg):
    """the former rule charged n-0 the daemon that selects single-pod-instance-type; the encoding no longer does"""
    prob = dict(CORPUS)["miscount"]
    _, ex, ids = _encode(pkg, prob, [], False)
    former = dict(dp.former_existing_overhead(prob))
    now = dict(dp.existing_overhead(prob))
    assert former[0].get("cpu") == 500 and "cpu" not in now[0]
    assert ex[0] == _row(now[0], ids) != _row(former[0], ids)
    assert ex[1] == _row(now[1], ids) == _row(former[1], ids)


@pytest.mark.parametrize("name,prob", dp.near_misses(), ids=[n for n, _ in dp.near_misses()])
def test_near_misses_are_refused(pkg, name, prob):
    for superset in (False, True):
        with pytest.raises(pkg.KschedError, match="daemonset pod with a hostname requirement") as e:
            _encode(pkg, prob, [], superset)
        assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED


# ---------------------------------------------------------------- the oracle's results
BATCHES = [(n, p) for n, p in CORPUS if p["pods"]]
BIDS = [n for n, _ in BATCHES]


@pytest.mark.parametrize("name,prob", BATCHES, ids=BIDS)
def test_oracle_holds_every_node_to_its_overhead(pkg, oracle, name, prob):
    """every option of every new node holds the node's pods plus its template's overhead; every existing node holds its new
    pods plus the remaining overhead within what its bound pods leave"""
    _, res = oracle.solve_dict(pkg, prob)
    d = res.to_dict()
    pods, its = prob["pods"], prob["instanceTypes"]
    overhead = dp.template_overhead(prob)
    for nn in d["newNodes"]:
        need = ea._merge(overhead[nn["provisioner"]], ea.requests_for_pods([pods[i] for i in nn["pods"]]))
        for t in nn["options"]:
            assert ea.fits(need, ea.allocatable(its[t])), (name, its[t]["name"], need)
    remaining = dict(dp.existing_overhead(prob))
    for k, e in enumerate(d["existing"]):
        n = prob["nodes"][e["node"]]
        mine = [pods[i] for i, a in enumerate(d["assign"]) if a == k]
        if not mine:
            continue
        need = ea._merge(remaining[e["node"]], ea.requests_for_pods(mine))
        avail = ea._subtract(ea._resources(n["allocatable"]), ea.requests_for_pods(n["pods"]))
        assert ea.fits(need, avail), (name, n["name"], need, avail)


def test_miscount_scenario_places_the_pod_on_n0(pkg, oracle):
    _, res = oracle.solve_dict(pkg, dict(CORPUS)["miscount"])
    assert res.to_dict()["assign"] == [0]


@pytest.mark.parametrize("name,prob", [b for b in BATCHES if not b[1].get("nodes")], ids=[n for n, p in BATCHES if not p.get("nodes")])
def test_oracle_results_keep_the_invariants(pkg, oracle, name, prob):
    problem, res = oracle.solve_dict(pkg, prob)
    d = res.to_dict(brief=True)
    overhead = dp.template_overhead(prob)
    for nn in d["newNodes"]:  # the invariants sum the pods only: take the template's overhead off first
        for r in ("cpu", "memory", "pods"):
            nn["requests"][r] = nn["requests"].get(r, 0) - int(overhead[nn["provisioner"]].get(r, 0))
    pi.check(problem, _Brief(res, d))


class _Brief:
    """a Result whose to_dict(brief=True) is the given dict"""

    def __init__(self, res, d):
        self.res, self.d = res, d

    def to_dict(self, brief=False):
        return self.d


@pytest.mark.parametrize("name,prob", BATCHES, ids=BIDS)
def test_oracle_fast_mode_equals_literal(pkg, oracle, name, prob):
    oracle.assert_fast_equals_literal(pkg, prob)


KNOWN = dp.known_answers()


@pytest.mark.parametrize("name,prob,want", KNOWN, ids=[k[0] for k in KNOWN])
def test_known_answers(pkg, oracle, name, prob, want):
    _, res = oracle.solve_dict(pkg, prob)
    d = res.to_dict()
    assert d["assign"] == [0]
    it = next(i for i in prob["instanceTypes"] if i["name"] == launched_type(prob, d, 0))
    assert (it["capacity"]["cpu"], it["capacity"]["memory"]) == want
    charged = dp.template_overhead(prob)[0]["pods"] == 1000
    assert charged == (want == ("4", "4Gi"))
    _encode(pkg, prob, [], False)  # encodes without refusal


def test_cluster_has_sixty_nodes_and_the_after_state_a_new_daemonset(pkg):
    c, a = dp.cluster(0), dp.after(0)
    assert len(c["nodes"]) == 60 and len(a["daemonSetPods"]) == len(c["daemonSetPods"]) + 1
    for prob in (c, a):
        cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
        for superset in (False, True):
            _encode(pkg, prob, cands, superset)
