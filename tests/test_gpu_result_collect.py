"""GPU: the results both simulation calls and a Solve's download collect on the device.

 * A simulation call whose first set has an empty batch still runs K1's class pass for the sets after it. Right before each
   call, a poison problem leaves class rows in the handle's K1 buffers that say no pod fits any instance type, so a set that
   read them instead of its own rows would open no replacement node. Checked on consolidation probes and searches,
   validation and full simulations, each against the oracle or a fresh Solve.
 * ksched_download returns the existing nodes' final requirements as rows, and the same new nodes as ksched_solve."""
import copy
import ctypes as C
import random

import pytest

import consolidation_answers as ca
import fixtures as fx
import many_key_problems as mk
from oracle_compare import compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu


def _cluster():
    """an empty node of the cheapest type, cheapest to disrupt, then three nodes of the most expensive on-demand type with
    one 24-CPU pod each: no such pod fits beside another, so removing any of the three needs a replacement node; no pod is
    pending"""
    its = ca.assorted()
    od = ca.on_demand_by_price(its)
    nodes = [ca.node_of_type("empty", od[0], [], 1.0)]
    nodes[0]["allocatable"] = dict(od[0]["capacity"])
    nodes += [ca.node_of_type(f"node{i}", od[-1], [fx.pod({"cpu": "24"}, nodeName=f"node{i}")], 1.0) for i in range(1, 4)]
    return fx.problem([], instance_types=its, provisioners=[fx.provisioner(consolidationEnabled=True)], nodes=nodes, deriveCandidates=True)


def _poison(cluster):
    """the cluster's catalog and provisioners with 32 pod classes that fit no instance type"""
    return fx.problem([fx.pod({"cpu": str(64 + i)}) for i in range(32)], instance_types=cluster["instanceTypes"],
                      provisioners=cluster["provisioners"])


def _whole(res):
    d = res.to_dict()
    d.pop("nodesVisited")  # a simulation also counts the removed nodes it skips
    return d


@pytest.mark.parametrize("threads", [32, 512])
def test_an_empty_first_set_keeps_the_class_pass(pkg, oracle, monkeypatch, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    before = _cluster()
    problem = pkg.Problem.from_dict(before)
    poison = pkg.Problem.from_dict(_poison(before))
    cands = oracle.rank_candidates(problem)[0]
    assert cands == [0, 1, 2, 3]  # the empty node first
    # as many classes as the cluster's superset encoding, so the K1 buffers keep their allocation and the poison's rows
    assert pkg.ResidentSolve(poison).dims["classes"] >= pkg.ResidentSolve(problem, candidates=cands).dims["classes"]
    assert pkg.Scheduler(poison).solve().num_new_nodes == 0
    # every single probe after the empty node's replaces its node, and so does the prefix of two
    assert [oracle.consolidate_single(problem, c)["action"] for c in cands] == [1, 2, 2, 2]
    assert oracle.consolidate_probe(problem, 2)[0] == 2

    pkg.Scheduler(poison).solve()
    compare_cluster(pkg, oracle, problem, min_candidates=4)  # every prefix in one call, every single in another

    pkg.Scheduler(poison).solve()
    compare_validation(pkg, before, copy.deepcopy(before), "empty first")

    pkg.Scheduler(poison).solve()
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    sets = [[0], [1], [2, 3], [0, 3]]
    got = [_whole(r) for r in cs.simulate(sets)]
    for s, g in zip(sets, got):
        assert g == _whole(pkg.Scheduler(problem).solve(candidates=s, count_visited=False)), s
    assert len(got[1]["newNodes"]) == 1


class _Result(C.Structure):  # ksched_result, include/ksched.h
    _fields_ = [("assign", C.c_void_p), ("relax_level", C.c_void_p), ("place_seq", C.c_void_p), ("new_nodes", C.c_void_p),
                ("new_node_types", C.c_void_p), ("existing_reqs", C.c_void_p), ("feasibility", C.c_void_p),
                ("best_column", C.c_void_p), ("n_new_nodes", C.c_int32), ("n_unscheduled", C.c_int32), ("nodes_visited", C.c_int64),
                ("add_calls", C.c_int64), ("launch", C.c_void_p), ("new_node_requests_ext", C.c_void_p),
                ("new_node_requests_ext_present", C.c_void_p), ("all_pods_scheduled", C.c_int32), ("uninitialized_existing", C.c_int32)]


NEW_NODE_BYTES = 216          # sizeof(ksched_new_node)
REQSET_BYTES = 136            # sizeof(ksched_reqset): 16 values, then meta
EXISTING_BYTES = 296          # sizeof(ksched_existing_node), whose reqs come first
PROBLEM_EXISTING_OFFSET = 56  # offsetof(ksched_problem, existing)


def _many_key_problem():
    """six existing nodes labelled on every key of the catalog's requirements and the provisioners' labels, and 60 pods
    without selector, affinity or topology terms that fill some of them and open new nodes. One more pod names every key
    and lands nowhere (no provisioner labels team "nobody"), so that all of them are mask keys."""
    rng = random.Random(7)
    its, _ = mk.types(7)
    mid = mk._mid(its)
    nodes = [mk._node(f"n{i}", rng.choice(mid), rng, prov=("ml", "web")[i % 2]) for i in range(6)]
    keys = [k for k in mk.TYPE_KEYS + mk.CUSTOM + (fx.ZONE, fx.CAPACITY_TYPE, fx.ARCH, fx.OS) if k != "team"]
    nowhere = mk._pods(1, {"cpu": "1"}, "nowhere", required=[[mk._r(k, "Exists") for k in keys] + [mk._r("team", "In", "nobody")]])
    return mk._problem([fx.pod({"cpu": "2", "memory": "2Gi"}) for _ in range(60)] + nowhere, its, nodes)


def _result(call, L, h, problem_ptr, dims):
    """(assign, n_new_nodes, new node rows, their option words, existing_reqs rows) of ksched_download or ksched_solve"""
    P, NE, W = dims["pods"], dims["existing"], dims["type_words"]
    assign, nodes, types = (C.c_int32 * P)(), C.create_string_buffer(P * NEW_NODE_BYTES), (C.c_uint64 * (P * W))()
    ex = C.create_string_buffer(max(NE, 1) * REQSET_BYTES)
    res = _Result()
    res.assign, res.new_nodes, res.new_node_types, res.existing_reqs = (C.addressof(b) for b in (assign, nodes, types, ex))
    assert call(h, problem_ptr, C.byref(res)) == 0, L.ksched_last_error(h)
    n = res.n_new_nodes
    return list(assign), n, nodes.raw[:n * NEW_NODE_BYTES], list(types[:n * W]), ex.raw[:NE * REQSET_BYTES]


def test_download_returns_existing_requirements_as_rows(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(_many_key_problem()))
    assert 12 <= rs.dims["keys"] <= 16
    NE = rs.dims["existing"]
    L = pkg.lib()
    L.kh_handle.restype = L.kh_encoded_problem.restype = C.c_void_p
    L.kh_encoded_problem.argtypes = [C.c_void_p]
    L.ksched_download.argtypes = L.ksched_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.ksched_last_error.restype = C.c_char_p
    L.ksched_last_error.argtypes = [C.c_void_p]
    problem_ptr = L.kh_encoded_problem(rs.enc)
    # the encoded input rows, meta masked to its low 32 bits as the upload does
    existing = C.c_void_p.from_address(problem_ptr + PROBLEM_EXISTING_OFFSET).value
    want = b""
    for e in range(NE):
        row = C.string_at(existing + e * EXISTING_BYTES, REQSET_BYTES)
        want += row[:128] + (int.from_bytes(row[128:], "little") & 0xFFFFFFFF).to_bytes(8, "little")
    rs.load()
    rs.run()
    h = L.kh_handle()
    got = _result(L.ksched_download, L, h, problem_ptr, rs.dims)
    assert any(0 <= a < NE for a in got[0]) and got[1] > 0  # pods landed on existing nodes and on new ones
    assert got[4] == want
    assert got[1:4] == _result(L.ksched_solve, L, h, problem_ptr, rs.dims)[1:4]
