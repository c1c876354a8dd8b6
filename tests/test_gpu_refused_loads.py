"""GPU: a refused ksched_upload or ksched_load_catalog leaves the handle as it was. The problem or catalog loaded before it stays
resident and gives the same answer, and the refused input is refused again instead of being taken for the resident one."""
import ctypes as C

import pytest

import fixtures as fx

pytestmark = pytest.mark.gpu

TYPE_ROW_BYTES = 256  # sizeof(ksched_type_row), include/ksched.h


class _Catalog(C.Structure):  # ksched_catalog, include/ksched.h
    _fields_ = [("n_keys", C.c_int32), ("n_res", C.c_int32), ("n_types", C.c_int32), ("n_templates", C.c_int32),
                ("keys", C.c_void_p), ("key_regions", C.c_void_p), ("key_int_values", C.c_void_p), ("types", C.c_void_p),
                ("type_bounds", C.c_void_p), ("type_capacity", C.c_void_p), ("templates", C.c_void_p),
                ("template_bounds", C.c_void_p), ("offering_keys", C.c_void_p), ("n_res_ext", C.c_int32), ("pad_ext", C.c_int32),
                ("type_alloc_ext", C.c_void_p)]


class _Result(C.Structure):  # ksched_result, include/ksched.h
    _fields_ = [("assign", C.c_void_p), ("relax_level", C.c_void_p), ("place_seq", C.c_void_p), ("new_nodes", C.c_void_p),
                ("new_node_types", C.c_void_p), ("existing_reqs", C.c_void_p), ("feasibility", C.c_void_p),
                ("best_column", C.c_void_p), ("n_new_nodes", C.c_int32), ("n_unscheduled", C.c_int32), ("nodes_visited", C.c_int64),
                ("add_calls", C.c_int64), ("launch", C.c_void_p), ("new_node_requests_ext", C.c_void_p),
                ("new_node_requests_ext_present", C.c_void_p)]


def _labelled(spread_keys):
    """a pod that every one of the ten groups k0..k9 counts, constrained by hostname spread over the groups named"""
    return fx.pod({"cpu": "100m"}, labels={f"k{j}": "v" for j in range(10)},
                  topologySpreadConstraints=[fx.spread(fx.HOSTNAME, {f"k{j}": "v"}) for j in spread_keys])


def _plain(n):
    return [fx.pod({"cpu": "1", "memory": "1Gi"}) for _ in range(n)]


def test_refused_upload_keeps_the_resident_problem(pkg, oracle):
    # A is at least as large as B in pods, classes, existing nodes, groups and class_topo entries, so a handle that kept
    # B's sizes on A's arrays would read nothing out of bounds; both share one catalog
    a = pkg.Problem.from_dict(fx.problem(_plain(6) + [_labelled(range(5)), _labelled(range(5, 10))]))
    b = pkg.Problem.from_dict(fx.problem(_plain(6) + [_labelled(range(10))]))
    want = pkg.Result()
    assert oracle.solve(a, want) == 0, want.error
    ra, rb = pkg.ResidentSolve(a), pkg.ResidentSolve(b)
    for k in ("pods", "classes", "existing", "groups", "class_topo", "hostname_reqs"):
        assert ra.dims[k] >= rb.dims[k], k
    ra.load()
    with pytest.raises(pkg.KschedError) as e:
        rb.load()  # ten topology groups constrain one pod class: more than the pack kernel carries
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED
    ra.run()
    g, w = ra.download().to_dict(), want.to_dict()
    assert g["assign"] == w["assign"] and g["relax"] == w["relax"]
    assert [(n["pods"], n["options"], n["requests"]) for n in g["newNodes"]] == \
           [(n["pods"], n["options"], n["requests"]) for n in w["newNodes"]]


def _solve(L, handle, cat, problem_ptr, n_pods):
    assert L.ksched_load_catalog(handle, C.byref(cat)) == 0
    assign, relax = (C.c_int32 * n_pods)(), (C.c_int32 * n_pods)()
    res = _Result()
    res.assign, res.relax_level = C.addressof(assign), C.addressof(relax)
    assert L.ksched_solve(handle, problem_ptr, C.byref(res)) == 0
    return list(assign), list(relax), res.n_new_nodes, res.n_unscheduled


def test_refused_catalog_is_refused_again(pkg, oracle):
    problem = pkg.Problem.from_dict(fx.problem(_plain(40)))
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    rs = pkg.ResidentSolve(problem)
    L = pkg.lib()
    L.kh_encoded_catalog.restype = L.kh_encoded_problem.restype = C.c_void_p
    L.kh_encoded_catalog.argtypes = L.kh_encoded_problem.argtypes = [C.c_void_p]
    good = _Catalog.from_address(L.kh_encoded_catalog(rs.enc))
    problem_ptr = C.c_void_p(L.kh_encoded_problem(rs.enc))
    n = good.n_types
    assert n >= 2
    # the same catalog with its cheapest and its most expensive instance type swapped: out of price order
    rows = (C.c_char * (n * TYPE_ROW_BYTES)).from_buffer_copy(C.string_at(good.types, n * TYPE_ROW_BYTES))
    first, last = bytes(rows[:TYPE_ROW_BYTES]), bytes(rows[(n - 1) * TYPE_ROW_BYTES:])
    rows[:TYPE_ROW_BYTES], rows[(n - 1) * TYPE_ROW_BYTES:] = last, first
    bad = _Catalog.from_buffer_copy(good)
    bad.types = C.addressof(rows)

    handles = [C.c_void_p(), C.c_void_p()]
    for h in handles:
        assert L.ksched_create(0, C.byref(h)) == 0
    try:
        used, fresh = handles
        assert L.ksched_load_catalog(used, C.byref(good)) == 0
        for _ in range(2):
            assert L.ksched_load_catalog(used, C.byref(bad)) == pkg.KSCHED_ERR_INVALID
        got = _solve(L, used, good, problem_ptr, rs.dims["pods"])
        assert got == _solve(L, fresh, good, problem_ptr, rs.dims["pods"])
        assert got[2] == want.num_new_nodes
    finally:
        for h in handles:
            L.ksched_destroy(h)
