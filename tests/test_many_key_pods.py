"""CPU: pod classes whose requirements and topology terms touch more than 8 label keys (tests/many_key_problems.py) encode,
each scenario has a class that the former limit of the pack kernel (8 touched keys, counted as the pod's keys plus one per
constraining group on a mask key) refused, the oracle places such classes on existing, in-flight and fresh nodes, its
results keep the placement invariants, and its fast mode equals the literal one. The near misses stay refused."""
import ctypes as C

import pytest

import many_key_problems as mk
import placement_invariants as pi

CORPUS = mk.corpus()
IDS = [n for n, _ in CORPUS]
HOSTNAME_KEY = 255  # KSCHED_KEY_HOSTNAME, include/ksched.h
CONSTRAINS = 1      # KSCHED_TOPO_CONSTRAINS


class _Problem(C.Structure):  # the leading fields of ksched_problem, include/ksched.h
    _fields_ = [("n_pods", C.c_int32), ("n_classes", C.c_int32), ("n_existing", C.c_int32), ("n_groups", C.c_int32),
                ("classes", C.c_void_p), ("class_bounds", C.c_void_p), ("pod_class", C.c_void_p), ("pod_timestamp", C.c_void_p),
                ("pod_uid_rank", C.c_void_p), ("existing", C.c_void_p), ("existing_bounds", C.c_void_p), ("groups", C.c_void_p),
                ("group_domain_counts", C.c_void_p), ("group_existing_counts", C.c_void_p), ("class_topo", C.c_void_p),
                ("n_class_topo", C.c_int32)]


class _PodRow(C.Structure):  # ksched_pod_row
    _fields_ = [("requests", C.c_int64 * 8), ("values", C.c_uint64 * 16), ("meta", C.c_uint64), ("tolerated", C.c_uint64),
                ("hp_conflicts", C.c_uint64), ("hp_entries", C.c_uint64), ("res_present", C.c_uint32), ("relax_next", C.c_uint32),
                ("itype_req", C.c_uint32), ("hostname_req", C.c_uint32), ("topo_begin", C.c_uint32), ("topo_end", C.c_uint32),
                ("reserved", C.c_uint64)]


class _Group(C.Structure):  # ksched_topo_group
    _fields_ = [("type", C.c_uint8), ("key", C.c_uint8), ("inverse", C.c_uint8), ("dormant", C.c_uint8), ("max_skew", C.c_int32),
                ("filter_begin", C.c_uint32), ("filter_end", C.c_uint32), ("registered", C.c_uint64), ("extra", C.c_int32), ("pad", C.c_int32)]


class _ClassTopo(C.Structure):  # ksched_class_topo
    _fields_ = [("group", C.c_uint32), ("flags", C.c_uint32)]


assert C.sizeof(_PodRow) == 256 and C.sizeof(_Group) == 32


def encoded_classes(pkg, rs):
    """[(distinct touched keys, former count, constraining groups, relax_next)] per class of the encoding: the keys are the
    pod's keys and the keys of its constraining mask-key groups; the former count adds one per such group"""
    L = pkg.lib()
    L.kh_encoded_problem.restype = C.c_void_p
    L.kh_encoded_problem.argtypes = [C.c_void_p]
    pb = _Problem.from_address(L.kh_encoded_problem(rs.enc))
    rows = (_PodRow * pb.n_classes).from_address(pb.classes) if pb.n_classes else []
    groups = (_Group * max(pb.n_groups, 1)).from_address(pb.groups) if pb.n_groups else []
    rels = (_ClassTopo * max(pb.n_class_topo, 1)).from_address(pb.class_topo) if pb.n_class_topo else []
    out = []
    for r in rows:
        keys = r.meta & 0xFFFF
        old = bin(keys).count("1")
        ncg = 0
        for e in range(r.topo_begin, r.topo_end):
            if rels[e].flags & CONSTRAINS:
                ncg += 1
                g = groups[rels[e].group]
                if g.key != HOSTNAME_KEY:
                    old += 1
                    keys |= 1 << g.key
        out.append((bin(keys).count("1"), old, ncg, r.relax_next))
    return out


def resident(pkg, prob):
    """the encoding of a batch, or of a cluster's candidates' pods"""
    cands = [i for i, n in enumerate(prob.get("nodes", [])) if n.get("candidate")]
    return pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands if not prob["pods"] else ())


def _solve(pkg, oracle, prob, fast=False):
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    oracle.lib.oracle_set_fast(1 if fast else 0)
    try:
        assert oracle.solve(problem, res) == 0, res.error
    finally:
        oracle.lib.oracle_set_fast(0)
    return problem, res


def _many_key_pods(pkg, prob, d):
    """pods whose class at their final relaxation level was refused by the former count"""
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    cls = encoded_classes(pkg, rs)
    out = set()
    for i, lvl in enumerate(d["relax"]):
        c = rs.pod_class(i)
        for _ in range(max(lvl, 0)):
            c = cls[c][3]
        if cls[c][1] > 8:
            out.add(i)
    return out


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_scenario_has_a_class_the_former_count_refused(pkg, name, prob):
    cls = encoded_classes(pkg, resident(pkg, prob))
    assert max(old for _, old, _, _ in cls) > 8
    assert all(keys <= 16 and ncg <= 8 for keys, _, ncg, _ in cls)


def test_sixteen_distinct_keys_where_the_former_count_was_nineteen(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(mk.sixteen(0)))
    assert rs.dims["keys"] == 16
    assert (16, 19, 3) in [c[:3] for c in encoded_classes(pkg, rs)]


def test_relaxation_crosses_the_former_count_both_ways(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(mk.relaxing(0)))
    cls = encoded_classes(pkg, rs)
    chains = [(c[1], cls[c[3]][1]) for c in cls if c[3] != 0xFFFFFFFF]
    assert (12, 8) in chains  # 11 keys + zone spread, relaxed to 7 keys + zone spread
    assert (6, 12) in chains  # 5 keys + capacity-type spread, relaxed to 11 keys + spread


def test_nine_groups_encode_with_nine_constraining_groups(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(mk.nine_groups(0)))
    assert max(ncg for _, _, ncg, _ in encoded_classes(pkg, rs)) == 9


def test_seventeen_keys_are_refused(pkg):
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(mk.seventeen_keys(0)))
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED


def test_oracle_places_many_key_classes_on_existing_in_flight_and_fresh_nodes(pkg, oracle):
    kinds = set()
    for name, prob in CORPUS:
        _, res = _solve(pkg, oracle, prob)
        d = res.to_dict()
        many = _many_key_pods(pkg, prob, d)
        n_ex = len(d["existing"])
        for i in many:
            if 0 <= d["assign"][i] < n_ex:
                kinds.add("existing")
        for n in d["newNodes"]:
            if n["pods"][0] in many:
                kinds.add("fresh")
            if any(p in many for p in n["pods"][1:]):
                kinds.add("in-flight")
    assert kinds == {"existing", "in-flight", "fresh"}


def test_grown_requirements_keep_in_pods_off_bare_nodes(pkg, oracle):
    """the NotIn / DoesNotExist pods land on the nodes without nvme / cost-center first; the later pods with nvme In [true]
    then never share such a node with them (a node without the well-known key would admit them), and the cost-center In
    pods never take a node without that custom key"""
    for seed in range(2):
        prob = mk.existing(seed)
        _, res = _solve(pkg, oracle, prob)
        d = res.to_dict()
        n_ex = len(d["existing"])
        app = lambda i: prob["pods"][i]["labels"]["app"]
        on = {}
        for i, a in enumerate(d["assign"]):
            if 0 <= a < n_ex:
                on.setdefault(prob["nodes"][d["existing"][a]["node"]]["name"], set()).add(app(i))
        bare = [apps for name, apps in on.items() if name.startswith("bare-")]
        assert any("avoid" in apps for apps in bare)
        assert not any({"avoid", "want-nvme"} <= apps for apps in bare)
        assert not any("want-cc" in apps for apps in bare)


# the invariants' zone-spread check reads the zones of new nodes: batches without existing nodes; inflight() allows 2 zones
BATCHES = [(n, p) for n, p in CORPUS if not p.get("nodes")]


@pytest.mark.parametrize("name,prob", BATCHES, ids=[n for n, _ in BATCHES])
def test_oracle_results_keep_the_invariants(pkg, oracle, name, prob):
    problem, res = _solve(pkg, oracle, prob)
    pi.check(problem, res, n_zones=2 if name.startswith("inflight") else 3)


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_oracle_fast_mode_equals_literal(pkg, oracle, name, prob):
    _, literal = _solve(pkg, oracle, prob)
    _, fast = _solve(pkg, oracle, prob, fast=True)
    assert fast.to_dict() == literal.to_dict()
