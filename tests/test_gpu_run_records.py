"""GPU: the class runs' relation tables (csrc/pack_kernel.cuh: run_rec_build), one record per class built in the row
gather's launch before the pack kernel. The records a resident Solve downloads are compared field by field with a
restatement of the rules from the encoder's class topology, for the run, shape, round-stretch, fill-stretch,
variant-table and many-provisioner corpora. A builder that is too strict would not change any placement (the class
takes the generic step), so only this comparison sees it.

The seeded corpus below reaches the entry's checks on the group state: later deployments whose hostname anti-affinity
or hostname spread selects an earlier deployment's pods (the group counts slots at the run's entry, grp_host_total > 0),
near misses whose selectors match nothing placed before them (total 0, the hostname counts are not loaded), and
preferred terms that are relaxed during the Solve. Each of its problems equals the oracle's whole result at 32, 128 and
512 threads and under each KSCHED_NO_* switch, KSCHED_NO_VARSTORE and KSCHED_NO_RUNDERIVE included."""
import ctypes as C

import pytest

import fill_stretch_problems as fsp
import fixtures as fx
import provisioner_problems as pp
import round_stretch_problems as rsp
import run_problems as rp
import shape_problems as sp
import variant_table_problems as vt
from fixtures import HOSTNAME, ZONE
from oracle_compare import MODE_SWITCHES, set_modes

pytestmark = pytest.mark.gpu

HOSTNAME_KEY, NONE = 255, 0xFFFFFFFF  # KSCHED_KEY_HOSTNAME, KSCHED_NONE, include/ksched.h
CONSTRAINS, SELECTS, RECORDS, RECORDS_INVERSE = 1, 2, 4, 8  # KSCHED_TOPO_*
RUN_HOST, RUN_MASK, RUN_DOM = 4, 2, 16  # kRunHost, kRunMask, kRunDom (csrc/pack_state.cuh, pack_kernel.cuh)


class _Problem(C.Structure):  # the leading fields of ksched_problem, include/ksched.h, up to filter_term_itype
    _fields_ = [("n_pods", C.c_int32), ("n_classes", C.c_int32), ("n_existing", C.c_int32), ("n_groups", C.c_int32),
                ("classes", C.c_void_p), ("class_bounds", C.c_void_p), ("pod_class", C.c_void_p), ("pod_timestamp", C.c_void_p),
                ("pod_uid_rank", C.c_void_p), ("existing", C.c_void_p), ("existing_bounds", C.c_void_p), ("groups", C.c_void_p),
                ("group_domain_counts", C.c_void_p), ("group_existing_counts", C.c_void_p), ("class_topo", C.c_void_p),
                ("n_class_topo", C.c_int32), ("filter_terms", C.c_void_p), ("n_filter_terms", C.c_int32), ("itype_req_sets", C.c_void_p),
                ("itype_req_complement", C.c_void_p), ("n_itype_reqs", C.c_int32), ("hostname_reqs", C.c_void_p),
                ("n_hostname_reqs", C.c_int32), ("max_new_nodes", C.c_int32), ("write_feasibility", C.c_int32),
                ("count_nodes_visited", C.c_int32), ("class_volumes", C.c_void_p), ("existing_volumes", C.c_void_p),
                ("volume_driver_mask", C.c_uint64 * 4), ("class_tolerated_ext", C.c_void_p), ("n_tolerated_ext_words", C.c_int32),
                ("pad_ext", C.c_int32), ("class_requests_ext", C.c_void_p), ("class_res_ext_present", C.c_void_p),
                ("existing_available_ext", C.c_void_p), ("class_hostport_conflicts_ext", C.c_void_p),
                ("class_hostport_entries_ext", C.c_void_p), ("existing_hostport_ext", C.c_void_p), ("n_hostport_ext_words", C.c_int32),
                ("pad_hostport", C.c_int32), ("hostname_slots", C.c_void_p), ("filter_term_hostname", C.c_void_p),
                ("n_hostname_words", C.c_int32), ("pad_hostname", C.c_int32), ("filter_term_itype", C.c_void_p)]


class _Catalog(C.Structure):  # the leading fields of ksched_catalog
    _fields_ = [("n_keys", C.c_int32), ("n_res", C.c_int32), ("n_types", C.c_int32), ("n_templates", C.c_int32),
                ("keys", C.c_void_p), ("key_regions", C.c_void_p), ("key_int_values", C.c_void_p), ("types", C.c_void_p),
                ("type_bounds", C.c_void_p), ("type_capacity", C.c_void_p), ("templates", C.c_void_p)]


class _KeyInfo(C.Structure):  # ksched_keyinfo
    _fields_ = [("dict_mask", C.c_uint64), ("int_mask", C.c_uint64), ("well_known", C.c_int32), ("is_zone", C.c_int32),
                ("is_ct", C.c_int32), ("pad", C.c_int32)]


class _ReqSet(C.Structure):  # ksched_reqset (also the head of ksched_template)
    _fields_ = [("values", C.c_uint64 * 16), ("meta", C.c_uint64)]


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


assert _Problem.filter_terms.offset == 112 and _Problem.filter_term_itype.offset == 320
assert C.sizeof(_PodRow) == 256 and C.sizeof(_Group) == 32 and C.sizeof(_KeyInfo) == 32


def expected_records(pkg, rs):
    """(records, key_regions): the relation tables of every class of the encoding, restated from its class topology, as
    run_rec_build must build them (fields that are not set stay 0; an ineligible class's record is all 0)"""
    L = pkg.lib()
    L.kh_encoded_catalog.restype = L.kh_encoded_problem.restype = C.c_void_p
    L.kh_encoded_catalog.argtypes = L.kh_encoded_problem.argtypes = [C.c_void_p]
    pb = _Problem.from_address(L.kh_encoded_problem(rs.enc))
    cat = _Catalog.from_address(L.kh_encoded_catalog(rs.enc))
    rows = (_PodRow * pb.n_classes).from_address(pb.classes)
    groups = (_Group * pb.n_groups).from_address(pb.groups) if pb.n_groups else []
    rels = (_ClassTopo * pb.n_class_topo).from_address(pb.class_topo) if pb.n_class_topo else []
    keys = (_KeyInfo * cat.n_keys).from_address(cat.keys) if cat.n_keys else []
    tmpl = _ReqSet.from_address(cat.templates)  # template 0: the one template of a topology class
    nf = pb.n_filter_terms
    terms = (_ReqSet * nf).from_address(pb.filter_terms) if nf else []
    f_host = (C.c_uint32 * nf).from_address(pb.filter_term_hostname) if nf and pb.filter_term_hostname else None
    f_itype = (C.c_uint32 * nf).from_address(pb.filter_term_itype) if nf and pb.filter_term_itype else None

    def has_filter(G):  # a TopologyNodeFilter, unless one of its terms has no requirement (it matches every node)
        for f in range(G.filter_begin, min(G.filter_end, nf)):
            if terms[f].meta & 0xFFFF == 0 and (f_host is None or f_host[f] == NONE) and (f_itype is None or f_itype[f] == NONE):
                return False
        return G.filter_begin != G.filter_end

    host_row, nh = {}, 0
    for g, G in enumerate(groups):  # the hostname counter rows, in group order (ksched_upload)
        if G.key == HOSTNAME_KEY:
            host_row[g] = nh
            nh += 1
    out = []
    for r in rows:
        rec = dict(ok=0, n_host=0, n_mask=0, h_row=[0] * 4, h_group=[0] * 4, h_lim=[0] * 4, h_times=[0] * 4, m_group=[0] * 2,
                   m_skew=[0] * 2, m_key=[0] * 2, m_self=[0] * 2, m_rec=[0] * 2, m_wk=[0] * 2, m_tallow=[0] * 2, m_dict=[0] * 2)
        ok = r.topo_begin == r.topo_end or cat.n_templates == 1
        for e in range(r.topo_begin, r.topo_end):
            if not ok:
                break
            flags, g = rels[e].flags, rels[e].group
            G = groups[g]
            if not flags & CONSTRAINS or (flags & RECORDS and has_filter(G)):
                ok = False
                break
            times = bool(flags & RECORDS) + bool(flags & RECORDS_INVERSE)
            self_ = 1 if flags & SELECTS else 0
            if G.key == HOSTNAME_KEY:
                j = rec["n_host"]
                if G.type == 1 or j == RUN_HOST:
                    ok = False
                    break
                lim = G.max_skew - self_ if G.type == 0 else 0
                rec["h_row"][j], rec["h_group"][j], rec["h_times"][j] = host_row[g], g, times
                rec["h_lim"][j] = min(lim, 0x10000) if lim >= -1 else -1
                rec["n_host"] += 1
            else:
                k, j = G.key, rec["n_mask"]
                dmask = keys[k].dict_mask
                if G.type != 0 or j == RUN_MASK or flags & RECORDS_INVERSE or dmask >> RUN_DOM or k in rec["m_key"][:j]:
                    ok = False
                    break
                present, comp = (tmpl.meta >> k) & 1, (tmpl.meta >> (16 + k)) & 1
                allowed = ((~tmpl.values[k] & dmask) if comp else tmpl.values[k]) if present else dmask
                rec["m_group"][j], rec["m_skew"][j], rec["m_key"][j] = g, G.max_skew, k
                rec["m_self"][j], rec["m_rec"][j], rec["m_wk"][j] = self_, 1 if flags & RECORDS else 0, 1 if keys[k].well_known else 0
                rec["m_dict"][j], rec["m_tallow"][j] = dmask & 0xFFFFFFFF, allowed & 0xFFFFFFFF
                rec["n_mask"] += 1
        if ok:
            rec["ok"] = 1
        else:
            rec = {k: (0 if isinstance(v, int) else [0] * len(v)) for k, v in rec.items()}
        out.append(rec)
    return out, bool(cat.key_regions), pb.n_existing


def check_records(pkg, problem):
    """one resident Solve of the problem; its downloaded records equal the restatement (None when the Solve builds none:
    the problem has existing nodes)"""
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    rs.run()
    got = rs.run_records()
    want, regions, n_existing = expected_records(pkg, rs)
    if n_existing:
        assert got is None
        return 0
    assert got is not None and len(got) == len(want)
    for c, (g, w) in enumerate(zip(got, want)):
        for f, v in w.items():
            have = [int(x) for x in g[f]] if isinstance(v, list) else int(g[f])
            if regions and f in ("m_dict", "m_tallow"):  # the library adds region bits to the dictionary masks
                continue
            assert have == v, (c, f, have, v)
        # pin_neutral (the catalog's own table): values of the key's dictionary only
        for j in range(w["n_mask"]):
            assert int(g["m_neutral"][j]) & ~int(g["m_dict"][j]) == 0, (c, j)
        assert [int(x) for x in g["m_neutral"][w["n_mask"]:]] == [0] * (2 - w["n_mask"]), c
    return sum(r["ok"] for r in want)


def _problem(pkg, mod, name, seed):
    built = mod.build(name, seed)
    return pkg.Problem.from_dict(built[0] if isinstance(built, tuple) else built)


CORPORA = [("run", rp, c) for c in rp.CORPUS] + [("shape", sp, c) for c in sp.CORPUS] + [("round", rsp, c) for c in rsp.CORPUS] + \
          [("fill", fsp, c) for c in fsp.CORPUS] + [("table", vt, c) for c in vt.CORPUS]


@pytest.mark.parametrize("corpus,mod,case", CORPORA, ids=[f"{k}-{c[0]}-{c[1]}" for k, _, c in CORPORA])
def test_records_match_restatement(pkg, monkeypatch, corpus, mod, case):
    set_modes(monkeypatch)
    check_records(pkg, _problem(pkg, mod, *case))


PROVISIONERS = pp.corpus()


@pytest.mark.parametrize("name,prob", PROVISIONERS, ids=[n for n, _ in PROVISIONERS])
def test_records_many_provisioners(pkg, monkeypatch, name, prob):
    set_modes(monkeypatch)
    check_records(pkg, pkg.Problem.from_dict(prob))


# ---------------------------------------------------------------- seeded corpus: the group state at a run's entry
def _anti(labels):
    return {"required": [fx.affinity_term(HOSTNAME, labels)]}


def cross_deployment(seed):
    """earlier deployments' pods are selected by later deployments' hostname anti-affinity and hostname spreads (their
    groups count slots when the later class's run starts), next to zone spreads of their own"""
    zs = rp.zone_names(3, "eu-south")
    its = rp.zonal_types(zs, [(4, 16), (8, 32), (16, 64)], pods_cap=[20, 110][seed % 2])
    r = rp.Runs(f"x{seed}")
    r.run("db", [31, 33, 129][seed % 3], {"cpu": "2", "memory": "2Gi"}, labels={"app": "db", "tier": "data"})
    r.run("cache", 32, {"cpu": "1", "memory": "1Gi"}, labels={"app": "cache", "tier": "data"},
          topologySpreadConstraints=[fx.spread(HOSTNAME, {"app": "cache"}, max_skew=1)])
    r.run("web", [127, 128, 250][seed % 3], {"cpu": "500m", "memory": "512Mi"}, labels={"app": "web"},
          podAntiAffinity=_anti({"app": "db"}), topologySpreadConstraints=[fx.spread(ZONE, {"app": "web"})])
    r.run("api", 129, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "api"},
          topologySpreadConstraints=[fx.spread(HOSTNAME, {"tier": "data"}, max_skew=1 + seed % 3), fx.spread(ZONE, {"app": "api"})])
    r.run("worker", 250, rp.SMALL, labels={"app": "worker"},
          topologySpreadConstraints=[fx.spread(HOSTNAME, {"app": "web"}, max_skew=2)])
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


def near_miss(seed):
    """the same shapes, but every selector of a later deployment matches no pod placed before it (a label nobody carries,
    or the deployment's own pods): the groups count no slot at the run's entry"""
    zs = rp.zone_names(3, "eu-south")
    its = rp.zonal_types(zs, [(4, 16), (8, 32)], pods_cap=[20, 110][seed % 2])
    r = rp.Runs(f"n{seed}")
    r.run("db", 33, {"cpu": "2", "memory": "2Gi"}, labels={"app": "db", "tier": "data"})
    r.run("web", [127, 250][seed % 2], {"cpu": "500m", "memory": "512Mi"}, labels={"app": "web"},
          podAntiAffinity=_anti({"app": "nobody"}), topologySpreadConstraints=[fx.spread(ZONE, {"app": "web"})])
    r.run("api", 129, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "api"},
          topologySpreadConstraints=[fx.spread(HOSTNAME, {"app": "api"}, max_skew=2), fx.spread(HOSTNAME, {"tier": "none"})])
    r.run("solo", 32, rp.SMALL, labels={"app": "solo"}, podAntiAffinity=_anti({"app": "solo"}))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


def relaxed_terms(seed):
    """preferred terms relaxed during the Solve: a preferred node affinity no zone satisfies, preferred hostname
    anti-affinity against an earlier deployment, a ScheduleAnyway spread whose relaxation leaves a class with other
    groups; a relaxed class's groups may be created then (dormant until the first pod that owns them is relaxed)"""
    zs = rp.zone_names(3, "eu-east")
    its = rp.zonal_types(zs, [(4, 16), (8, 32)])
    r = rp.Runs(f"r{seed}")
    r.run("db", 32, {"cpu": "2", "memory": "2Gi"}, labels={"app": "db"})
    r.run("prefer", 127, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "prefer"},
          nodeAffinity={"preferred": [{"weight": 50, "terms": [{"key": ZONE, "operator": "In", "values": ["no-such-zone"]}]}]},
          podAntiAffinity={"preferred": [{"weight": 10, "term": fx.affinity_term(HOSTNAME, {"app": "db"})}]},
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "prefer"})])
    r.run("anyway", [128, 250][seed % 2], rp.SMALL, labels={"app": "anyway"},
          topologySpreadConstraints=[fx.spread(ZONE, {"app": "anyway"}, when="ScheduleAnyway"),
                                     fx.spread(HOSTNAME, {"app": "db"}, max_skew=3)])
    r.run("soft", 33, rp.SMALL, labels={"app": "soft"},
          podAntiAffinity={"preferred": [{"weight": 10, "term": fx.affinity_term(HOSTNAME, {"app": "prefer"})}]},
          nodeAffinity={"preferred": [{"weight": 5, "terms": [{"key": ZONE, "operator": "In", "values": [zs[seed % 3]]}]}]})
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


SEEDED = {"cross_deployment": cross_deployment, "near_miss": near_miss, "relaxed_terms": relaxed_terms}
SEEDED_CASES = [(n, s) for n in SEEDED for s in (0, 1, 2)]


@pytest.mark.parametrize("name,seed", SEEDED_CASES, ids=[f"{n}-{s}" for n, s in SEEDED_CASES])
def test_seeded_records_match_restatement(pkg, monkeypatch, name, seed):
    set_modes(monkeypatch)
    assert check_records(pkg, pkg.Problem.from_dict(SEEDED[name](seed))) > 0  # some class reaches a class run's entry


@pytest.mark.parametrize("name,seed", SEEDED_CASES, ids=[f"{n}-{s}" for n, s in SEEDED_CASES])
def test_seeded_every_block_size_and_switch(pkg, oracle, monkeypatch, name, seed):
    problem = pkg.Problem.from_dict(SEEDED[name](seed))
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    run = pkg.ResidentSolve(problem)
    run.set_count_visited(False)
    run.load()
    envs = [f"KSCHED_PACK_THREADS={t}" for t in (32, 128, 512)] + list(MODE_SWITCHES) + ["KSCHED_NO_RUNDERIVE"]
    for env in envs:
        set_modes(monkeypatch, env)
        monkeypatch.delenv("KSCHED_NO_RUNDERIVE", raising=False)
        if env == "KSCHED_NO_RUNDERIVE":
            monkeypatch.setenv(env, "1")
        run.run()
        res = run.download()
        assert (res.assign == want.assign).all(), env
        assert (res.relax_level == want.relax_level).all(), env
        assert res.digest() == want.digest(), env
    set_modes(monkeypatch)
