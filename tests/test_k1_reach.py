"""CPU: every scenario of tests/k1_problems.py reaches the K1 path it is built for, on a 114-SM and a 132-SM H100. What the
class pass does with each row is restated from the kernel's launch rule (k1_problems.k1_grid / paths) over the encoder's own
class rows (kh_encoded_class_row); test_gpu_feasibility_paths.py confirms the launch with the kernel's own plan."""
import pytest

import k1_problems as kp

N_SM = (114, 132)


def _encode(pkg, s):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(s["prob"]))
    nc = rs.dims["classes"]
    if s["class_shape"] is not None:
        assert nc == len(s["class_shape"])
        for i in range(0, len(s["pod_shape"]), 97):  # the builder's class table is the encoder's
            assert s["class_shape"][rs.pod_class(i)] == s["pod_shape"][i], i
    rows = [rs.class_row(c) for c in range(nc)]
    return rs, rows


def _paths(rs, rows, n_sm, cacheable=True):
    ext = rs.dims["resources_ext"] > 0
    return kp.paths([kp.cmp_words(r, ext) for r in rows], n_sm, cacheable)


def _differing_words(a, b):
    return [w for w in range(32) if w != 31 and a[w] != b[w]]


def _check_near_misses(rows, paths, s, chunk, offsets):
    seen = {}
    for j, kind in s["near"].items():
        d = _differing_words(rows[j - 1], rows[j])
        assert len(d) == 1, (kind, j, d)  # one compared word and nothing else
        w = d[0]
        if kind == "value":
            assert 8 <= w < 24, (kind, w)
        else:
            assert w == kp.NEAR_WORD[kind], (kind, w)
            if kind == "itype":
                assert (int(rows[j - 1][29]) ^ int(rows[j][29])) >> 32 == 0  # the low half only
        assert paths[j] == "compute", (kind, j, paths[j])
        seen.setdefault(kind, set()).add(j % chunk)
    assert set(seen) == set(kp.NEAR)
    for kind, offs in seen.items():
        assert offs == set(offsets), (kind, offs)
    return seen


@pytest.mark.parametrize("n_sm", N_SM)
def test_job_chunks_reach_the_row_cache(pkg, n_sm):
    s = kp.job_chunks(n_sm)
    rs, rows = _encode(pkg, s)
    nc = len(rows)
    blocks, warps, chunk = kp.k1_grid(nc, n_sm)
    assert blocks == 2 * n_sm and chunk == 3 and 2 * warps <= nc <= 3 * warps
    paths = _paths(rs, rows, n_sm)
    assert paths.count("row") > warps // 2 and "batch" not in paths
    _check_near_misses(rows, paths, s, chunk, (0, 1, 2))
    for j, kind in s["near"].items():
        if j % chunk == 2:
            assert paths[j - 1] == "row", (kind, j)  # right after a cache-served row
    nofit = s["shapes"].index(kp.NOFIT)
    assert sum(1 for j in range(nc) if s["class_shape"][j] == nofit and paths[j] == "row") >= 3
    prefer = s["shapes"].index(kp.PREFER)
    j = s["class_shape"].index(prefer)
    assert paths[j] == paths[j + 1] == paths[j + 2] == "compute"  # the relaxed class follows and breaks the run
    assert s["shapes"][s["class_shape"][j + 1]] == kp._with(kp.PREFER, nodeAffinity=None)
    assert _differing_words(rows[j + 1], rows[j + 2]) == []  # ... and equals the run it interrupts


@pytest.mark.parametrize("n_sm", N_SM)
def test_whole_batches_are_served_from_the_cache(pkg, n_sm):
    s = kp.whole_batches(n_sm)
    rs, rows = _encode(pkg, s)
    nc = len(rows)
    _, warps, chunk = kp.k1_grid(nc, n_sm)
    assert chunk == 50 and nc > 2 * 16 * warps
    paths = _paths(rs, rows, n_sm)
    _check_near_misses(rows, paths, s, chunk, (0, 1, 15, 16, 31, 32, 47, 49))
    for j, kind in s["near"].items():
        if j % chunk == 32:
            assert paths[j - 16:j] == ["batch"] * 16, (kind, j)  # right after a full-batch repeat
        if j % chunk in (31, 47):
            assert paths[j - 15:j] == ["row"] * 15, (kind, j)  # the last row of a batch the vote turned down
    full = [w for w in range(warps) if paths[w * chunk + 16:w * chunk + 48] == ["batch"] * 32]
    assert len(full) > warps // 2  # two consecutive full-batch repeats
    assert sum(1 for w in full if paths[w * chunk + 48:w * chunk + 50] == ["batch"] * 2) > warps // 2  # a partial batch (nb = 2)
    mixed = [w for w in range(warps) if "row" in paths[w * chunk + 16:w * chunk + 32] and "compute" in paths[w * chunk + 16:w * chunk + 32]]
    assert mixed
    nofit = s["shapes"].index(kp.NOFIT)
    assert sum(1 for j in range(nc) if s["class_shape"][j] == nofit and paths[j] == "batch") >= 32


@pytest.mark.parametrize("n_sm", N_SM)
def test_wide_batches_use_two_column_words_per_lane(pkg, n_sm):
    s = kp.wide_batches(n_sm)
    rs, rows = _encode(pkg, s)
    _, warps, chunk = kp.k1_grid(len(rows), n_sm)
    W32 = 2 * rs.dims["type_words"]
    assert chunk == 20 and -(-W32 // 32) == 2 and rs.dims["templates"] == 2
    paths = _paths(rs, rows, n_sm)
    assert sum(1 for w in range(warps) if paths[w * chunk + 16:w * chunk + 20] == ["batch"] * 4) > warps // 2
    for j, kind in s["near"].items():
        assert paths[j] == "compute" and len(_differing_words(rows[j - 1], rows[j])) == 1, (kind, j)


@pytest.mark.parametrize("n_sm", N_SM)
def test_layouts_sit_on_the_intended_side_of_each_threshold(pkg, n_sm):
    odd = False
    for s in kp.layout(n_sm):
        rs, rows = _encode(pkg, s)
        d = rs.dims
        assert d["resources"] == s["n_res"] and d["resources_ext"] == 0
        V, T = d["templates"], d["types"]
        W32 = 2 * d["type_words"]
        wpl = -(-W32 // 32)
        assert (V * wpl <= kp.K1_CACHE_WORDS) == s["cache"], s["name"]
        alloc_in, (tables_surely, tables_maybe) = kp.smem_plan(d["resources"], T, V, d["keys"])
        assert alloc_in == s["alloc"], s["name"]
        if s["tables"] is True:
            assert tables_surely, s["name"]
        elif s["tables"] is False:
            assert not tables_maybe, s["name"]
        nc = len(rows)
        _, warps, _ = kp.k1_grid(nc, n_sm)
        assert nc > warps
        paths = _paths(rs, rows, n_sm, s["cache"])
        assert (paths.count("row") > warps // 8) == s["cache"], s["name"]
        odd = odd or T % 64 != 0
    names = {s["name"]: s for s in kp.layout(n_sm)}
    assert kp.smem_plan(8, 2048, 1, 4)[0] and not kp.smem_plan(8, 2049, 1, 4)[0]  # exactly 128 KiB, and one type more
    assert {"v8_t2048", "v4_t4000", "v9_t2048", "v17_t1000", "r8_t2048_v50", "r8_t2049"} <= set(names) and odd


@pytest.mark.parametrize("n_sm", N_SM)
def test_best_edges_and_stream_shapes(pkg, n_sm):
    s = kp.best_edges(n_sm)
    rs, rows = _encode(pkg, s)
    _, warps, _ = kp.k1_grid(len(rows), n_sm)
    assert len(rows) > warps and "row" in _paths(rs, rows, n_sm)
    st = kp.stream(n_sm)
    P = len(st["prob"]["pods"])
    assert P % 32 != 0 and P > 2048 * n_sm
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(st["prob"]))
    assert rs.dims["pods"] == P and rs.dims["classes"] == len(st["shapes"]) <= 8
    # feasibility_kernel: min(8 * n_sm, ceil(ceil(P / 32) / 8)) CTAs of 8 warps, one 32-row block per warp and iteration
    nblk = -(-P // 32)
    warps = min(8 * n_sm, -(-nblk // 8)) * 8
    assert nblk > warps


def test_every_near_miss_changes_the_reference_columns(pkg, oracle):
    s = kp.job_chunks(132)
    F, best = kp.reference(pkg, oracle, s)
    base = s["shapes"].index(kp.BASE)
    for kind, spec in kp.NEAR.items():
        k = s["shapes"].index(spec)
        assert (F[k] != F[base]).any(), kind
    assert best[s["shapes"].index(kp.NOFIT)] == kp.NO_BEST and not F[s["shapes"].index(kp.NOFIT)].any()
    assert (F[s["shapes"].index(kp.PREFER)] != F[base]).any()
    e = kp.best_edges(132)
    Fe, be = kp.reference(pkg, oracle, e)
    names = [it["name"] for it in e["prob"]["instanceTypes"]]
    pos, p32 = kp.column_order(e["prob"])
    shape = {g: next(i for i, sp in enumerate(e["shapes"]) if sp["nodeSelector"]["grp"] == g) for g in ("eq", "f32", "zero", "dead")}
    assert int(be[shape["eq"]]) & 0xFFFFFF == pos[names.index("eq-a")] < pos[names.index("eq-b")]
    hi, lo = names.index("f32-hi"), names.index("f32-lo")
    assert p32[hi] == p32[lo] and pos[lo] < pos[hi]  # one float32, two columns
    assert int(be[shape["f32"]]) == (p32[hi] << 32) | (0 << 24) | pos[hi]  # template 0 wins against the earlier column
    assert int(be[shape["zero"]]) >> 32 == 0
    assert be[shape["dead"]] == kp.NO_BEST and pos[names.index("dead")] == len(names) - 1
    dead = e["prob"]["instanceTypes"][names.index("dead")]  # its requirements admit the pod: only availability turns it away
    assert all(r["values"] for r in dead["requirements"]) and not any(o["available"] for o in dead["offerings"])


def _corpora():
    import extended_resource_problems as xp
    import fuzz_problems
    import hostname_problems, hostport_problems, itype_filter_problems, many_key_problems, namespace_problems
    import numeric_problems, provisioner_problems, taint_problems, volume_problems, wide_problems, zone_problems
    out = [(c[0], next(x for x in c[1:] if isinstance(x, dict)))
           for m in (xp, hostname_problems, hostport_problems, itype_filter_problems, many_key_problems, namespace_problems,
                     numeric_problems, provisioner_problems, taint_problems, volume_problems, wide_problems, zone_problems)
           for c in m.corpus()]
    out += xp.fresh_corpus() + [("pairs", xp.pairs())] + [(f"fuzz-{s}", fuzz_problems.random_problem(s)) for s in range(20)]
    return out


def test_existing_corpora_and_baseline_configs_never_reach_the_row_cache(pkg):
    """what this file's scenarios add: no problem of the other corpora nor of C2-C5 has a row K1 serves from its cache"""
    checked = 0
    for name, prob in _corpora():
        try:
            rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
        except pkg.KschedError:
            continue  # corpora that also hold refused near misses
        rows = [rs.class_row(c) for c in range(rs.dims["classes"])]
        for n_sm in N_SM:
            assert set(_paths(rs, rows, n_sm)) <= {"compute"}, name
        checked += 1
    for config, pods, types, nodes in ((2, 10000, 500, 0), (3, 50000, 1000, 0), (4, 100000, 1000, 0), (5, 600, 1000, 60)):
        rs = pkg.ResidentSolve(pkg.Problem.synth(config, pods, types, 42, nodes))
        rows = [rs.class_row(c) for c in range(rs.dims["classes"])]
        for n_sm in N_SM:
            assert set(_paths(rs, rows, n_sm)) <= {"compute"}, config
        checked += 1
    assert checked > 30
