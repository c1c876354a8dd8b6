"""GPU: K1's feasibility matrix F and best_column on the paths tests/k1_problems.py reaches (the consecutive-row cache, whole
16-row batches, the cache layouts and shared-memory staging choices, best_column's key at its edges, the pod-row stream)
equal a fresh-node reference built from the oracle, pod by pod, and so does every column shard of them. The scenarios are
sized from this device's SM count and the kernel's own launch plan (kh_gpu_k1_plan) confirms the path.

Before each check a different problem of the same size runs on the handle, so that no result of an earlier run of the same
problem can stand in for the one under test."""
import numpy as np
import pytest

import k1_problems as kp
import placement_invariants
from oracle_compare import compare

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def n_sm():
    return kp.device_sm_count()


@pytest.fixture
def shard(pkg):
    """the process handle's column shard; restored to (0, 1) afterwards (the handle serves the whole session)"""
    yield lambda rank, world: pkg.set_shard(rank, world)
    pkg.set_shard(0, 1)


_REF = {}


def _reference(pkg, oracle, s):
    key = (s["name"], s["n_sm"])
    if key not in _REF:
        _REF[key] = kp.reference(pkg, oracle, s)
    return _REF[key]


def _scrub(pkg, s):
    """a different problem with the same catalog, templates and number of classes (every pod fits almost anywhere)"""
    prob = s["prob"]
    n = len(prob["pods"]) if s["class_shape"] is None else len(s["class_shape"])
    pods = [{"name": f"scrub-{i}", "uid": f"scrub-{i}", "requests": {"cpu": "10m"}, "labels": {"scrub": str(i)}} for i in range(n)]
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(dict(prob, pods=pods)))
    rs.set_count_visited(False)
    rs.load()
    rs.run()


def _run(pkg, s):
    _scrub(pkg, s)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(s["prob"]))
    rs.set_count_visited(False)
    rs.load()
    rs.run()
    res, feas, best = rs.download(want_feasibility=True)
    return rs, res, feas, best, rs.k1_plan()


def _assert_rows(s, feas, best, F, B, what=""):
    """every pod's F row and best_column against its shape's reference"""
    shape = np.asarray(s["pod_shape"])
    want_f, want_b = F[shape], B[shape]
    bad = np.nonzero((feas != want_f).any(axis=(1, 2)) | (best != want_b))[0]
    if len(bad):
        p = int(bad[0])
        pytest.fail(f"{s['name']}{what}: {len(bad)} pods differ from the reference, first pod {p} (shape {shape[p]}): "
                    f"F {feas[p].tolist()} != {want_f[p].tolist()}, best {int(best[p]):#x} != {int(want_b[p]):#x}")


def _assert_plan(s, rs, plan, n_sm):
    nc = rs.dims["classes"]
    blocks, _, chunk = kp.k1_grid(nc, n_sm)
    assert (plan["blocks"], plan["chunk"]) == (blocks, chunk), plan
    assert plan["cacheable"] == int(s.get("cache", True)), plan
    if "alloc" in s:
        assert plan["alloc_in_smem"] == int(s["alloc"]), plan
    if s.get("tables") is not None:
        assert plan["tables_in_smem"] == int(s["tables"]), plan


def _check(pkg, oracle, s, n_sm, with_oracle=True):
    rs, res, feas, best, plan = _run(pkg, s)
    _assert_plan(s, rs, plan, n_sm)
    F, B = _reference(pkg, oracle, s)
    _assert_rows(s, feas, best, F, B)
    if with_oracle:
        compare(pkg, oracle, pkg.Problem.from_dict(s["prob"]))
    return res


def test_job_chunks(pkg, oracle, n_sm):
    _check(pkg, oracle, kp.job_chunks(n_sm), n_sm)


@pytest.mark.parametrize("i", range(6), ids=["v8_t2048", "v4_t4000", "v9_t2048", "v17_t1000", "r8_t2048_v50", "r8_t2049"])
def test_cache_layouts_and_staging(pkg, oracle, n_sm, i):
    s = kp.layout(n_sm)[i]
    _check(pkg, oracle, s, n_sm)


def test_best_column_edges(pkg, oracle, n_sm):
    s = kp.best_edges(n_sm)
    _check(pkg, oracle, s, n_sm)
    # the reference keys themselves: input order at equal prices, the template field at equal float32 prices, price 0
    F, B = _reference(pkg, oracle, s)
    assert kp.NO_BEST in B.tolist() and any(int(b) >> 32 == 0 for b in B)


def _large(pkg, oracle, s, n_sm, shard, with_oracle):
    """the large scenarios: F and best_column against the reference, and the whole result as the same Solve with sharded
    columns (world 3: the pack kernel's path without F). The batch scenarios are compared with the oracle too (one CPU oracle
    Solve of their 84 000-211 000 single-pod classes takes 13-25 s); stream (270 000+ pods of five classes) is not: its CPU
    oracle Solve did not finish in 5 minutes. placement_invariants checks the same batch without its daemonset, whose
    overhead it does not model."""
    res = _check(pkg, oracle, s, n_sm, with_oracle=with_oracle)
    problem = pkg.Problem.from_dict(s["prob"])
    one = pkg.Scheduler(problem).solve(count_visited=False)
    assert one.to_dict(brief=True)["assign"] == res.to_dict(brief=True)["assign"]
    shard(1, 3)
    three = pkg.Scheduler(problem).solve(count_visited=False)
    shard(0, 1)
    assert int(three.digest()) == int(one.digest())
    bare = pkg.Problem.from_dict(dict(s["prob"], daemonSetPods=[]))
    placement_invariants.check(bare, pkg.Scheduler(bare).solve(count_visited=False))


def test_whole_batches(pkg, oracle, n_sm, shard):
    _large(pkg, oracle, kp.whole_batches(n_sm), n_sm, shard, with_oracle=True)


def test_whole_batches_two_words_per_lane(pkg, oracle, n_sm, shard):
    _large(pkg, oracle, kp.wide_batches(n_sm), n_sm, shard, with_oracle=True)


def test_stream_of_many_pod_rows(pkg, oracle, n_sm, shard):
    _large(pkg, oracle, kp.stream(n_sm), n_sm, shard, with_oracle=False)


SHARDED = ["job_chunks", "best_edges", "v17_t1000"]


def _scenario(name, n_sm):
    if name == "job_chunks":
        return kp.job_chunks(n_sm)
    if name == "best_edges":
        return kp.best_edges(n_sm)
    return next(s for s in kp.layout(n_sm) if s["name"] == name)


@pytest.mark.parametrize("world", [2, 3, 7])
@pytest.mark.parametrize("name", SHARDED)
def test_column_shards(pkg, oracle, n_sm, shard, name, world):
    """rank r computes only its u32 words of F (the rest reads 0) and its best key; the ranks' minimum is world 1's best.
    job_chunks has W32 = 2 (world 3: a shard of one u32 word, half of a u64 word, and an empty one), v17_t1000 W32 = 32 (world
    3: 11 words, so a shard boundary splits a u64 word)."""
    s = _scenario(name, n_sm)
    F, B = _reference(pkg, oracle, s)
    W32 = 2 * F.shape[2]
    shape = np.asarray(s["pod_shape"])
    lowest = None
    spans = [pkg.shard_range(W32, r, world) for r in range(world)]
    if name == "job_chunks" and world == 3:
        assert spans == [(0, 1), (1, 2), (2, 2)]
    if name == "v17_t1000" and world == 3:
        assert spans[0] == (0, 11)
    for rank, (b, e) in enumerate(spans):
        shard(rank, world)
        rs, res, feas, best, plan = _run(pkg, s)
        mask = kp.shard_columns(s["prob"], b, e)
        _assert_rows(s, feas, best, F & mask[None, None, :], kp.shard_best(F, s["prob"], b, e), f" rank {rank} of {world}")
        lowest = best if lowest is None else np.minimum(lowest, best)
    assert np.array_equal(lowest, B[shape])
    shard(world - 1, world)  # the Solve without F (use_F = 0): every fresh node through the column words
    compare(pkg, oracle, pkg.Problem.from_dict(s["prob"]))
