"""GPU: consolidation validation on the device (a second device-resident snapshot of the cluster after the TTL) must return
exactly what the oracle's restatement of validation.go returns - action, node, options and the validation trace - and
sessions that share the scheduler handle must stay correct when they are interleaved."""
import ctypes as C

import pytest

import validation_answers as va
import validation_oracle as vo
import validation_problems as vp
import fixtures as fx
import consolidation_answers as ca
from oracle_compare import VALIDATION_KEYS, compare_validation

pytestmark = pytest.mark.gpu


def _pp(pkg, d):
    return d, pkg.Problem.from_dict(d)


@pytest.mark.parametrize("name,ref,build", va.CASES, ids=[c[0] for c in va.CASES])
def test_known_answer_on_device(pkg, oracle, name, ref, build):
    (b, a), check = build()
    check(*compare_validation(pkg, b, a, name))


PAIRS = vp.pairs()


@pytest.mark.parametrize("i", range(len(PAIRS)), ids=[p[0] for p in PAIRS])
def test_corpus_pair_on_device(pkg, oracle, i):
    name, b, a = PAIRS[i]
    try:
        compare_validation(pkg, b, a, name)
    except pkg.KschedError as e:
        if e.code == pkg.KSCHED_ERR_UNSUPPORTED:
            pytest.skip(f"refused loudly: {e}")
        raise


def test_single_node_shares_merge_on_device(pkg, oracle):
    for name, b, a in PAIRS[::6]:
        before, after = _pp(pkg, b), _pp(pkg, a)
        n = len(oracle.rank_candidates(before[1])[0])
        sn = pkg.SingleNodeConsolidation(before[1])
        merged = pkg.merge_single_node_shares([sn.compute_command(0, n // 2, 64, after=after[1]), sn.compute_command(n // 2, -1, 64, after=after[1])])
        whole = sn.compute_command(batch=64, after=after[1])
        assert {k: merged[k] for k in VALIDATION_KEYS} == {k: whole[k] for k in VALIDATION_KEYS}, name


def test_cluster_validate_batches_of_64(pkg, oracle):
    """70 single-node deletes in one kh_cluster_validate call, against an unchanged cluster and one with nodes nominated"""
    b = va._cluster(70)
    a = va._cluster(70)
    for n in a["nodes"][::9]:
        n["nominated"] = True
    before, after = _pp(pkg, b), _pp(pkg, a)
    cs = pkg.ClusterSession(before[1])
    order = cs.candidate_nodes()
    res = cs.probe_sets([[i] for i in range(len(order))], False)
    cmds = [([i], act, o) for i, (act, o) in enumerate(res) if act in (1, 2)]
    assert len(cmds) >= 64
    assert all(cs.validate(before[1], cmds))
    got = cs.validate(after[1], cmds)
    want = [vo.is_valid(before, after, [order[i] for i in s_], act, o) for s_, act, o in cmds]
    assert got == want and not all(got)


def test_cluster_validate_equals_the_oracle(pkg, oracle):
    for name, b, a in PAIRS[::3]:
        before, after = _pp(pkg, b), _pp(pkg, a)
        try:
            cs = pkg.ClusterSession(before[1])
        except pkg.KschedError as e:
            if e.code == pkg.KSCHED_ERR_UNSUPPORTED:
                continue
            raise
        order = cs.candidate_nodes()
        sets = [[i] for i in range(len(order))] + [list(range(c)) for c in range(2, len(order) + 1)]
        res = cs.probe_sets(sets[:len(order)], False) + cs.probe_sets(sets[len(order):], True)
        cmds = [(s_, act, o) for s_, (act, o) in zip(sets, res) if act in (1, 2)]
        got = cs.validate(after[1], cmds)
        want = [vo.is_valid(before, after, [order[i] for i in s_], act, o) for s_, act, o in cmds]
        assert got == want, name


def test_refused_snapshot_validates_through_fresh_solves(pkg, oracle):
    """a node in `after` hosts a pod with more topology groups than the pack kernel carries: the snapshot refuses `after`
    (its pods are batch pods there), each validation is a freshly encoded solve that leaves that node's pods bound"""
    b = va._cluster()
    a = va._cluster()
    its = a["instanceTypes"]
    big = ca.on_demand_by_price(its)[-1]
    crowd = fx.pod({"cpu": "100m"}, nodeName="crowd", labels={f"k{j}": "v" for j in range(10)},
                   topologySpreadConstraints=[fx.spread(fx.HOSTNAME, {f"k{j}": "v"}) for j in range(10)])
    a["nodes"].append(ca.node_of_type("crowd", big, [crowd], 1.0))
    assert not pkg.ClusterSession(pkg.Problem.from_dict(a)).resident
    got, got_m = compare_validation(pkg, b, a, "refused")
    assert got["validations"] == [(0, True)]


def _probe_problem(n_small):
    """nodes of one expensive type; n_small of them carry a pod too big for their neighbours, so the probes differ"""
    d = va._cluster(4)
    for n in d["nodes"][:n_small]:
        n["pods"] = [fx.pod({"cpu": "31"}, nodeName=n["name"])]
    return d


def test_interleaved_sessions_equal_the_oracle(pkg, oracle):
    da, db = _probe_problem(0), _probe_problem(4)
    pa, pb = pkg.Problem.from_dict(da), pkg.Problem.from_dict(db)
    sa, sb = pkg.ClusterSession(pa), pkg.ClusterSession(pb)
    assert sa.resident and sb.resident
    other = pkg.Problem.synth(1, 100, 10, 42, 0)
    differ = False
    for round_ in range(3):
        for sess, prob in ((sa, pa), (sb, pb)):
            for c in range(1, sess.n_candidates + 1):
                got = sess.probe_sets([list(range(c))], True)[0]
                assert got == oracle.consolidate_probe(prob, c), (round_, c)
            pkg.Scheduler(other).solve()
        differ = differ or [sa.probe_sets([[i]], False)[0] for i in range(4)] != [sb.probe_sets([[i]], False)[0] for i in range(4)]
    assert differ, "the two problems must give different probe answers"


def test_upload_drops_the_handle_snapshot(pkg, oracle):
    problem = pkg.Problem.synth(5, 600, 1000, 42, 60)
    cs = pkg.ClusterSession(problem)
    L = pkg.lib()
    dummy = (C.c_byte * 64)()
    assert L.ksched_simulate_batch(C.c_void_p(L.kh_handle()), dummy, 0, dummy, None) == 0
    pkg.ResidentSolve(pkg.Problem.synth(1, 100, 10, 42, 0)).load()
    assert L.ksched_simulate_batch(C.c_void_p(L.kh_handle()), dummy, 0, dummy, None) == pkg.KSCHED_ERR_INVALID
    # the session loads its snapshot again before its next batch
    w = oracle.consolidate_single(problem, 0)
    assert cs.probe_sets([[0]], False)[0] == (w["action"], w["options"])


def test_resident_solve_runs_its_own_problem_after_a_session(pkg, oracle):
    """a consolidation session between ResidentSolve.load() and run() takes the handle; the run loads its problem again"""
    problem = pkg.Problem.synth(1, 100, 10, 42, 0)
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0
    rs = pkg.ResidentSolve(problem)
    rs.load()
    pkg.ClusterSession(pkg.Problem.synth(5, 600, 1000, 42, 60)).probe_sets([[0]], False)
    with pytest.raises(pkg.KschedError):
        rs.download()   # nothing of this problem's run is on the handle
    rs.run()
    assert (rs.download().assign == want.assign).all()


def test_validation_snapshot_follows_a_new_after_at_a_reused_address(pkg, oracle):
    """`after` problems created one after the other, the first freed before the second exists: the second is validated
    against its own cluster even when the allocator hands it the first one's address"""
    b = va._cluster(6)
    a1 = va._cluster(6)
    a2 = va._cluster(3)          # fewer nodes: a stale candidate list would index past them
    a2["pods"] = [fx.pod({"cpu": "1000"})]
    before = _pp(pkg, b)
    cs = pkg.ClusterSession(before[1])
    order = cs.candidate_nodes()
    res = cs.probe_sets([[i] for i in range(len(order))], False)
    cmds = [([i], act, o) for i, (act, o) in enumerate(res) if act in (1, 2)]
    p1 = pkg.Problem.from_dict(a1)
    addr1 = p1.ptr
    assert all(cs.validate(p1, cmds))
    cs._after = None
    del p1
    after2 = _pp(pkg, a2)
    got = cs.validate(after2[1], cmds)
    want = [vo.is_valid(before, after2, [order[i] for i in s_], act, o) for s_, act, o in cmds]
    assert got == want and not any(got), ("reused address" if after2[1].ptr == addr1 else "new address")
