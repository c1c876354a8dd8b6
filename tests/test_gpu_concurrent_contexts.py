"""Two scheduler contexts on one device, driven from two threads at once (the provisioning and the deprovisioning
controller): every answer equals the oracle's and the same call made alone, the two handles' pack kernels overlap in device
time, handles that share a parameter slot keep their order, and the process-wide handle is unaffected."""
import copy
import threading
import time

import pytest

import consolidation_answers as ca
import fixtures as fx
import validation_oracle as vo
from known_answers import CASES
from oracle_compare import compare

pytestmark = pytest.mark.gpu

INSTANCE_TYPE = "node.kubernetes.io/instance-type"


def _solve_key(r):
    d = r.to_dict()
    return d["assign"], d["relax"], d["existing"], d["newNodes"]


def _oracle_key(r):
    """what the oracle and the device must agree on: every field but the new nodes' instance-type requirement, which the
    oracle renders and the device leaves to the options"""
    d = r.to_dict()
    nodes = [(n["provisioner"], n["pods"], n["options"], n["requests"], {k: v for k, v in n["requirements"].items() if k != INSTANCE_TYPE},
              n.get("launch")) for n in d["newNodes"]]
    return d["assign"], d["relax"], d["existing"], nodes


def topology_cluster(n_nodes=600):
    """~600 nodes in three zones: a zone-spread web pod on every node and a hostname anti-affinity pod on every fourth, so
    the session holds topology groups and every simulation re-places spread-constrained pods"""
    od = {it["offerings"][0]["zone"]: it for it in ca.on_demand_by_price(ca.assorted()) if it["name"].startswith("32c-32g-")}
    zones = sorted(od)
    assert len(zones) == 3
    web = {"app": "web"}
    nodes = []
    for i in range(n_nodes):
        name = f"n{i:03d}"
        pods_ = [fx.pod({"cpu": "2", "memory": "1Gi"}, nodeName=name, labels=web, topologySpreadConstraints=[fx.spread(fx.ZONE, web)])]
        if i % 4 == 0:
            pods_.append(fx.pod({"cpu": "1", "memory": "1Gi"}, nodeName=name, labels={"app": "solo"},
                                podAntiAffinity={"required": [fx.affinity_term(fx.HOSTNAME, {"app": "solo"})]}))
        nodes.append(ca.node_of_type(name, od[zones[i % len(zones)]], pods_, float(i % 97) + i / 1000.0))
    return fx.problem([], instance_types=ca.assorted(), provisioners=[fx.provisioner(consolidationEnabled=True)], nodes=nodes,
                      deriveCandidates=True)


def after_the_ttl(before):
    """the cluster when the TTL ends: one node gone and a 28-cpu pod bound to every seventh of the first 140 nodes, so
    commands that remove those nodes no longer validate"""
    after = copy.deepcopy(before)
    for i in range(0, 140, 7):
        n = after["nodes"][i]
        n["pods"].append(fx.pod({"cpu": "28", "memory": "1Gi"}, nodeName=n["name"]))
    del after["nodes"][5]
    return after


def _search(pkg, cs):
    """firstNNodeConsolidationOption on the session's probes: (action, nodes removed, options, probe trace, probe actions)"""
    seen = {}

    def probe_many(counts):
        for c in counts:
            seen[c] = tuple(cs.probe_sets([list(range(c))], True)[0])
        return {c: seen[c] for c in counts}
    action, count, options, _, path = pkg.speculative_binary_search(cs.n_candidates, probe_many, 1)
    return action, count, list(options), path, [seen[c][0] for c in path]


def deprovisioning(pkg, ctx, before, after):
    """thread B: the multi-node search, the single-node sweep at batch 64, 20 full simulations and the validation of the
    commands found against the cluster after the TTL, all on one session of `ctx`"""
    cs = pkg.ClusterSession(before[1], context=ctx)
    n = cs.n_candidates
    search = _search(pkg, cs)
    sweep = []
    for b in range(0, n, 64):
        sweep += [(a, list(o)) for a, o in cs.probe_sets([[i] for i in range(b, min(n, b + 64))], False)]
    nodes = cs.candidate_nodes()
    sets = [[nodes[i]] for i in range(10)] + [[nodes[i + 1], nodes[i]] for i in range(0, 20, 2)]
    sims = [_oracle_key(r) + (r.all_pods_scheduled, r.uninitialized_existing) for r in cs.simulate(sets)]
    cmds = [([i], a, o) for i, (a, o) in enumerate(sweep) if a in (1, 2)][:48]
    if search[0] in (1, 2):
        cmds.append((list(range(search[1])), search[0], search[2]))
    valid = cs.validate(after[1], cmds)
    cs.close()
    return {"nodes": nodes, "search": search, "sweep": sweep, "sets": sets, "sims": sims, "cmds": cmds, "valid": valid}


def provisioning(pkg, ctx, problems):
    """thread A: Solves of the known answers and of the synthetic batches"""
    return [_oracle_key(pkg.Scheduler(p, context=ctx).solve(count_visited=False)) for p in problems]


def _run_together(*jobs):
    out, errs = [None] * len(jobs), []
    barrier = threading.Barrier(len(jobs))

    def run(i, fn):
        try:
            barrier.wait()
            out[i] = fn()
        except BaseException as e:  # surfaced below
            errs.append(e)
    ts = [threading.Thread(target=run, args=(i, fn)) for i, fn in enumerate(jobs)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]
    return out


@pytest.fixture(scope="module")
def prov(pkg):
    known = []
    for _, _, build in CASES:
        prob, _ = build()
        known += [pkg.Problem.from_dict(d) for d in prob.get("multi", [prob])]
    synth = [pkg.Problem.synth(1, 100, 10, 42, 0), pkg.Problem.synth(4, 500, 1000, 42, 0), pkg.Problem.synth(2, 10_000, 500, 42, 0)]
    return known, synth


@pytest.fixture(scope="module")
def cluster(pkg):
    b = topology_cluster()
    a = after_the_ttl(b)
    return (b, pkg.Problem.from_dict(b)), (a, pkg.Problem.from_dict(a))


def _check_deprovisioning_against_the_oracle(pkg, oracle, got, before, after):
    problem = before[1]
    want = oracle.consolidate(problem)
    assert got["search"] == (want["action"], want["nodes_removed"], want["options"], want["probes"], want["probe_actions"])
    for i, g in enumerate(got["sweep"]):
        w = oracle.consolidate_single(problem, i)
        assert g == (w["action"], w["options"]), ("single", i)
    assert any(a in (1, 2) for a, _ in got["sweep"])
    for s, g in zip(got["sets"], got["sims"]):
        want = pkg.Result()
        assert oracle.solve(problem, want, s) == 0, want.error
        assert g[:4] == _oracle_key(want), s
        w = want.to_dict()  # simulateScheduling's verdicts, derived from the oracle's placements
        init = [n["labels"].get("karpenter.sh/initialized") == "true" for n in before[0]["nodes"]]
        assert (g[4], g[5]) == (all(a >= 0 for a in w["assign"]), any(not init[e["node"]] for e in w["existing"])), s
    nodes = got["nodes"]
    verdicts = [vo.is_valid(before, after, [nodes[p] for p in pos], a, o) for pos, a, o in got["cmds"]]
    assert got["valid"] == verdicts
    assert True in verdicts and False in verdicts  # the state after the TTL really changed some verdicts


def test_two_contexts_concurrently_equal_the_oracle(pkg, oracle, prov, cluster):
    known, synth = prov
    before, after = cluster
    a, b = pkg.Context(0), pkg.Context(0)
    alone_a = provisioning(pkg, a, known + synth)
    alone_b = deprovisioning(pkg, b, before, after)
    _check_deprovisioning_against_the_oracle(pkg, oracle, alone_b, before, after)
    for p, got in zip(known + synth[:2], alone_a):
        want = pkg.Result()
        assert oracle.solve(p, want) == 0, want.error
        assert got == _oracle_key(want)
    # the C2 batch against the process-wide handle (the oracle needs tens of seconds for it)
    assert alone_a[-1] == _oracle_key(pkg.Scheduler(synth[2]).solve(count_visited=False))
    for _ in range(2):
        got_a, got_b = _run_together(lambda: provisioning(pkg, a, known + synth), lambda: deprovisioning(pkg, b, before, after))
        assert got_a == alone_a
        assert got_b == alone_b
    b.destroy()
    a.destroy()


def test_contexts_sharing_a_slot_keep_their_answers(pkg, prov):
    _, synth = prov
    ctxs = [pkg.Context(0) for _ in range(3)]  # two parameter slots: at least two of them share one
    jobs = [synth[:2], synth[1:], synth[::2]]
    alone = [provisioning(pkg, c, j) for c, j in zip(ctxs, jobs)]
    got = _run_together(*[(lambda c=c, j=j: provisioning(pkg, c, j)) for c, j in zip(ctxs, jobs)])
    assert got == alone
    for c in ctxs:
        c.destroy()


def test_two_contexts_repeat_their_own_solves(pkg, oracle):
    """Two contexts driven by two host threads, each solving its own problem six times: every repetition equals that
    context's first result bit for bit (assignment, new nodes and their options), and the process-wide handle still agrees
    with the oracle afterwards."""
    problems = [pkg.Problem.synth(4, 1500, 1000, 5, 0), pkg.Problem.synth(3, 2000, 1000, 6, 0)]
    ctxs = [pkg.Context(0), pkg.Context(0)]

    def repeat(ctx, problem):
        return [_solve_key(pkg.Scheduler(problem, context=ctx).solve(count_visited=False)) for _ in range(6)]
    got = _run_together(*[(lambda c=c, p=p: repeat(c, p)) for c, p in zip(ctxs, problems)])
    for runs in got:
        assert all(r == runs[0] for r in runs[1:])
    compare(pkg, oracle, problems[0])
    for c in ctxs:
        c.destroy()


def test_pack_kernels_of_two_contexts_overlap(pkg):
    """A C4 Solve on one context while a single-node sweep runs on another: the Solve's pack launch intersects one of the
    sweep's. The sweep probes one candidate per call, so every one of its pack launches is recorded."""
    long_solve = pkg.Problem.synth(4, 100_000, 1000, 42, 0)
    cluster = pkg.Problem.synth(5, 20_000, 1000, 42, 2000)
    a, b = pkg.Context(0), pkg.Context(0)
    pkg.Scheduler(long_solve, context=a).solve(count_visited=False)  # warm both handles
    cs = pkg.ClusterSession(cluster, context=b)
    cs.probe_sets([[0]], False)
    done = threading.Event()
    sweep_intervals = []

    def provision():
        ivs, walls = [], []
        for _ in range(3):
            t0 = time.perf_counter()
            pkg.Scheduler(long_solve, context=a).solve(count_visited=False)
            walls.append(time.perf_counter() - t0)
            ivs.append(a.timings()["pack_interval_ns"])
        done.set()
        return ivs, walls

    def sweep():
        t0, i = time.perf_counter(), 0
        while not done.is_set():
            cs.probe_sets([[i % cs.n_candidates]], False)
            sweep_intervals.append(b.timings()["pack_interval_ns"])
            i += 1
        return time.perf_counter() - t0
    (solve_intervals, walls), sweep_s = _run_together(provision, sweep)
    assert min(walls) >= 0.05 and sweep_s >= 0.05, (walls, sweep_s)  # both workloads run for at least 50 ms
    assert all(e > s > 0 for s, e in solve_intervals + sweep_intervals)
    assert any(s1 < e2 and s2 < e1 for s1, e1 in solve_intervals for s2, e2 in sweep_intervals), (solve_intervals, sweep_intervals[:8])
    cs.close()
    b.destroy()
    a.destroy()


def test_contexts_interleaved_with_the_process_handle(pkg, prov, cluster):
    _, synth = prov
    before, _ = cluster
    ctx = pkg.Context(0)
    sets = [[0], [1], [0, 1]]
    legacy_solve = _solve_key(pkg.Scheduler(synth[1]).solve(count_visited=False))
    legacy_cs = pkg.ClusterSession(before[1])
    legacy_probe = legacy_cs.probe_sets(sets, False)
    ctx_cs = pkg.ClusterSession(before[1], context=ctx)
    ctx_probe = ctx_cs.probe_sets(sets, False)
    assert _solve_key(pkg.Scheduler(synth[1], context=ctx).solve(count_visited=False)) == legacy_solve
    assert legacy_cs.probe_sets(sets, False) == legacy_probe == ctx_probe
    assert _solve_key(pkg.Scheduler(synth[1]).solve(count_visited=False)) == legacy_solve
    assert ctx_cs.probe_sets(sets, False) == ctx_probe
    got = _run_together(lambda: _solve_key(pkg.Scheduler(synth[1]).solve(count_visited=False)),
                        lambda: ctx_cs.probe_sets(sets, False),
                        lambda: legacy_cs.probe_sets(sets, False))
    assert got == [legacy_solve, ctx_probe, legacy_probe]
    with pytest.raises(pkg.KschedError):
        ctx.destroy()  # a session is still open on it
    ctx_cs.close()
    legacy_cs.close()
    ctx.destroy()
