"""GPU: simulateScheduling's whole result from the device-resident cluster (ClusterSession.simulate, ksched_simulate_full)
is, set for set, what a freshly encoded Solve with that set as the candidates returns (Scheduler.solve(candidates=set)) and
what the oracle returns: the whole result in the fresh problem's numbering and both verdicts. nodes_visited is the one
field left out: a simulation also counts the removed nodes the pack kernel skips. Checked at three pack-kernel block
sizes, under every mode switch, with one and with 64 sets per call, on a refused snapshot, at C5's full size, and for the
snapshot's state: probes and validations before and after a simulation agree. A refused snapshot's probes and single-node
search equal the oracle too."""
import copy
import ctypes as C

import pytest

import consolidation_answers as ca
import fixtures as fx
import full_simulation_problems as fp
import validation_answers as va
from oracle_compare import INSTANCE_TYPE, MODE_SWITCHES, compare_probes, set_modes

pytestmark = pytest.mark.gpu

CORPUS = fp.corpus()
IDS = [c[0] for c in CORPUS]


def _verdicts(prob, d):
    """(all pods scheduled, an existing node of the result not initialised) of a result dict, from the problem dict"""
    init = [n["labels"].get("karpenter.sh/initialized") == "true" for n in prob["nodes"]]
    return all(a >= 0 for a in d["assign"]), any(not init[e["node"]] for e in d["existing"])


def _whole(res, brief=False):
    d = res.to_dict(brief)
    d.pop("nodesVisited")
    return d, (res.all_pods_scheduled, res.uninitialized_existing)


def _sets(pkg, oracle, prob, sets):
    problem = pkg.Problem.from_dict(prob)
    return problem, fp.resolve_sets(prob, sets, oracle.rank_candidates(problem)[0])


def _against_solve_and_oracle(pkg, oracle, prob, problem, s, got):
    want = pkg.Scheduler(problem).solve(candidates=s, count_visited=False)
    assert _whole(got) == _whole(want), s
    o = pkg.Result()
    assert oracle.solve(problem, o, s) == 0, o.error
    g, w = got.to_dict(), o.to_dict()
    for k in ("assign", "relax", "existing", "addCalls"):
        assert g[k] == w[k], (s, k)
    assert len(g["newNodes"]) == len(w["newNodes"]), s
    for a, b in zip(g["newNodes"], w["newNodes"]):
        b = dict(b, requirements={k: v for k, v in b["requirements"].items() if k != INSTANCE_TYPE})
        assert a == b, s
    assert (got.all_pods_scheduled, got.uninitialized_existing) == _verdicts(prob, w), s


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob,sets,prop", CORPUS, ids=IDS)
def test_simulate_equals_fresh_solve_and_oracle(pkg, oracle, monkeypatch, threads, name, prob, sets, prop):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    problem, resolved = _sets(pkg, oracle, prob, sets)
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    for s in resolved:
        _against_solve_and_oracle(pkg, oracle, prob, problem, s, cs.simulate([s])[0])
    # 64 sets in one call: the scenario's sets over and over, each result its own set's
    many = [resolved[q % len(resolved)] for q in range(64)]
    singles = [_whole(r) for r in (cs.simulate([s])[0] for s in resolved)]
    for q, r in enumerate(cs.simulate(many)):
        assert _whole(r) == singles[q % len(resolved)], (name, q)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob,sets,prop", CORPUS, ids=IDS)
def test_simulate_under_mode_switches(pkg, oracle, monkeypatch, switch, name, prob, sets, prop):
    set_modes(monkeypatch, switch)
    problem, resolved = _sets(pkg, oracle, prob, sets)
    cs = pkg.ClusterSession(problem)
    for s, got in zip(resolved, cs.simulate(resolved)):
        _against_solve_and_oracle(pkg, oracle, prob, problem, s, got)


def test_simulation_leaves_the_snapshot_as_it_found_it(pkg, oracle):
    prob = fp.topology()
    problem = pkg.Problem.from_dict(prob)
    cs = pkg.ClusterSession(problem)
    n = cs.n_candidates
    probes = [list(range(c)) for c in range(1, n + 1)] + [[i] for i in range(n)]
    before = [cs.probe_sets(probes[:n], True), cs.probe_sets(probes[n:], False)]
    commands = [([i], a, o) for i, (a, o) in enumerate(before[1]) if a in (1, 2)]
    valid = cs.validate(problem, commands)
    order = cs.candidate_nodes()
    cs.simulate([order[::-1], order[:1], order[1:]])
    assert [cs.probe_sets(probes[:n], True), cs.probe_sets(probes[n:], False)] == before
    assert cs.validate(problem, commands) == valid


def _crowded_cluster(pod_cpu="1"):
    """a cluster the snapshot refuses: node "crowd" (the last in the node list) hosts a pod with more topology groups than
    the pack kernel carries"""
    a = va._cluster(pod_cpu=pod_cpu)
    big = ca.on_demand_by_price(a["instanceTypes"])[-1]
    crowd = fx.pod({"cpu": "100m"}, nodeName="crowd", labels={f"k{j}": "v" for j in range(10)},
                   topologySpreadConstraints=[fx.spread(fx.HOSTNAME, {f"k{j}": "v"}) for j in range(10)])
    a["nodes"].append(ca.node_of_type("crowd", big, [crowd], 1.0))
    return a


def test_refused_snapshot_simulates_through_fresh_solves(pkg, oracle):
    a = _crowded_cluster()
    problem = pkg.Problem.from_dict(a)
    cs = pkg.ClusterSession(problem)
    assert not cs.resident
    crowd = len(a["nodes"]) - 1  # its pod stays bound: a set that removed it would put the pod in the batch
    order = [i for i in cs.candidate_nodes() if i != crowd]
    sets = [order[:1], order[::-1], order[1:2]]
    for s, got in zip(sets, cs.simulate(sets)):
        want = pkg.Scheduler(problem).solve(candidates=s)
        assert _whole(got) == _whole(want), s


@pytest.mark.parametrize("pod_cpu", ["1", "24"])
def test_refused_snapshot_consolidates_through_fresh_solves(pkg, oracle, pod_cpu):
    """computeConsolidation on a session whose snapshot is refused, each set a freshly encoded solve: every probe that
    leaves the crowd node's pod bound, and the single-node search, equal the oracle. With 1-CPU pods every probe deletes;
    with 24-CPU pods the two cheapest nodes are replaced by one and removing three does nothing."""
    a = _crowded_cluster(pod_cpu)
    problem = pkg.Problem.from_dict(a)
    cs = pkg.ClusterSession(problem)
    assert not cs.resident
    order = cs.candidate_nodes()
    assert order[-1] == len(a["nodes"]) - 1
    n = len(order) - 1
    compare_probes(pkg, oracle, problem, cs, [list(range(c)) for c in range(1, n + 1)], [[i] for i in range(n)])
    got = pkg.SingleNodeConsolidation(problem).compute_command(batch=1)
    want = oracle.consolidate_single(problem)
    keys = ("action", "node", "options")
    assert {k: got[k] for k in keys} == {k: want[k] for k in keys}


def test_refusals(pkg, oracle):
    prob = fp.uninitialized()  # node "cold" is not initialised: it stays in every simulation, no set may remove it
    problem = pkg.Problem.from_dict(prob)
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    cold = [n["name"] for n in prob["nodes"]].index("cold")
    with pytest.raises(pkg.KschedError) as e:
        cs.simulate([[cold]])
    assert e.value.code == pkg.KSCHED_ERR_INVALID
    gone = copy.deepcopy(prob)
    c0 = [n["name"] for n in gone["nodes"]].index("c0")
    cs2 = pkg.ClusterSession(pkg.Problem.from_dict(gone))
    gone["nodes"][c0]["markedForDeletion"] = True
    cs3 = pkg.ClusterSession(pkg.Problem.from_dict(gone))
    with pytest.raises(pkg.KschedError) as e:
        cs3.simulate([[c0]])
    assert e.value.code == pkg.KSCHED_ERR_INVALID and "marked for deletion" in str(e.value)
    assert cs2.simulate([[c0]])[0].all_pods_scheduled
    # the flat C-ABI on the snapshot the scheduler handle holds: a slot that is not removable, one out of range, and a
    # result smaller than the set's batch
    cs.simulate([[c0]])
    L = pkg.lib()
    L.kh_handle.restype = C.c_void_p
    L.ksched_simulate_full.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.ksched_last_error.restype = C.c_char_p
    L.ksched_last_error.argtypes = [C.c_void_p]

    class CandidateSet(C.Structure):
        _fields_ = [("nodes", C.POINTER(C.c_int32)), ("n_nodes", C.c_int32), ("capacity", C.c_int32), ("remaining", C.c_void_p)]

    h = L.kh_handle()
    result = C.create_string_buffer(1024)  # a zeroed ksched_result: every refusal comes before a result is touched
    slot_c0 = 2  # slots: full, cold, c0, c1 (node-list order)
    for slot, capacity, why in ((1, 64, "not removable"), (9, 64, "out of range"), (slot_c0, 1, "holds 1 pods")):
        nodes = (C.c_int32 * 1)(slot)
        cset = CandidateSet(nodes, 1, capacity, None)
        assert L.ksched_simulate_full(h, C.byref(cset), 1, result) == pkg.KSCHED_ERR_INVALID, why
        assert why in L.ksched_last_error(h).decode()


def test_c5_full_size_single_node_sets(pkg):
    problem = pkg.Problem.synth(5, 50000, 1000, 42, 5000)
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    sets = [[n] for n in cs.candidate_nodes()[:20]]
    for s, got in zip(sets, cs.simulate(sets)):
        want = pkg.Scheduler(problem).solve(candidates=s, count_visited=False)
        assert _whole(got, brief=True) == _whole(want, brief=True), s
        assert got.assign.tolist() == want.assign.tolist()
