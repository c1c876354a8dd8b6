"""GPU: the consolidation data plane - device-resident cluster snapshot + batched simulations (ksched_load_cluster /
ksched_simulate_batch), single-node consolidation, candidate ranking - must return exactly what the oracle returns."""
import random

import pytest

import consolidation_answers as ca
import fixtures as fx
import run_problems
from ranking_answers import CASES as RANK_CASES, SINGLE

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,ref,build", RANK_CASES, ids=[c[0] for c in RANK_CASES])
def test_ranking_known_answer_on_device(pkg, oracle, name, ref, build):
    prob, check = build()
    problem = pkg.Problem.from_dict(prob)
    order, cost = pkg.rank_candidates(problem)
    check(order, cost)
    assert (order, cost) == oracle.rank_candidates(problem)   # bit-exact doubles


def test_ranking_random_costs_match_the_oracle(pkg, oracle):
    rng = random.Random(5)
    its = ca.assorted()
    it = ca.on_demand_by_price(its)[-1]
    of = it["offerings"][0]
    nodes = []
    for i in range(700):
        pods_ = [fx.pod({"cpu": "100m"}, nodeName=f"n{i}", **({"deletionCost": rng.choice([-3.5e9, -1000, 7, 12345.678, 2.2e9])} if rng.random() < 0.5 else {}),
                        **({"priority": rng.choice([-2147483648, -5, 3, 1000000000])} if rng.random() < 0.5 else {}),
                        **({"doNotEvict": True} if rng.random() < 0.03 else {})) for _ in range(rng.choice([0, 1, 2, 5, 9]))]
        nodes.append(fx.state_node(f"n{i}", it["name"], zone=of["zone"], capacity_type=of["capacityType"], allocatable={"cpu": "32", "memory": "64Gi", "pods": "100"},
                                   pods_=pods_, creationTimestamp=float(rng.choice([0, 10, 500, 999, 2000]))))
    prob = fx.problem([], instance_types=its, provisioners=[fx.provisioner(consolidationEnabled=True, ttlSecondsUntilExpired=1000)], nodes=nodes,
                      deriveCandidates=True, now=1000.5)
    problem = pkg.Problem.from_dict(prob)
    assert pkg.rank_candidates(problem) == oracle.rank_candidates(problem)


@pytest.mark.parametrize("name,ref,build", SINGLE, ids=[c[0] for c in SINGLE])
def test_single_node_known_answer_on_device(pkg, oracle, name, ref, build):
    prob, check = build()
    problem = pkg.Problem.from_dict(prob)
    got = pkg.SingleNodeConsolidation(problem).compute_command(batch=1)
    check(got)
    want = oracle.consolidate_single(problem)
    assert (got["action"], got["node"], got["options"]) == (want["action"], want["node"], want["options"])
    wide = pkg.SingleNodeConsolidation(problem).compute_command(batch=64)   # speculative batches find the same first hit
    assert (wide["action"], wide["node"], wide["options"]) == (want["action"], want["node"], want["options"])


def _cluster(seed, n_nodes=96, pods_per_node=6):
    return pkg_synth_args(seed, n_nodes, pods_per_node)


def pkg_synth_args(seed, n_nodes, pods_per_node):
    return (5, n_nodes * pods_per_node, 1000, seed, n_nodes)


def test_batched_simulations_equal_the_oracle_probe_for_probe(pkg, oracle):
    """>= 64 candidate sets in ONE ksched_simulate_batch call: prefixes (multi-node) and single nodes"""
    problem = pkg.Problem.synth(*pkg_synth_args(42, 96, 6))
    cs = pkg.ClusterSession(problem)
    assert cs.resident, "the synthetic C5 cluster has no topology groups: the snapshot path must take it"
    n = cs.n_candidates
    prefixes = [list(range(c)) for c in range(1, n, max(1, n // 40))]
    singles = [[i] for i in range(0, n, 2)]
    assert len(prefixes) + len(singles) >= 64
    got_multi = cs.probe_sets(prefixes, True)
    got_single = cs.probe_sets(singles, False)
    for s_, g in zip(prefixes, got_multi):
        assert g == oracle.consolidate_probe(problem, len(s_)), len(s_)
    for s_, g in zip(singles, got_single):
        w = oracle.consolidate_single(problem, s_[0])
        assert g == (w["action"], w["options"]), s_


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_searches_on_the_snapshot_equal_the_oracle(pkg, oracle, seed):
    problem = pkg.Problem.synth(*pkg_synth_args(seed, 150, 8))
    got = pkg.MultiNodeConsolidation(problem).first_n_node_consolidation_option()
    want = oracle.consolidate(problem)
    assert (got["action"], got["nodes_removed"], got["options"], got["probes"], got["probe_actions"]) == \
           (want["action"], want["nodes_removed"], want["options"], want["probes"], want["probe_actions"])
    got1 = pkg.SingleNodeConsolidation(problem).compute_command()
    want1 = oracle.consolidate_single(problem)
    assert (got1["action"], got1["node"], got1["options"]) == (want1["action"], want1["node"], want1["options"])


def test_snapshot_with_provisioner_limits_and_uninitialised_nodes(pkg, oracle):
    """limits: the removed nodes' capacity is given back per simulation; an uninitialised node that stays blocks the command"""
    its = ca.assorted()
    big = ca.on_demand_by_price(its)[-1]
    nodes = [ca.node_of_type(f"n{i}", big, [fx.pod({"cpu": "20"}, nodeName=f"n{i}")], float(i + 1)) for i in range(4)]
    for n in nodes:
        n["capacity"] = {"cpu": "32", "memory": "64Gi", "pods": "100"}
    prob = fx.problem([], instance_types=its, provisioners=[fx.provisioner(limits={"cpu": "150"})], nodes=nodes)
    problem = pkg.Problem.from_dict(prob)
    cs = pkg.ClusterSession(problem)
    sets = [[0], [0, 1], [0, 1, 2], [3], [1, 2]]
    assert cs.probe_sets([s_ for s_ in sets if s_ == list(range(len(s_)))], True) == [oracle.consolidate_probe(problem, c) for c in (1, 2, 3)]
    nodes[2]["labels"].pop(fx.INITIALIZED)
    nodes[2]["candidate"] = False
    problem2 = pkg.Problem.from_dict(prob)
    cs2 = pkg.ClusterSession(problem2)
    assert cs2.probe_sets([[0], [0, 1]], True) == [oracle.consolidate_probe(problem2, 1), oracle.consolidate_probe(problem2, 2)]


# ---------------------------------------------------------------- clusters WITH topology groups on the snapshot path
from consolidation_answers import CASES as _CONS, CPU_ONLY_CASES as _CONS_LATE
from fuzz_problems import random_problem


@pytest.mark.parametrize("name,ref,build", _CONS + _CONS_LATE, ids=[c[0] for c in _CONS + _CONS_LATE])
def test_consolidation_known_answers_run_on_the_snapshot(pkg, oracle, name, ref, build):
    """every consolidation known answer (the topology-aware ones included, suite_test.go:1827-2030) is taken by the
    device-resident cluster - no probe falls back to a re-encoded ksched_solve - and equals the oracle probe for probe"""
    prob, _ = build()
    problem = pkg.Problem.from_dict(prob)
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    sets = [list(range(c)) for c in range(1, cs.n_candidates + 1)]
    if sets:
        assert cs.probe_sets(sets, True) == [oracle.consolidate_probe(problem, len(s_)) for s_ in sets]


def _candidate_cluster(seed):
    """a fuzz problem (pending pods, bound pods with selectors / anti-affinity, spread constraints, several provisioners) whose
    owned nodes are consolidation candidates"""
    prob = random_problem(seed)
    rng = random.Random(seed * 31 + 7)
    offered = {(it["name"], o["capacityType"], o["zone"]) for it in prob["instanceTypes"] for o in it["offerings"]}
    n = 0
    for node in prob.get("nodes", []):
        lab = node["labels"]
        if lab.get(fx.PROVISIONER_NAME) and not node.get("markedForDeletion") and \
                (lab.get(fx.INSTANCE_TYPE), lab.get(fx.CAPACITY_TYPE), lab.get(fx.ZONE)) in offered:  # getNodePrices needs the node's offering
            node["candidate"] = True
            node["disruptionCost"] = float(rng.choice([0, 1, 1, 2, 3]))
            n += 1
    return prob, n


@pytest.mark.parametrize("seed,zones,ct_spread", [(1, 9, False), (2, 16, False), (3, 9, True)])
def test_snapshot_equals_oracle_on_wide_zone_clusters(pkg, oracle, seed, zones, ct_spread):
    """run-shaped clusters: zone spread over 9 or 16 zones, and zone plus capacity-type spread (two mask relations)"""
    problem = pkg.Problem.from_dict(run_problems.cluster(seed, zones, ct_spread))
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    n = cs.n_candidates
    assert n == 3 * zones
    prefixes = [list(range(c)) for c in range(1, n + 1)]
    for s_, g in zip(prefixes, cs.probe_sets(prefixes, True)):
        assert g == oracle.consolidate_probe(problem, len(s_)), ("prefix", len(s_))
    singles = [[i] for i in range(n)]
    for s_, g in zip(singles, cs.probe_sets(singles, False)):
        w = oracle.consolidate_single(problem, s_[0])
        assert g == (w["action"], w["options"]), ("single", s_)


@pytest.mark.parametrize("seed", [s for s in range(400) if _candidate_cluster(s)[1] >= 2][:60])
def test_snapshot_equals_oracle_on_random_clusters_with_topology(pkg, oracle, seed):
    prob, n = _candidate_cluster(seed)
    problem = pkg.Problem.from_dict(prob)
    try:
        cs = pkg.ClusterSession(problem)
    except pkg.KschedError as e:
        if e.code == pkg.KSCHED_ERR_UNSUPPORTED:
            pytest.skip(f"refused loudly: {e}")
        raise
    assert cs.resident
    order = cs.candidate_nodes()
    prefixes = [list(range(c)) for c in range(1, len(order) + 1)]
    singles = [[i] for i in range(len(order))]
    for s_, g in zip(prefixes, cs.probe_sets(prefixes, True)):
        assert g == oracle.consolidate_probe(problem, len(s_)), ("prefix", len(s_))
    for s_, g in zip(singles, cs.probe_sets(singles, False)):
        w = oracle.consolidate_single(problem, s_[0])
        assert g == (w["action"], w["options"]), ("single", s_)
