"""GPU: daemonsets whose requirements name node.kubernetes.io/instance-type (tests/daemonset_itype_problems.py) reach the
device as template and existing-node overhead, and the results equal the oracle, none of them refused: whole results at
every pack-kernel block size and with each class-run step switched off, a daemonset problem solved again after one without
daemonsets on the same device state, the restated known answers, the consolidation session probe for probe, and validation
against the cluster after the TTL at batch 1 and 64."""
import pytest

import daemonset_itype_problems as dp
import fixtures as fx
import validation_oracle as vo
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu

CORPUS = dp.corpus() + [(n, p) for n, p, _ in dp.known_answers()]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_daemonset_itype_equals_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_daemonset_itype_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_daemonsets_then_none_then_daemonsets_again(pkg, oracle, monkeypatch):
    set_modes(monkeypatch)
    plain = fx.problem(fx.pods(12, requests={"cpu": "1", "memory": "1Gi"}), instance_types=dp.TYPES)
    for prob in (dp.efa(0), plain, dp.efa(0)):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_miscount_scenario_places_the_pod_on_n0(pkg):
    got = pkg.Scheduler(pkg.Problem.from_dict(dp.miscount(0))).solve()
    assert list(got.assign) == [0]


def test_daemonset_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    problem = pkg.Problem.from_dict(dp.cluster(0))
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    order = cs.candidate_nodes()
    assert len(order) >= 2
    prefixes = [list(range(c)) for c in range(1, len(order) + 1)]
    for s_, g in zip(prefixes, cs.probe_sets(prefixes, True)):
        assert g == oracle.consolidate_probe(problem, len(s_)), ("prefix", len(s_))
    singles = [[i] for i in range(len(order))]
    for s_, g in zip(singles, cs.probe_sets(singles, False)):
        w = oracle.consolidate_single(problem, s_[0])
        assert g == (w["action"], w["options"]), ("single", s_)
    got = pkg.MultiNodeConsolidation(problem).first_n_node_consolidation_option()
    want = oracle.consolidate(problem)
    assert (got["action"], got["nodes_removed"], got["options"], got["probes"]) == \
           (want["action"], want["nodes_removed"], want["options"], want["probes"])
    one = pkg.SingleNodeConsolidation(problem).compute_command()
    want1 = oracle.consolidate_single(problem)
    assert (one["action"], one["node"], one["options"]) == (want1["action"], want1["node"], want1["options"])


def test_daemonset_validation_equals_oracle(pkg, oracle):
    b, a = dp.cluster(0), dp.after(0)
    before, after = (b, pkg.Problem.from_dict(b)), (a, pkg.Problem.from_dict(a))
    keys = ("action", "position", "node", "options", "validations", "failed_validation")
    want = vo.single_compute_command(before, after)
    for batch in (1, 64):
        got = pkg.SingleNodeConsolidation(before[1]).compute_command(batch=batch, after=after[1])
        assert {k: got[k] for k in keys} == {k: want[k] for k in keys}, batch
    mkeys = ("action", "nodes_removed", "options", "probes", "probe_actions", "validations")
    got_m = pkg.MultiNodeConsolidation(before[1]).compute_command(after[1])
    want_m = vo.multi_compute_command(before, after)
    assert {k: got_m[k] for k in mkeys} == {k: want_m[k] for k in mkeys}
