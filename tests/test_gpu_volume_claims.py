"""GPU: clusters and batches whose pods mount more than 64 volume claims that the sharing rule would track
(tests/volume_problems.py) are solved on the device and equal the oracle, none of them refused: whole results at every
pack-kernel block size and with each class-run step switched off, a problem with the claim table solved again after one
without it on the same device state, the consolidation session probe for probe, and validation against the cluster after
the TTL."""
import pytest

import validation_oracle as vo
import volume_problems as vp
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu

CORPUS = [(n, p) for n, p, _ in vp.corpus()]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_volume_claims_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
    assert vp.volume_violations(prob, got.to_dict()) == []


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_volume_claims_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_table_then_no_table_then_table_again(pkg, oracle, monkeypatch):
    """the existing nodes' extra words are restored on every Solve: a table problem after a table-free one on the same device
    state gives the same result as the first time"""
    set_modes(monkeypatch)
    for prob in (vp.traps(0), vp.bound_only(0), vp.traps(0)):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


CLUSTERS = [("sts-60x3", vp.statefulsets(60, 3, 0)), ("shared-60x3", vp.shared(60, 3, 120, 0))]


@pytest.mark.parametrize("name,prob", CLUSTERS, ids=[c[0] for c in CLUSTERS])
def test_volume_cluster_equals_oracle_probe_for_probe(pkg, oracle, name, prob):
    problem = pkg.Problem.from_dict(prob)
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


@pytest.mark.parametrize("name,prob", CLUSTERS, ids=[c[0] for c in CLUSTERS])
def test_volume_validation_equals_oracle(pkg, oracle, name, prob):
    a = vp.after(prob, 0)
    before, after = (prob, pkg.Problem.from_dict(prob)), (a, pkg.Problem.from_dict(a))
    keys = ("action", "position", "node", "options", "validations", "failed_validation")
    want = vo.single_compute_command(before, after)
    for batch in (1, 64):
        got = pkg.SingleNodeConsolidation(before[1]).compute_command(batch=batch, after=after[1])
        assert {k: got[k] for k in keys} == {k: want[k] for k in keys}, batch
    mkeys = ("action", "nodes_removed", "options", "probes", "probe_actions", "validations")
    got_m = pkg.MultiNodeConsolidation(before[1]).compute_command(after[1])
    want_m = vo.multi_compute_command(before, after)
    assert {k: got_m[k] for k in mkeys} == {k: want_m[k] for k in mkeys}
