"""GPU: pod affinity and anti-affinity terms with a namespaceSelector (tests/namespace_problems.py) on the device. The
namespaces are resolved into groups and class x group relations on the host, so the device sees relation shapes it did not
see before: classes selected by groups that other namespaces' pods own, and bound pods' inverse groups that span
namespaces. Whole results equal the oracle at every pack-kernel block size and with each class-run step switched off; the
consolidation session equals the oracle probe for probe; validation against the cluster after the TTL, where one namespace
was relabelled, equals the validation oracle."""
import pytest

import namespace_problems as nsp
import validation_oracle as vo
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu

CORPUS = nsp.corpus()
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,doc", CORPUS, ids=IDS)
def test_corpus_equals_oracle(pkg, oracle, monkeypatch, name, doc, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(doc), refusal_skips=False)
    nsp.check(doc, got.to_dict())


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,doc", CORPUS, ids=IDS)
def test_corpus_with_a_step_switched_off(pkg, oracle, monkeypatch, name, doc, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(doc), refusal_skips=False)


@pytest.mark.parametrize("which", ["cluster", "after"])
def test_cluster_equals_oracle_probe_for_probe(pkg, oracle, which):
    problem = pkg.Problem.from_dict(getattr(nsp, which)())
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
    assert (got["action"], got["nodes_removed"], got["options"], got["probes"], got["probe_actions"]) == \
           (want["action"], want["nodes_removed"], want["options"], want["probes"], want["probe_actions"])


def test_validation_against_the_relabelled_cluster_equals_oracle(pkg, oracle):
    b, a = nsp.cluster(), nsp.after()
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
