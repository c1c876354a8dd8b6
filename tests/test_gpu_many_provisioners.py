"""GPU: clusters with up to 64 provisioners and template-only keys folded into the templates' instance-type lists
(tests/provisioner_problems.py) are solved on the device and equal the oracle, none of them refused: whole results (the new
nodes' requirements on the folded keys included) at every pack-kernel block size and with each class-run step switched
off, the consolidation session probe for probe, and validation against the cluster after the TTL."""
import pytest

import provisioner_problems as pp
import validation_oracle as vo
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu

CORPUS = pp.corpus()


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=[c[0] for c in CORPUS])
def test_many_provisioners_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
    folded = pp.template_keys(prob) - pp.pod_side_keys(prob)
    assert any(k in n["requirements"] for n in got.to_dict()["newNodes"] for k in folded), "no folded requirement was rendered"


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS[::3], ids=[c[0] for c in CORPUS[::3]])
def test_many_provisioners_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_many_provisioner_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    problem = pkg.Problem.from_dict(pp.cluster(0))
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


def test_many_provisioner_validation_equals_oracle(pkg, oracle):
    b, a = pp.cluster(0), pp.after(0)
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
