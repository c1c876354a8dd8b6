"""GPU: batches whose pods request 9 to 32 distinct resources (tests/extended_resource_problems.py) are solved on the device
and equal the oracle, none of them refused: whole results (the ext requests of new nodes included) at every pack-kernel
block size and with each class-run step switched off, the GPU consolidation cluster probe for probe, and validation against
the cluster after the TTL."""
import pytest

import extended_resource_problems as xp
import k1_problems as kp
import validation_oracle as vo
from oracle_compare import MODE_SWITCHES, compare, set_modes

pytestmark = pytest.mark.gpu

CORPUS = xp.corpus()
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_extended_resources_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
    assert _ext_on_new_nodes(got) > 0


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS[::2], ids=IDS[::2])
def test_extended_resources_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


FRESH = xp.fresh_corpus()


def _ext_on_new_nodes(got):
    return sum(1 for n in got.to_dict()["newNodes"] if any(k in xp.EXT_RESOURCES for k in n["requests"]))


@pytest.mark.parametrize("switch", (None,) + MODE_SWITCHES)
@pytest.mark.parametrize("threads", [32, 128, 512])
def test_fresh_fleets_back_to_back_equal_oracle(pkg, oracle, monkeypatch, threads, switch):
    """no existing nodes: the closed-form modes place the classes that request no ext resource and open nodes of their
    own between the generic steps of those that do. Different problems run one after the other on the same device state,
    so a node slot that keeps an earlier problem's ext sums would show."""
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}", switch)
    for name, prob in FRESH + CORPUS[:1] + FRESH[::-1]:
        got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
        assert _ext_on_new_nodes(got) > 0, name


def test_gpu_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    problem = pkg.Problem.from_dict(xp.cluster(0))
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


def test_gpu_cluster_validation_equals_oracle(pkg, oracle):
    b, a = xp.cluster(0), xp.after(0)
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


def test_neighbouring_classes_that_differ_in_an_ext_amount(pkg, oracle):
    """more classes than K1 has warps: one warp evaluates both classes of a pair back to back (extended_resource_problems.pairs)"""
    k1_warps = kp.max_warps(kp.device_sm_count())
    prob = xp.pairs()
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["classes"] == len(prob["pods"]) > k1_warps and rs.resource_id("aws.amazon.com/neuron") >= 8
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
