"""GPU: clusters and batches whose pods mount more than 64 volume claims that the sharing rule would track
(tests/volume_problems.py) are solved on the device and equal the oracle, none of them refused: whole results at every
pack-kernel block size and with each class-run step switched off, a problem with the claim table solved again after one
without it on the same device state, the consolidation session probe for probe, and validation against the cluster after
the TTL."""
import pytest

import volume_problems as vp
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

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
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(prob))


@pytest.mark.parametrize("name,prob", CLUSTERS, ids=[c[0] for c in CLUSTERS])
def test_volume_validation_equals_oracle(pkg, oracle, name, prob):
    compare_validation(pkg, prob, vp.after(prob, 0))
