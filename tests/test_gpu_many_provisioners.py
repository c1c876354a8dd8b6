"""GPU: clusters with up to 64 provisioners and template-only keys folded into the templates' instance-type lists
(tests/provisioner_problems.py) are solved on the device and equal the oracle, none of them refused: whole results (the new
nodes' requirements on the folded keys included) at every pack-kernel block size and with each class-run step switched
off, the consolidation session probe for probe, and validation against the cluster after the TTL."""
import pytest

import provisioner_problems as pp
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

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
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(pp.cluster(0)))


def test_many_provisioner_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, pp.cluster(0), pp.after(0))
