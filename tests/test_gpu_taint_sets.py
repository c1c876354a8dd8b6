"""GPU: clusters whose owned existing nodes carry more than 64 distinct taint sets (tests/taint_problems.py) are solved on
the device and equal the oracle, none of them refused: whole results at every pack-kernel block size and with each class-run
step switched off, the consolidation session probe for probe, and validation against the cluster after the TTL."""
import pytest

import taint_problems as tp
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = tp.corpus()
IDS = [c[0] for c in CORPUS]


def _beyond_template_sets(prob, got):
    """pods the device put on existing nodes whose taint set no template has"""
    tmpl = tp.template_sets(prob)
    return sum(len(e["pods"]) for e in got.to_dict()["existing"]
               if tp.taint_set(tp.node_taints(prob["nodes"][e["node"]])) not in tmpl)


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_taint_sets_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
    assert _beyond_template_sets(prob, got) > 0


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS[::2], ids=IDS[::2])
def test_taint_sets_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_taint_set_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(tp.cluster(0)))


def test_taint_set_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, tp.cluster(0), tp.after(0))
