"""GPU: clusters whose pods name more than 64 distinct host-port entries (tests/hostport_problems.py) are solved on the device
and equal the oracle, none of them refused: whole results at every pack-kernel block size and with each class-run step
switched off, the consolidation session probe for probe, validation against the cluster after the TTL, and a problem with
the entry table solved again after one without it on the same device state."""
import pytest

import hostport_problems as hp
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = [(n, p) for n, p, _ in hp.corpus()]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_host_ports_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
    assert hp.node_conflicts(prob, got.to_dict()) == []


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_host_ports_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_table_then_no_table_then_table_again(pkg, oracle, monkeypatch):
    """the existing nodes' extra words are restored and the new nodes' written on every Solve: a table problem after a
    table-free one on the same device state gives the same result as the first time"""
    set_modes(monkeypatch)
    for prob in (hp.traps(0), hp.daemonsets(60, 0, "few"), hp.traps(0)):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_host_port_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(hp.cluster(0)))


def test_host_port_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, hp.cluster(0), hp.after(0))
