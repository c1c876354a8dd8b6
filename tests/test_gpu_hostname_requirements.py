"""GPU: pods whose kubernetes.io/hostname requirements go beyond one In / NotIn value (tests/hostname_problems.py) are solved
on the device and equal the oracle, none of them refused: whole results at every pack-kernel block size and with each
class-run step switched off, a problem with the hostname table solved again after one without it on the same device state,
the consolidation session probe for probe, and validation against the cluster after the TTL."""
import pytest

import hostname_problems as hn
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = [(n, p) for n, p, _ in hn.corpus()]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_hostname_requirements_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_hostname_requirements_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_table_then_no_table_then_table_again(pkg, oracle, monkeypatch):
    set_modes(monkeypatch)
    for prob in (hn.local_pv(0), hn.old_forms(0), hn.local_pv(0)):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_hostname_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(hn.cluster(0)))


def test_hostname_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, hn.cluster(0), hn.after(0))
