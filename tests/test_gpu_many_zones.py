"""GPU: catalogs that offer instance types in more than 16 zones or 4 capacity types (tests/zone_problems.py) are solved on the
device with dense offering slots and equal the oracle, launch choice included: whole results at every pack-kernel block
size and with each class-run step switched off, a catalog with slot tables solved after one without them on the same
device state and back, the consolidation session probe for probe, and validation against the cluster after the TTL."""
import pytest

import zone_problems as zp
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = [(n, p) for n, p, _ in zp.corpus()]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_many_zones_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_many_zones_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_table_then_old_layout_then_table_again(pkg, oracle, monkeypatch):
    set_modes(monkeypatch)
    table, old = zp.spread_all(1), zp.zonal(16, cts=("capacity-block", "on-demand", "reserved", "spot"))
    for prob in (table, old, table):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_many_zones_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(zp.cluster(0)))


def test_many_zones_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, zp.cluster(0), zp.after(0))
