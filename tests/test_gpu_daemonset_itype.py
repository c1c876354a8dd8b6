"""GPU: daemonsets whose requirements name node.kubernetes.io/instance-type (tests/daemonset_itype_problems.py) reach the
device as template and existing-node overhead, and the results equal the oracle, none of them refused: whole results at
every pack-kernel block size and with each class-run step switched off, a daemonset problem solved again after one without
daemonsets on the same device state, the restated known answers, the consolidation session probe for probe, and validation
against the cluster after the TTL at batch 1 and 64."""
import pytest

import daemonset_itype_problems as dp
import fixtures as fx
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = dp.corpus() + [(n, p) for n, p, _ in dp.known_answers()]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_daemonset_itype_equals_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_daemonset_itype_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_daemonsets_then_none_then_daemonsets_again(pkg, oracle, monkeypatch):
    set_modes(monkeypatch)
    plain = fx.problem(fx.pods(12, requests={"cpu": "1", "memory": "1Gi"}), instance_types=dp.TYPES)
    for prob in (dp.efa(0), plain, dp.efa(0)):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_miscount_scenario_places_the_pod_on_n0(pkg):
    got = pkg.Scheduler(pkg.Problem.from_dict(dp.miscount(0))).solve()
    assert list(got.assign) == [0]


def test_daemonset_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(dp.cluster(0)))


def test_daemonset_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, dp.cluster(0), dp.after(0))
