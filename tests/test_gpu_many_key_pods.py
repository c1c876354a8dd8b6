"""GPU: pod classes whose requirements and topology terms touch more than 8 label keys (tests/many_key_problems.py) are
placed on the device and the results equal the oracle, none of them refused: whole results at every pack-kernel block size
and with each class-run step switched off, a many-key problem solved again after an 8-key one on the same handle, the
consolidation session probe for probe, and validation against the cluster after the TTL. A class constrained by 9 topology
groups is still refused at upload."""
import pytest

import many_key_problems as mk
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = [(n, p) for n, p in mk.corpus() if p["pods"]]
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_many_key_pods_equal_oracle(pkg, oracle, monkeypatch, name, prob, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_many_key_pods_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def _eight_keys():
    """deployments(0) cut down to classes of at most 8 keys by the former count"""
    prob = mk.deployments(0)
    prob["pods"] = [p for p in prob["pods"] if p["labels"]["app"] in ("nine", "plain")]
    for p in prob["pods"]:
        p.pop("nodeAffinity", None)
    return prob


def test_many_keys_then_eight_then_many_again(pkg, oracle, monkeypatch):
    set_modes(monkeypatch)
    for prob in (mk.sixteen(0), _eight_keys(), mk.sixteen(0)):
        compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_nine_groups_are_refused_at_upload(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(mk.nine_groups(0)))
    with pytest.raises(pkg.KschedError) as e:
        rs.load()
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED


def test_many_key_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(mk.cluster(0)))


def test_many_key_validation_equals_oracle(pkg, oracle):
    compare_validation(pkg, mk.cluster(0), mk.after(0))
