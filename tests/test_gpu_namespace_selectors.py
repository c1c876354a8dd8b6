"""GPU: pod affinity and anti-affinity terms with a namespaceSelector (tests/namespace_problems.py) on the device. The
namespaces are resolved into groups and class x group relations on the host, so the device sees relation shapes it did not
see before: classes selected by groups that other namespaces' pods own, and bound pods' inverse groups that span
namespaces. Whole results equal the oracle at every pack-kernel block size and with each class-run step switched off; the
consolidation session equals the oracle probe for probe; validation against the cluster after the TTL, where one namespace
was relabelled, equals the validation oracle."""
import pytest

import namespace_problems as nsp
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, compare_validation, set_modes

pytestmark = pytest.mark.gpu

CORPUS = nsp.corpus()
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,doc", CORPUS, ids=IDS)
def test_corpus_equals_oracle(pkg, oracle, monkeypatch, name, doc, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(doc), refusal_skips=False)
    nsp.check(doc, got.to_dict())


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,doc", CORPUS, ids=IDS)
def test_corpus_with_a_step_switched_off(pkg, oracle, monkeypatch, name, doc, switch):
    set_modes(monkeypatch, switch)
    compare(pkg, oracle, pkg.Problem.from_dict(doc), refusal_skips=False)


@pytest.mark.parametrize("which", ["cluster", "after"])
def test_cluster_equals_oracle_probe_for_probe(pkg, oracle, which):
    compare_cluster(pkg, oracle, pkg.Problem.from_dict(getattr(nsp, which)()))


def test_validation_against_the_relabelled_cluster_equals_oracle(pkg, oracle):
    compare_validation(pkg, nsp.cluster(), nsp.after())
