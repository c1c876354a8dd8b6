"""GPU: problems whose label keys or resource lists are wider than the device word (tests/wide_problems.py) are solved on the
device and equal the oracle, none of them refused: whole results, the consolidation session probe for probe, and the
random_problem_with_bounds seeds whose `integer` key has more than 63 values."""
import pytest

import wide_problems as wp
from fuzz_problems import random_problem_with_bounds
from oracle_compare import compare

pytestmark = pytest.mark.gpu

CORPUS = wp.corpus()


@pytest.mark.parametrize("name,prob", CORPUS, ids=[c[0] for c in CORPUS])
def test_wide_problem_equals_oracle(pkg, oracle, name, prob):
    compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)


def test_wide_cluster_equals_oracle_probe_for_probe(pkg, oracle):
    problem = pkg.Problem.from_dict(wp.cluster(0))
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
    one = pkg.SingleNodeConsolidation(problem).compute_command()
    want1 = oracle.consolidate_single(problem)
    assert (one["action"], one["node"], one["options"]) == (want1["action"], want1["node"], want1["options"])


def _wide_bound_seeds():
    """random_problem_with_bounds seeds with more than 63 `integer` values (70 fake types): refused before value classes"""
    out = []
    for seed in range(150):
        prob = random_problem_with_bounds(seed)
        vals = {v for it in prob["instanceTypes"] for r in it["requirements"] if r["key"] == "integer" and r["operator"] == "In" for v in r["values"]}
        if len(vals) > 63:
            out.append(seed)
    return out


WIDE_SEEDS = _wide_bound_seeds()


def test_wide_bound_seeds_exist():
    assert len(WIDE_SEEDS) >= 10


@pytest.mark.parametrize("seed", WIDE_SEEDS)
def test_wide_fuzz_seed_equals_oracle(pkg, oracle, seed):
    compare(pkg, oracle, pkg.Problem.from_dict(random_problem_with_bounds(seed)), add_calls=False, refusal_skips=False)
