"""GPU: the numeric-edge corpus (tests/numeric_problems.py) on the CUDA path. Problems the product takes equal the oracle,
whole result, and pass the exact-arithmetic check (tests/exact_arith.py), at every pack-kernel block size and with each
class-run step switched off; the queue cases, whose packed key only fits with the timestamps ranked, give the oracle's
order; the 4Pi limit clusters equal the oracle probe for probe and on both consolidations; and rank_candidates returns a
permutation of the eligible nodes equal to the float64 restatement, NaN rule (R8) included."""
import pytest

import exact_arith as ea
import numeric_problems as nprob
from oracle_compare import MODE_SWITCHES, compare, compare_cluster, set_modes
from test_numeric_edges import same_costs

pytestmark = pytest.mark.gpu

CORPUS = [c for c in nprob.corpus() if c[2] is not None]
IDS = [c[0] for c in CORPUS]
RANKING = nprob.ranking_corpus()


def _check(pkg, oracle, prob, answer):
    got, _ = compare(pkg, oracle, pkg.Problem.from_dict(prob), refusal_skips=False)
    assert ea.check_exact(prob, got.to_dict(), answer) == []


@pytest.mark.parametrize("threads", [32, 128, 512])
@pytest.mark.parametrize("name,prob,answer", CORPUS, ids=IDS)
def test_numeric_edges_equal_oracle(pkg, oracle, monkeypatch, name, prob, answer, threads):
    set_modes(monkeypatch, f"KSCHED_PACK_THREADS={threads}")
    _check(pkg, oracle, prob, answer)


@pytest.mark.parametrize("switch", MODE_SWITCHES)
@pytest.mark.parametrize("name,prob,answer", CORPUS, ids=IDS)
def test_numeric_edges_with_a_step_switched_off(pkg, oracle, monkeypatch, name, prob, answer, switch):
    set_modes(monkeypatch, switch)
    _check(pkg, oracle, prob, answer)


@pytest.mark.parametrize("name,prob,answer", [c for c in nprob.corpus() if c[2] is None], ids=[c[0] for c in nprob.corpus() if c[2] is None])
def test_sums_past_the_bound_are_refused(pkg, name, prob, answer):
    try:
        problem = pkg.Problem.from_dict(prob)
    except ValueError as e:
        assert "out of range" in str(e)
        return
    with pytest.raises(pkg.KschedError, match="out of range"):
        pkg.Scheduler(problem).solve()


@pytest.mark.parametrize("kept", [0, 2])
def test_limit_cluster_equals_oracle_probe_for_probe(pkg, oracle, kept):
    assert compare_cluster(pkg, oracle, pkg.Problem.from_dict(nprob.limit_cluster(kept)), 3).n_candidates == 3


@pytest.mark.parametrize("name,prob", RANKING, ids=[r[0] for r in RANKING])
def test_rank_candidates_equal_restatement(pkg, oracle, name, prob):
    problem = pkg.Problem.from_dict(prob)
    order, cost = pkg.rank_candidates(problem)
    assert sorted(order) == list(range(len(prob["nodes"])))  # a permutation of the eligible nodes: every slot written
    want_order, want_cost = ea.ranked(prob, list(range(len(prob["nodes"]))))
    assert order == want_order and same_costs(cost, want_cost)
    o_order, o_cost = oracle.rank_candidates(problem)
    assert order == o_order and same_costs(cost, o_cost)
