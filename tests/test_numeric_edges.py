"""CPU: the numeric-edge corpus (tests/numeric_problems.py) against exact arithmetic (tests/exact_arith.py). Every quantity
string parses to its exact milli value or is refused; every problem is refused by the loader or the encoder exactly when a
sum crosses 2^62, and otherwise the oracle's result fits on every resource, keeps every provisioner within its limits and
equals the stated answer; the oracle's candidate ranking equals the float64 restatement bit for bit, NaN rule (R8)
included; and the limit cluster's probes give a replacement only where the exact remaining allows one."""
import math
import struct

import pytest

import exact_arith as ea
import numeric_problems as nprob

INT64_MIN = -2 ** 63
CORPUS = nprob.corpus()
IDS = [c[0] for c in CORPUS]
RANKING = nprob.ranking_corpus()


def same_costs(a, b):
    """float64 lists equal bit for bit, any NaN equal to any NaN (R8 orders NaNs; their payload is not part of the order)"""
    return len(a) == len(b) and all((math.isnan(x) and math.isnan(y)) or struct.pack("<d", x) == struct.pack("<d", y) for x, y in zip(a, b))


def load(pkg, prob):
    """the Problem and its ResidentSolve encoding, or None where the loader or the encoder refuses it"""
    try:
        problem = pkg.Problem.from_dict(prob)
    except ValueError:
        return None, None
    try:
        return problem, pkg.ResidentSolve(problem)
    except pkg.KschedError:
        return problem, None


@pytest.mark.parametrize("text,want", nprob.QUANTITIES, ids=[q[0][:24] for q in nprob.QUANTITIES])
def test_quantity_is_exact_or_refused(pkg, text, want):
    exact = ea.quantity_milli(text)
    short = len(text.lstrip("+-").replace(".", "").lstrip("0")) <= 20
    if want is not None:
        assert exact == want  # the table itself
    got = pkg.model_lib().kh_parse_quantity(text.encode())
    if want is None:
        assert got == INT64_MIN, f"{text} parsed to {got}, exact value {exact}"
    else:
        assert got in (want, INT64_MIN), f"{text} parsed to {got}, exact value {want}"
        if short:
            assert got == want  # short forms are never refused


def test_refusal_names_the_resource(pkg):
    bad = nprob.limit_wrap(1, "5Pi")
    with pytest.raises(ValueError, match="resource memory: quantity out of range"):
        pkg.Problem.from_dict(bad)
    with pytest.raises(ValueError, match="resource memory: quantity has too many digits"):
        pkg.Problem.from_dict(nprob.limit_wrap(1, "340282366920938463463374607431768211456m"))
    with pytest.raises(ValueError, match="negative request"):
        pkg.Problem.from_dict(nprob._one_type_problem([{"name": "p", "uid": "p", "requests": {"cpu": "-1"}}]))
    with pytest.raises(ValueError, match="negative capacity"):
        pkg.Problem.from_dict(nprob.limit_wrap(1, "-4Ti"))


@pytest.mark.parametrize("name,prob,answer", CORPUS, ids=IDS)
def test_refused_or_exact(pkg, oracle, name, prob, answer):
    problem, enc = load(pkg, prob)
    if answer is None:  # a sum crosses 2^62: refused by the product and by the oracle
        assert enc is None, name
        if problem is not None:
            res = pkg.Result()
            assert oracle.solve(problem, res) != 0 and "out of range" in res.error
        return
    assert enc is not None, name
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    assert ea.check_exact(prob, res.to_dict(), answer) == []


def test_limit_wrap_pair(pkg, oracle):
    """2 090 and 2 100 owned 4Ti nodes under a 1Ti memory limit: neither opens a node (the capacity sum of 2 100 passes
    INT64_MAX in milli-bytes)"""
    for n in (2090, 2100):
        prob = nprob.limit_wrap(n)
        assert ea.remaining_after_existing(prob, prob["provisioners"][0])["memory"] == 2 ** 40 * 1000 - n * 4 * 2 ** 40 * 1000
        res = pkg.Result()
        assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0
        assert res.to_dict()["newNodes"] == [] and list(res.assign) == [-1], n


@pytest.mark.parametrize("kept", [0, 2])
def test_limit_cluster_probes(pkg, oracle, kept):
    """computeConsolidation over the k cheapest candidates of the 4Pi cluster gives a replacement only where the exact
    remaining, with their capacity given back, holds the replacement's options"""
    prob = nprob.limit_cluster(kept)
    problem = pkg.Problem.from_dict(prob)
    its = prob["instanceTypes"]
    for k in (1, 2, 3):
        rem = ea.remaining_after_existing(prob, prob["provisioners"][0], removed=set(range(k)))["memory"]
        action, options = oracle.consolidate_probe(problem, k)
        if action == 2:
            assert all(ea._resources(its[t]["capacity"])["memory"] <= rem for t in options), (kept, k, rem)
        if kept == 2:
            assert action != 2 and rem < 0, k


@pytest.mark.parametrize("name,prob", RANKING, ids=[r[0] for r in RANKING])
def test_oracle_ranking_equals_restatement(pkg, oracle, name, prob):
    order, cost = oracle.rank_candidates(pkg.Problem.from_dict(prob))
    want_order, want_cost = ea.ranked(prob, list(range(len(prob["nodes"]))))
    assert order == want_order
    assert same_costs(cost, want_cost)


def test_nan_sorts_last():
    prob = nprob.ranking_corpus()[0][1]  # costs 1, NaN, 0
    order, cost = ea.ranked(prob, [0, 1, 2])
    assert order == [2, 0, 1] and cost[:2] == [0.0, 1.0] and math.isnan(cost[2])


@pytest.mark.parametrize("name,prob,answer", nprob.queue_corpus(), ids=[q[0] for q in nprob.queue_corpus()])
def test_queue_answers_on_the_oracle(pkg, oracle, name, prob, answer):
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    assert answer(res.to_dict())
