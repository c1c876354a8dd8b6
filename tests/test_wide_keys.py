"""CPU: label keys and resource lists wider than the device word (tests/wide_problems.py). The encoder accepts every problem
of the corpus, keeps at most m + 2 representatives on a collapsed key (m = its Gt/Lt thresholds), still refuses what the
word cannot hold, and the value classes agree with the exact string algebra (kh_value_class_selftest)."""
import pytest

import placement_invariants
import wide_problems as wp

CORPUS = wp.corpus()


def _wide_keys(prob):
    """label keys on which the catalog and the nodes carry more than 63 distinct values"""
    vals = {}
    for it in prob["instanceTypes"]:
        for r in it["requirements"]:
            if r["operator"] in ("In", "NotIn"):
                vals.setdefault(r["key"], set()).update(r["values"])
    for n in prob.get("nodes", []):
        for k, v in n["labels"].items():
            vals.setdefault(k, set()).add(v)
    return {k for k, v in vals.items() if len(v) > 63}


def _distinct_resources(prob):
    return {k for it in prob["instanceTypes"] for k in it["capacity"]}


@pytest.mark.parametrize("name,prob", CORPUS, ids=[c[0] for c in CORPUS])
def test_encoder_accepts_wide_problem(pkg, name, prob):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["pods"] == len(prob["pods"])
    collapsed = 0
    for key in _wide_keys(prob):
        info = rs.key_info(key)
        if info is None:
            continue  # no requirement of the problem names the key: it is not a mask key at all
        assert info["values"] <= 63
        assert 0 < info["representatives"] <= info["thresholds"] + 2, (key, info)
        collapsed += 1
    if name.startswith("extended"):
        assert len(_distinct_resources(prob)) > 8 and rs.dims["resources"] <= 8
    else:
        assert collapsed > 0, "the corpus problem exercises no collapsed key"


@pytest.mark.parametrize("name,prob", wp.NEAR_MISSES, ids=[c[0] for c in wp.NEAR_MISSES])
def test_near_misses_are_still_refused(pkg, name, prob):
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED
    assert "more than 63 distinct values" in str(e.value)


def test_keys_that_fit_are_not_collapsed(pkg):
    prob = wp.fake(40, 0)  # 40 type values + the pods' own + at most 8 regions: fits the word as it is
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    info = rs.key_info("integer")
    assert info["representatives"] == 0 and info["values"] >= 40


def test_cluster_is_accepted(pkg):
    prob = wp.cluster(0)
    assert _wide_keys(prob)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=[0, 1, 2])
    assert rs.key_info("memory")["representatives"] >= 1


@pytest.mark.parametrize("name,prob", [c for c in CORPUS if not c[1].get("nodes")], ids=[c[0] for c in CORPUS if not c[1].get("nodes")])
def test_oracle_results_pass_placement_invariants(pkg, oracle, name, prob):
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    stats = placement_invariants.check(problem, res)
    assert stats["scheduled"] > 0


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_value_class_selftest(pkg, seed):
    assert pkg.lib().kh_value_class_selftest(seed, 20000) == 0
