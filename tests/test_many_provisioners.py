"""CPU: clusters with up to 64 provisioners whose requirements and labels name keys no pod names (tests/provisioner_problems.py).
The encoder accepts every problem of the corpus with one template per provisioner, keeps exactly the pod-side keys (plus
zone and capacity-type) as mask keys, folds the others, still refuses what the device cannot hold, and the oracle's results
are sound placements."""
import pytest

import placement_invariants
import provisioner_problems as pp

CORPUS = pp.corpus()


@pytest.mark.parametrize("name,prob", CORPUS, ids=[c[0] for c in CORPUS])
def test_encoder_folds_template_only_keys(pkg, name, prob):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["templates"] == len(prob["provisioners"])
    mask = pp.pod_side_keys(prob)
    assert rs.dims["keys"] == len(mask), sorted(mask)
    folded = pp.template_keys(prob) - mask
    assert folded, "the corpus problem folds no key"
    for key in folded:
        assert rs.key_info(key) is None, key
    for key in mask:
        assert rs.key_info(key) is not None, key


def test_the_fold_is_needed(pkg):
    """every corpus problem has more than 16 active keys or more than 63 provisioner names: none fits the word unfolded"""
    for name, prob in CORPUS:
        active = pp.pod_side_keys(prob) | pp.template_keys(prob)
        assert len(active) > 16 or len(prob["provisioners"]) > 63, name


def test_names_only_problem_has_few_keys(pkg):
    prob = pp.names_only(0)
    assert len(pp.pod_side_keys(prob) | pp.template_keys(prob)) <= 16
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.key_info(pp.PROVISIONER_NAME) is None and rs.dims["templates"] == 64


def test_cluster_is_accepted(pkg):
    prob = pp.cluster(0)
    cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands[:3])
    assert rs.dims["templates"] == 40 and rs.key_info("family") is None
    pkg.ResidentSolve(pkg.Problem.from_dict(pp.after(0)))


@pytest.mark.parametrize("name,prob,message", pp.NEAR_MISSES, ids=[c[0] for c in pp.NEAR_MISSES])
def test_near_misses_are_still_refused(pkg, name, prob, message):
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED
    assert message in str(e.value)


@pytest.mark.parametrize("name,prob", [c for c in CORPUS if not c[1].get("nodes")], ids=[c[0] for c in CORPUS if not c[1].get("nodes")])
def test_oracle_results_pass_placement_invariants(pkg, oracle, name, prob):
    prob = dict(prob, daemonSetPods=[])  # the invariants sum the pods' own requests: no daemonset overhead
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    stats = placement_invariants.check(problem, res)
    assert stats["scheduled"] > 0
