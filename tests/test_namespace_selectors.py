"""CPU: namespaceSelector on pod affinity and anti-affinity terms (tests/namespace_problems.py). The oracle reproduces the
reference's answer and an independent restatement of the semantics on every corpus problem; the encoder accepts the corpus,
merges groups by their resolved namespace sets and keeps pods that differ only in their selector in separate classes; the
loader refuses selectors it cannot resolve."""
import pytest

import namespace_problems as nsp
import validation_oracle as vo

CORPUS = nsp.corpus()
IDS = [c[0] for c in CORPUS]


def run_oracle(pkg, oracle, doc):
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(doc), res) == 0, res.error
    return res.to_dict()


def test_empty_selector_reaches_another_namespace(pkg, oracle):
    """topology_test.go:2131-2168: the pod with affinity lands on its target's node, in another namespace"""
    a = run_oracle(pkg, oracle, nsp.restated_empty_selector())["assign"]
    assert a[10] >= 0 and a[11] == a[10]


# what each scenario must come to, beyond the restated semantics of nsp.check
def _expect(name, doc, res):
    a = res["assign"]
    if name.startswith("match_labels_target_unlabelled"):
        assert a[0] >= 0 and all(x < 0 for x in a[1:])           # the followers' selector misses the target's namespace
    elif name.startswith("match_labels_target_labelled"):
        assert min(a) >= 0 and len(set(a)) == 1
    elif name.startswith("selects_nothing_self_affinity"):
        assert all(x < 0 for x in a)                             # an empty set selects not even the pod itself
    elif name.startswith("selects_nothing_anti"):
        assert min(a) >= 0 and len(set(a)) == 1                  # nobody is repelled: one node takes them all
    elif name.startswith("three_namespaces_zone"):
        assert 1 <= sum(x >= 0 for x in a) <= 3                  # at most one db pod per zone, whichever namespace it is in
    elif name.startswith("three_namespaces_hostname"):
        assert min(a) >= 0 and len(set(a)) == len(a)
    elif name.startswith("preferred_relaxed"):
        assert min(a) >= 0 and max(res["relax"]) > 0
    elif name.startswith("bound_inverse"):
        n_existing = len(res["existing"])
        agent_nodes = {e for e, ex in enumerate(res["existing"]) if doc["nodes"][ex["node"]]["pods"]}
        web = [x for p, x in zip(doc["pods"], a) if p.get("labels") == {"app": "web"}]
        assert min(web) >= 0 and not agent_nodes & set(web) and n_existing == 4
        others = [x for p, x in zip(doc["pods"], a) if p.get("labels") == {"app": "other"}]
        assert min(others) >= 0


@pytest.mark.parametrize("name,doc", CORPUS, ids=IDS)
def test_oracle_holds_the_restated_semantics(pkg, oracle, name, doc):
    res = run_oracle(pkg, oracle, doc)
    nsp.check(doc, res)
    _expect(name, doc, res)


@pytest.mark.parametrize("name,doc", CORPUS, ids=IDS)
def test_encoder_accepts_the_corpus(pkg, name, doc):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(doc))
    assert rs.dims["pods"] == len(doc["pods"]) and rs.dims["groups"] > 0


@pytest.mark.parametrize("name,doc", [c for c in CORPUS if nsp.explicit(c[1]) is not None],
                         ids=[c[0] for c in CORPUS if nsp.explicit(c[1]) is not None])
def test_groups_merge_by_their_resolved_namespaces(pkg, oracle, name, doc):
    """the same problem with each selector written out as the namespace list it resolves to: the same groups, the same result"""
    plain = nsp.explicit(doc)
    assert pkg.ResidentSolve(pkg.Problem.from_dict(doc)).dims["groups"] == pkg.ResidentSolve(pkg.Problem.from_dict(plain)).dims["groups"]
    assert run_oracle(pkg, oracle, doc) == run_oracle(pkg, oracle, plain)


def test_selectors_that_resolve_alike_share_a_group(pkg):
    """`{}` and a selector every namespace matches resolve to one set: the two deployments' anti-affinity terms share a group"""
    import fixtures as fx
    web = {"app": "web"}
    spaces = [nsp.ns("default", zone="any"), nsp.ns("a", zone="any")]
    one = [fx.pod({"cpu": "1"}, labels=web, podAntiAffinity={"required": [nsp.term(fx.HOSTNAME, web, nsp.EVERY)]})]
    two = [fx.pod({"cpu": "1"}, labels=web, podAntiAffinity={"required": [nsp.term(fx.HOSTNAME, web, {"matchLabels": {"zone": "any"}})]})]
    dims = lambda pods_: pkg.ResidentSolve(pkg.Problem.from_dict(fx.problem(pods_, namespaces=spaces))).dims
    assert dims(one + two)["groups"] == dims(one)["groups"]
    assert dims(one + two)["classes"] == 2


def test_pods_that_differ_only_in_their_selector_get_different_classes(pkg):
    import fixtures as fx
    web = {"app": "web"}
    spaces = [nsp.ns("default"), nsp.ns("a", team="x"), nsp.ns("b", team="y")]
    pod = lambda sel: fx.pod({"cpu": "1"}, labels=web, podAntiAffinity={"required": [nsp.term(fx.HOSTNAME, web, sel)]})
    dims = lambda pods_: pkg.ResidentSolve(pkg.Problem.from_dict(fx.problem(pods_, namespaces=spaces))).dims
    same = dims([pod({"matchLabels": {"team": "x"}}) for _ in range(4)])
    differ = dims([pod({"matchLabels": {"team": "x"}}) for _ in range(2)] + [pod({"matchLabels": {"team": "y"}}) for _ in range(2)])
    nil = dims([pod({"matchLabels": {"team": "x"}}) for _ in range(2)] + [pod(None) for _ in range(2)])
    assert same["classes"] == 1 and differ["classes"] == 2 and nil["classes"] == 2
    assert differ["groups"] == nil["groups"] == 2 * same["groups"]   # a group (and its inverse) per resolved set


@pytest.mark.parametrize("name,doc", nsp.near_misses(), ids=[c[0] for c in nsp.near_misses()])
def test_near_misses_are_refused_loudly(pkg, name, doc):
    with pytest.raises(ValueError, match="namespace"):
        pkg.Problem.from_dict(doc)


def test_relabelled_namespace_changes_validation(pkg):
    """the consolidation pair: relabelling one namespace after the TTL changes which commands validate"""
    b, a = nsp.cluster(), nsp.after()
    before, after = (b, pkg.Problem.from_dict(b)), (a, pkg.Problem.from_dict(a))
    unchanged = (b, pkg.Problem.from_dict(b))
    assert vo.single_compute_command(before, after) != vo.single_compute_command(before, unchanged)
