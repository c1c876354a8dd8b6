"""CPU: topology spread node filters that name node.kubernetes.io/instance-type (tests/itype_filter_problems.py) encode without
refusal and get the instance-type filter tables; problems without such a term get none and encode as before. Terms that differ
only in their instance-type part make different groups, countDomains counts what TopologyNodeFilter.Matches restated on
strings admits, and the oracle's results keep its invariants. The near misses are refused."""
import pytest

import fixtures as fx
import itype_filter_problems as itf
from fixtures import INSTANCE_TYPE, ZONE

CORPUS = itf.corpus()
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_encoder_takes_the_scenario(pkg, name, prob, table):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert (rs.dims["itype_filter_terms"] > 0) == table


@pytest.mark.parametrize("name,prob", itf.near_misses(), ids=[n for n, _ in itf.near_misses()])
def test_near_misses_are_refused(pkg, name, prob):
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED


def test_old_forms_get_no_table_and_keep_their_entries(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(itf.old_forms(0)))
    assert rs.dims["itype_filter_terms"] == 0 and rs.dims["itype_reqs"] == 2


def _two_spreads(types_a, types_b):
    lab = {"app": "g"}
    pods = fx.pods(3, requests={"cpu": "1"}, labels=lab, nodeAffinity={"required": [[itf._it("In", types_a)]]},
                   topologySpreadConstraints=[fx.spread(ZONE, lab)])
    pods += fx.pods(3, requests={"cpu": "1"}, labels=lab, nodeAffinity={"required": [[itf._it("In", types_b)]]},
                    topologySpreadConstraints=[fx.spread(ZONE, lab)])
    return itf._problem(pods)


def test_terms_that_differ_only_in_the_instance_type_are_different_groups(pkg):
    same = pkg.ResidentSolve(pkg.Problem.from_dict(_two_spreads(["fake-it-3"], ["fake-it-3"])))
    diff = pkg.ResidentSolve(pkg.Problem.from_dict(_two_spreads(["fake-it-3"], ["fake-it-4"])))
    assert same.dims["groups"] == 1 and diff.dims["groups"] == 2


@pytest.mark.parametrize("name,prob,table", [c for c in CORPUS if c[2]], ids=[c[0] for c in CORPUS if c[2]])
def test_counted_domains_equal_the_string_restatement(pkg, name, prob, table):
    """for a single-spread owner class whose group is the only one of its selector, countDomains counts the bound pods the
    selector picks on nodes whose labels a term of the owner's filter matches (TopologyNodeFilter.Matches restated)"""
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    if name not in ("listed-unlisted", "unlabelled", "two-terms"):
        return
    owner = next(p for p in prob["pods"] if p.get("topologySpreadConstraints") and p["topologySpreadConstraints"][0]["topologyKey"] == ZONE)
    sel = owner["topologySpreadConstraints"][0]["labelSelector"]["matchLabels"]
    na = owner.get("nodeAffinity") or {}
    sel_reqs = [{"key": k, "operator": "In", "values": [v]} for k, v in (owner.get("nodeSelector") or {}).items()]
    terms = [sel_reqs + t for t in (na.get("required") or [[]])]
    want = 0
    for n in prob["nodes"]:
        if ZONE not in n["labels"] or not n["labels"].get(fx.PROVISIONER_NAME):
            continue
        zone_ok = lambda t: all(r["key"] != ZONE or n["labels"][ZONE] in r["values"] for r in t)
        if any(itf.term_matches(t, n["labels"]) and zone_ok(t) for t in terms):
            want += sum(all(p["labels"].get(k) == v for k, v in sel.items()) for p in n["pods"])
    totals = [rs.group_total(g) for g in range(rs.dims["groups"])]
    assert want in totals, (want, totals)


def test_listed_and_unlisted_types_are_told_apart(pkg, oracle):
    """topology_test.go:661-695 with instance types: only the pods on the listed type's nodes are counted, so the spread pods
    balance against 2 + 1 and not against the 5 on the other types"""
    prob = itf.listed_unlisted(0)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert 3 in [rs.group_total(g) for g in range(rs.dims["groups"])]


def test_cloud_lists_reach_beyond_the_first_word(pkg):
    prob = itf.cloud_lists(0)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["types"] == 720 and rs.dims["type_words"] > 1 and rs.dims["itype_filter_terms"] > 0


def _check_placements(prob, res):
    """each placed pod sits on an existing node whose instance-type label its own (unrelaxed) requirement admits, or a new one"""
    n_ex = len(res["existing"])
    for i, a in enumerate(res["assign"]):
        p = prob["pods"][i]
        if not (0 <= a < n_ex):
            continue
        labels = prob["nodes"][res["existing"][a]["node"]]["labels"]
        na = p.get("nodeAffinity") or {}
        req = na.get("required") or [[]]
        sel = [{"key": k, "operator": "In", "values": [v]} for k, v in (p.get("nodeSelector") or {}).items() if k == INSTANCE_TYPE]
        assert any(itf.term_matches(sel + t, labels) for t in req), (i, labels.get(INSTANCE_TYPE))


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_places_pods_only_where_admitted(pkg, oracle, name, prob, table):
    _check_placements(prob, oracle.solve_dict(pkg, prob)[1].to_dict())


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_fast_mode_equals_literal(pkg, oracle, name, prob, table):
    oracle.assert_fast_equals_literal(pkg, prob)


def test_narrowed_nodes_are_not_recorded(pkg, oracle):
    """the scenario reaches what it was built for: some small selector pods share a node with a pod that excluded the listed
    types, and some spread pods land on new nodes"""
    prob = itf.narrowed(0)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    n_ex = len(d["existing"])
    by_node = {}
    for i, a in enumerate(d["assign"]):
        if a >= n_ex:
            by_node.setdefault(a, set()).add(prob["pods"][i]["labels"]["app"])
    assert any({"big", "s"} <= apps for apps in by_node.values())


def test_cluster_candidates_encode(pkg):
    for prob in (itf.cluster(0), itf.after(0)):
        cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands)
        assert rs.dims["itype_filter_terms"] > 0
