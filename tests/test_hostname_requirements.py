"""CPU: pods whose kubernetes.io/hostname requirements go beyond one In / NotIn value (tests/hostname_problems.py) encode
without refusal. Each class's admitted existing slots equal the reference's Requirement.Has on the problem's strings, the
single-value forms keep their {complement, slot} pair and get no table, and the oracle's results only put a pod where its
requirement admits it. The near misses are refused."""
import pytest

import fixtures as fx
import hostname_problems as hn

CORPUS = hn.corpus()
IDS = [c[0] for c in CORPUS]
TABLE = [c for c in CORPUS if c[2]]


def _admitted(prob, reqs):
    """(admits a new node, existing slots admitted) of a list of requirements intersected (requirements.go:87-94); every
    provisioner-owned node is an existing slot in this corpus"""
    owned = [n for n in prob["nodes"] if n["labels"].get(fx.PROVISIONER_NAME)]
    slots = [e for e, n in enumerate(owned) if all(hn.admits(r, hn.node_hostname(n)) for r in reqs)]
    new = all(hn.admits(r, hn.PLACEHOLDER + "0001") for r in reqs)
    return new, slots


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_encoder_takes_the_scenario(pkg, name, prob, table):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert (rs.dims["hostname_words"] > 0) == table
    if table:
        assert rs.dims["hostname_words"] == max(1, (rs.dims["existing"] + 63) // 64)


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_admitted_slots_equal_the_string_restatement(pkg, name, prob, table):
    """each pod's own class (before any relaxation) points to the entry that restates its hostname requirements on
    strings; a pod without one has a class without an entry"""
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["pods"] == len(prob["pods"])
    entries = rs.hostname_reqs()
    checked = 0
    for i, p in enumerate(prob["pods"]):
        reqs = hn.hostname_reqs(p)
        e = rs.class_hostname_req(rs.pod_class(i))
        if not reqs:
            assert e is None, p["name"]
            continue
        new, slots = _admitted(prob, reqs)
        assert e is not None and entries[e] == (new, slots), (p["name"], reqs)
        checked += 1
    assert checked > 0


def test_old_forms_get_no_table(pkg):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(hn.old_forms(0)))
    assert rs.dims["hostname_words"] == 0 and rs.dims["hostname_reqs"] > 0


def test_in_lists_reach_beyond_the_first_word(pkg):
    for k in (2, 5, 40):
        prob = hn.in_list(k, k)
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
        assert any(not new and len(slots) == k and max(slots) >= 64 for new, slots in rs.hostname_reqs())


@pytest.mark.parametrize("name,prob", hn.near_misses(), ids=[n for n, _ in hn.near_misses()])
def test_near_misses_are_refused(pkg, name, prob):
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED


def _check_placements(prob, res):
    """each placed pod without preferred terms sits on a node admitted by its hostname requirements with one of its required
    terms in force (relaxation drops them in order): an existing node's hostname, or a new node's placeholder"""
    n_ex = len(res["existing"])
    checked = 0
    for i, a in enumerate(res["assign"]):
        p = prob["pods"][i]
        na = p.get("nodeAffinity") or {}
        if a < 0 or na.get("preferred"):
            continue
        levels = [hn.hostname_reqs(p, t) for t in range(max(1, len(na.get("required") or [])))]
        host = hn.node_hostname(prob["nodes"][res["existing"][a]["node"]]) if a < n_ex else hn.PLACEHOLDER + "0001"
        assert any(all(hn.admits(r, host) for r in lv) for lv in levels), (i, host)
        checked += 1
    return checked


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_places_pods_only_where_admitted(pkg, oracle, name, prob, table):
    _check_placements(prob, oracle.solve_dict(pkg, prob)[1].to_dict())


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_fast_mode_equals_literal(pkg, oracle, name, prob, table):
    oracle.assert_fast_equals_literal(pkg, prob)


def test_scenarios_cross_what_they_were_built_for(pkg, oracle):
    # In lists: the listed nodes fill (slots >= 64 used), the rest stay unscheduled and no new node opens for them
    prob = hn.in_list(5, 1)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    pinned = [i for i, p in enumerate(prob["pods"]) if p["labels"]["app"] == "pinned"]
    on = {d["existing"][d["assign"][i]]["node"] for i in pinned if 0 <= d["assign"][i] < len(d["existing"])}
    assert any(s >= 64 for s in on)
    assert any(d["assign"][i] < 0 for i in pinned)
    assert all(d["assign"][i] < len(d["existing"]) for i in pinned)
    # NotIn: pods go to new nodes while the excluded nodes still have room
    prob = hn.not_in(2000, 3, 0)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    web = [i for i, p in enumerate(prob["pods"]) if p["labels"]["app"] == "web"]
    assert any(d["assign"][i] >= len(d["existing"]) for i in web)
    excluded = set(prob["pods"][web[0]]["nodeAffinity"]["required"][0][0]["values"])
    assert not any(0 <= d["assign"][i] < len(d["existing"]) and
                   prob["nodes"][d["existing"][d["assign"][i]]["node"]]["name"] in excluded for i in web)
    # selector a plus NotIn [a] admits nothing
    prob = hn.selector_and_affinity(0)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    assert all(d["assign"][i] < 0 for i, p in enumerate(prob["pods"]) if p["labels"]["app"] == "none")
    assert any(d["assign"][i] >= 0 for i, p in enumerate(prob["pods"]) if p["labels"]["app"] == "one")
    # hostname affinity: matching pods only on excluded nodes still bootstrap onto an admitted node (lists and the pair
    # form); a matching pod on an admitted node draws the pods there; the extra-domain flag is set for the unowned node
    prob = hn.affinity_lists(0)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    host = {i: prob["nodes"][d["existing"][a]["node"]]["name"] for i, a in enumerate(d["assign"]) if 0 <= a < len(d["existing"])}
    app = {i: p["labels"]["app"] for i, p in enumerate(prob["pods"])}
    assert {host[i] for i in host if app[i] == "a1"} and {host[i] for i in host if app[i] == "a1"} <= {"n-004", "n-005", "n-012"}
    assert {host[i] for i in host if app[i] == "a2"} == {"n-006"}
    assert {host[i] for i in host if app[i] == "a3"} == {"n-010"}
    # two terms: some pods land on the second list after the first is full
    prob = hn.two_terms(0)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    second = {n["name"] for n in prob["nodes"][5:8]}
    assert any(0 <= a < len(d["existing"]) and prob["nodes"][d["existing"][a]["node"]]["name"] in second for a in d["assign"])


def test_cluster_candidates_encode(pkg):
    for prob in (hn.cluster(0), hn.after(0)):
        cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands)
        assert rs.dims["hostname_reqs"] > 0
