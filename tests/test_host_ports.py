"""CPU: clusters whose pods name more than 64 distinct host-port entries (tests/hostport_problems.py) encode without refusal.
The encoder's entry table is the one restated from the problem's strings (first appearance, and with more than 64 entries
only those a different pod of the batch can match); problems that fit the word keep their ids and get no table. The
oracle's results never put a pod next to a different pod holding an entry its ports match, and where the table exists its
entries from id 64 on turn pods away from nodes."""
import copy

import pytest

import hostport_problems as hp

CORPUS = hp.corpus()
IDS = [c[0] for c in CORPUS]
TABLE = [c for c in CORPUS if c[2]]


def _words(n):
    return (n - 64 + 63) // 64 if n > 64 else 0


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_encoder_keeps_the_entries_a_pod_can_match(pkg, name, prob, table):
    seen, kept = hp.kept_entries(prob)
    assert len(seen) > 64 or name in ("fit64",), len(seen)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.hostports() == kept
    assert rs.dims["hostports"] == len(kept)
    assert rs.dims["hostport_ext_words"] == _words(len(kept))
    assert (rs.dims["hostport_ext_words"] > 0) == table


def test_boundaries():
    assert [len(x) for x in hp.kept_entries(hp.boundary("fit64"))] == [64, 64]
    assert [len(x) for x in hp.kept_entries(hp.boundary("prune65"))] == [65, 64]
    assert [len(x) for x in hp.kept_entries(hp.boundary("keep65"))] == [65, 65]


def test_daemonset_clusters_without_batch_ports_keep_no_entry(pkg):
    prob = hp.daemonsets(60, 0, "none")
    assert len(hp.kept_entries(prob)[0]) > 80
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["hostports"] == 0 and rs.dims["hostport_ext_words"] == 0


def test_traps_have_a_class_whose_entries_are_all_beyond_64(pkg):
    prob = hp.traps(0)
    kept = pkg.ResidentSolve(pkg.Problem.from_dict(prob)).hostports()
    assert kept.index(("0.0.0.0", 9500, "TCP")) >= 64
    # 9500 matches nothing below 64: the class's row words are both zero
    assert not any(hp.matches(("0.0.0.0", 9500, "TCP"), e) for e in kept[:64])
    # the two-container pod holds one entry, and 10.9.0.1:8081 / 10.9.0.2:8081 are two entries that 0.0.0.0:8081 both matches
    assert kept.count(("0.0.0.0", 9000, "TCP")) == 1
    assert {("10.9.0.1", 8081, "TCP"), ("10.9.0.2", 8081, "TCP"), ("0.0.0.0", 8081, "TCP")} <= set(kept)


def test_cluster_candidates_keep_more_than_64_entries(pkg):
    for prob in (hp.cluster(0), hp.after(0)):
        cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
        seen, kept = hp.kept_entries(prob, cands)
        assert len(kept) > 64
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands)
        assert rs.hostports() == kept and rs.dims["hostport_ext_words"] == _words(len(kept))


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_never_puts_matching_ports_together(pkg, oracle, name, prob, table):
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    assert hp.node_conflicts(prob, d) == []
    with_ports = [i for i, p in enumerate(prob["pods"]) if hp.pod_ports(p)]
    assert with_ports == [] or any(d["assign"][i] >= 0 for i in with_ports)


def _on_existing(d):
    return {i: e["node"] for e in d["existing"] for i in e["pods"]}


def _strip(prob, high):
    """the problem with every port declaration whose entry has an id from 64 on removed (pending and bound pods)"""
    out = copy.deepcopy(prob)
    for p in out["pods"] + [q for n in out["nodes"] for q in n["pods"]]:
        for c in [p] + p.get("containers", []):
            if "ports" in c:
                c["ports"] = [x for x in c["ports"] if (x.get("hostIP") or "0.0.0.0", x["hostPort"], x.get("protocol", "TCP")) not in high]
    return out


@pytest.mark.parametrize("name,prob,table", TABLE, ids=[c[0] for c in TABLE])
def test_entries_beyond_64_turn_pods_away(pkg, oracle, name, prob, table):
    """some pod that the oracle puts on an existing node once the entries from id 64 on are gone is turned away from that
    node, which holds such an entry matching one of its ports, and placed elsewhere or left unscheduled"""
    high = set(pkg.ResidentSolve(pkg.Problem.from_dict(prob)).hostports()[64:])
    real, stripped = oracle.solve_dict(pkg, prob)[1].to_dict(), oracle.solve_dict(pkg, _strip(prob, high))[1].to_dict()
    on, on_s = _on_existing(real), _on_existing(stripped)
    turned = 0
    for i, node in on_s.items():
        if on.get(i) == node:
            continue
        held = [e for q in prob["nodes"][node]["pods"] for e in hp.pod_ports(q)]
        held += [e for j, n in on.items() if n == node for e in hp.pod_ports(prob["pods"][j])]
        turned += any(e in high and hp.matches(a, e) for a in hp.pod_ports(prob["pods"][i]) for e in held)
    assert turned > 0
