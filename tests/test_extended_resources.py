"""CPU: batches whose pods request 9 to 32 distinct resources (tests/extended_resource_problems.py) encode without refusal,
with the resources a daemonset requests or a limit names in row slots and the rest as ext resources; the near misses are
refused; and the oracle's placements are sound on every resource (Fits restated over the existing nodes)."""
import pytest

import extended_resource_problems as xp
import placement_invariants

CORPUS = xp.corpus()
IDS = [c[0] for c in CORPUS]


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_encoder_accepts_up_to_32_resources(pkg, name, prob):
    n = len(xp.read_resources(prob) | {r for nd in prob["nodes"] for p in nd["pods"] for r in p.get("requests", {})})
    assert 9 <= n <= 32
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["resources"] == 8 and rs.dims["resources"] + rs.dims["resources_ext"] == n
    # the GPU limit and the hugepages daemonset's resource take row slots, the MIG profiles and the other rare ones are ext
    assert sorted(rs.resource_id(r) for r in xp.SLOTS) == list(range(8))
    assert all(rs.resource_id(r) >= 8 for r in xp.EXT_RESOURCES)


def test_fresh_fleet_is_accepted(pkg):
    for _, prob in xp.fresh_corpus():
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
        assert rs.dims["existing"] == 0 and rs.dims["resources_ext"] >= 6


def test_cluster_and_after_are_accepted(pkg):
    for prob in (xp.cluster(0), xp.after(0)):
        cands = [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands[:3])
        assert rs.dims["resources_ext"] > 0


@pytest.mark.parametrize("make,msg", [(xp.too_many_resources, "more than 32 resources"),
                                      (xp.too_many_slot_resources, "more than 8 resources that a daemonset requests or a provisioner limit names")])
def test_near_misses_are_refused(pkg, make, msg):
    with pytest.raises(pkg.KschedError, match=msg):
        pkg.ResidentSolve(pkg.Problem.from_dict(make()))


def pkg_qty(s):
    s = str(s)
    units = {"Ki": 2 ** 10, "Mi": 2 ** 20, "Gi": 2 ** 30, "Ti": 2 ** 40, "m": 1e-3}
    for u, f in units.items():
        if s.endswith(u):
            return float(s[: -len(u)]) * f
    return float(s)


def _requests(pod):
    """resources.RequestsForPods: the containers' sum, raised to each init container's request (the ceiling)"""
    if "requests" in pod:
        return {k: pkg_qty(v) for k, v in pod["requests"].items()}
    out = {}
    for c in pod.get("containers", []):
        for k, v in c.get("requests", {}).items():
            out[k] = out.get(k, 0.0) + pkg_qty(v)
    for c in pod.get("initContainers", []):
        for k, v in c.get("requests", {}).items():
            out[k] = max(out.get(k, 0.0), pkg_qty(v))
    return out


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_oracle_placements_fit_on_every_resource(pkg, oracle, name, prob):
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    d = res.to_dict()
    on_existing = ext_on_existing = 0
    for e in d["existing"]:
        node = prob["nodes"][e["node"]]
        used = {}
        for p in node["pods"] + [prob["pods"][i] for i in e["pods"]]:
            for k, v in _requests(p).items():
                used[k] = used.get(k, 0.0) + v
        for i in e["pods"]:
            for k in _requests(prob["pods"][i]):  # Fits over the keys of the requests (resources.go:138-145)
                assert used[k] <= pkg_qty(node["allocatable"].get(k, "0")) + 1e-9, (node["name"], k)
            on_existing += 1
            ext_on_existing += any(k.startswith("nvidia.com/mig") for k in _requests(prob["pods"][i]))
    assert on_existing > 0 and ext_on_existing > 0
    _new_nodes_fit(prob, d)


def _allocatable(it):
    """capacity less the overhead, over the keys of capacity (the encoder's allocatable of an instance type)"""
    ov = it.get("overhead", {})
    out = {k: pkg_qty(v) for k, v in it["capacity"].items()}
    for part in ("kubeReserved", "systemReserved", "evictionThreshold"):
        for k, v in ov.get(part, {}).items():
            if k in out:
                out[k] -= pkg_qty(v)
    return out


def _new_nodes_fit(prob, d):
    """every option of every new node covers the node's requests on every resource, and the node's ext requests are the sum
    of its pods' (no daemonset requests an ext resource)"""
    ext_nodes = 0
    for n in d["newNodes"]:
        req = {k: v / 1000.0 for k, v in n["requests"].items()}
        assert n["options"]
        for t in n["options"]:
            alloc = _allocatable(prob["instanceTypes"][t])
            for k, v in req.items():
                assert v <= alloc.get(k, 0.0) + 1e-6, (prob["instanceTypes"][t]["name"], k, v)
        own = {}
        for p in n["pods"]:
            for k, v in _requests(prob["pods"][p]).items():
                own[k] = own.get(k, 0.0) + v
        for k in xp.EXT_RESOURCES:
            assert abs(req.get(k, 0.0) - own.get(k, 0.0)) < 1e-6, (k, req.get(k), own.get(k))
        ext_nodes += any(k in req for k in xp.EXT_RESOURCES)
    assert ext_nodes > 0


@pytest.mark.parametrize("name,prob", xp.fresh_corpus(), ids=[c[0] for c in xp.fresh_corpus()])
def test_oracle_new_nodes_fit_without_existing_nodes(pkg, oracle, name, prob):
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    _new_nodes_fit(prob, res.to_dict())


@pytest.mark.parametrize("name,prob", CORPUS, ids=IDS)
def test_oracle_results_pass_placement_invariants(pkg, oracle, name, prob):
    # the invariants sum the pods' own requests (no daemonset overhead) and know the zones of new nodes only
    prob = dict(prob, daemonSetPods=[], pods=[{k: v for k, v in p.items() if k != "topologySpreadConstraints"} for p in prob["pods"]])
    problem = pkg.Problem.from_dict(prob)
    res = pkg.Result()
    assert oracle.solve(problem, res) == 0, res.error
    stats = placement_invariants.check(problem, res)
    assert stats["scheduled"] > 0
