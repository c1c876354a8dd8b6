"""CPU: every scenario of tests/run_problems.py really reaches the capacity of the pack kernel's run paths it was built
for. Each predicate is computed from the problem and the literal oracle's result alone, so a generator edit that misses
its boundary fails here. The oracle's fast mode (the one that made the full-size golden digests) must also equal the
literal path on the whole corpus: it had only been checked on 3-zone shapes before."""
import pytest

import fixtures as fx
import run_problems as rp
from fixtures import CAPACITY_TYPE, HOSTNAME, ZONE

K_ACT_CAP = 1280      # pack_kernel.cuh kActCap: open nodes whose hot state is in shared memory
K_M1_LV = 12          # kM1Lv: pod counts the mask run's lists represent
K_RUN_VARIANTS = 4    # kRunVariants: fresh-node variants one class keeps
K_RUN_HOST = 4        # kRunHost: hostname relations of a run-eligible class
K_RUN_W32 = 64        # kRunW32: option words of a variant


def _single(req):
    op, _, rest = (req or "").partition(" ")
    vals = rest.strip()[1:-1].split()
    return vals[0] if op == "In" and len(vals) == 1 else None


class Placed:
    """where the oracle put every pod: node ids (existing e < n_existing, else new), and each node's label values"""

    def __init__(self, prob, res):
        self.prob, self.res = prob, res
        self.assign = res["assign"]
        self.ne = len(res["existing"])

    def value(self, node, key):
        if node < self.ne:
            return self.prob["nodes"][self.res["existing"][node]["node"]]["labels"].get(key)
        nn = self.res["newNodes"][node - self.ne]
        v = _single(nn["requirements"].get(key))
        if v is None and key in (ZONE, CAPACITY_TYPE):
            v = nn["launch"]["zone" if key == ZONE else "capacityType"]
        return v

    def nodes_of(self, pods):
        return [self.assign[i] for i in pods if self.assign[i] >= 0]


def queue_order(prob):
    """the queue's order (queue.go:74-110): cpu desc, memory desc, creationTimestamp, UID"""
    def key(i):
        p = prob["pods"][i]
        r = p.get("requests", {})
        return (-fx._qty_float(r.get("cpu", "0")), -fx._qty_float(r.get("memory", "0")), p.get("creationTimestamp", 0), p["uid"])
    return sorted(range(len(prob["pods"])), key=key)


def class_of(facts):
    return {i: c for c, idx in facts["classes"].items() for i in idx}


def hostname_relations(pod):
    n = sum(1 for s in pod.get("topologySpreadConstraints", []) if s["topologyKey"] == HOSTNAME)
    for kind in ("podAffinity", "podAntiAffinity"):
        n += sum(1 for t in pod.get(kind, {}).get("required", []) if t["topologyKey"] == HOSTNAME)
    return n


# ---------------------------------------------------------------- one predicate per scenario
def reach_zones(prob, facts, pl):
    nz = facts["zones"]
    spread = [c for c in facts["classes"] if c.startswith("spread")]
    most = max(len({pl.value(n, ZONE) for n in pl.nodes_of(facts["classes"][c])}) for c in spread)
    assert most == nz, f"one zone-spread class should hold pods in all {nz} zones, got {most}"
    if nz >= 9:
        assert most >= 9  # registered domains beyond kM1Dom = 8: the mask run is refused
    if nz == 17:
        assert len({o["zone"] for it in prob["instanceTypes"] for o in it["offerings"]}) == 16  # the 17th comes from nodes


def reach_pods_capacity(prob, facts, pl):
    spread = set(facts["classes"]["spread-a"]) | set(facts["classes"]["spread-b"])
    most = max(sum(1 for p in nn["pods"] if p in spread) for nn in pl.res["newNodes"])
    assert most >= K_M1_LV, f"a zone-spread node should reach {K_M1_LV} pods, got {most}"


def reach_pinned_nodes(prob, facts, pl):
    pinned, spread = set(facts["classes"]["pinned"]), set(facts["classes"]["spread"])
    shared = [nn for nn in pl.res["newNodes"] if pinned & set(nn["pods"]) and spread & set(nn["pods"])]
    assert shared, "no zone-spread pod landed on a node opened In [z0 z1] by the earlier class"


def reach_two_masks(prob, facts, pl):
    for cls, second in (("zc", facts["second"]), ("zr", rp.RACK)):
        pairs = {(pl.value(n, ZONE), pl.value(n, second)) for n in pl.nodes_of(facts["classes"][cls])}
        assert None not in {b for _, b in pairs}, (cls, pairs)
        assert len(pairs) > K_RUN_VARIANTS, f"{cls}: {len(pairs)} (zone, {second}) pairs, the variant ring needs more than {K_RUN_VARIANTS}"


def reach_hostname_relations(prob, facts, pl):
    cls = class_of(facts)
    for n_rel in (3, 4, 5):
        idx = facts["classes"][f"h{n_rel}"]
        assert hostname_relations(prob["pods"][idx[0]]) == n_rel
        assert all(pl.assign[i] >= 0 for i in idx)
    assert hostname_relations(prob["pods"][facts["classes"]["h5"][0]]) > K_RUN_HOST
    # the relations constrain: pods of the classes share nodes with each other (counts above zero are evaluated)
    mixed = [nn for nn in pl.res["newNodes"] if len({cls[p] for p in nn["pods"]} - {"db"}) >= 2]
    assert mixed


def reach_big_active_set(prob, facts, pl):
    cls = class_of(facts)
    anti = [nn for nn in pl.res["newNodes"] if cls[nn["pods"][0]] == "anti"]
    assert len(anti) > K_ACT_CAP
    # every anti-affinity node holds one pod of the same shape, so before the zone run they are all alike: one that takes a
    # zone-spread pod shows that more than kActCap open nodes could still take the next topology run's pod
    assert all(sum(cls[p] == "anti" for p in nn["pods"]) == 1 for nn in anti)
    assert len({tuple(nn["options"]) for nn in anti}) == 1
    for later in ("zone", "host"):
        took = {n - pl.ne for n in pl.nodes_of(facts["classes"][later])}
        assert any(cls[pl.res["newNodes"][t]["pods"][0]] == "anti" for t in took), f"no {later}-spread pod landed on an anti-affinity node"


def reach_limits(prob, facts, pl):
    if "big" in facts["classes"]:
        big = facts["classes"]["big"]
        placed = sum(pl.assign[i] >= 0 for i in big)
        assert 0 < placed < len(big), f"the limit should bind inside the run: {placed} of {len(big)} placed"
    else:
        assert len({nn["provisioner"] for nn in pl.res["newNodes"]}) >= 3


def reach_many_existing(prob, facts, pl):
    live = [n for n in prob["nodes"] if not n.get("markedForDeletion")]
    assert len(live) >= 2048 and pl.ne == len(live)
    assert any(n.get("taints") for n in live) and len(live) < len(prob["nodes"])
    hit = {n for n in pl.nodes_of(facts["classes"]["plain"]) if n < pl.ne}
    assert len(hit) > 512, f"the plain run should span more than 512 existing nodes, got {len(hit)}"


def reach_huge_catalog(prob, facts, pl):
    assert (len(prob["instanceTypes"]) + 31) // 32 > K_RUN_W32
    spread = set(facts["classes"]["spread"])
    assert max(sum(1 for p in nn["pods"] if p in spread) for nn in pl.res["newNodes"]) >= 2  # fresh nodes the variants would replay


def reach_extended_resources(prob, facts, pl):
    for cls in ("ext", "ext-spread"):
        nodes = pl.nodes_of(facts["classes"][cls])
        assert len(nodes) == len(facts["classes"][cls])
        best = max(set(nodes), key=nodes.count)
        req = pl.res["newNodes"][best - pl.ne]["requests"]
        assert nodes.count(best) >= 2 and "fake.com/vendor-a" in req and "fake.com/vendor-b" in req


def reach_relaxation(prob, facts, pl):
    cls = class_of(facts)
    order = [i for i in queue_order(prob) if cls[i] in ("ok", "nowhere")]
    assert [cls[i] for i in order[:6]] == ["ok", "nowhere"] * 3
    assert all((pl.assign[i] >= 0) == (cls[i] == "ok") for i in order)  # placed and unschedulable alternate pod by pod
    assert all(pl.assign[i] < 0 for i in facts["classes"]["too-big"])
    prefer = facts["classes"]["prefer"]
    assert all(pl.assign[i] >= 0 and pl.res["relax"][i] > 0 for i in prefer)
    assert all(pl.assign[i] >= 0 for i in facts["classes"]["anyway"])


def reach_chunk_edges(prob, facts, pl):
    cls = class_of(facts)
    seq = [cls[i] for i in queue_order(prob)]
    k = facts["k"]
    assert seq[:k + 1] == ["a"] * k + ["b"], "the class change should sit at index k of the first run"
    x = seq.index("x")
    assert seq[x:x + 6] == ["x", "y"] * 3
    assert all(a >= 0 for a in pl.assign)


REACH = {name: globals()["reach_" + ("zones" if name.startswith("zones") else name)] for name in rp.SCENARIOS}


@pytest.mark.parametrize("name,seed", rp.CORPUS, ids=[f"{n}-{s}" for n, s in rp.CORPUS])
def test_scenario_reaches_its_boundary(pkg, oracle, name, seed):
    prob, facts = rp.build(name, seed)
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    REACH[name](prob, facts, Placed(prob, res.to_dict()))


@pytest.mark.parametrize("name,seed", rp.CORPUS, ids=[f"{n}-{s}" for n, s in rp.CORPUS])
def test_fast_mode_equals_literal_on_run_corpus(pkg, oracle, name, seed):
    a, b = oracle.assert_fast_equals_literal(pkg, rp.build(name, seed)[0])
    assert a.nodes_visited == b.nodes_visited and a.add_calls == b.add_calls
