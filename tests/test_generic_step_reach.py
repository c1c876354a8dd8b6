"""CPU: every scenario of tests/generic_step_problems.py reaches the generic-step mechanism it is built for. Each predicate
is restated on the problem's strings and the literal oracle's result (integers in milli-units, tests/exact_arith.py), with
no product code. The state before a pod comes from the oracle's Solve of the queue-order prefix before it: queue order is a
total order, so dropping the later pods reorders nothing, and the prefix's placements must equal the full run's."""
import re
from pathlib import Path

import pytest

import exact_arith as ea
import generic_step_problems as gp
from fixtures import ARCH, PROVISIONER_NAME, ZONE

IDS = [n for n, _ in gp.CORPUS]


def queue_order(prob):
    """the queue's order (queue.go:74-110): cpu desc, memory desc, creationTimestamp, UID"""
    def key(i):
        p = prob["pods"][i]
        r = ea.pod_requests(p)
        return (-r.get("cpu", 0), -r.get("memory", 0), p.get("creationTimestamp", 0), p["uid"])
    return sorted(range(len(prob["pods"])), key=key)


def _solve(pkg, oracle, prob):
    res = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(prob), res) == 0, res.error
    return res.to_dict()


def _prefix(pkg, oracle, prob, full, pos):
    """(prefix problem, its result): the pods before queue position pos; their placements equal the full run's"""
    order = queue_order(prob)[:pos]
    sub = dict(prob, pods=[prob["pods"][i] for i in order])
    res = _solve(pkg, oracle, sub)
    assert res["assign"] == [full["assign"][i] for i in order]
    return sub, res


def scan_order(prob, res):
    """new nodes in the order the reference scans them after the last pod of `res` (scheduler.go:183-190): a stable sort by
    pod count after every Add (every pod of these scenarios is placed in its first pass)"""
    assert all(a >= 0 for a in res["assign"]) and not any(res["relax"])
    ne = len(res["existing"])
    nodes, count = [], {}
    for i in queue_order(prob):
        n = res["assign"][i] - ne
        if n < 0:
            continue
        if n not in count:
            nodes.append(n)
            count[n] = 0
        count[n] += 1
        nodes.sort(key=lambda m: count[m])
    return nodes


def _alloc(prob, t):
    return ea.allocatable(prob["instanceTypes"][t])


def _type_arch(prob, t):
    return next(r["values"][0] for r in prob["instanceTypes"][t]["requirements"] if r["key"] == ARCH)


def _any_option_holds(prob, nn, extra, arch=None):
    """some option (of architecture `arch`, if given) holds the node's requests plus `extra`"""
    need = ea._merge(dict(nn["requests"]), extra)
    return any(ea.fits(need, _alloc(prob, t)) for t in nn["options"] if arch is None or _type_arch(prob, t) == arch)


def _arch_allows(nn, arch):
    req = nn["requirements"].get(ARCH)
    return req is None or arch in req.split("[", 1)[1].rstrip("]").split()


def _hot_fit(prob, nn, extra):
    """some option holds the requests in cpu, memory and pods (what the quick fit tests)"""
    need = ea._merge(dict(nn["requests"]), extra)
    need = {k: v for k, v in need.items() if k in ("cpu", "memory", "pods")}
    return any(ea.fits(need, _alloc(prob, t)) for t in nn["options"])


# ---------------------------------------------------------------- a. exclusions
def excluded_before(pkg, oracle, prob, facts, full, pod):
    """(count of in-flight nodes the pod's step excludes ahead of where the pod goes, position of the accepting node in the
    scan order or None for a fresh node): nodes whose quick fit passes and whose full check fails - requirement-compatible
    with no option holding the requests (or, for the zone-spread P, refused by the arch requirement)"""
    pos = queue_order(prob).index(pod)
    sub, res = _prefix(pkg, oracle, prob, full, pos)
    ne = len(res["existing"])
    target = full["assign"][pod] - ne
    preq = ea.pod_requests(prob["pods"][pod])
    n_excl, at = 0, None
    for k, n in enumerate(scan_order(sub, res)):
        if n == target:
            at = k
            break
        nn = res["newNodes"][n]
        if not _hot_fit(sub, nn, preq):
            continue
        if facts["spread"]:
            n_excl += not _arch_allows(nn, "arm64")
        elif facts["ext"]:
            n_excl += not _any_option_holds(sub, nn, preq)
        else:
            n_excl += _arch_allows(nn, "arm64") and not _any_option_holds(sub, nn, preq, "arm64")
    return n_excl, at


def reach_exclusions(pkg, oracle, prob, facts, full, name):
    firsts = [facts["classes"][p][0] for p in facts["p"]]
    seen = [excluded_before(pkg, oracle, prob, facts, full, pod) for pod in firsts]
    counts = [c for c, _ in seen]
    q = facts["q"]
    if name in ("excl15", "excl16", "excl17", "excl40", "excl_wide"):
        assert counts == [q] * len(firsts), counts
    else:  # (a zone-spread or ext P also meets the fresh nodes of the P classes before it)
        assert min(counts) >= max(q, gp.K_MAX_EXCL + 1), counts
    landed = [at for _, at in seen if at is not None]
    assert landed, seen  # a P class lands on an in-flight node behind the excluded ones
    if name == "excl_overflow":
        assert min(landed) >= gp.K_ACT_CAP, seen  # the accepting slot is in the ov_* arrays
    if facts["spread"]:  # no rejected memo for a topology class: its second pod meets them again
        c, _ = excluded_before(pkg, oracle, prob, facts, full, facts["classes"][facts["p"][0]][1])
        assert c == q


def reach_excl_wide(pkg, oracle, prob, facts, full, name):
    reach_exclusions(pkg, oracle, prob, facts, full, name)
    pos = column_positions(prob)
    names = [it["name"] for it in prob["instanceTypes"]]
    amd = [pos[i] for i, nm in enumerate(names) if nm.startswith("amd")]
    assert min(amd) >= 32 * 32 and -(-len(names) // 32) == 35
    # the accepting node held amd64 options (in words >= 32) before P narrowed them away
    a = full["assign"][facts["classes"]["a"][0]] - len(full["existing"])
    p_pods = [i for c in facts["p"] for i in facts["classes"][c]]
    assert any(full["assign"][i] - len(full["existing"]) == a for i in p_pods)
    pos_a = queue_order(prob).index(facts["classes"]["a"][0])
    sub, res = _prefix(pkg, oracle, prob, full, pos_a + 1)
    assert any(pos[t] >= 32 * 32 for t in res["newNodes"][a]["options"])
    assert all(names[t].startswith("arm") for t in full["newNodes"][a]["options"])


def column_positions(prob):
    """the encoder's type numbering (host/encoder.cc, instance_types): a stable sort by the cheapest available offering"""
    price = [min(o["price"] for o in it["offerings"] if o.get("available", True)) for it in prob["instanceTypes"]]
    order = sorted(range(len(price)), key=lambda i: price[i])
    pos = [0] * len(price)
    for t, i in enumerate(order):
        pos[i] = t
    return pos


# ---------------------------------------------------------------- b. fronts
HOT = ("cpu", "memory", "pods")


def front(prob, options, keys=HOT):
    """Pareto front (distinct maximal vectors) of the options' allocatable vectors over `keys`"""
    vecs = {tuple(_alloc(prob, t).get(k, 0) for k in keys) for t in options}
    return {v for v in vecs if not any(w != v and all(a >= b for a, b in zip(w, v)) for w in vecs)}


def min_requests(prob):
    reqs = [ea.pod_requests(p) for p in prob["pods"]]
    return {k: min(r.get(k, 0) for r in reqs) for k in HOT}


def reach_fronts(pkg, oracle, prob, facts, full, name):
    shape = facts["shape"]
    sizes = [len(front(prob, nn["options"])) for nn in full["newNodes"]]
    first = full["newNodes"][0]
    want = {"one": 1, "two": 2, "three": 3, "tie": 1, "dup": 2, "wide": 3}[shape]
    # the first node's options before its later pods: the prefix up to its second pod
    pods = sorted(first["pods"], key=queue_order(prob).index)
    sub, res = _prefix(pkg, oracle, prob, full, queue_order(prob).index(pods[0]) + 1)
    opened = res["newNodes"][0]["options"]
    assert len(front(sub, opened)) == want, (shape, front(sub, opened))
    assert len(full["newNodes"]) >= 2 and max(sizes) >= 1
    if shape == "tie":
        pos = column_positions(prob)
        cpu_max = max(_alloc(prob, t)["cpu"] for t in opened)
        first_cpu = min((t for t in opened if _alloc(prob, t)["cpu"] == cpu_max), key=lambda t: pos[t])
        assert front(sub, [first_cpu]) != front(sub, opened)  # the first cpu-maximal type is not the dominant one
    if shape == "dup":
        vecs = [tuple(_alloc(prob, t)[k] for k in HOT) for t in opened]
        assert len(set(vecs)) < len(vecs)
    if shape == "wide":
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
        assert rs.dims["resources"] > gp.K_HOT_RES
    # node_closed: some node ends with no option holding one more pod of the smallest requests, and some does not
    mr = min_requests(prob)
    closed = [not _any_option_holds(prob, nn, mr) for nn in full["newNodes"]]
    assert any(closed) and not all(closed), closed


def reach_front_warps(pkg, oracle, prob, facts, full, name):
    pos = column_positions(prob)
    names = [it["name"] for it in prob["instanceTypes"]]
    c = names.index("big-c")
    assert pos[c] >= 32 * 32 and pos[names.index("big-a")] < 32 and pos[names.index("big-b")] < 32
    x = facts["classes"]["x"][0]
    y = facts["classes"]["y"][0]
    assert full["assign"][y] == full["assign"][x]  # Y lands on X's node, through C alone
    sub, res = _prefix(pkg, oracle, prob, full, queue_order(prob).index(x) + 1)
    opened = res["newNodes"][0]["options"]
    assert len(front(sub, opened)) == 3 and c in opened
    assert full["newNodes"][full["assign"][x]]["options"] == [c]


# ---------------------------------------------------------------- c. memos
def reach_class_memo(pkg, oracle, prob, facts, full, name):
    provs = [p["name"] for p in prob["provisioners"]]  # already in weight order
    by_kind = {}
    for cls, idx in facts["classes"].items():
        kind = cls.rstrip("0123456789")
        for i in idx:
            nn = full["newNodes"][full["assign"][i]]
            by_kind.setdefault(kind, []).append((provs[nn["provisioner"]], full["relax"][i]))
    assert len(facts["classes"]) * len(provs) >= 96
    assert "tainted" in {p for p, _ in by_kind["tol"]}                      # tolerated template
    assert "tainted" not in {p for k in ("big", "small", "rlx") for p, _ in by_kind[k]}  # untolerated: rejected, memoised empty
    assert {p for p, _ in by_kind["big"]} == {"large"}                      # nothing on 'small' fits: cached-empty, hit again
    assert "small" in {p for p, _ in by_kind["small"]}
    assert all(r > 0 for _, r in by_kind["rlx"])                            # placed after relaxing (no K1 row)
    big = facts["classes"]["big0"]
    assert len({full["assign"][i] for i in big}) >= 2                       # the class opens more than one node


def reach_limit_front(pkg, oracle, prob, facts, full, name):
    names = [it["name"] for it in prob["instanceTypes"]]
    limited = [nn for nn in full["newNodes"] if nn["provisioner"] == 0]
    assert len(limited) >= 2 and any(nn["provisioner"] == 1 for nn in full["newNodes"])
    fronts_ = [front(prob, nn["options"]) for nn in limited]
    assert names.index("lim-16") in limited[0]["options"] and names.index("lim-16") not in limited[1]["options"]
    assert fronts_[0] != fronts_[1]
    # subtractMax: the limit binds once the largest option capacities of the limited nodes exceed it
    cap = sum(max(ea._resources(prob["instanceTypes"][t]["capacity"])["cpu"] for t in nn["options"]) for nn in limited)
    assert cap <= facts["limit_cpu_milli"] < cap + 16000


def fd_visits(prob, full):
    """the fd_* keys every pod's fresh-node attempt visits, in order: (class, template, zone requirement) for each template up
    to the one that opens the pod's node; the first 15 fail on resources (restated: no type of theirs holds the pod)"""
    ne = len(full["existing"])
    provs = sorted(range(len(prob["provisioners"])), key=lambda i: -prob["provisioners"][i].get("weight", 0))
    out = []
    for i in queue_order(prob):
        nn = full["newNodes"][full["assign"][i] - ne]
        cls = prob["pods"][i]["labels"]["app"]
        zone = nn["requirements"][ZONE]
        for v in range(nn["provisioner"] + 1):
            if v < nn["provisioner"]:
                pool = prob["provisioners"][provs[v]]["requirements"][0]["values"][0]
                its = [it for it in prob["instanceTypes"] if {"key": gp.POOL, "operator": "In", "values": [pool]} in it["requirements"]]
                assert its and not any(ea.fits(ea.pod_requests(prob["pods"][i]), ea.allocatable(it)) for it in its)
            out.append((cls, v, zone))
    return out


def reach_fresh_memo(pkg, oracle, prob, facts, full, name):
    visits = fd_visits(prob, full)
    assert len(set(visits)) > gp.K_FRESH_MEMO_SLOTS
    last, between, revisited = {}, [], 0
    for j, key in enumerate(visits):
        if key in last:
            between.append(len(set(visits[last[key] + 1:j]) - {key}))
            revisited += 1
        last[key] = j
    assert revisited >= gp.FD_CLASSES * gp.FD_TEMPLATES and min(between) > gp.K_FRESH_MEMO_SLOTS, (revisited, min(between))
    # the zone pin changes the options: the last template's nodes in different zones keep different type sets
    assert len({(nn["requirements"][ZONE], tuple(nn["options"])) for nn in full["newNodes"]}) == 3
    assert len({tuple(nn["options"]) for nn in full["newNodes"]}) == 3


def reach_fresh_memo_collision(pkg, oracle, prob, facts, full, name):
    """the fd_* keys restated over the encoder's own key numbering and value bits: each spread class visits two keys that
    differ only in the zone value, share one slot (gp.fd_slot) with nothing else written to it in between, and have different
    outcomes"""
    zs = facts["zones"]
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.dims["keys"] == 2 and rs.dims["templates"] == 1
    # key ids and value bits, from the class rows of helper pods appended to the same problem (the class table is in pod
    # order, so the scenario's classes keep their indices): provisioner name = key 0 (In [default] = bit 0), zone = key 1
    # (the dictionary in sorted order); a row's meta word carries the present bits from bit 0
    helpers = [fx_pod(f"h-{i}", {ZONE: z}) for i, z in enumerate(zs)] + [fx_pod("h-pn", {PROVISIONER_NAME: "default"})]
    var = dict(prob, pods=prob["pods"] + helpers)
    vs = pkg.ResidentSolve(pkg.Problem.from_dict(var))
    assert vs.key_info(ZONE) == rs.key_info(ZONE) and vs.key_info(PROVISIONER_NAME) == rs.key_info(PROVISIONER_NAME)
    base = len(prob["pods"])
    for i in range(len(zs)):
        row = vs.class_row(vs.pod_class(base + i))
        assert (int(row[8]), int(row[9]), int(row[24])) == (0, 1 << i, 0b10), i
    row = vs.class_row(vs.pod_class(base + len(zs)))
    assert (int(row[8]), int(row[9]), int(row[24])) == (1, 0, 0b01)
    # every fresh-node attempt of a spread pod, in queue order: its class, zone pin and options (one pod per node)
    visits = []
    for i in queue_order(prob):
        app = prob["pods"][i]["labels"]["app"]
        if not app.startswith("d"):
            continue
        nn = full["newNodes"][full["assign"][i] - len(full["existing"])]
        assert nn["pods"] == [i] or nn["pods"][0] == i  # the spread pod opened this node
        z = zs.index(nn["requirements"][ZONE].split("[", 1)[1].rstrip("]"))
        c = rs.pod_class(i)
        visits.append((c, z, tuple(nn["options"]), gp.fd_slot(c, 0b11, [1, 1 << z])))
    for at in gp.FDC_AT:
        mine = [(j, v) for j, v in enumerate(visits) if v[0] == at]
        assert [v[1] for _, v in mine] == list(range(gp.FDC_ZONES))  # one zone per round, in sorted order
        pairs = [(ja, jb) for ja, a in mine for jb, b in mine if ja < jb and a[3] == b[3]]
        assert pairs, at
        for ja, jb in pairs:
            a, b = visits[ja], visits[jb]
            assert a[1] != b[1] and a[2] != b[2]  # different zone values, different outcomes
            assert not any(v[3] == a[3] for v in visits[ja + 1:jb])  # the first key's entry is still in the slot


def fx_pod(name, selector):
    return {"name": name, "uid": name, "requests": {"cpu": "5m"}, "nodeSelector": dict(selector)}


# ---------------------------------------------------------------- d. cursor
def reach_cursor(pkg, oracle, prob, facts, full, name):
    ex = [e["node"] for e in full["existing"]]
    at = lambda i: ex[full["assign"][i]]
    spread = facts["classes"]["spread"]
    seq = [at(i) for i in sorted(spread, key=queue_order(prob).index)]
    e4 = facts["spread_old_node"]
    assert seq[:3] == [5, 6, e4], seq  # e4 refused for now (zone skew) before the acceptor e5, then taken
    # e0-e3 refuse the class for good: pod slots full, untolerated taint, its host port taken, too little cpu
    nodes = prob["nodes"]
    assert len(nodes[0]["pods"]) == int(nodes[0]["allocatable"]["pods"]) and nodes[1]["taints"]
    assert any(p.get("ports") for p in nodes[2]["pods"]) and ea.quantity_milli(nodes[3]["allocatable"]["cpu"]) < 1000
    # the instance-type class is refused by e0-e6 for its type and accepted by e7
    assert {at(i) for i in facts["classes"]["itype"]} == {7}
    # the plain class's first run ends in the middle of the node list; its later pods continue from there
    order = [i for i in queue_order(prob) if i in set(facts["classes"]["plain"])]
    first_run = [at(i) for i in order[:20]]
    assert 0 < max(first_run) < len(nodes) - 1 and max(at(i) for i in order[20:]) > max(first_run)


# ---------------------------------------------------------------- e. tables
def reach_alloc(pkg, oracle, prob, facts, full, name):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    d = rs.dims
    assert d["resources"] == 4 and d["types"] == facts["n_types"]
    assert gp.ALLOC_SMEM_LIMIT == smem_limit_from_source() == 39424
    assert gp.alloc_in_smem(4, facts["n_types"]) == (facts["n_types"] <= 1232)
    it_pods = facts["classes"]["itype"]
    assert all(full["assign"][i] >= 0 for i in it_pods)


ROOT = Path(__file__).resolve().parent.parent
_CTYPES = {"unsigned long long": 8, "long long": 8, "unsigned short": 2, "unsigned": 4, "int": 4}


def smem_limit_from_source():
    """run_pack's shared-memory budget for the allocatable table, computed from the declarations themselves: HotSmem's
    members (pack_kernel.cuh, natural alignment), kRunArrayBytes and the 227 KiB / 14 KiB terms of ksched.cu"""
    csrc = ROOT / "karpenter-core_b200" / "csrc"
    pk = (csrc / "pack_kernel.cuh").read_text()
    const = {m[1]: int(m[2]) for m in re.finditer(r"constexpr int (k\w+) = (\d+);", pk)}
    body = re.search(r"struct HotSmem \{(.*?)\n\};", pk, re.S).group(1)
    size = 0
    for m in re.finditer(r"^\s*(unsigned long long|long long|unsigned short|unsigned|int)\s+\w+((?:\[\w+\])+);", body, re.M):
        n = 1
        for d in re.findall(r"\[(\w+)\]", m[2]):
            n *= const[d] if d in const else int(d)
        w = _CTYPES[m[1]]
        size = -(-size // w) * w + w * n
    size = -(-size // 8) * 8
    assert "constexpr size_t kRunArrayBytes = (size_t)kTopoCap * (kRunMask * 4 + kRunHost * 2) + (size_t)kActCap * 4;" in pk
    run = const["kTopoCap"] * (const["kRunMask"] * 4 + const["kRunHost"] * 2) + const["kActCap"] * 4
    ks = (csrc / "ksched.cu").read_text()
    assert "static_smem = (size_t)(14 << 10);" in ks
    assert "smem_left = (size_t)(227 << 10) - sizeof(HotSmem) - kRunArrayBytes - static_smem;" in ks
    assert "s.alloc_in_smem = alloc_bytes <= smem_left ? 1 : 0;" in ks
    assert size == gp.HOT_SMEM_BYTES and run == gp.RUN_ARRAY_BYTES
    return (227 << 10) - size - run - (14 << 10)


REACH = {
    **{n: reach_exclusions for n in gp.SCENARIOS if n.startswith("excl")},
    "excl_wide": reach_excl_wide,
    **{n: reach_fronts for n in gp.SCENARIOS if n.startswith("front_")},
    "front_warps": reach_front_warps,
    "class_memo": reach_class_memo,
    "limit_front": reach_limit_front,
    "fresh_memo": reach_fresh_memo,
    "fresh_memo_collision": reach_fresh_memo_collision,
    "cursor": reach_cursor,
    "alloc_1232": reach_alloc,
    "alloc_1233": reach_alloc,
}


@pytest.mark.parametrize("name", IDS)
def test_scenario_reaches_its_mechanism(pkg, oracle, name):
    prob, facts = gp.build(name)
    full = _solve(pkg, oracle, prob)
    REACH[name](pkg, oracle, prob, facts, full, name)


@pytest.mark.parametrize("name", IDS)
def test_every_option_holds_its_node(pkg, oracle, name):
    """independently of the oracle's Fits: every option of every new node holds the node's final requests"""
    prob, _ = gp.build(name)
    full = _solve(pkg, oracle, prob)
    ds = ea.daemon_overhead(prob)
    for k, nn in enumerate(full["newNodes"]):
        pods = [prob["pods"][i] for i in nn["pods"]]
        need = ea._merge(ea.requests_for_pods(pods), ds) if prob.get("daemonSetPods") else ea.requests_for_pods(pods)
        assert {r: v for r, v in need.items() if v} == {r: v for r, v in nn["requests"].items() if v}, k
        assert nn["options"] and all(ea.fits(need, _alloc(prob, t)) for t in nn["options"]), k


@pytest.mark.parametrize("name", IDS)
def test_fast_mode_equals_literal(pkg, oracle, name):
    problem = pkg.Problem.from_dict(gp.build(name)[0])
    out = []
    for fast in (0, 1):
        oracle.lib.oracle_set_fast(fast)
        try:
            res = pkg.Result()
            assert oracle.solve(problem, res) == 0, res.error
        finally:
            oracle.lib.oracle_set_fast(0)
        out.append(res)
    assert out[0].to_dict() == out[1].to_dict()
    assert out[0].digest() == out[1].digest()
