"""Scenarios for the pack kernel's generic step (csrc/pack_kernel.cuh: generic_step), each built to reach one of its
device-only mechanisms: the exclusion list of in-flight winners that fail their full check, the Pareto-front resource test
and node closure, the fresh-node outcome memos (fc_* per class and template, fd_* keyed by the node's requirement set), the
existing-node cursor and the block-size and table edges of the cooperative instance-type check.

Every scenario reaches the generic step: with nodes_visited counted the pack kernel runs no class run or existing-node run
at all (ksched.cu: fast_allowed needs count_visited off), and the GPU test also runs each one under KSCHED_NO_CLASSRUN.
Pods are written with rp.Runs: the queue orders them by cpu, then memory, then creationTimestamp, then UID.
tests/test_generic_step_reach.py shows on the oracle's result that each scenario gets where it is built to go."""
import copy

import fixtures as fx
import run_problems as rp
from fixtures import ARCH, HOSTNAME, ZONE

# ---------------------------------------------------------------- device constants, restated
K_MAX_EXCL = 16          # pack_kernel.cuh kMaxExcl: in-flight winners one step excludes before every thread checks in full
K_ACT_CAP = 1280         # pack_kernel.cuh kActCap: open nodes whose hot state is in shared memory (the rest: ov_*)
K_HOT_RES = 4            # pack_kernel.cuh kHotRes: resources of the hot request and front vectors
K_FRESH_MEMO_SLOTS = 8192  # ksched.cu kFreshMemoSlots: slots of the topology memo PackState::fd_*
# ksched.cu run_pack: alloc_in_smem = n_res * n_types * 8 <= 227 KiB - sizeof(HotSmem) - kRunArrayBytes - 14 KiB, with
#   sizeof(HotSmem) = kActCap * (8 key + 3 * kHotRes * 8 q / bound / bound2 + 4 node + 2 flags + 4 absorbed + 4 rejected + 8 nn_last)
#   kRunArrayBytes  = kTopoCap * (kRunMask * 4 + kRunHost * 2) + kActCap * 4, kTopoCap = 768, kRunMask = 2, kRunHost = 4
HOT_SMEM_BYTES = K_ACT_CAP * (8 + 3 * K_HOT_RES * 8 + 4 + 2 + 4 + 4 + 8)
RUN_ARRAY_BYTES = 768 * (2 * 4 + 4 * 2) + K_ACT_CAP * 4
ALLOC_SMEM_LIMIT = (227 << 10) - HOT_SMEM_BYTES - RUN_ARRAY_BYTES - (14 << 10)


def alloc_in_smem(n_res, n_types):
    return n_res * n_types * 8 <= ALLOC_SMEM_LIMIT


ZS = rp.zone_names(3, "gs-west")
POOL = "example.com/pool"


def itype(name, cpu, mem_gi, price, arch="amd64", zones=ZS, extra=None, labels=None, pods=110):
    """one instance type offered spot (cheaper) and on-demand in `zones`; columns are ordered by price (host/encoder.cc)"""
    res = {"cpu": str(cpu), "memory": f"{mem_gi}Gi", "pods": str(pods), **(extra or {})}
    offers = [{"capacityType": ct, "zone": z, "price": round(price * (0.6 if ct == "spot" else 1.0), 6), "available": True}
              for z in zones for ct in ("spot", "on-demand")]
    it = fx.instance_type(name, res, offerings=offers, arch=arch, oses=("linux",))
    for k, v in (labels or {}).items():
        it["requirements"].append({"key": k, "operator": "In", "values": [v]})
    return it


def _problem(runs, its, provs=None, **kw):
    prob = fx.problem(runs.pods, instance_types=its, provisioners=provs or [rp.unlimited()], **kw)
    prob["wellKnownLabels"] = list(prob["wellKnownLabels"]) + [POOL]
    return prob


ARM = {ARCH: "arm64"}
AMD = {ARCH: "amd64"}


# ---------------------------------------------------------------- a. in-flight exclusions
# Q (3 cpu, 33Gi, no arch requirement): one pod per node (two exceed every type's memory), options of both arches.
# A (1.5 cpu, anti-affinity to Q): opens the node that later accepts. P_i (1 cpu, arch arm64): on a Q node the quick fit passes
# through the amd64 types, the requirements are compatible, and no arm64 type (3.9 cpu allocatable) holds 4 cpu: the node wins
# the argmin, fails the cooperative check and is excluded. Each P class's `rejected` memo hides the Q nodes from its own later
# pods, so several classes each meet all of them.
Q_REQ = {"cpu": "3", "memory": "33Gi"}
A_REQ = {"cpu": "1500m", "memory": "1Gi"}  # before P in the queue, and A + P fits an arm64 type


def _excl_catalog(wide=False):
    if not wide:
        return [itype("arm-a", 4, 64, 0.10, "arm64"), itype("arm-b", 4, 96, 0.12, "arm64"),
                itype("amd-a", 16, 40, 0.50), itype("amd-b", 32, 48, 0.80)]
    # 1 100 types (W32 = 35): 1 030 arm64 types of one allocatable vector (duplicates) in words 0-32, then the amd64 ones,
    # the most expensive, at column 1 030 and on: the types P's arch requirement removes sit in words >= 32
    its = [itype(f"arm-{i:04d}", 4, 64, round(0.10 + i * 1e-4, 6), "arm64") for i in range(1030)]
    return its + [itype(f"amd-{i:02d}", 16, 40, round(0.50 + i * 1e-3, 6)) for i in range(70)]


def exclusions(n_q, n_p=3, spread=False, ext=False, wide=False, accept=True, q_anti=False):
    r = rp.Runs(f"x{n_q}")
    q_spec = {"labels": {"app": "q"}}
    if q_anti:  # a topology refusal is cheap for the literal oracle, which would otherwise try every type of every Q node
        q_spec["podAntiAffinity"] = {"required": [fx.affinity_term(HOSTNAME, {"app": "q"})]}
    if spread:
        q_spec["nodeSelector"] = dict(AMD)  # Q nodes are amd64 only: the full requirement check refuses P (win_fail)
    r.run("q", n_q, Q_REQ, **q_spec)
    if accept:
        r.run("a", 1, A_REQ, labels={"app": "a"}, podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "q"})]})
    for i in range(n_p):
        req = {"cpu": "1", "memory": f"{1024 - 64 * i}Mi"}
        spec = {"labels": {"app": f"p{i}"}, "nodeSelector": dict(ARM)}
        if spread:
            spec = dict(rp.zone_spread(f"p{i}"), nodeSelector=dict(ARM))
        if ext:  # no arch requirement: the ext fit of narrow_word removes every type that could hold the requests
            req = dict(req, **{EXT: "1"})
            spec = {"labels": {"app": f"p{i}"}}
        r.run(f"p{i}", 2, req, **spec)
    its = _excl_catalog(wide)
    kw = {}
    if ext:
        its = _ext_catalog()
        kw["daemonSetPods"] = [fx.pod({"cpu": "10m", **{k: "1" for k in DS_RES}}, name="ds-agent", isDaemonSet=True)]
    facts = {"classes": r.classes, "q": n_q, "p": [f"p{i}" for i in range(n_p)], "spread": spread, "ext": ext}
    return _problem(r, its, **kw), facts


# ext resources: resources beyond the KSCHED_MAX_RES = 8 row slots (include/ksched.h). A daemonset that requests five
# resources fills the row slots (cpu, memory, pods and its five); the pods' accelerator is an ext resource.
DS_RES = tuple(f"example.com/slot{i}" for i in range(5))
EXT = "example.com/accel"


def _ext_catalog():
    slots = {k: "8" for k in DS_RES}
    # arm-x holds the accelerator but not Q + P's cpu; amd-a holds the cpu and has no accelerator
    return [itype("arm-x", 4, 64, 0.10, "arm64", extra=dict(slots, **{EXT: "2"})), itype("arm-b", 4, 96, 0.12, "arm64", extra=slots),
            itype("amd-a", 16, 40, 0.50, extra=slots)]


# ---------------------------------------------------------------- b. Pareto-front shapes and node closure
# (cpu, memory GiB) of each shape's types, cheapest first; X (opener) pods open nodes whose options are all of them, small
# pods of several shapes fill them, and the last class's requests (min_req) decide when node_closed closes a node.
FRONTS = {
    "one": [(4, 16), (8, 32), (16, 64)],                               # (16, 64) dominates
    "two": [(2, 8), (16, 16), (4, 64), (8, 12)],                         # cpu-heavy and memory-heavy families
    "three": [(16, 16), (4, 64), (10, 40), (2, 2)],                      # three incomparable families: necessary test only
    "tie": [(16, 32), (16, 64), (8, 16)],                                # equal cpu: perm_desc's first cpu type is not dominant
    "dup": [(8, 32), (8, 32), (8, 32), (4, 64), (4, 64), (2, 4)],        # duplicate allocatable vectors
    "wide": [(16, 16), (4, 64), (8, 32)],                                # 7 row resources (n_res > kHotRes)
}
FRONT_PODS = [  # (cpu milli, memory MiB, count) in queue order (FFD: cpu, then memory, descending)
    (3500, 2048, 3), (3000, 30000, 3), (2500, 9000, 4), (1500, 1024, 6), (1200, 40000, 2), (700, 6000, 8), (400, 500, 10),
    (300, 14000, 4), (250, 256, 12)]


def fronts(shape):
    wide = shape == "wide"
    extra = {f"example.com/w{i}": "4" for i in range(4)} if wide else None
    its = [itype(f"{shape}-{i}", cpu, mem, 0.05 * (i + 1), extra=extra) for i, (cpu, mem) in enumerate(FRONTS[shape])]
    r = rp.Runs(f"f{shape}")
    for j, (cpu, mem, k) in enumerate(FRONT_PODS):
        req = {"cpu": f"{cpu}m", "memory": f"{mem}Mi"}
        if wide:
            req.update({f"example.com/w{i}": "1" for i in range(j % 4 + 1)})
        r.run(f"s{j}", k, req, labels={"app": f"s{j}"})
    return _problem(r, its), {"classes": r.classes, "shape": shape}


def front_across_warps():
    """1 100 types: 1 097 dominated fillers, A (32 cpu, 32Gi) and B (8 cpu, 128Gi) among the first columns and C (20 cpu, 80Gi)
    the most expensive, in option word 34: at 128 threads warp 0 reads words 0-31 only, where A and B cover every option. X
    opens a node with all three families; Y fits that node only through C."""
    its = [itype("big-a", 32, 32, 0.01), itype("big-b", 8, 128, 0.011)]
    its += [itype(f"fill-{i:04d}", 1, 1, round(0.02 + i * 1e-4, 6)) for i in range(1097)]
    its.append(itype("big-c", 20, 80, 5.0))
    r = rp.Runs("fw")
    r.run("x", 1, {"cpu": "7", "memory": "1Gi"}, labels={"app": "x"})
    r.run("y", 2, {"cpu": "6", "memory": "60Gi"}, labels={"app": "y"})
    return _problem(r, its), {"classes": r.classes}


# ---------------------------------------------------------------- c. fresh-node memos
def class_memo():
    """fc_*: 24 classes x 4 templates. Template 0 (weight 40) is tainted and only 'tol' classes tolerate it; template 1 offers
    small types only, where the large classes fit nowhere (cached-empty, hit again by their later pods); 'rlx' classes
    prefer a zone no type is offered in and are placed only after relaxing (no K1 row: the dynamic path with the memo)."""
    small = [itype(f"sm-{i}", 2, 4, 0.02 + 0.01 * i, labels={POOL: "small"}) for i in range(3)]
    big = [itype(f"lg-{i}", 8 * (i + 1), 16 * (i + 1), 0.2 * (i + 1), labels={POOL: "large"}) for i in range(3)]
    taint = {"key": "dedicated", "value": "x", "effect": "NoSchedule"}
    provs = [rp.unlimited("tainted", weight=40, taints=[taint]),
             rp.unlimited("small", weight=30, requirements=[{"key": POOL, "operator": "In", "values": ["small"]}]),
             rp.unlimited("large", weight=20, requirements=[{"key": POOL, "operator": "In", "values": ["large"]}]),
             rp.unlimited("any", weight=10)]
    r = rp.Runs("fc")
    for i in range(24):
        kind = ("big", "small", "tol", "rlx")[i % 4]
        cpu = {"big": 5000 - 40 * i, "small": 1500 - 20 * i, "tol": 1200 - 10 * i, "rlx": 3000 - 30 * i}[kind]
        spec = {"labels": {"app": f"c{i}"}}
        if kind == "tol":
            spec["tolerations"] = [{"key": "dedicated", "operator": "Exists"}]
        if kind == "rlx":
            spec["nodeAffinity"] = {"preferred": [{"weight": 10, "terms": [{"key": ZONE, "operator": "In", "values": ["nowhere"]}]}]}
        r.run(f"{kind}{i}", 5, {"cpu": f"{cpu}m", "memory": f"{1 + i % 3}Gi"}, **spec)
    return _problem(r, small + big, provs), {"classes": r.classes}


def limit_front():
    """the K1-row path's front memo next to a provisioner whose cpu limit (24) binds in the middle of the batch: the first
    node keeps the 16-cpu type (front: that type), the limit then cuts it from the next nodes (front: the 8-cpu type)"""
    its = [itype("lim-4", 4, 16, 0.05), itype("lim-8", 8, 32, 0.1), itype("lim-16", 16, 64, 0.2)]
    provs = [fx.provisioner("limited", weight=20, limits={"cpu": "24"}), rp.unlimited("spill", weight=10)]
    r = rp.Runs("lf")
    r.run("k", 14, {"cpu": "3500m", "memory": "1Gi"}, labels={"app": "k"})
    r.run("m", 10, {"cpu": "1200m", "memory": "2Gi"}, labels={"app": "m"})
    return _problem(r, its, provs), {"classes": r.classes, "limit_cpu_milli": 24000}


FD_CLASSES = 180
FD_ROUNDS = 4
FD_TEMPLATES = 16


def fresh_memo():
    """fd_*: 180 zone-spread deployments of 4 pods with equal requests, pod k of every class before pod k + 1 of any
    (timestamps); 16 weighted provisioners, the first 15 offering 1-cpu types only (each attempt writes an empty entry),
    the last one types offered in different pairs of zones (the zone pin changes the option set). Requests above half the
    largest type: every pod opens a node. Rounds 1 and 4 of a class meet the same zone counts, so the same keys, with more
    than kFreshMemoSlots other keys in between. 720 pods: the only large scenario of the corpus."""
    its = []
    for v in range(FD_TEMPLATES - 1):
        its.append(itype(f"tiny-{v:02d}", 1, 2, 0.01 + 0.001 * v, labels={POOL: f"p{v:02d}"}))
    for j, zs in enumerate(([ZS[0], ZS[1]], [ZS[1], ZS[2]], [ZS[0], ZS[2]], ZS)):
        its.append(itype(f"wide-{j}", 16, 64, 0.3 + 0.05 * j, zones=zs, labels={POOL: f"p{FD_TEMPLATES - 1:02d}"}))
    provs = [rp.unlimited(f"pool-{v:02d}", weight=100 - v, requirements=[{"key": POOL, "operator": "In", "values": [f"p{v:02d}"]}])
             for v in range(FD_TEMPLATES)]
    r = rp.Runs("fd")
    for k in range(FD_ROUNDS):
        for c in range(FD_CLASSES):
            r._pod(f"d{c:03d}", {"cpu": "9", "memory": "2Gi"}, 1 + k * FD_CLASSES + c, rp.zone_spread(f"d{c:03d}"))
    return _problem(r, its, provs), {"classes": r.classes}


# The fd_* slot of a fresh-node attempt, restated from pack_kernel.cuh (generic_step, step 3): fc = class * V + template,
# meta = the template's requirement meta (low 32 bits) with the touched keys' final present / complement bits, vals = the
# final value mask of every mask key (touched keys) or the template's (the rest).
def fd_slot(fc, meta, vals):
    m64 = (1 << 64) - 1
    h = (((fc + 1) * 0x9E3779B97F4A7C15) & m64) ^ meta
    for v in vals:
        h = ((h ^ v) * 0xBF58476D1CE4E5B9) & m64
        h ^= h >> 29
    return (h >> 13) & (K_FRESH_MEMO_SLOTS - 1)


FDC_ZONES = 8
FDC_AT = (115, 144)  # class indices whose zone keys share a slot (fd_slot): zones 1 and 7, and zones 2 and 5


def fresh_memo_collision():
    """two keys of one (class, template) that differ only in the zone pin and share an fd_* slot, with different outcomes.
    One provisioner without requirements: the mask keys are the provisioner name (key 0, the template's own In [default])
    and the zone (key 1, pinned by the spread), so a fresh node's key is (class, meta 0b11, [1, 1 << zone]). Two 8-pod
    zone-spread deployments sit at class indices FDC_AT (plain one-pod filler classes before them; the class table is in
    pod order) and visit the 8 zones one per round; instance type j < 3 is offered in the zones whose index has bit j set,
    type 3 everywhere, so every zone pin keeps a different option set. The second key of each colliding pair finds the
    first one's entry in its slot: only the value compare tells them apart."""
    zs = rp.zone_names(FDC_ZONES, "fc-north")
    its = [itype(f"zb-{j}", 16, 64, 0.3 + 0.05 * j, zones=[z for i, z in enumerate(zs) if j == 3 or (i >> j) & 1]) for j in range(4)]
    r = rp.Runs("fdc")
    n = 0
    for at in FDC_AT:
        while n < at:
            r._pod(f"f{n:03d}", {"cpu": "10m", "memory": "16Mi"}, 0, {"labels": {"app": f"f{n:03d}"}})
            n += 1
        for k in range(FDC_ZONES):
            r._pod(f"d{at}", {"cpu": "9", "memory": "2Gi"}, 1 + k, rp.zone_spread(f"d{at}"))
        n += 1
    return _problem(r, its), {"classes": r.classes, "zones": zs}


# ---------------------------------------------------------------- d. existing-node cursor
def cursor():
    """existing nodes in caller order: e0 closed (its pod slots are taken), e1 tainted, e2 with the class's host port taken,
    e3 too small, then e4-e6 in zones 0-2 (e4 already holds a pod of the spread class, so its zone's skew refuses the next
    two pods for now), e7 of an instance type the 'itype' class does not name. 'spread' takes e5, e6, then e4 again once
    the other zones have caught up. 'plain' runs before and after 'other' (same requests, later timestamp): with
    nodes_visited off the existing-node run places both of its segments, the first one ending in the middle of the node
    list (its cursor, last_used); with nodes_visited on the generic step places them from the cursor its own steps keep.
    No pod of 'plain' reaches the generic step after an existing-node run of its class: that hand-off is not built here."""
    its = [itype("ex-8", 8, 32, 0.1), itype("ex-16", 16, 64, 0.2)]
    nodes = []
    taint = [{"key": "dedicated", "value": "x", "effect": "NoSchedule"}]
    spread_spec = rp.zone_spread("spread")
    spread_spec["ports"] = [{"hostPort": 9000, "protocol": "TCP"}]

    def node(i, zone, alloc_cpu="7900m", pods=None, **kw):
        return fx.state_node(f"e{i}", "ex-8", zone=zone, allocatable={"cpu": alloc_cpu, "memory": "31Gi", "pods": "10"}, pods_=pods or [], **kw)

    nodes.append(node(0, ZS[0], pods=[fx.pod({"cpu": "10m"}, name=f"full-{j}", uid=f"full-{j}", nodeName="e0") for j in range(10)]))
    nodes.append(node(1, ZS[1], taints=taint))
    nodes.append(node(2, ZS[2], pods=[fx.pod({"cpu": "10m"}, name="port-user", uid="port-user", nodeName="e2", labels={"app": "agent"},
                                             ports=[{"hostPort": 9000, "protocol": "TCP"}])]))
    nodes.append(node(3, ZS[0], alloc_cpu="300m"))
    nodes.append(node(4, ZS[0], pods=[fx.pod({"cpu": "500m", "memory": "512Mi"}, name="spread-old", uid="spread-old", nodeName="e4",
                                             labels={"app": "spread"})]))
    nodes.append(node(5, ZS[1]))
    nodes.append(node(6, ZS[2]))
    nodes.append(fx.state_node("e7", "ex-16", zone=ZS[1], allocatable={"cpu": "15900m", "memory": "63Gi", "pods": "10"}))
    for i in range(8, 14):
        nodes.append(node(i, ZS[i % 3]))
    r = rp.Runs("cur")
    r.run("spread", 4, {"cpu": "1", "memory": "1Gi"}, **copy.deepcopy(spread_spec))
    r.run("itype", 3, {"cpu": "900m", "memory": "1Gi"}, labels={"app": "itype"},
          nodeAffinity={"required": [[{"key": fx.INSTANCE_TYPE, "operator": "In", "values": ["ex-16"]}]]})
    r.run("plain", 20, {"cpu": "700m", "memory": "1Gi"}, labels={"app": "plain"})
    r.run("other", 4, {"cpu": "700m", "memory": "1Gi"}, **rp.zone_spread("other"))
    r.run("plain", 30, {"cpu": "700m", "memory": "1Gi"}, labels={"app": "plain"})
    return _problem(r, its, nodes=nodes), {"classes": r.classes, "spread_old_node": 4}


# ---------------------------------------------------------------- e. block-size and table edges
def alloc_edge(n_types):
    """4 row resources (cpu, memory, pods and one the daemonset requests) x n_types: the sorted allocatable table is staged
    in shared memory up to 1 232 types and read from global memory from 1 233 on (alloc_in_smem)"""
    its = [itype(f"al-{i:04d}", 1 + i % 16, 2 * (1 + i % 23), round(0.01 + i * 1e-4, 6), extra={"example.com/slot": "4"}) for i in range(n_types)]
    ds = [fx.pod({"cpu": "10m", "example.com/slot": "1"}, name="ds-agent", isDaemonSet=True)]
    r = rp.Runs(f"al{n_types}")
    for j, (cpu, mem, k) in enumerate(FRONT_PODS):
        r.run(f"s{j}", k, {"cpu": f"{cpu}m", "memory": f"{mem}Mi"}, labels={"app": f"s{j}"})
    r.run("itype", 3, {"cpu": "2", "memory": "3Gi"}, labels={"app": "itype"},
          nodeAffinity={"required": [[{"key": fx.INSTANCE_TYPE, "operator": "In", "values": [f"al-{i:04d}" for i in range(0, n_types, 7)]}]]})
    return _problem(r, its, daemonSetPods=ds), {"classes": r.classes, "n_types": n_types}


# ---------------------------------------------------------------- the corpus
SCENARIOS = {
    "excl15": lambda: exclusions(15),
    "excl16": lambda: exclusions(16),
    "excl17": lambda: exclusions(17),
    "excl40": lambda: exclusions(40),
    "excl_spread": lambda: exclusions(20, n_p=2, spread=True),
    "excl_ext": lambda: exclusions(20, ext=True),
    "excl_overflow": lambda: exclusions(K_ACT_CAP + 30, n_p=2, q_anti=True),
    "excl_wide": lambda: exclusions(15, wide=True),  # < kMaxExcl: the accepting winner still takes the cooperative check
    **{f"front_{k}": (lambda k=k: fronts(k)) for k in FRONTS},
    "front_warps": front_across_warps,
    "class_memo": class_memo,
    "limit_front": limit_front,
    "fresh_memo": fresh_memo,
    "fresh_memo_collision": fresh_memo_collision,
    "cursor": cursor,
    "alloc_1232": lambda: alloc_edge(1232),
    "alloc_1233": lambda: alloc_edge(1233),
}
CORPUS = [(name, 0) for name in SCENARIOS]


def build(name, seed=0):
    """(problem dict, facts): facts names the classes (pod indices per class) the scenario's predicate talks about"""
    return SCENARIOS[name]()
