"""Scenarios for K1's class pass (csrc/feasibility_kernel.cuh: class_feasibility_kernel) and its stream to pod rows
(feasibility_kernel), sized from the device's SM count so that each one reaches the path it names:

 * job_chunks: single-pod Jobs (every pod its own class through its unique labels, rows identical apart from the class
   index), about 2.5 class rows per warp, with near misses - classes that differ from their predecessor in exactly one row
   word the kernel's cmp_mask covers - at the first row of a chunk, right after a computed row and right after a
   cache-served one; a run that nothing fits (kNoBest) and a class with a preference, whose relaxed class follows it;
 * whole_batches: more than 2 x 16 class rows per warp on a narrow catalog, so that whole 16-row batches repeat the cached
   row; near misses at offsets 0, 1, 15, 16, 31, 32, 47 and 49 of a chunk (31 and 47: the last row of a voted batch; 32:
   right after a full-batch repeat) and a partial last batch;
 * wide_batches: whole batches on a catalog of two column words per lane, so that the cache's layout matters;
 * layout: the consecutive-row cache at V * wpl = 16 (wpl = 2 and 4 column words per lane) and just above, the sorted
   allocatable arrays at exactly 128 KiB and one type above, the column tables on both sides of their 160 KiB budget;
 * best_edges: best_column's key at equal double prices, at prices one float32 apart only as doubles, at price 0, and on
   instance types without an available offering;
 * stream: more than 2048 pod rows per SM with few classes and a pod count that is not a multiple of 32.

Every scenario keeps a daemonset (K1 adds the template's daemon overhead) and has no existing nodes and no limits (K1 reads
neither). A scenario is a dict: name, prob (problem document), shapes (pod specs without identity), pod_shape (shape of each
pod), class_shape (shape of each class in class-table order; a relaxed class has the shape of its pod with the preference
dropped), near (class index -> near-miss kind) and the launch facts it is built for."""
import copy

import fixtures as fx

ZONE, CT, INSTANCE_TYPE = fx.ZONE, fx.CAPACITY_TYPE, fx.INSTANCE_TYPE
TAINT = {"key": "dedicated", "value": "batch", "effect": "NoSchedule"}

# ---------------------------------------------------------------- K1's launch, restated from csrc/ksched.cu
# run_class_feasibility: blocks = max(1, min(2 * n_sm, ceil(NC / 16))) of kK1Threads = 512 threads (16 warps); the kernel
# gives each warp the contiguous chunk ceil(NC / warps) of class rows and reads them kBatch = 16 at a time.
K1_WARPS_PER_BLOCK = 16
K1_BATCH = 16
K1_CACHE_WORDS = 16       # kK1Cache: the cache holds V * wpl <= 16 words per lane
ALLOC_SMEM_BYTES = 128 << 10
TABLE_SMEM_BYTES = 160 << 10
TEMPLATE_BYTES = 280      # sizeof(ksched_template)
KEYINFO_BYTES = 32        # sizeof(ksched_keyinfo)
MAX_KEYS = 16


def k1_grid(n_classes, n_sm):
    """(blocks, warps, chunk) of the class pass over n_classes rows on an n_sm-SM device"""
    blocks = max(1, min(2 * n_sm, -(-n_classes // K1_WARPS_PER_BLOCK)))
    warps = blocks * K1_WARPS_PER_BLOCK
    return blocks, warps, -(-n_classes // warps)


def device_sm_count(ordinal=0):
    """streaming multiprocessors of CUDA device `ordinal`, from the driver API. (torch.cuda would do, but importing torch
    after libksched.so has loaded the system NCCL fails to resolve torch's newer NCCL symbols.)"""
    import ctypes
    cu = ctypes.CDLL("libcuda.so.1")
    dev, n = ctypes.c_int(), ctypes.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), ordinal) == 0
    assert cu.cuDeviceGetAttribute(ctypes.byref(n), 16, dev) == 0  # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return n.value


def max_warps(n_sm):
    return 2 * n_sm * K1_WARPS_PER_BLOCK


def cmp_words(row, ext_present):
    """the parts of a class row the kernel compares with its predecessor: words 0-25, the low halves of 28 and 29, and
    word 31 (the class index) when the problem has ext resources"""
    out = [int(row[w]) for w in range(26)] + [int(row[28]) & 0xFFFFFFFF, int(row[29]) & 0xFFFFFFFF]
    return tuple(out + [int(row[31])]) if ext_present else tuple(out)


def paths(keys, n_sm, cacheable=True):
    """what class_feasibility_kernel does with each class row, given each row's comparison key (cmp_words): 'compute',
    'row' (copied from the cache after the per-row vote) or 'batch' (a whole 16-row batch voted equal to the cached row)"""
    nc = len(keys)
    _, warps, chunk = k1_grid(nc, n_sm)
    out = [None] * nc
    for w in range(warps):
        j0, j1 = w * chunk, min(nc, (w + 1) * chunk)
        prev = None
        for jb in range(j0, j1, K1_BATCH):
            je = min(j1, jb + K1_BATCH)
            if prev is not None and cacheable and all(keys[j] == prev for j in range(jb, je)):
                out[jb:je] = ["batch"] * (je - jb)
                continue
            for j in range(jb, je):
                if prev is not None and cacheable and keys[j] == prev:
                    out[j] = "row"
                else:
                    out[j] = "compute"
                    prev = keys[j]
    return out


def smem_plan(n_res, n_types, n_templates, n_keys):
    """alloc_in_smem, and (lower, upper) bounds of the column-table staging decision: the table rows are the valset rows
    (1 .. 64 per key), 2 per key, the offering rows (1 .. 64), anyoffer and one per template"""
    W32 = 2 * max(1, -(-n_types // 64))
    alloc = n_res * n_types * 8
    alloc_in = alloc <= ALLOC_SMEM_BYTES
    base = TEMPLATE_BYTES * n_templates + KEYINFO_BYTES * MAX_KEYS + (alloc if alloc_in else 0) + 2 * MAX_KEYS * 64 + 2 * 64 + 8 * 128
    lo = base + (1 + 2 * n_keys + 1 + 1 + n_templates) * W32 * 4
    hi = base + (64 * n_keys + 2 * n_keys + 64 + 1 + n_templates) * W32 * 4
    return alloc_in, (hi <= TABLE_SMEM_BYTES, lo <= TABLE_SMEM_BYTES)


# ---------------------------------------------------------------- catalogs
def itype(name, cpu_m, price, size="small", tier="t0", grp=None, extra=None, available=True, zones=("test-zone-1", "test-zone-2")):
    cap = {"cpu": f"{cpu_m}m", "memory": "64Gi", "pods": "1000"}
    cap.update(extra or {})
    offers = [{"capacityType": ct, "zone": z, "price": price, "available": available} for ct in ("spot", "on-demand") for z in zones]
    # the zone and capacity-type requirements name every offering, available or not: a type without an available offering
    # is then turned away by the offering check alone, not by its requirements
    reqs = [{"key": INSTANCE_TYPE, "operator": "In", "values": [name]},
            {"key": ZONE, "operator": "In", "values": sorted({o["zone"] for o in offers})},
            {"key": CT, "operator": "In", "values": sorted({o["capacityType"] for o in offers})},
            {"key": "size", "operator": "In", "values": [size]},
            {"key": "tier", "operator": "In", "values": [tier]}]
    if grp is not None:
        reqs.append({"key": "grp", "operator": "In", "values": [grp]})
    return {"name": name, "requirements": reqs, "offerings": offers, "capacity": cap,
            "overhead": {"kubeReserved": {"cpu": "100m", "memory": "10Mi"}}}


def catalog(n_types, extra=None):
    """n_types instance types: cpu 700m + 100m * ((i - 1) % 40) (type 1, of tier t1, is the smallest) except type 40k + 2,
    of 64 cores (so that a node holds about 100 pods of a Job); three tiers, every fourth one `size: large`, type 5k + 4
    offered in zone 3 only (zone-1 preferences remove it). Prices rise with cpu, ties broken by input order."""
    out = []
    for i in range(n_types):
        z = ("test-zone-3",) if i % 5 == 4 else ("test-zone-1", "test-zone-2")
        cpu = 64000 if i % 40 == 2 else 700 + 100 * ((i - 1) % 40)
        out.append(itype(f"it-{i:04d}", cpu, round(0.01 * (1 + (i - 1) % 40), 4), "large" if i % 4 == 3 else "small",
                         f"t{i % 3}", extra=extra, zones=z))
    return out


def templates(n, taint_last=False):
    """n provisioners in weight order; template v admits the tiers other than t(v % 3) (a template-only key, folded into
    membership), so neighbouring templates have different columns"""
    out = []
    for v in range(n):
        pr = {"name": f"pool-{v:02d}", "weight": 100 - v, "requirements": [{"key": "tier", "operator": "NotIn", "values": [f"t{v % 3}"]}]}
        if taint_last and v == n - 1:
            pr["taints"] = [dict(TAINT)]
        out.append(pr)
    return out


def daemonset(extra=None):
    req = {"cpu": "100m", "memory": "64Mi"}
    req.update(extra or {})
    return [fx.pod(req, name="ds-node-agent", isDaemonSet=True)]


def problem(pods, its, provs, ds):
    return {"wellKnownLabels": ["size", "tier", "grp"], "instanceTypes": its, "provisioners": provs, "pods": pods, "daemonSetPods": ds}


# ---------------------------------------------------------------- shapes and near misses
BASE = {"requests": {"cpu": "500m", "memory": "256Mi"}, "nodeSelector": {"size": "small"}}


def _with(base, **kw):
    s = copy.deepcopy(base)
    for k, v in kw.items():
        if v is None:
            s.pop(k, None)
        else:
            s[k] = v
    return s


# each near miss differs from BASE in exactly one compared row word, and in the columns it admits:
#   request   cpu + 1 milli: no longer fits the 700m types (word 0)
#   value     size: large instead of small (the key's value word, 8-23)
#   op        size NotIn [small] instead of In [small]: the meta word only (24)
#   toleration  tolerates the tainted template's taint (25)
#   itype     an instance-type requirement (the low half of word 29)
NEAR = {
    "request": _with(BASE, requests={"cpu": "501m", "memory": "256Mi"}),
    "value": _with(BASE, nodeSelector={"size": "large"}),
    "op": _with(BASE, nodeSelector=None, nodeAffinity={"required": [[{"key": "size", "operator": "NotIn", "values": ["small"]}]]}),
    "toleration": _with(BASE, tolerations=[{"key": "dedicated", "operator": "Exists"}]),
    "itype": _with(BASE, nodeAffinity={"required": [[{"key": INSTANCE_TYPE, "operator": "In", "values": ["it-0001", "it-0006", "it-0010"]}]]}),
}
NEAR_WORD = {"request": 0, "op": 24, "toleration": 25, "itype": 29}  # "value": the size key's value word (8 + key id)
NOFIT = _with(BASE, requests={"cpu": "100", "memory": "256Mi"})
PREFER = _with(BASE, nodeAffinity={"preferred": [{"weight": 10, "terms": [{"key": ZONE, "operator": "In", "values": ["test-zone-1"]}]}]})


class Builder:
    """class-table layout -> pods: slot j of `layout` is the shape of class j; PREFER takes two slots (its relaxed class)"""

    def __init__(self):
        self.shapes, self.ids = [], {}
        self.pod_shape, self.class_shape, self.pods, self.near = [], [], [], {}

    def shape(self, spec):
        key = repr(sorted(spec.items()))
        if key not in self.ids:
            self.ids[key] = len(self.shapes)
            self.shapes.append(copy.deepcopy(spec))
        return self.ids[key]

    def add(self, spec, labels=None, near=None):
        s = self.shape(spec)
        if near:
            self.near[len(self.class_shape)] = near
        i = len(self.pods)
        p = fx.pod(**copy.deepcopy(spec))
        p["labels"] = labels if labels is not None else {"job-name": f"job-{i}", "controller-uid": f"cu-{i:07d}"}
        self.pods.append(p)
        self.pod_shape.append(s)
        self.class_shape.append(s)
        if "preferred" in spec.get("nodeAffinity", {}):
            self.class_shape.append(self.shape(_with(spec, nodeAffinity=None)))

    def done(self, name, prob, **facts):
        prob["pods"] = self.pods
        return dict(name=name, prob=prob, shapes=self.shapes, pod_shape=self.pod_shape, class_shape=self.class_shape, near=self.near,
                    **facts)


def _jobs(b, nc, chunk, near_at, fill=BASE, special=None):
    """nc classes of `fill`, near misses at {class index: kind}, special = {class index: spec} (runs, preferences)"""
    special = special or {}
    while len(b.class_shape) < nc:
        j = len(b.class_shape)
        if j in near_at:
            b.add(NEAR[near_at[j]], near=near_at[j])
        elif j in special:
            b.add(special[j])
        else:
            b.add(fill)


def job_chunks(n_sm):
    """about 2.5 single-pod Jobs per K1 warp (chunks of 3), two templates (the second tainted) on 40 instance types"""
    warps = max_warps(n_sm)
    nc = 3 * warps - warps // 2
    _, _, chunk = k1_grid(nc, n_sm)
    assert chunk == 3
    near_at, special = {}, {}
    w = 10
    for kind in NEAR:
        for off in (0, 1, 2):  # first row of a chunk; after a computed row; after a cache-served row
            near_at[w * chunk + off] = kind
            w += 7
    for j in range(200 * chunk, 203 * chunk):  # whole chunks that nothing fits: kNoBest from the cache
        special[j] = NOFIT
    special[300 * chunk + 1] = PREFER  # its relaxed class takes slot 300 * chunk + 2
    b = Builder()
    _jobs(b, nc, chunk, near_at, special=special)
    return b.done("job_chunks", problem([], catalog(40), templates(2, taint_last=True), daemonset()), n_sm=n_sm)


def whole_batches(n_sm):
    """50 single-pod Jobs per warp (batches at offsets 0, 16, 32 and a partial one of 2 at 48) on 48 instance types and
    two templates: every warp without a near miss serves batches 1 and 2 whole"""
    warps = max_warps(n_sm)
    nc = 50 * warps
    _, _, chunk = k1_grid(nc, n_sm)
    assert chunk == 50
    near_at, special = {}, {}
    w = 20
    for kind in NEAR:
        for off in (0, 1, 15, 16, 31, 32, 47, 49):
            near_at[w * chunk + off] = kind
            w += 11
    for j in range(500 * chunk, 502 * chunk):
        special[j] = NOFIT
    special[600 * chunk + 40] = PREFER
    b = Builder()
    _jobs(b, nc, chunk, near_at, special=special)
    return b.done("whole_batches", problem([], catalog(48), templates(2, taint_last=True), daemonset()), n_sm=n_sm)


def wide_batches(n_sm):
    """20 single-pod Jobs per warp on 2048 instance types (two column words per lane) and two templates: the second batch of
    every chunk (4 rows) is served whole from a cache of V * wpl = 4 words per lane; near misses at offsets 0, 16 and 17"""
    warps = max_warps(n_sm)
    nc = 20 * warps
    _, _, chunk = k1_grid(nc, n_sm)
    assert chunk == 20
    near_at = {}
    w = 30
    for kind in ("request", "value", "toleration"):
        for off in (0, 16, 17):
            near_at[w * chunk + off] = kind
            w += 13
    b = Builder()
    _jobs(b, nc, chunk, near_at)
    return b.done("wide_batches", problem([], catalog(2048), templates(2, taint_last=True), daemonset()), n_sm=n_sm)


def _layout(name, n_sm, n_types, n_templates, n_res=3, **facts):
    """NC = warps + warps / 4 single-pod Jobs (chunks of 2) with request and value near misses at offset 1"""
    warps = max_warps(n_sm)
    nc = warps + warps // 4
    extra = {f"example.com/r{i}": "100" for i in range(n_res - 3)}
    ds = daemonset({f"example.com/r{i}": "1" for i in range(n_res - 3)})
    _, _, chunk = k1_grid(nc, n_sm)
    near_at = {(w * 97 % (nc // chunk)) * chunk + 1: kind for w, kind in enumerate(("request", "value", "request", "value"))}
    b = Builder()
    _jobs(b, nc, chunk, near_at, special={5 * chunk: NOFIT, 5 * chunk + 1: NOFIT})
    return b.done(name, problem([], catalog(n_types, extra), templates(n_templates), ds), n_sm=n_sm, n_res=n_res, **facts)


def layout(n_sm):
    """[(scenario)]: cache / staging edges. Facts: cache (V * wpl <= 16), alloc (allocatable staged), tables (True / False /
    None = either)"""
    return [
        _layout("v8_t2048", n_sm, 2048, 8, cache=True, alloc=True, tables=None),
        _layout("v4_t4000", n_sm, 4000, 4, cache=True, alloc=True, tables=None),
        _layout("v9_t2048", n_sm, 2048, 9, cache=False, alloc=True, tables=None),
        _layout("v17_t1000", n_sm, 1000, 17, cache=False, alloc=True, tables=True),
        _layout("r8_t2048_v50", n_sm, 2048, 50, n_res=8, cache=False, alloc=True, tables=False),
        _layout("r8_t2049", n_sm, 2049, 2, n_res=8, cache=True, alloc=False, tables=True),
    ]


def best_edges(n_sm):
    """best_column's key: `eq-a` / `eq-b` cost the same double (input order decides), `f32-hi` (template 0 only) and
    `f32-lo` (template 1 only) differ as doubles but not as float32 (the template field decides, against the column order),
    `free` costs 0, `dead` has no available offering. Filler types take the other columns."""
    its = [itype("f32-hi", 64000, 0.3 + 1e-12, tier="a", grp="f32"), itype("eq-b", 64000, 0.5, tier="c", grp="eq"),
           itype("dead", 64000, 0.05, tier="c", grp="dead", available=False), itype("f32-lo", 64000, 0.3, tier="b", grp="f32"),
           itype("eq-a", 64000, 0.5, tier="c", grp="eq"), itype("free", 64000, 0.0, tier="c", grp="zero")]
    its[1], its[4] = its[4], its[1]  # eq-a before eq-b in input order
    its += [itype(f"fill-{i}", 1000 + 500 * i, 0.1 + 0.1 * i, tier="c", grp="fill") for i in range(90)]
    provs = [{"name": "hi", "weight": 20, "requirements": [{"key": "tier", "operator": "In", "values": ["a", "c"]}]},
             {"name": "lo", "weight": 10, "requirements": [{"key": "tier", "operator": "In", "values": ["b", "c"]}]}]
    edge = {g: {"requests": {"cpu": "1", "memory": "256Mi"}, "nodeSelector": {"grp": g}} for g in ("eq", "f32", "zero", "dead", "fill")}
    warps = max_warps(n_sm)
    nc = warps + warps // 2
    _, _, chunk = k1_grid(nc, n_sm)
    b = Builder()
    order = ("fill", "eq", "f32", "zero", "dead")
    while len(b.class_shape) < nc:  # runs of each edge across chunk boundaries
        b.add(edge[order[(len(b.class_shape) // 5) % len(order)]])
    return b.done("best_edges", problem([], its, provs, daemonset()), n_sm=n_sm)


def stream(n_sm):
    """2048 * n_sm + 37 pods of five deployments (five classes) on 40 instance types"""
    n = 2048 * n_sm + 37
    specs = [BASE, NEAR["request"], NEAR["value"], NOFIT, NEAR["toleration"]]
    b = Builder()
    for i in range(n):
        s = (i * 7 // 3) % len(specs)
        b.pods.append(dict(fx.pod(**copy.deepcopy(specs[s])), labels={"app": f"deploy-{s}"}))
        b.pod_shape.append(b.shape(specs[s]))
    b.class_shape = None  # the class table is in first-appearance order: reach tests read it from the encoding
    return b.done("stream", problem([], catalog(40), templates(2, taint_last=True), daemonset()), n_sm=n_sm)


# ---------------------------------------------------------------- the reference
NO_BEST = 2 ** 64 - 1


def fresh_node_options(pkg, oracle, prob, spec, prov):
    """input indices of the instance types a fresh node of provisioner `prov` keeps for one pod of `spec` (Node.Add on a new
    node, node.go:62-107): one single-pod, single-provisioner oracle Solve, daemonsets kept. A pod the oracle could only
    place after relaxing it has no option unrelaxed, and neither has one it cannot place at all."""
    single = dict(prob, pods=[fx.pod(**copy.deepcopy(spec))], provisioners=[prov], nodes=[])
    want = pkg.Result()
    assert oracle.solve(pkg.Problem.from_dict(single), want) == 0, want.error
    w = want.to_dict()
    return w["newNodes"][0]["options"] if w["assign"][0] >= 0 and w["relax"][0] == 0 else []


def column_order(prob):
    """(position of each input type among the price-ordered columns, float32 bits of its cheapest available offering):
    the columns are a stable sort by that price (host/encoder.cc, instance_types); no available offering prices +inf"""
    import numpy as np
    price = [min([o["price"] for o in it["offerings"] if o.get("available", True)], default=float("inf")) for it in prob["instanceTypes"]]
    order = sorted(range(len(price)), key=lambda i: price[i])
    pos = [0] * len(price)
    for t, i in enumerate(order):
        pos[i] = t
    return pos, [int(np.float32(p).view(np.uint32)) for p in price]


def reference(pkg, oracle, scenario):
    """(F [shapes][templates][type words] uint64 in caller column order, best [shapes] uint64) of every shape: one fresh-node
    Solve per (shape, template), templates in weight order; best = min over feasible columns t of template v of
    (f32 price bits << 32 | v << 24 | t)"""
    import numpy as np
    prob = scenario["prob"]
    provs = sorted(prob["provisioners"], key=lambda p: -p.get("weight", 0))
    n_types = len(prob["instanceTypes"])
    tw = max(1, -(-n_types // 64))
    pos, p32 = column_order(prob)
    F = np.zeros((len(scenario["shapes"]), len(provs), tw), dtype=np.uint64)
    best = np.full(len(scenario["shapes"]), NO_BEST, dtype=np.uint64)
    for s, spec in enumerate(scenario["shapes"]):
        for v, prov in enumerate(provs):
            for i in fresh_node_options(pkg, oracle, prob, spec, prov):
                F[s, v, i // 64] |= np.uint64(1 << (i % 64))
                best[s] = min(int(best[s]), (p32[i] << 32) | (v << 24) | pos[i])
    return F, best


def shard_columns(prob, b, e):
    """[type words] uint64 mask (caller column order) of the columns in u32 words [b, e) of the price-ordered columns"""
    import numpy as np
    pos, _ = column_order(prob)
    m = np.zeros(max(1, -(-len(pos) // 64)), dtype=np.uint64)
    for i, t in enumerate(pos):
        if b * 32 <= t < e * 32:
            m[i // 64] |= np.uint64(1 << (i % 64))
    return m


def shard_best(F, prob, b, e):
    """best of one shard: the minimum key over the columns in u32 words [b, e) only"""
    import numpy as np
    pos, p32 = column_order(prob)
    out = np.full(F.shape[0], NO_BEST, dtype=np.uint64)
    for s in range(F.shape[0]):
        for v in range(F.shape[1]):
            for i, t in enumerate(pos):
                if b * 32 <= t < e * 32 and (int(F[s, v, i // 64]) >> (i % 64)) & 1:
                    out[s] = min(int(out[s]), (p32[i] << 32) | (v << 24) | t)
    return out
