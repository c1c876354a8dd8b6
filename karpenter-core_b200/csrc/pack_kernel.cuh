// K2 — pack_kernel: Scheduler.add's sequential first-fit (scheduler.go:174-219) in one persistent CTA.
//
// Design (latency-bound integer work; DESIGN.md section 4 has the long form):
//  * one CTA (128..512 threads), four modes: the failure memo (pods of the class that has just failed are requeued in
//    one step), the class run over the shared-memory window of open nodes (consecutive pods of one class whose accept
//    test is exact there; class_run), the existing-node run (identical plain pods fill the existing nodes in one
//    prefix-sum pass; existing_run), and the out-of-line generic step (staging: gen_stage, existing nodes,
//    requirement / topology evaluation, fresh nodes, relaxation: gen_requeue);
//  * candidate nodes are examined one per thread and the reference's scan order is recovered by an argmin over
//    (pod count, stable tie-break) = the position under sort.Slice(newNodes, len(Pods)<) treated as a stable sort;
//  * the state every candidate check needs (order key, request vector, Pareto front of the allocatable vectors of the
//    node's surviving instance types) lives in SHARED MEMORY for the first kActCap open nodes; everything colder
//    (requirement masks, instance-type bitsets, host ports) stays in global memory / L2;
//  * the instance-type bitset of a node is filtered LAZILY by resources: Fits() is monotone in the request vector, so
//    options_true = options_stored AND FIT(requests) and the AND is applied once, by finalize_options_kernel;
//  * generic step: cheap per-candidate filter -> block argmin -> full evaluation of the winner only -> the whole CTA
//    checks / narrows the winner's instance-type words (exclude + retry when it fails);
//  * parameters come from __constant__ memory (g_k2), the per-CTA working set is file-scope __shared__: out-of-line
//    functions reach both with immediate addresses.
// Part of the single translation unit ksched.cu, which includes it once per parameter slot (after topology.cuh).

constexpr int kActCap = 1280;  // open in-flight nodes whose hot state is held in shared memory
constexpr int kHotRes = 4;     // resources covered by the hot request / bound vectors (cpu, memory, pods, +1)

struct HotSmem {
  unsigned long long key[kActCap];     // (pod count << 32) | biased tie-break  == position under a stable sort
  long long q[kHotRes][kActCap];       // node.Requests
  // Exact resource test without touching the option bitsets: when the Pareto front of the allocatable vectors of a
  // node's stored options has one or two members (flags bit0 "exact"; bit5 "two members"), a request vector fits some
  // option iff it fits a front member. Otherwise bound holds per-resource maxima (a necessary test only).
  long long bound[kHotRes][kActCap];
  long long bound2[kHotRes][kActCap];
  int node[kActCap];
  unsigned short flags[kActCap];       // bit0 dominant option exists; bits 1..4 request-map keys; bits 8.. template
  // Requirement verdict memo per open node, valid for topology-free pod classes without host ports:
  //  absorbed: the node's requirements already contain this class's requirements (a further pod of the class changes
  //            nothing: Compatible holds, the merge is the identity, the stored options are untouched);
  //  rejected: the last requirement / instance-type evaluation of this class against the node failed and nothing has
  //            been committed to the node since.
  unsigned absorbed[kActCap];
  unsigned rejected[kActCap];
  unsigned long long nn_last[kActCap];  // class_run: the key a tombstoned node had when it left the active set
};

struct Hot {
  HotSmem* sm;
  unsigned long long* ov_key;
  long long* ov_q;      // [kHotRes][ov_stride]
  long long* ov_bound;  // [kHotRes][ov_stride]
  long long* ov_bound2;
  int* ov_node;
  unsigned short* ov_flags;
  unsigned* ov_absorbed;
  unsigned* ov_rejected;
  int ov_stride;
  __device__ __forceinline__ unsigned long long& key(int a) const { return a < kActCap ? sm->key[a] : ov_key[a - kActCap]; }
  __device__ __forceinline__ long long& q(int r, int a) const { return a < kActCap ? sm->q[r][a] : ov_q[(size_t)r * ov_stride + (a - kActCap)]; }
  __device__ __forceinline__ long long& bound(int r, int a) const { return a < kActCap ? sm->bound[r][a] : ov_bound[(size_t)r * ov_stride + (a - kActCap)]; }
  __device__ __forceinline__ long long& bound2(int r, int a) const { return a < kActCap ? sm->bound2[r][a] : ov_bound2[(size_t)r * ov_stride + (a - kActCap)]; }
  __device__ __forceinline__ int& node(int a) const { return a < kActCap ? sm->node[a] : ov_node[a - kActCap]; }
  __device__ __forceinline__ unsigned short& flags(int a) const { return a < kActCap ? sm->flags[a] : ov_flags[a - kActCap]; }
  __device__ __forceinline__ unsigned& absorbed(int a) const { return a < kActCap ? sm->absorbed[a] : ov_absorbed[a - kActCap]; }
  __device__ __forceinline__ unsigned& rejected(int a) const { return a < kActCap ? sm->rejected[a] : ov_rejected[a - kActCap]; }
  __device__ void move(int dst, int src) const {
    key(dst) = key(src);
    for (int r = 0; r < kHotRes; ++r) { q(r, dst) = q(r, src); bound(r, dst) = bound(r, src); bound2(r, dst) = bound2(r, src); }
    node(dst) = node(src);
    flags(dst) = flags(src);
    absorbed(dst) = absorbed(src);
    rejected(dst) = rejected(src);
  }
};

__device__ __forceinline__ unsigned long long order_key(int count, int tb) {
  return ((unsigned long long)(unsigned)count << 32) | (unsigned)(tb ^ 0x80000000);
}

constexpr unsigned short kFlExact = 1, kFlTwo = 0x20;

// Pareto front (size <= 2) of the allocatable vectors of a node's stored options, or per-resource maxima when the front
// is larger. Candidates are the per-resource arg-max types (found by probing each resource's descending order); a
// candidate pair is a front iff every stored option is dominated by one of the two.
__device__ __noinline__ void compute_front(const uint32_t* opts, int stride, int n, long long* b1, long long* b2, unsigned short* bits) {
  KS_K2
  const int R = c.n_res < kHotRes ? c.n_res : kHotRes;
  const int T = c.n_types;
  int arg[kHotRes];
  for (int r = 0; r < kHotRes; ++r) { b1[r] = INT64_MIN; b2[r] = INT64_MIN; arg[r] = -1; }
  *bits = 0;
  for (int r = 0; r < R; ++r) {
    const int32_t* perm = c.perm_desc + (size_t)r * T;
    for (int i = 0; i < T; ++i) {
      const int t = perm[i];
      if ((opts[(size_t)(t >> 5) * stride + n] >> (t & 31)) & 1) { arg[r] = t; b1[r] = c.alloc_rt[(size_t)r * T + t]; break; }
    }
  }
  if (arg[0] < 0 || c.n_res > kHotRes) return;  // no option left / resources beyond the hot vectors: necessary test only
  auto dominates = [&](int a, const long long* v) {  // alloc(a) >= v in every hot resource
    for (int r = 0; r < R; ++r) if (c.alloc_rt[(size_t)r * T + a] < v[r]) return false;
    return true;
  };
  if (dominates(arg[0], b1)) { *bits = kFlExact; return; }  // one option is maximal in every resource
  // distinct candidates
  int cand[kHotRes], nc = 0;
  for (int r = 0; r < R; ++r) {
    bool seen = false;
    for (int i = 0; i < nc; ++i) seen = seen || cand[i] == arg[r];
    if (!seen) cand[nc++] = arg[r];
  }
  // which candidate pairs cover every option?  opts ⊆ domset[ci] ∪ domset[cj], word by word
  unsigned pair_ok = 0;  // bit (i*4+j), i<j
  for (int i = 0; i < nc; ++i) for (int j = i + 1; j < nc; ++j) pair_ok |= 1u << (i * 4 + j);
  const int W32 = c.W32;
  for (int w = 0; w < W32 && pair_ok; ++w) {
    const uint32_t m = opts[(size_t)w * stride + n];
    if (!m) continue;
    uint32_t d[kHotRes];
    for (int i = 0; i < nc; ++i) d[i] = c.domset[(size_t)cand[i] * W32 + w];
    for (int i = 0; i < nc; ++i) for (int j = i + 1; j < nc; ++j)
      if (m & ~(d[i] | d[j])) pair_ok &= ~(1u << (i * 4 + j));
  }
  if (!pair_ok) return;  // front larger than two: b1 keeps the per-resource maxima
  const int pi = (__ffs(pair_ok) - 1) / 4, pj = (__ffs(pair_ok) - 1) % 4;
  for (int r = 0; r < R; ++r) { b1[r] = c.alloc_rt[(size_t)r * T + cand[pi]]; b2[r] = c.alloc_rt[(size_t)r * T + cand[pj]]; }
  *bits = kFlExact | kFlTwo;
}

// 0 = no option can hold the requests, 1 = some option holds them (exact), 2 = unknown (per-resource maxima pass)
__device__ __forceinline__ int quick_fit(const long long* q, uint32_t qp, int RH, const long long* b1, const long long* b2, unsigned short fl) {
  bool f1 = true, f2 = true;
#pragma unroll
  for (int r = 0; r < kHotRes; ++r)
    if (r < RH && ((qp >> r) & 1)) { f1 = f1 && q[r] <= b1[r]; f2 = f2 && q[r] <= b2[r]; }
  if (fl & kFlExact) return (f1 || ((fl & kFlTwo) && f2)) ? 1 : 0;
  return f1 ? 2 : 0;
}
// no pod of the batch can ever fit again (min_req: per-resource minimum request over all pod classes)
__device__ __forceinline__ bool node_closed(const long long* q, const long long* min_req, int RH, const long long* b1, const long long* b2, unsigned short fl) {
  bool o1 = false, o2 = false;
#pragma unroll
  for (int r = 0; r < kHotRes; ++r)
    if (r < RH && min_req[r] > 0) { o1 = o1 || q[r] + min_req[r] > b1[r]; o2 = o2 || q[r] + min_req[r] > b2[r]; }
  return (fl & kFlTwo) ? (o1 && o2) : o1;
}

// single-sync block argmin (double-buffered scratch)
__device__ __forceinline__ unsigned long long block_min_u64_db(unsigned long long v, unsigned long long (*red)[32], int& parity) {
  v = warp_min_u64(v);
  if (blockDim.x == 32) return v;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long* buf = red[parity];
  parity ^= 1;
  if (lane == 0) buf[warp] = v;
  __syncthreads();
  const unsigned long long r = lane < (int)(blockDim.x >> 5) ? buf[lane] : ~0ull;
  return warp_min_u64(r);
}

// two independent u32 minima with one barrier (double-buffered scratch, same protocol as block_min_u64_db)
__device__ __forceinline__ void block_min2_u32_db(unsigned a, unsigned b, unsigned long long (*red)[32], int& parity, unsigned* ra, unsigned* rb) {
  a = __reduce_min_sync(0xffffffffu, a);
  b = __reduce_min_sync(0xffffffffu, b);
  if (blockDim.x == 32) { *ra = a; *rb = b; return; }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long* buf = red[parity];
  parity ^= 1;
  if (lane == 0) buf[warp] = ((unsigned long long)a << 32) | b;
  __syncthreads();
  const unsigned long long r = lane < (int)(blockDim.x >> 5) ? buf[lane] : ~0ull;
  *ra = __reduce_min_sync(0xffffffffu, (unsigned)(r >> 32));
  *rb = __reduce_min_sync(0xffffffffu, (unsigned)r);
}

// compute_front with the whole CTA (same result, every thread calls it): the per-resource arg-max types are found by
// probing each resource's descending order T positions at a time (block minimum of the first hit), the pair coverage test
// runs one option word per thread. The serial version walks the orders and the words through dependent L2 loads, tens of
// thousands of cycles per fresh node of a new shape on the 1 000-type catalog.
__shared__ unsigned g_front_pairs;
__device__ __noinline__ void compute_front_block(const uint32_t* opts, int stride, int n, long long* b1, long long* b2, unsigned short* bits,
                                                 unsigned long long (*red)[32], int& parity) {
  KS_K2
  const int R = c.n_res < kHotRes ? c.n_res : kHotRes;
  const int T = c.n_types, tid = threadIdx.x, NT = blockDim.x, W32 = c.W32;
  unsigned pos[kHotRes] = {~0u, ~0u, ~0u, ~0u};
  for (int r = 0; r < R; ++r) {
    const int32_t* perm = c.perm_desc + (size_t)r * T;
    for (int i = tid; i < T; i += NT) {
      const int t = perm[i];
      if ((opts[(size_t)(t >> 5) * stride + n] >> (t & 31)) & 1) { pos[r] = (unsigned)i; break; }
    }
  }
  unsigned pm[kHotRes];
  block_min2_u32_db(pos[0], pos[1], red, parity, &pm[0], &pm[1]);
  block_min2_u32_db(pos[2], pos[3], red, parity, &pm[2], &pm[3]);
  if (tid == 0) g_front_pairs = ~0u;
  int arg[kHotRes];
  long long m1v[kHotRes];
  for (int r = 0; r < kHotRes; ++r) {
    arg[r] = (r < R && pm[r] != ~0u) ? c.perm_desc[(size_t)r * T + pm[r]] : -1;
    m1v[r] = arg[r] >= 0 ? c.alloc_rt[(size_t)r * T + arg[r]] : INT64_MIN;
  }
  bool done = arg[0] < 0 || c.n_res > kHotRes;  // no option left / resources beyond the hot vectors: necessary test only
  unsigned short fb = 0;
  if (!done) {
    bool dom0 = true;  // one option is maximal in every resource
    for (int r = 0; r < R; ++r) dom0 = dom0 && c.alloc_rt[(size_t)r * T + arg[0]] >= m1v[r];
    if (dom0) { fb = kFlExact; done = true; }
  }
  if (done) {
    if (tid == 0) {
      for (int r = 0; r < kHotRes; ++r) { b1[r] = m1v[r]; b2[r] = INT64_MIN; }
      *bits = fb;
    }
    return;  // (uniform: every thread holds the same values)
  }
  int cand[kHotRes], nc = 0;
  for (int r = 0; r < R; ++r) {
    bool seen = false;
    for (int i = 0; i < nc; ++i) seen = seen || cand[i] == arg[r];
    if (!seen) cand[nc++] = arg[r];
  }
  unsigned pair_ok = 0;  // bit (i*4+j), i<j: every option is dominated by candidate i or j
  for (int i = 0; i < nc; ++i) for (int j = i + 1; j < nc; ++j) pair_ok |= 1u << (i * 4 + j);
  unsigned mine = pair_ok;
  for (int w = tid; w < W32; w += NT) {
    const uint32_t m = opts[(size_t)w * stride + n];
    if (!m) continue;
    uint32_t d[kHotRes];
    for (int i = 0; i < nc; ++i) d[i] = c.domset[(size_t)cand[i] * W32 + w];
    for (int i = 0; i < nc; ++i) for (int j = i + 1; j < nc; ++j)
      if (m & ~(d[i] | d[j])) mine &= ~(1u << (i * 4 + j));
  }
  mine = __reduce_and_sync(0xffffffffu, mine);
  __syncthreads();  // g_front_pairs initialised
  if ((tid & 31) == 0) atomicAnd(&g_front_pairs, mine);
  __syncthreads();
  pair_ok &= g_front_pairs;
  if (tid == 0) {
    for (int r = 0; r < kHotRes; ++r) { b1[r] = m1v[r]; b2[r] = INT64_MIN; }
    *bits = 0;
    if (pair_ok) {
      const int pi = (__ffs(pair_ok) - 1) / 4, pj = (__ffs(pair_ok) - 1) % 4;
      for (int r = 0; r < R; ++r) { b1[r] = c.alloc_rt[(size_t)r * T + cand[pi]]; b2[r] = c.alloc_rt[(size_t)r * T + cand[pj]]; }
      *bits = kFlExact | kFlTwo;
    }
  }
}

struct StepShared {
  int placed_closed;   // commit outcome: 1 = the accepting node became full and left the active set
  int path;            // fresh-node path
  unsigned any;
  long long q[KSCHED_MAX_RES];
  unsigned qp;
  long long bound[kHotRes], bound2[kHotRes];
  unsigned short front_bits;
  long long visited;
  // in-flight winner posted for the cooperative instance-type check / commit
  int win_a, win_n, win_need, win_commit, win_fail;
  int excl[16];        // nodes that won the argmin of this step but failed the instance-type check
  // fresh node of a topology-constrained class: slot of the outcome memo (PackState::fd_*), new node's requirement meta
  int fd_slot;
  uint64_t meta;
};
constexpr int kMaxExcl = 16;

enum { kPathReject = 0, kPathCached = 1, kPathRow = 2, kPathDynamic = 3, kPathCachedEmpty = 4, kPathDynCached = 5, kPathDynEmpty = 6 };

// The words of a pod row every candidate check needs. Loaded RAW one iteration ahead for first-pass pods (anything
// derived from them is computed by the consuming iteration, so the prefetch never waits on its own loads).
struct PodRegs {
  const ksched_pod_row* row;
  uint32_t pod, res, itype, hostname, topo_begin, topo_end;
  long long req[kHotRes];
  uint64_t tol, hpc, hpe, meta, cls64;
};
__device__ __forceinline__ PodRegs load_pod_regs(const ksched_pod_row* row, uint32_t pod) {
  PodRegs r;
  r.row = row;
  r.pod = pod;
  r.res = row->res_present;
#pragma unroll
  for (int i = 0; i < kHotRes; ++i) r.req[i] = row->requests[i];  // 0 where the resource is absent
  r.tol = row->tolerated_taintsets;
  r.hpc = row->hostport_conflicts;
  r.hpe = row->hostport_entries;
  r.meta = row->meta;
  r.itype = row->itype_req;
  r.hostname = row->hostname_req;
  r.topo_begin = row->topo_begin;
  r.topo_end = row->topo_end;
  r.cls64 = row->reserved;
  return r;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// Ext resources the class requests (DESIGN.md §3). Such classes take the generic step only: every closed-form mode below
// reads the 8 row slots alone (the variant table builds no entry for them).
__device__ __forceinline__ uint32_t class_ext(const PackState& s, unsigned cls) {
  return s.cls_ext_present ? s.cls_ext_present[cls] : 0u;
}

// Slow part of a candidate check (requirement keys / topology / instance-type words), kept out of line so that the
// common path (no requirement can change, dominant option fits) stays in registers.
struct SlowEval {
  Touched t;
  TypeCtx x;
  long long q[KSCHED_MAX_RES];
  uint32_t qp;
  bool changed;
  bool need_types;  // with_types == false: the instance-type options still have to be checked (by the whole CTA, for the winner only)
};
// `t` receives the touched requirement keys: the thread's own e.t, or the CTA's shared Touched when the caller is the argmin winner
template <bool kExt>
__device__ __noinline__ bool evaluate_slow(bool plain,
                                           int n, unsigned short fl, const long long* q_hot, const int64_t* alloc_sorted, bool with_types, Touched& t,
                                           SlowEval& e) {
  KS_K2
  KS_ROW
  const int MAXN = s.max_new, NE = s.n_existing, R = c.n_res, W32 = c.W32;
  const uint32_t p_res = row.res_present, p_ext = kExt ? class_ext(s, (unsigned)row.reserved) : 0u;
  t.clear();
  e.changed = false;
  bool need_types = !(fl & 1) || row.itype_req != KSCHED_NONE || p_ext;
  if (!plain) {
    if (!requirements_phase(s.nn_vals, s.nn_meta[n], MAXN, n, NE + n, false, t)) return false;
    e.changed = t.changed != 0;
    need_types = need_types || e.changed;
  }
  for (int r = 0; r < kHotRes; ++r) e.q[r] = q_hot[r];
  for (int r = kHotRes; r < R; ++r) e.q[r] = s.nn_req[(size_t)r * MAXN + n] + (((p_res >> r) & 1) ? row.requests[r] : 0);
  e.qp = s.nn_req_present[n] | p_res;
  e.need_types = need_types && !with_types;
  if (!need_types || !with_types) return true;  // the dominant option fits and no requirement changed / checked later
  build_type_ctx(t, e.q, e.qp, s.nn_vals, s.nn_meta[n], MAXN, n, false, alloc_sorted, e.x);
  for (int w = 0; w < W32; ++w) {
    const uint32_t base = s.nn_opts[(size_t)w * MAXN + n];
    uint32_t sw = base ? type_word(c, s, e.x, base, w) : 0;
    if (sw && p_ext)
      sw = ext_fit_word(c, s.nn_req_ext + (size_t)n * c.n_res_ext, s.cls_req_ext + (size_t)row.reserved * c.n_res_ext, p_ext, sw, w);
    if (sw) return true;
  }
  return false;
}
// Requirement part of a commit into a node's requirement set (SoA vals / meta, column idx): its new masks.
__device__ __forceinline__ uint64_t commit_touched(const Touched& t, uint64_t* vals, uint64_t* metas, int stride, int idx) {
  for (uint32_t m = t.keys; m; m &= m - 1) {
    const int k = __ffs(m) - 1;
    vals[(size_t)k * stride + idx] = t.fin[k];
  }
  const uint64_t meta = t.overlay_meta(metas[idx]);
  metas[idx] = meta;
  return meta;
}
__device__ __forceinline__ uint64_t commit_reqs(int n, const Touched& t) {
  KS_K2
  return commit_touched(t, s.nn_vals, s.nn_meta, s.max_new, n);
}
// Requirement-changing commit done by ONE thread (fallback mode): new masks, requirement-driven narrowing of the stored
// options, new bounds.
template <bool kExt>
__device__ __noinline__ void commit_slow(int n, SlowEval& e, long long* bound,
                                         long long* bound2, unsigned short* front_bits, uint64_t* meta_out) {
  KS_K2
  KS_ROW
  const int MAXN = s.max_new, W32 = c.W32;
  *meta_out = commit_reqs(n, e.t);
  e.x.res_mask = 0;  // resources stay lazy (finalize_options_kernel), except ext resources: narrowed eagerly (DESIGN.md §3)
  const uint32_t p_ext = kExt ? class_ext(s, (unsigned)row.reserved) : 0u;
  for (int w = 0; w < W32; ++w) {
    const uint32_t base = s.nn_opts[(size_t)w * MAXN + n];
    uint32_t sw = base ? type_word(c, s, e.x, base, w) : 0;
    if (sw && p_ext)
      sw = ext_fit_word(c, s.nn_req_ext + (size_t)n * c.n_res_ext, s.cls_req_ext + (size_t)row.reserved * c.n_res_ext, p_ext, sw, w);
    if (base) s.nn_opts[(size_t)w * MAXN + n] = sw;
  }
  compute_front(s.nn_opts, MAXN, n, bound, bound2, front_bits);
}

// per-CTA objects of the generic step (file scope: see g_row / g_pt in ksched.cu)
__shared__ Touched g_fresh_t;
__shared__ TypeCtx g_fresh_x;
__shared__ unsigned long long g_red[2][32];
__shared__ StepShared g_sh;
__shared__ uint32_t g_tmpl_taintset[KSCHED_MAX_TEMPLATES];
extern __shared__ __align__(16) unsigned char dyn_smem[];  // HotSmem, then (optionally) the sorted allocatable arrays
__device__ __forceinline__ Hot make_hot(const PackState& s) {
  return Hot{reinterpret_cast<HotSmem*>(dyn_smem), s.ov_key, s.ov_q, s.ov_bound, s.ov_bound2, s.ov_node, s.ov_flags, s.ov_absorbed, s.ov_rejected, s.max_new};
}
__device__ __forceinline__ const int64_t* alloc_table(const DevCatalog& c, const PackState& s) {
  return s.alloc_in_smem ? reinterpret_cast<const int64_t*>(dyn_smem + sizeof(HotSmem)) : c.alloc_sorted;
}
struct LoopVars {
  int head, qlen, n_new, n_active, tick, seq, parity, fatal;
  uint32_t epoch;
  bool pt_nonempty;
  long long nodes_visited;
  uint32_t pt_class;   // class the shared PodTopo was built for (KSCHED_NONE: none)
  uint32_t row_class;  // class whose row g_row holds
  // the step has just opened node slot fresh_a for a pod of class fresh_cls and the node is still open (class_run captures it)
  int fresh_valid, fresh_a;
  uint32_t fresh_cls;
  // the step failed and depends on nothing but (class, placements so far, relaxations so far): no topology relation of
  // any kind, no relaxation left. pack_kernel requeues the following pods of the class without evaluating them again.
  int fail_memo;
  // in: class_run asks for a fresh node only (run_derive): no in-flight node is tried, the pod is neither assigned nor
  // recorded in the topology counters nor requeued, and the caller keeps its tick / seq. Out: n_new / n_active as the
  // step would have left them.
  int derive;
};

// ---- existing-node run ("water-fill") --------------------------------------------------------------------------------
// A run of consecutive first-pass pods of ONE plain class (no requirement key, no topology relation, no host port, no
// volume, no instance-type requirement) is placed on the existing nodes in one pass. A hostname requirement only removes the
// slots it does not admit (K_e = 0): that verdict never changes for the class, so the cursor stays exact. First fit over existing
// nodes in slice order (scheduler.go:176-180) sends identical pods to the first node that still fits one, until it does not:
// node e takes K_e = min over requested resources of floor((available - requests) / request) of them, so the run is an
// exclusive prefix sum of K over the nodes from the class's cursor on. Every effect of the sequential commits is reproduced
// (requests, closed flag, assign, place_seq); what the existing nodes cannot take is left to the generic step.
constexpr int kExRunMax = 1 << 20;
// CSI volume limits (ksched.h: ksched_class_volumes). Tracked claims 0-63 are bits of the row's and the nodes' words; from 64
// on they are words of the per-class table and of the nodes' [word][node] array (ksched.h: class_volumes_shared_ext). A class
// whose tracked claims all have ids from 64 on and that has no private claim has a zero row, so the gates read the per-class
// "mounts a claim" byte the upload derives from the row and the table (one byte load where the row test took 16 bytes).
__device__ __forceinline__ bool class_has_volumes(const PackState& s, unsigned cls) { return s.cls_has_vol && s.cls_has_vol[cls]; }
// Both volume helpers are out of line, like hostname_table_allows: the generic step carries a call, not the driver loop and
// the table loops (DESIGN.md §3).
// volumeUsage.Validate(pod).Exceeds(volumeLimits) of existing node e for a class with volumes (existingnode.go:88-96)
__device__ __noinline__ bool node_vol_over(unsigned cls, int e) {
  KS_K2
  const ksched_node_volumes nv = s.ex_vol[e];
  const ksched_class_volumes pv = s.cls_vol[cls];
  const uint64_t all = nv.mounted | pv.shared;
  const int W = s.vol_ext_words, NE = s.n_existing;
  const uint64_t* cw = s.cls_vol_ext + (size_t)cls * W;
  for (int d = 0; d < KSCHED_MAX_VOLUME_DRIVERS; ++d) {
    if (nv.limit[d] < 0) continue;
    const uint64_t* mw = s.vol_mask_ext + (size_t)d * W;
    int n = nv.used[d] + __popcll(all & s.vol_mask[d]) + (int)pv.priv[d];
    for (int w = 0; w < W; ++w) n += __popcll((s.ex_vol_ext[(size_t)w * NE + e] | cw[w]) & mw[w]);
    if (n > nv.limit[d]) return true;
  }
  return false;
}
// volumeUsage.Add (existingnode.go:128): the class's claims join those existing node e mounts
__device__ __noinline__ void node_vol_commit(unsigned cls, int e) {
  KS_K2
  ksched_node_volumes nv = s.ex_vol[e];
  const ksched_class_volumes pv = s.cls_vol[cls];
  nv.mounted |= pv.shared;
#pragma unroll
  for (int d = 0; d < KSCHED_MAX_VOLUME_DRIVERS; ++d) nv.used[d] += (int)pv.priv[d];
  s.ex_vol[e] = nv;
  const int W = s.vol_ext_words, NE = s.n_existing;
  for (int w = 0; w < W; ++w) s.ex_vol_ext[(size_t)w * NE + e] |= s.cls_vol_ext[(size_t)cls * W + w];
}
// Taints.Tolerates (taints.go:28-40) of an existing node's taint set. Ids below 64 are bits of the row's word; ids from 64 on
// only existing nodes carry (ksched.h: class_tolerated_ext), and they live in the per-class table.
__device__ __forceinline__ bool tolerates_node_set(const PackState& s, uint64_t tol, unsigned cls, uint32_t ts) {
  const uint64_t w = ts < 64 ? tol : s.cls_tol_ext[(size_t)cls * s.tol_ext_words + ((ts - 64) >> 6)];
  return (w >> (ts & 63)) & 1;
}
// Host ports (HostPortUsage, hostportusage.go:65-93). Entries 0-63 are bits of the row's and the nodes' words; entries from
// 64 on are words of the per-class tables and of the nodes' [word][node] arrays (ksched.h: class_hostport_conflicts_ext).
// A class whose entries all have ids from 64 on has zero row words, so every gate that means "no host port" asks
// has_host_ports: such a class takes the generic step, the only one that checks and commits entries.
__device__ __forceinline__ bool class_hp_ext(const PackState& s, unsigned cls) { return s.cls_hp_ext && s.cls_hp_ext[cls]; }
__device__ __forceinline__ bool has_host_ports(const PackState& s, const PodRegs& p) {
  return (p.hpc | p.hpe) != 0 || class_hp_ext(s, (unsigned)p.cls64);
}
// HostPortUsage.validate: node idx of `words` / `ext` (`stride` nodes per ext word) holds an entry the class conflicts with.
// hpx: class_hp_ext of the class.
__device__ __forceinline__ bool node_hp_conflict(const PackState& s, uint64_t hpc, bool hpx, unsigned cls, const uint64_t* words,
                                                 const uint64_t* ext, int stride, int idx) {
  if (hpc && (words[idx] & hpc)) return true;
  if (!hpx) return false;
  const uint64_t* cw = s.cls_hpc_ext + (size_t)cls * s.hp_ext_words;
  for (int w = 0; w < s.hp_ext_words; ++w)
    if (cw[w] & ext[(size_t)w * stride + idx]) return true;
  return false;
}
// HostPortUsage.Add: the class's entries join those node idx holds
__device__ __forceinline__ void node_hp_commit(const PackState& s, uint64_t hpe, bool hpx, unsigned cls, uint64_t* words, uint64_t* ext,
                                               int stride, int idx) {
  if (hpe) words[idx] |= hpe;
  if (!hpx) return;
  const uint64_t* ce = s.cls_hpe_ext + (size_t)cls * s.hp_ext_words;
  for (int w = 0; w < s.hp_ext_words; ++w) ext[(size_t)w * stride + idx] |= ce[w];
}
// A new node holds its first pod's entries and nothing else. Every site that opens a node writes all its words (the class
// runs' nodes with hpe = 0, hpx = false), so a later host-port pod's in-flight scan never reads a word of an earlier Solve.
__device__ __forceinline__ void fresh_node_hp(const PackState& s, uint64_t hpe, bool hpx, unsigned cls, int n) {
  s.nn_hp[n] = hpe;
  for (int w = 0; w < s.hp_ext_words; ++w)
    s.nn_hp_ext[(size_t)w * s.max_new + n] = hpx ? s.cls_hpe_ext[(size_t)cls * s.hp_ext_words + w] : 0;
}
// The scalar global state of new node n, opened from template v: requirement meta, template, request keys, host-port
// entries, instance-type slot state and, when `count` is set, the pod count and tie-break of its first pod. The class runs
// open nodes with hpe = 0, hpx = false and itype = KSCHED_NONE.
__device__ __forceinline__ void open_node(const PackState& s, int n, int v, uint64_t meta, uint32_t qp, uint64_t hpe, bool hpx, unsigned cls,
                                          uint32_t itype, bool count, int tb) {
  s.nn_meta[n] = meta;
  s.nn_tmpl[n] = (uint8_t)v;
  s.nn_req_present[n] = qp;
  fresh_node_hp(s, hpe, hpx, cls, n);
  if (s.nn_it) itype_state_open(n, v, itype);
  if (count) {
    s.nn_count[n] = 1;
    s.nn_tb[n] = tb;
  }
}
// Ext sums of one node, resource x at sums[x * stride], against / plus the class's ext requests creq (ext bits p_ext)
__device__ __forceinline__ bool ext_fits(const int64_t* sums, const int64_t* avail, size_t stride, const int64_t* creq, uint32_t p_ext) {
  for (uint32_t m = p_ext; m; m &= m - 1) {
    const int x = __ffs(m) - 1;
    if (sums[x * stride] + creq[x] > avail[x * stride]) return false;
  }
  return true;
}
__device__ __forceinline__ void ext_add(int64_t* sums, size_t stride, const int64_t* creq, uint32_t p_ext) {
  for (uint32_t m = p_ext; m; m &= m - 1) { const int x = __ffs(m) - 1; sums[x * stride] += creq[x]; }
}
// k pods requesting req (resources res) join existing node e. Returns its closed flag: no pod of the batch fits it any more
// (min_req: per-resource minimum request over all pod classes).
template <class Req>
__device__ __forceinline__ bool existing_add(const PackState& s, int R, int e, uint32_t res, const Req* req, long long k) {
  const int NE = s.n_existing;
  bool closed = false;
  for (int r = 0; r < R; ++r) {
    if ((res >> r) & 1) s.ex_req[(size_t)r * NE + e] += k * req[r];
    const long long a = ((s.ex_avail_present[e] >> r) & 1) ? s.ex_avail[(size_t)r * NE + e] : 0;
    if (s.min_req[r] > 0 && s.ex_req[(size_t)r * NE + e] + s.min_req[r] > a) closed = true;
  }
  s.ex_req_present[e] |= res;
  return closed;
}
struct ExRunIO { int qi, head, qlen, seq, parity, placed; long long add_calls; };
__shared__ ExRunIO g_xio;
// one partial sum per warp, double-buffered: every warp of the largest block the kernel is launched with needs a slot
constexpr int kScanWarps = kPackThreads / 32;
static_assert(kScanWarps * 32 == kPackThreads, "block_scan_incl: kPackThreads is a whole number of warps");
__shared__ int g_xscan[2][kScanWarps];
__device__ __forceinline__ int block_scan_incl(int v, int* total, int& xpar) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
  int* buf = g_xscan[xpar];
  xpar ^= 1;
  if (lane == 31) buf[warp] = x;
  __syncthreads();
  int base = 0, tot = 0;
  for (int w = 0; w < nw; ++w) { const int t = buf[w]; if (w < warp) base += t; tot += t; }
  *total = tot;
  return x + base;
}
__device__ __noinline__ void existing_run(const PodRegs& first) {
  KS_K2
  const int tid = threadIdx.x, T = blockDim.x, NE = s.n_existing, R = c.n_res;
  ExRunIO& io = g_xio;
  const unsigned cls = (unsigned)first.cls64;
  const ksched_pod_row* ffd_rows = reinterpret_cast<const ksched_pod_row*>(s.rows);
  const int qi = io.qi, seq0 = io.seq;
  int parity = io.parity, xpar = 0;
  __syncthreads();  // everybody has read g_xio
  // run length: consecutive queue entries of this class
  const int lim = min(s.n_pods - qi, kExRunMax);
  unsigned long long stop = ~0ull;
  for (int j = tid; j < lim; j += T)
    if ((unsigned)ffd_rows[qi + j].reserved != cls) { stop = (unsigned long long)j; break; }
  const unsigned long long st = block_min_u64_db(stop, g_red, parity);
  const int m = st == ~0ull ? lim : (int)st;
  int e0 = s.cls_cursor[cls], placed = 0, last_used = -1;
  while (placed < m && e0 < NE) {
    const int e = e0 + tid;
    int k = 0;
    if (e < NE && !s.ex_closed[e] && tolerates_node_set(s, first.tol, cls, s.ex_taintset[e]) &&
        (first.hostname == KSCHED_NONE || hostname_req_allows(s, first.hostname, e, true))) {
      long long K = m - placed;
      const uint32_t qp = s.ex_req_present[e] | first.res, ap = s.ex_avail_present[e];
      for (int r = 0; r < R && K > 0; ++r) {
        if (!((qp >> r) & 1)) continue;
        const long long a = ((ap >> r) & 1) ? s.ex_avail[(size_t)r * NE + e] : 0;
        const long long q = s.ex_req[(size_t)r * NE + e];
        const long long pr = (r < kHotRes && ((first.res >> r) & 1)) ? first.req[r] : 0;
        if (q + pr > a) { K = 0; break; }  // Fits(requests + pod, available) fails for the very next pod (existingnode.go:98-102)
        if (pr > 0) { const long long kk = (a - q) / pr; if (kk < K) K = kk; }
      }
      k = (int)K;
    }
    int total;
    const int incl = block_scan_incl(k, &total, xpar);
    const int excl = incl - k, want = m - placed;
    const int take = excl < want ? min(k, want - excl) : 0;
    if (take > 0) {
      // (the run's pods request hot resources only: its gate admits no class with res >> kHotRes)
      s.ex_closed[e] = existing_add(s, R, e, first.res & ((1u << kHotRes) - 1), first.req, take);
      for (int j = 0; j < take; ++j) {
        const uint32_t pod = s.order[qi + placed + excl + j];
        s.assign[pod] = e;
        s.place_seq[pod] = seq0 + placed + excl + j;
      }
    }
    const unsigned long long lu = block_min_u64_db(take > 0 ? (unsigned long long)(0x7fffffff - e) : ~0ull, g_red, parity);  // max e that took pods
    if (lu != ~0ull) last_used = 0x7fffffff - (int)lu;
    placed += min(total, want);
    if (placed < m) e0 += T;
  }
  if (tid == 0) {
    // nodes passed over took nothing for a monotone reason (closed, taint, requests), nodes filled are full for this class
    s.cls_cursor[cls] = placed < m ? NE : (last_used >= 0 ? last_used : s.cls_cursor[cls]);
    const int qcap = s.n_pods + 1;
    io.qi = qi + placed;
    io.head = (io.head + placed) % qcap;
    io.qlen -= placed;
    io.seq = seq0 + placed;
    io.add_calls += placed;
    io.placed = placed;
    io.parity = parity;
  }
  __syncthreads();
}

// Cycle and event counters of the profiling build (KSCHED_PROFILE_PACK): PK_T in pack_kernel (pk_acc / pk_last), GK_T / GK_C
// in the generic step (gk_last, the PackState s)
#ifdef KSCHED_PROFILE_PACK
#define PK_T(i) { long long _now = clock64(); pk_acc[i] += _now - pk_last; pk_last = _now; }
#define GK_T(i) { if (threadIdx.x == 0) { long long _n = clock64(); s.counters[i] += _n - gk_last; gk_last = _n; } }
#define GK_C(i) { if (threadIdx.x == 0) s.counters[i] += 1; }
#else
#define PK_T(i)
#define GK_T(i)
#define GK_C(i)
#endif

// generic step, staging: the pod's row into g_row and its topology constraints into g_pt. false: PodTopo overflowed
// (L.fatal is set).
__device__ __forceinline__ bool gen_stage(const ksched_pod_row* src, uint32_t cls, bool has_topo, LoopVars& L) {
  const int tid = threadIdx.x;
  PodTopo& pt = g_pt;
  // The pod's 256-byte row lives in shared memory (everything below reads it with immediate addresses); rows of one
  // class are identical, so it is copied on a class change only.
  const bool new_row = L.row_class != cls;
  const bool topo_step = has_topo || L.pt_nonempty;
  if (new_row || topo_step) {
    __syncthreads();  // previous step's readers of g_row / g_pt are done
    if (tid < 32) {
      if (new_row) {
        reinterpret_cast<uint64_t*>(&g_row)[tid] = reinterpret_cast<const uint64_t*>(src)[tid];
        __syncwarp();
      }
      if (topo_step) {
        if (L.pt_class == cls && !pt.overflow) refresh_pod_topo();  // same relations as the previous step, new counters
        else build_pod_topo();
      }
    }
    L.row_class = cls;
    if (topo_step) L.pt_class = cls;
    __syncthreads();
    if (topo_step) {
      L.pt_nonempty = pt.n != 0;
      if (pt.overflow) { L.fatal = KSCHED_ERR_UNSUPPORTED; return false; }
    }
  }
  return true;
}
// generic step, failure: relax + requeue (scheduler.go:117-123, queue.go:61-68)
__device__ __forceinline__ void gen_requeue(uint32_t pod, bool has_topo, LoopVars& L) {
  KS_K2
  KS_ROW
  const int qcap = s.n_pods + 1;
  GK_C(kCtrGenFailures)
  const uint32_t nx = row.relax_next;
  int tail = L.head + L.qlen;
  if (tail >= qcap) tail -= qcap;
  if (threadIdx.x == 0) {
    s.queue[tail] = pod;
    if (nx != KSCHED_NONE) {
      s.pod_class[pod] = nx;
      s.relax_level[pod] += 1;
      // Topology.Update(pod): groups that only the relaxed spec owns come into existence now
      const ksched_pod_row& nrow = s.classes[nx];
      for (uint32_t e = nrow.topo_begin; e < nrow.topo_end; ++e) {
        const ksched_class_topo ct = s.class_topo[e];
        if ((ct.flags & KSCHED_TOPO_CONSTRAINS) && !s.grp_active[ct.group]) {
          s.grp_active[ct.group] = 1;
          s.grp_min_slot[ct.group] = s.n_existing + L.n_new;
        }
      }
    } else {
      s.last_len[pod] = L.qlen + 1;
      s.last_epoch[pod] = L.epoch;
    }
  }
  ++L.qlen;
  if (nx != KSCHED_NONE) ++L.epoch;  // a successful relaxation resets the lastLen map
  L.fail_memo = nx == KSCHED_NONE && !has_topo && !L.pt_nonempty;
  __syncthreads();
}

// generic step, in-flight winner that failed its full check: no later argmin of this step picks it again
__device__ __forceinline__ void exclude_winner(const Hot& H, int wa, bool simple, unsigned cls, int& n_excl, bool& full_eval) {
  if (threadIdx.x == 0) {
    if (n_excl < kMaxExcl) g_sh.excl[n_excl] = wa;
    if (simple) H.rejected(wa) = cls;
  }
  ++n_excl;
  if (n_excl >= kMaxExcl) full_eval = true;
  __syncthreads();
}
// generic step, option word w of in-flight node: narrowed by the winner's requirements and, for an ext class, its ext sums
__device__ __forceinline__ uint32_t narrow_word(const DevCatalog& c, const PackState& s, const TypeCtx& x, uint32_t base, int w,
                                                const int64_t* node_ext, const int64_t* cls_ext, uint32_t p_ext) {
  uint32_t sw = type_word_keys(c, s, x, base, w);
  if (sw && p_ext) sw = ext_fit_word(c, node_ext, cls_ext, p_ext, sw, w);
  return sw;
}
// generic step, Pareto front of a memoised option set: entry i of (bound, bound2, dom) in the fc_* or fd_* tables, to / from g_sh
__device__ __forceinline__ void front_load(const long long* b1, const long long* b2, const uint8_t* dom, size_t i) {
  StepShared& sh = g_sh;
  for (int r = 0; r < kHotRes; ++r) { sh.bound[r] = b1[i * kHotRes + r]; sh.bound2[r] = b2[i * kHotRes + r]; }
  sh.front_bits = dom[i];
}
__device__ __forceinline__ void front_store(long long* b1, long long* b2, uint8_t* dom, size_t i) {
  const StepShared& sh = g_sh;
  for (int r = 0; r < kHotRes; ++r) { b1[i * kHotRes + r] = sh.bound[r]; b2[i * kHotRes + r] = sh.bound2[r]; }
  dom[i] = (uint8_t)sh.front_bits;
}

// NewNode + Add of template tm for the pod in g_row / g_pt, requirement part (thread 0): Tolerates, then Compatible + merge
// and the topology pin (t), on node slot `slot`. On success g_sh holds the node's requests (q, qp) and its requirement set's
// meta word: the template's, overlaid by what this Add touched. Shared by the generic step and the variant table.
__device__ __forceinline__ bool fresh_node_reqs(const ksched_template& tm, uint64_t p_tol, bool plain, uint32_t p_res, int slot, Touched& t) {
  KS_K2
  KS_ROW
  StepShared& sh = g_sh;
  const int R = c.n_res;
  bool ok = (p_tol >> tm.taintset) & 1;
  t.clear();
  if (ok && !plain) ok = requirements_phase(tm.reqs.values, tm.reqs.meta & 0xFFFFFFFFull, 1, 0, slot, false, t);
  if (!ok) return false;
  sh.qp = tm.daemon_res_present | p_res;
  for (int r = 0; r < KSCHED_MAX_RES; ++r) sh.q[r] = r < R ? tm.daemon_requests[r] + (((p_res >> r) & 1) ? row.requests[r] : 0) : 0;
  sh.meta = t.overlay_meta(tm.reqs.meta & 0xFFFFFFFFull);
  return true;
}

// One full Scheduler.add for one pod (existing nodes -> in-flight nodes -> new node -> relax/requeue). Every thread of
// the CTA calls it together. Kept out of line: the steady-state path in pack_kernel must stay a few KB of code, because a
// single resident CTA runs straight out of the instruction cache hierarchy (L0 ~6 KB, L1.5 32 KB).
// kExt: the problem has ext resources (DESIGN.md §3); without them every ext branch is compiled out.
template <bool kExt>
__device__ __noinline__ void generic_step(const PodRegs& cur, bool first_pass, int fpos_first, LoopVars& L) {
  KS_K2
  const int tid = threadIdx.x, lane = tid & 31;
  const int W32 = c.W32, V = c.n_templates, NE = s.n_existing, MAXN = s.max_new;
  const int R = c.n_res, RH = R < kHotRes ? R : kHotRes;
  Touched& fresh_t = g_fresh_t;
  TypeCtx& fresh_x = g_fresh_x;
  unsigned long long (*red)[32] = g_red;
  StepShared& sh = g_sh;
  const uint32_t* tmpl_taintset = g_tmpl_taintset;
  const Hot H = make_hot(s);
  const int64_t* alloc_sorted = alloc_table(c, s);
  int &n_new = L.n_new, &n_active = L.n_active, &tick = L.tick, &seq = L.seq, &parity = L.parity, &fatal = L.fatal;
  bool& pt_nonempty = L.pt_nonempty;
  long long& nodes_visited = L.nodes_visited;
#ifdef KSCHED_PROFILE_PACK
  long long gk_last = clock64();
#endif
    const uint32_t pod = cur.pod, cls = (uint32_t)cur.cls64;
    L.fresh_valid = 0;
    L.fail_memo = 0;
    const ksched_pod_row& row = g_row;
    const uint32_t p_res = cur.res;
    long long preq[kHotRes];
#pragma unroll
    for (int r = 0; r < kHotRes; ++r) preq[r] = cur.req[r];
    const uint64_t p_tol = cur.tol, p_hpc = cur.hpc, p_hpe = cur.hpe;
    const uint32_t p_keys = (uint32_t)(cur.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF, p_itype = cur.itype, p_hostname = cur.hostname;
    const bool has_topo = cur.topo_begin != cur.topo_end;
    if (!gen_stage(cur.row, cls, has_topo, L)) return;
    // ext resources (DESIGN.md §3): checked on every node this class is placed on, narrowed eagerly into new nodes' options.
    // A class that requests one is neither plain nor simple: no in-flight node accepts it without the full check.
    const uint32_t p_ext = kExt ? class_ext(s, cls) : 0u;
    const int X = c.n_res_ext;
    const bool plain = p_keys == 0 && !pt_nonempty && p_itype == KSCHED_NONE && p_hostname == KSCHED_NONE && !p_ext;  // no requirement can change
    const bool p_hpx = class_hp_ext(s, cls);  // host-port entries from id 64 on
    const bool simple = !has_topo && p_hpc == 0 && p_hpe == 0 && !p_hpx && !p_ext;  // the requirement verdict memo (HotSmem::absorbed/rejected) applies

    bool placed = false;
    const bool has_vol = class_has_volumes(s, cls);
    GK_T(kCtrGenTopo)
    // ------------------------------------------------------------ 1) existing nodes in caller order (scheduler.go:176-180)
    if (NE > 0) {
      // Every existing node below the class's cursor refuses this class for good: it is closed, its taints are not
      // tolerated, a host port or a volume limit is taken, or the requests no longer fit - all of which only get worse as
      // pods are added (existingnode.go:79-102). Rejections by requirements / topology can be lifted later and stop the cursor.
      const int start = s.cls_cursor[cls];
      unsigned mine = ~0u, soft = ~0u;  // first node this thread accepts / first node it did not refuse for good
      Touched t;
      t.clear();
      for (int e = start + tid; e < NE; e += blockDim.x) {
        if (s.ex_closed[e]) continue;
        if (!tolerates_node_set(s, p_tol, cls, s.ex_taintset[e])) continue;
        if (node_hp_conflict(s, p_hpc, p_hpx, cls, s.ex_hp, s.ex_hp_ext, NE, e)) continue;
        if (has_vol && node_vol_over(cls, e)) continue;
        bool ok = true;  // Fits(requests, available) comes first (existingnode.go:98-102)
        const uint32_t qp = s.ex_req_present[e] | p_res;
        for (int r = 0; r < R && ok; ++r) {
          if (!((qp >> r) & 1)) continue;
          long long q = s.ex_req[(size_t)r * NE + e] + (((p_res >> r) & 1) ? row.requests[r] : 0);
          long long a = ((s.ex_avail_present[e] >> r) & 1) ? s.ex_avail[(size_t)r * NE + e] : 0;
          ok = q <= a;
        }
        if (!ok || !ext_fits(s.ex_req_ext + e, s.ex_avail_ext + e, NE, s.cls_req_ext + (size_t)cls * X, p_ext)) continue;
        if (soft == ~0u) soft = (unsigned)e;
        if (p_itype != KSCHED_NONE) {
          const uint32_t it = s.ex_itype[e];
          bool allowed = it == KSCHED_NONE ? (s.itype_complement[p_itype] != 0) : ((s.itype_sets[(size_t)p_itype * W32 + (it >> 5)] >> (it & 31)) & 1);
          if (!allowed) continue;
        }
        if (!plain && !requirements_phase(s.ex_vals, s.ex_meta[e], NE, e, e, true, t)) continue;
        mine = (unsigned)e;
        break;  // this thread's remaining nodes have larger indices
      }
      unsigned w32, soft_min;
      block_min2_u32_db(mine, soft, red, parity, &w32, &soft_min);
      if (tid == 0) s.cls_cursor[cls] = soft_min == ~0u ? NE : (int)soft_min;  // read again only after the next step's barriers
      const unsigned long long w = w32 == ~0u ? ~0ull : (unsigned long long)w32;
      if (w != ~0ull) {
        const int e = (int)w;
        nodes_visited += e + 1;
        if (mine == w32) {  // the winning thread commits its own candidate
          if (!plain) commit_touched(t, s.ex_vals, s.ex_meta, NE, e);
          const bool closed = existing_add(s, R, e, p_res, row.requests, 1);
          ext_add(s.ex_req_ext + e, NE, s.cls_req_ext + (size_t)cls * X, p_ext);
          node_hp_commit(s, p_hpe, p_hpx, cls, s.ex_hp, s.ex_hp_ext, NE, e);
          if (s.ex_it && p_itype != KSCHED_NONE) itype_state_add(e, p_itype);
          if (has_vol) node_vol_commit(cls, e);
          s.ex_closed[e] = closed;
          s.assign[pod] = e;
          s.place_seq[pod] = seq;
        }
        ++seq;
        placed = true;
        __syncthreads();  // the commit is read by every thread in the next step
        if (has_topo) topo_record_block(s.ex_vals, s.ex_meta[e], NE, e, e);
      } else {
        nodes_visited += NE;
      }
    }
    GK_T(kCtrGenExisting)
    // ------------------------------------------------------------ 2) in-flight nodes, fewest pods first (scheduler.go:183-190)
    // Every thread checks candidates for everything except the instance-type options (requirements, topology, the
    // resource pre-test); the block argmin picks the first such node in the reference's order; the whole CTA then
    // verifies the winner's instance-type options word-parallel and, if they survive, narrows them in place. A winner
    // whose options do not survive is excluded and the argmin is repeated (after kMaxExcl such failures every candidate is
    // checked in full by its own thread, which needs no verification).
    if (!placed && n_active > 0 && !L.derive) {
      int n_excl = 0;
      bool full_eval = false;
      const bool two_stage = pt_nonempty;  // topology-constrained pod
      while (true) {
        unsigned long long mine = ~0ull;
        int best_a = -1, last_slow = -1;
        long long bq[kHotRes] = {0, 0, 0, 0};
        SlowEval ev;
        bool best_slow = false;
        for (int a = tid; a < n_active; a += blockDim.x) {
          const unsigned long long key = H.key(a);
          if (key >= mine) continue;  // cannot beat this thread's current candidate
          if (n_excl) {
            bool excluded = false;
            for (int i = 0; i < n_excl && i < kMaxExcl; ++i) excluded = excluded || sh.excl[i] == a;
            if (excluded) continue;
          }
          const unsigned short fl = H.flags(a);
          if (!((p_tol >> tmpl_taintset[fl >> 8]) & 1)) continue;  // Taints.Tolerates
          const uint32_t qp = ((fl >> 1) & 0xF) | p_res;
          long long q[kHotRes], b1[kHotRes], b2[kHotRes];
#pragma unroll
          for (int r = 0; r < kHotRes; ++r) { q[r] = H.q(r, a) + preq[r]; b1[r] = H.bound(r, a); b2[r] = H.bound2(r, a); }
          const int qf = quick_fit(q, qp, RH, b1, b2, fl);
          if (qf == 0) continue;
          if ((p_hpc || p_hpx) && node_hp_conflict(s, p_hpc, p_hpx, cls, s.nn_hp, s.nn_hp_ext, MAXN, H.node(a))) continue;
          if (simple && H.rejected(a) == cls) continue;  // memo: same class, node untouched since it was refused
          const bool fast = (plain || (simple && H.absorbed(a) == cls)) && qf == 1;  // nothing can change and an option holds the requests
          if (!fast) {
            if (two_stage && !full_eval) {  // necessary condition only; the winner is checked in full
              const int n = H.node(a);
              if (!topo_prefilter(s.nn_vals, s.nn_meta[n], MAXN, n, NE + n)) continue;
            } else {
              last_slow = a;
              if (!evaluate_slow<kExt>(plain, H.node(a), fl, q, alloc_sorted, full_eval, ev.t, ev)) {
                if (simple) H.rejected(a) = cls;
                continue;
              }
            }
          }
          mine = key;
          best_a = a;
          best_slow = !fast;
#pragma unroll
          for (int r = 0; r < kHotRes; ++r) bq[r] = q[r];
        }
        GK_T(kCtrGenEval)
        const unsigned long long wkey = block_min_u64_db(mine, red, parity);
        if (wkey == ~0ull) {
          nodes_visited += n_new;
          break;
        }
        const bool winner = mine == wkey;
        if (winner) {  // post the candidate for the cooperative instance-type check
          const int a = best_a;
          bool okw = true, in_shared = false;
          if (best_slow && last_slow != a) {
            // without the instance-type part the touched keys go straight into the CTA's shared Touched
            in_shared = !full_eval;
            okw = evaluate_slow<kExt>(plain, H.node(a), H.flags(a), bq, alloc_sorted, full_eval, in_shared ? fresh_t : ev.t, ev);
          }
          sh.win_a = a;
          sh.win_n = H.node(a);
          sh.win_fail = okw ? 0 : 1;
          sh.win_need = (okw && best_slow && ev.need_types) ? 1 : 0;
          sh.win_commit = (okw && best_slow && (ev.changed || p_itype != KSCHED_NONE || p_ext)) ? 1 : 0;
          if (sh.win_need) {
            if (!in_shared) fresh_t = ev.t;
            for (int r = 0; r < KSCHED_MAX_RES; ++r) sh.q[r] = r < R ? ev.q[r] : 0;
            sh.qp = ev.qp;
          }
        }
        __syncthreads();
        const int wa = sh.win_a, wn = sh.win_n;
        if (sh.win_fail) {  // the prefilter let through a node the full requirement check refuses
          exclude_winner(H, wa, simple, cls, n_excl, full_eval);
          continue;
        }
        const bool coop = sh.win_need != 0;
        bool opts_changed = false;
        if (coop) {
          // TypeCtx of the winner: requirement part by thread 0, one Fits rank per resource by the first lanes of warp 1
          const int rbase = blockDim.x >= 64 ? 32 : 0;
          if (tid == 0) build_type_ctx(fresh_t, sh.q, sh.qp, s.nn_vals, s.nn_meta[wn], MAXN, wn, false, alloc_sorted, fresh_x, rbase == 0);
          if (rbase && tid >= rbase && tid < rbase + R) {
            const int r = tid - rbase;
            fresh_x.rank[r] = ((sh.qp >> r) & 1) ? fit_rank(alloc_sorted, c.n_types, r, sh.q[r]) : 0;
          }
          __syncthreads();
          // one pass: requirement-narrowed word kept in a register, resource test on top of it
          uint32_t keep_base = 0, keep = 0;
          int local_any = 0;
          const int64_t* wn_ext = p_ext ? s.nn_req_ext + (size_t)wn * X : nullptr;
          for (int w = tid; w < W32; w += blockDim.x) {
            const uint32_t base = s.nn_opts[(size_t)w * MAXN + wn];
            if (!base) continue;
            const uint32_t sw = narrow_word(c, s, fresh_x, base, w, wn_ext, s.cls_req_ext + (size_t)cls * X, p_ext);
            if (w == tid) { keep_base = base; keep = sw; }
            if (sw && type_word_res(c, fresh_x, sw, w)) local_any = 1;
          }
          if (!__syncthreads_or(local_any)) {  // no option survives: Node.Add fails on this node (node.go:92-95)
            exclude_winner(H, wa, simple, cls, n_excl, full_eval);
            continue;
          }
          if (sh.win_commit) {  // requirement-driven narrowing of the stored options; resources stay lazy
            int local_changed = 0;
            if (tid < W32 && keep != keep_base) { s.nn_opts[(size_t)tid * MAXN + wn] = keep; local_changed = 1; }
            for (int w = tid + blockDim.x; w < W32; w += blockDim.x) {
              const uint32_t base = s.nn_opts[(size_t)w * MAXN + wn];
              if (!base) continue;
              const uint32_t sw = narrow_word(c, s, fresh_x, base, w, wn_ext, s.cls_req_ext + (size_t)cls * X, p_ext);
              if (sw != base) { s.nn_opts[(size_t)w * MAXN + wn] = sw; local_changed = 1; }
            }
            opts_changed = __syncthreads_or(local_changed) != 0;
          }
        }
        GK_T(kCtrGenInflightVerify)
        GK_C(kCtrGenInflightPlaced)
        if (s.count_visited) {  // rank of the winner among ALL in-flight nodes (the reference also walks the full ones)
          int less = 0;
          for (int i = tid; i < n_new; i += blockDim.x) less += order_key(s.nn_count[i], s.nn_tb[i]) < wkey;
          for (int o = 16; o; o >>= 1) less += __shfl_xor_sync(0xffffffffu, less, o);
          __syncthreads();
          if (tid == 0) sh.visited = 0;
          __syncthreads();
          if (lane == 0 && less) atomicAdd((unsigned long long*)&sh.visited, (unsigned long long)less);
          __syncthreads();
          nodes_visited += sh.visited + 1;
        }
        if (winner) {  // the winning thread commits its own candidate
          const int a = best_a;
          const int n = wn;
          unsigned short fl = H.flags(a);
#pragma unroll
          for (int r = 0; r < kHotRes; ++r) H.q(r, a) = bq[r];
          for (int r = kHotRes; r < R; ++r)
            if ((p_res >> r) & 1) s.nn_req[(size_t)r * MAXN + n] += row.requests[r];
          if ((p_res >> kHotRes) || ((p_res & 0xF) & ~((fl >> 1) & 0xF))) s.nn_req_present[n] |= p_res;
          fl |= (unsigned short)((p_res & 0xF) << 1);
          node_hp_commit(s, p_hpe, p_hpx, cls, s.nn_hp, s.nn_hp_ext, MAXN, n);
          if (s.nn_it && p_itype != KSCHED_NONE) itype_state_add(NE + n, p_itype);  // idempotent on a node that absorbed the class
          const int count = (int)(wkey >> 32) + 1;
          s.nn_count[n] = count;
          s.nn_tb[n] = -(tick + 1);  // front of the next pod-count block under a stable sort
          H.key(a) = order_key(count, -(tick + 1));
          if (best_slow && (ev.changed || p_itype != KSCHED_NONE || p_ext)) {
            long long nb1[kHotRes], nb2[kHotRes];
            unsigned short fb;
            bool new_front = true;
            if (coop) {
              commit_reqs(n, fresh_t);
              if (opts_changed) compute_front(s.nn_opts, MAXN, n, nb1, nb2, &fb);
              else new_front = false;  // same option set, same Pareto front
            } else {
              uint64_t meta;
              commit_slow<kExt>(n, ev, nb1, nb2, &fb, &meta);
            }
            if (new_front) {
#pragma unroll
              for (int r = 0; r < kHotRes; ++r) { H.bound(r, a) = nb1[r]; H.bound2(r, a) = nb2[r]; }
              fl = (unsigned short)((fl & ~(kFlExact | kFlTwo)) | fb);
            }
          }
          if (p_ext) {  // after the narrowing above, which read the node's sums before this pod
            ext_add(s.nn_req_ext + (size_t)n * X, 1, s.cls_req_ext + (size_t)cls * X, p_ext);
            s.nn_ext_present[n] |= p_ext;
          }
          H.flags(a) = fl;
          H.rejected(a) = KSCHED_NONE;
          if (simple) H.absorbed(a) = cls;
          long long cb1[kHotRes], cb2[kHotRes];
#pragma unroll
          for (int r = 0; r < kHotRes; ++r) { cb1[r] = H.bound(r, a); cb2[r] = H.bound2(r, a); }
          const bool closed = node_closed(bq, s.min_req, RH, cb1, cb2, fl);
          s.assign[pod] = NE + n;
          s.place_seq[pod] = seq;
          if (closed) {  // the node leaves the active set: its request vector goes back to global memory
            for (int r = 0; r < RH; ++r) s.nn_req[(size_t)r * MAXN + n] = bq[r];
            if (a != n_active - 1) H.move(a, n_active - 1);
          }
          sh.placed_closed = closed ? 1 : 0;
        }
        ++tick;
        ++seq;
        placed = true;
        __syncthreads();
        GK_T(kCtrGenInflightWinner)
        if (sh.placed_closed) --n_active;
        if (has_topo) topo_record_block(s.nn_vals, s.nn_meta[wn], MAXN, wn, NE + wn);  // Topology.Record, one relation per thread
        GK_T(kCtrGenInflightRecord)
        break;
      }
    } else if (!placed) {
      nodes_visited += n_new;  // every in-flight node is full; the reference still walks them
    }
    GK_T(kCtrGenCommit)
    // ------------------------------------------------------------ 3) open a new node, templates in weight order (scheduler.go:194-217)
    if (!placed) {
      if (!L.derive) { GK_C(kCtrGenFreshSteps) }
      const bool f_valid = s.use_F && (first_pass || s.relax_level[pod] == 0);  // K1's row is valid while the pod has its original class
      const uint32_t fpos = first_pass ? (uint32_t)fpos_first : s.pod_pos[pod];
      const bool no_column = f_valid && s.best[fpos] == kNoBest;  // no feasible (template, type) column at all
      if (no_column) nodes_visited += V;
      for (int v = 0; v < V && !placed && !no_column; ++v) {
        const ksched_template& tm = c.templates[v];
        ++nodes_visited;
        if (n_new >= MAXN) { fatal = KSCHED_ERR_OVERFLOW; break; }
        const int n = n_new;  // tentative slot: the hostname placeholder of this attempt (node.go:46)
        const bool limits_active = tm.has_limits && tm.limit_present;
        // Without topology and provisioner limits the outcome of NewNode+Add depends on (class, template) only: memoised.
        const bool memo = !pt_nonempty && !limits_active;
        const size_t fc = ((size_t)cls * V + v);
        __syncthreads();
        if (tid == 0) {
          int path = kPathReject;
          const uint8_t st = memo ? s.fc_state[fc] : 0;
          if (st == 1) path = kPathCached;
          else if (st == 2) path = kPathCachedEmpty;
          else {
            if (fresh_node_reqs(tm, p_tol, plain, p_res, NE + n, fresh_t)) {
              const bool same = f_valid && fresh_t.fin_is_merged();  // topology left every requirement exactly as K1 saw it
              const uint64_t meta = sh.meta;
              sh.fd_slot = -1;
              if (same) path = kPathRow;
              else {
                path = kPathDynamic;
                if (!memo && !limits_active) {  // topology-constrained class: outcome memo keyed by the node's requirement set
                  uint64_t vals[KSCHED_MAX_KEYS];
                  uint64_t hsh = ((uint64_t)fc + 1) * 0x9E3779B97F4A7C15ull ^ meta;
                  for (int k = 0; k < c.n_keys; ++k) {
                    const uint64_t val = ((fresh_t.keys >> k) & 1) ? fresh_t.fin[k] : tm.reqs.values[k];
                    vals[k] = val;
                    hsh = (hsh ^ val) * 0xBF58476D1CE4E5B9ull;
                    hsh ^= hsh >> 29;
                  }
                  const int slot = (int)((hsh >> 13) & (uint64_t)(s.fd_cap - 1));
                  const uint8_t st = s.fd_state[slot];
                  bool hit = st != 0 && s.fd_fc[slot] == (uint32_t)fc && s.fd_meta[slot] == meta;
                  for (int k = 0; k < c.n_keys && hit; ++k) hit = s.fd_vals[(size_t)slot * KSCHED_MAX_KEYS + k] == vals[k];
                  sh.fd_slot = slot;
                  if (hit) path = st == 1 ? kPathDynCached : kPathDynEmpty;
                  else {
                    s.fd_state[slot] = 0;  // being refilled: tags now, state when the outcome is known
                    s.fd_fc[slot] = (uint32_t)fc;
                    s.fd_meta[slot] = meta;
                    for (int k = 0; k < c.n_keys; ++k) s.fd_vals[(size_t)slot * KSCHED_MAX_KEYS + k] = vals[k];
                  }
                }
                if (path == kPathDynamic)
                  build_type_ctx(fresh_t, sh.q, sh.qp, tm.reqs.values, tm.reqs.meta & 0xFFFFFFFFull, 1, 0, true, alloc_sorted, fresh_x);
              }
            } else if (memo) {
              s.fc_state[fc] = 2;
            }
          }
          sh.path = path;
          sh.any = 0;
        }
        __syncthreads();
        const int path = sh.path;
        GK_C(kCtrGenPath + (path > 4 ? 4 : path))
        GK_T(kCtrGenFreshDecide)
        if (path == kPathReject || path == kPathCachedEmpty || path == kPathDynEmpty) continue;
        const int fd_slot = (path == kPathDynamic || path == kPathDynCached) ? sh.fd_slot : -1;
        const int a = n_active;
        if (path == kPathCached) {
          for (int w = tid; w < W32; w += blockDim.x) s.nn_opts[(size_t)w * MAXN + n] = s.fc_opts[fc * W32 + w];
          if (tid < c.n_keys) s.nn_vals[(size_t)tid * MAXN + n] = s.fc_vals[fc * KSCHED_MAX_KEYS + tid];
        } else {
          bool local_any = false;
          for (int w = tid; w < W32; w += blockDim.x) {
            uint32_t base = c.member[(size_t)v * W32 + w];
            if (base && limits_active) {  // filterByRemainingResources (scheduler.go:293-309)
              uint32_t m = base;
              while (m) {
                const int b = __ffs(m) - 1;
                m &= m - 1;
                const int t = w * 32 + b;
                for (int r = 0; r < R; ++r)
                  if (((tm.limit_present >> r) & 1) && c.capacity[(size_t)t * KSCHED_MAX_RES + r] > s.remaining[(size_t)v * KSCHED_MAX_RES + r]) base &= ~(1u << b);
              }
            }
            uint32_t sw = 0;
            if (path == kPathDynCached) sw = s.fd_opts[(size_t)fd_slot * W32 + w];
            else if (base) sw = path == kPathRow ? (base & s.F[((size_t)fpos * V + v) * W32 + w]) : type_word(c, s, fresh_x, base, w);
            if (sw && p_ext && path == kPathDynamic) sw = ext_fit_word(c, nullptr, s.cls_req_ext + (size_t)cls * X, p_ext, sw, w);  // (F has them)
            s.nn_opts[(size_t)w * MAXN + n] = sw;
            if (memo) s.fc_opts[fc * W32 + w] = sw;
            if (path == kPathDynamic && fd_slot >= 0) s.fd_opts[(size_t)fd_slot * W32 + w] = sw;
            local_any = local_any || sw;
          }
          if (local_any) atomicOr(&sh.any, 1u);
          if (tid < c.n_keys) {
            const uint64_t val = ((fresh_t.keys >> tid) & 1) ? fresh_t.fin[tid] : tm.reqs.values[tid];
            s.nn_vals[(size_t)tid * MAXN + n] = val;
            if (memo) s.fc_vals[fc * KSCHED_MAX_KEYS + tid] = val;
          }
          __syncthreads();
          if (!sh.any) {
            if (memo && tid == 0) s.fc_state[fc] = 2;
            if (path == kPathDynamic && fd_slot >= 0 && tid == 0) s.fd_state[fd_slot] = 2;
            continue;
          }
        }
        GK_T(kCtrGenFreshWords)
        // the Pareto front of a new option set, with every thread (the words were stored before the barrier above)
        const bool front_memo_hit = path == kPathRow && !limits_active && s.fc_front_state[fc];
        const bool front_fresh = path != kPathCached && path != kPathDynCached && !front_memo_hit;
        if (front_fresh) compute_front_block(s.nn_opts, MAXN, n, sh.bound, sh.bound2, &sh.front_bits, red, parity);
        // ---- commit the new node (NewNode + Add, node.go:44-107) — one thread, everything else was written above
        __syncthreads();
        if (tid == 0) {
          uint64_t meta;
          if (path == kPathCached) {
            meta = s.fc_meta[fc];
            front_load(s.fc_bound, s.fc_bound2, s.fc_dom, fc);
            sh.qp = s.fc_qp[fc];
            for (int r = 0; r < KSCHED_MAX_RES; ++r) sh.q[r] = s.fc_q[fc * KSCHED_MAX_RES + r];
          } else {
            meta = sh.meta;
            // K1-row path without limits: the option set, hence its Pareto front, depends on (class, template) only
            const bool front_memo = path == kPathRow && !limits_active;
            if (front_memo && s.fc_front_state[fc]) {
              front_load(s.fc_bound, s.fc_bound2, s.fc_dom, fc);
            } else if (path == kPathDynCached) {
              front_load(s.fd_bound, s.fd_bound2, s.fd_dom, fd_slot);
            } else {  // (front_fresh: computed by the CTA above)
              if (front_memo) {
                front_store(s.fc_bound, s.fc_bound2, s.fc_dom, fc);
                s.fc_front_state[fc] = 1;
              }
              if (path == kPathDynamic && fd_slot >= 0) {
                front_store(s.fd_bound, s.fd_bound2, s.fd_dom, fd_slot);
                s.fd_state[fd_slot] = 1;
              }
            }
            if (memo) {
              s.fc_meta[fc] = meta;
              front_store(s.fc_bound, s.fc_bound2, s.fc_dom, fc);
              s.fc_qp[fc] = sh.qp;
              for (int r = 0; r < KSCHED_MAX_RES; ++r) s.fc_q[fc * KSCHED_MAX_RES + r] = sh.q[r];
              s.fc_state[fc] = 1;
            }
          }
          // requests and ext sums first, as the class runs write them (the same thread, no barrier before open_node)
          for (int r = 0; r < KSCHED_MAX_RES; ++r) s.nn_req[(size_t)r * MAXN + n] = sh.q[r];
          if (kExt) {  // a fresh node's ext sums are the pod's: no daemonset requests an ext resource
            for (int x = 0; x < X; ++x) s.nn_req_ext[(size_t)n * X + x] = ((p_ext >> x) & 1) ? s.cls_req_ext[(size_t)cls * X + x] : 0;
            s.nn_ext_present[n] = p_ext;
          }
          open_node(s, n, v, meta, sh.qp, p_hpe, p_hpx, cls, p_itype, true, tick + 1);  // appended: last of the one-pod block
          const bool closed = node_closed(sh.q, s.min_req, RH, sh.bound, sh.bound2, sh.front_bits);
          if (!closed) {
            H.key(a) = order_key(1, tick + 1);
            for (int r = 0; r < kHotRes; ++r) { H.q(r, a) = sh.q[r]; H.bound(r, a) = sh.bound[r]; H.bound2(r, a) = sh.bound2[r]; }
            H.node(a) = n;
            H.flags(a) = (unsigned short)(sh.front_bits | ((sh.qp & 0xF) << 1) | (v << 8));
            H.absorbed(a) = simple ? cls : KSCHED_NONE;
            H.rejected(a) = KSCHED_NONE;
          }
          sh.placed_closed = closed ? 1 : 0;
          if (!L.derive) {
            s.assign[pod] = NE + n;
            s.place_seq[pod] = seq;
          }
          if (limits_active) {  // subtractMax (scheduler.go:273-290): largest capacity among the surviving options
            for (int r = 0; r < R; ++r) {
              if (!((tm.limit_present >> r) & 1)) continue;
              long long mx = INT64_MIN;
              for (int w = 0; w < W32; ++w) {
                uint32_t m = s.nn_opts[(size_t)w * MAXN + n];
                while (m) {
                  const int b = __ffs(m) - 1;
                  m &= m - 1;
                  const long long cp = c.capacity[(size_t)(w * 32 + b) * KSCHED_MAX_RES + r];
                  mx = cp > mx ? cp : mx;
                }
              }
              if (mx != INT64_MIN) s.remaining[(size_t)v * KSCHED_MAX_RES + r] -= mx;
            }
          }
        }
        ++tick;
        ++seq;
        __syncthreads();
        if (has_topo && !L.derive) topo_record_block(s.nn_vals, s.nn_meta[n], MAXN, n, NE + n);  // Topology.Record, one relation per thread
        ++n_new;
        if (!sh.placed_closed) { L.fresh_valid = 1; L.fresh_a = n_active; L.fresh_cls = cls; ++n_active; }
        placed = true;
        GK_T(kCtrGenFreshCommit)
      }
      if (fatal) return;
    }
    GK_T(kCtrGenFresh)
    if (!placed && !L.derive) gen_requeue(pod, has_topo, L);
  }

// no requirement of the pod can change a node's requirements
__device__ __forceinline__ bool plain_pod_regs(const PodRegs& r) {
  return ((r.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF) == 0 && r.itype == KSCHED_NONE && r.hostname == KSCHED_NONE && r.topo_begin == r.topo_end;
}

// ---- class-run loop ------------------------------------------------------------------------------------------------
// Consecutive pods of the queue usually belong to ONE class (a deployment: identical row, identical topology terms). For
// such a run the whole CTA stays in this loop: ONE block barrier per pod, no global load and (almost) no global store on
// the chain, ~120 instructions per warp and pod.
//  * every open node is owned by thread (slot % blockDim): only its owner ever reads or writes its state, so a commit
//    needs no barrier to become visible; the block argmin carries a payload (slot, domains) from which every warp updates
//    its own copy of the spread counters;
//  * everything the accept test of a run needs from a node collapses into ONE word per node, `rp`:
//      room   = how many more pods of THIS class fit by the exact Pareto-front resource test (computed once per run with
//               integer divisions, decremented by the commits; 0 also covers untolerated taints / a memoised refusal,
//               kRoomSlow = "verdict not exact here"),
//      dead   = a hostname-keyed group of the class (anti-affinity, hostname spread) no longer admits the node - known at
//               the commit that fills it, because only this run's commits change those counts,
//      placed = pods of the run the node took; requests, order statistics and hostname counters are written back from it
//               when the run ends;
//    plus, per spread key of the class, the node's admissible domains (`zv`);
//  * a candidate is accepted here only when the verdict is EXACT and nothing but counters changes: requirements untouched
//    (plain / absorbed classes) or a spread domain that is already pinned on the node - or that can be pinned without
//    touching the option set (DevCatalog::pin_neutral). Any other winner or a pod that fails hands the pod to generic_step
//    (status 1); a fresh node of a shape not seen before in the run has its variant derived first (run_derive, status 3);
//  * a node that becomes full is tombstoned (key = ~0) and the active list is compacted when the run ends; assignments
//    are staged per queue chunk and stored coalesced;
//  * fresh nodes replay a VARIANT: NewNode+Add for (class, template, resulting requirement masks) is a pure function
//    when no provisioner limit is active (same argument as PackState::fd_*), so a node generic_step created for this
//    class (last before the run, or in derive mode for the run) is captured (options, masks, requests, Pareto front) and
//    replayed for every later pod of the run whose spread domains come out the same.
constexpr int kRunHost = 4;      // hostname-keyed relations of a run-eligible class
constexpr int kRunMask = 2;      // spread relations over a mask key
constexpr int kRunDom = 16;      // domains of such a key
constexpr int kTopoCap = 768;    // open nodes whose per-class topology inputs fit in shared memory
constexpr int kRunVariants = 4;
constexpr int kRunW32 = 64;      // option words a variant holds (T <= 2048)
constexpr int kRunWarps = kPackThreads / 32;
constexpr int kRunChunk = 128;   // queue entries staged in shared memory at a time
constexpr unsigned kRoomSlow = 0xFFFFu, kRoomMax = 0x7FFEu, kRpDead = 0x80000000u;
// why a class run stopped with status 1 (profile: kCtrNoVariantStops + cause - 1): no variant for the fresh node's domain, a
// winner whose verdict is not exact (kRoomSlow), a capacity guard (MAXN, kActCap, kTopoCap), anything else (a pin that is not
// neutral, no admissible domain or hostname for a fresh node)
enum StopCause : int { kStopNone, kStopNoVariant, kStopRoomSlow, kStopCapacity, kStopOther };
constexpr size_t kRunArrayBytes = (size_t)kTopoCap * (kRunMask * 4 + kRunHost * 2) + (size_t)kActCap * 4;

// RunVariant lives in pack_state.cuh (PackState points at the variant table) with the same three sizes
static_assert(sizeof(RunVariant::b1) == kHotRes * sizeof(long long) && sizeof(RunVariant::dom) == kRunMask && sizeof(RunVariant::opts) == kRunW32 * 4,
              "RunVariant is sized by kHotRes, kRunMask and kRunW32");
static_assert(sizeof(RunRec::h_row) == kRunHost * 4 && sizeof(RunRec::m_group) == kRunMask * 4, "RunRec is sized by kRunHost and kRunMask");
struct RunCtx {
  uint32_t cls;           // class the variants belong to (KSCHED_NONE: none)
  int eligible;
  int n_var, var_next;
  int tomb;               // nodes tombstoned by the current run
  RunRec rec;             // the class's relation tables (PackState::run_rec)
  int h_inc[kRunHost];    // hostnames that got their first matching pod in this run (grp_host_total)
  int h_zero;             // bit j: hostname relation j's group counted no slot at entry (grp_host_total 0: every count is 0)
  uint32_t m_registered[kRunMask];
  int32_t cnt[kRunWarps][kRunMask][kRunDom];  // one copy of the spread counters per warp (updated by its lane 0)
  unsigned long long red_key[2][32];
  unsigned red_pay[2][32];
  uint32_t q_pod[2][kRunChunk], q_cls[2][kRunChunk];  // upcoming queue entries (pod, class), double-buffered
  int32_t q_node[2][kRunChunk];                        // where the entry was placed (ksched_result.assign)
  int q_end[2];           // first staged entry of another class (or the chunk length), per buffer
  int lv_cnt[2];          // level step: members appended to the tie list (double-buffered)
  int lv_fill[2];         // fill step: pods the only eligible node takes
  RunVariant var[kRunVariants];
  int vt_got;             // block-wide fetch: ring slot the variant table filled, or -1
};
__shared__ RunCtx g_rc;

// ---- mask run: the class-run loop for ONE spread relation over a mask key (zone spread), driven by warp 0 alone ----------
// The accepting nodes are kept in singly linked lists in the reference's order (pod count, then tie-break), one per
// domain they are pinned to plus one for the nodes not pinned yet; they are sorted once per run (buckets by list and count,
// ranks by counting inside the bucket). An accepting node moves to the FRONT of the block of count + 1 of its domain's
// list (its new tie-break is the smallest so far), a fresh node goes to the END of the block of count 1. Each lane keeps
// the head of its list, the node after it and the tail of the head's bucket in registers, so a pod's node is the smallest
// head key over the lists of the admissible domains: a few warp reductions, no block barrier and no shared-memory load on
// the critical path instead of a scan of every open node. Anything the lists cannot represent hands the run back to the
// per-pod loop.
constexpr int kM1Dom = 8;             // domains with ids < kM1Dom; list kM1Dom holds the nodes that admit every registered domain
constexpr int kM1Lists = kM1Dom + 1;
constexpr int kM1Lv = 12;             // pod counts < kM1Lv
constexpr uint16_t kM1None = 0xFFFF;
struct M1Ctx {
  uint16_t tl[kM1Lv][kM1Lists];       // last node of the bucket (kM1None: empty)
  uint16_t head[kM1Lists];            // first node of the list (between two entries of the mask run)
  uint16_t ap[kM1Lv][kM1Lists];       // build: the bucket is arr[ap .. ae)
  uint16_t ae[kM1Lv][kM1Lists];
  union {
    int bcnt[kM1Lv * kM1Lists];       // build: members per bucket (bucket = list * kM1Lv + count)
    unsigned long long rk[32];        // round stretch (after the build): the key of each node, round by round
  };
  int bad;                            // build: a node the lists cannot represent
  int upos;                           // position of the unpinned list's head in arr: that list never gains a member (a node
                                      // leaves it when a pod pins it, fresh nodes are pinned), so it is the rest of the
                                      // segment the build sorted, and the pin step reads its next members without the links
  uint16_t ps[32];                    // pin step: the node of each pod; round stretch: the node of each (round, domain)
  int out_adv, out_reason, out_tick, out_n_new, out_n_active, out_why;  // out_why: StopCause of out_reason 1
  int n_fresh;                        // nodes created by this entry of the mask run: slot | variant << 16; their global
  uint32_t fr[kRunChunk];             // state (option words, requirement values, requests, ...) is stored by the CTA afterwards
};
__shared__ M1Ctx g_m1;

// ---- variant table: every fresh-node variant a class run can replay, built before the pack kernel (vt_build_block) ------
// With no provisioner limit NewNode + Add of a run class's fresh node depends on the class row, the template and the domain
// its mask relation pins (the fresh hostname's counts are the relations' times), so entry (cls, d) is the variant that
// run_derive + run_capture would store for the class and domain d (d = 0 without a mask relation), or none (vt_ok 0).
constexpr int kVtClasses = 1024;  // classes the table covers (ids below; the others derive their variants)
__device__ __forceinline__ size_t vt_index(unsigned cls, int d) { return (size_t)cls * kM1Dom + d; }
// the table holds the variant of (cls, d) (uniform: every thread reads the same flag)
__device__ __forceinline__ bool vt_has(const PackState& s, unsigned cls, int n_mask, int d) {
  return n_mask < 2 && cls < (unsigned)s.vt_classes && d < s.vt_ndom && s.vt_ok[vt_index(cls, d)] != 0;
}
// warp-wide: copies the table's variant of (cls, d) into ring slot rc.var_next; returns the slot, or -1 when vt_has is false
__device__ int vt_fetch(RunCtx& rc, unsigned cls, int n_mask, int d, int lane) {
  KS_K2
  if (!vt_has(s, cls, n_mask, d)) return -1;
  const int slot = rc.var_next;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&s.vtable[vt_index(cls, d)]);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&rc.var[slot]);
  for (int w = lane; w < (int)(sizeof(RunVariant) / 4); w += 32) dst[w] = src[w];
  __syncwarp();
  if (lane == 0) {
    rc.var_next = (slot + 1) % kRunVariants;
    if (rc.n_var < kRunVariants) rc.n_var++;
    s.counters[kCtrVtFetches] += 1;
  }
  __syncwarp();
  return slot;
}

struct RunIO {
  int qi, head, qlen, tick, seq, n_active, n_new, parity;
  long long add_calls;
  int placed;        // pods this call consumed
  int status;        // 0 the run ended (class change / end of the first pass); 1 the pod at qi needs generic_step; 2 class not
                     // eligible; 3 the pod at qi needs a variant derived (see resume)
  int fresh_valid, fresh_a;  // in: generic_step has just created node slot fresh_a for fresh_cls (nothing happened since)
  uint32_t fresh_cls;
  int staged;        // out: a variant was derived in the run (run_derive), so g_row and g_pt hold this class's row and topology
  // status 3: the pod at qi needs a variant the run does not have. Nothing is written back: the pack loop derives the variant
  // (run_derive) and re-enters with `resume`, and the run goes on from the state it left in shared memory and in these fields
  // (its first queue position and seq, the staged chunk, the level parity, the mask-run flags, the pod derived for)
  int resume;
  int r_qi0, r_seq0, r_cb, r_buf, r_lvp, r_m1, r_derived;
};
__shared__ RunIO g_rio;

constexpr unsigned kFull = 0xffffffffu;
// first domain in (count, id) order among `cand` (non-empty)
__device__ __forceinline__ int run_pick(uint32_t cand, const int32_t* cn) {
  int d = __ffs(cand) - 1;
  cand &= cand - 1;
  int32_t best = cn[d];
  while (cand) {
    const int e = __ffs(cand) - 1;
    cand &= cand - 1;
    if (cn[e] < best) { best = cn[e]; d = e; }
  }
  return d;
}
// run_pick with one domain per lane (warp-wide): the lowest lane among those `in` with the fewest count
__device__ __forceinline__ int warp_pick(bool in, int cnt) {
  const int mc = __reduce_min_sync(0xffffffffu, in ? cnt : INT32_MAX);
  return __ffs(__ballot_sync(0xffffffffu, in && cnt == mc)) - 1;
}
// How many more pods with request vector `req` (keys `res`) the node at slot a can take: exact by the Pareto front of its
// options (quick_fit for the k-th pod <=> k <= room); kRoomSlow when the front is not exact.
// Room of a node with flags fl, hot requests q and front (b1, b2).
__device__ __forceinline__ unsigned room_of(unsigned short fl, const long long* q, const long long* b1, const long long* b2, const long long* req,
                                            uint32_t res, int RH) {
  const uint32_t qp = ((fl >> 1) & 0xF) | res;
  long long best = 0;
  bool inexact_ok = true;
  for (int f = 0; f < 2; ++f) {
    if (f == 1 && !(fl & kFlTwo)) break;
    long long rf = kRoomMax;
    for (int r = 0; r < RH; ++r) {
      if (!((qp >> r) & 1)) continue;
      const long long slack = (f ? b2[r] : b1[r]) - q[r];
      if (req[r] > 0) {
        const long long k = slack < req[r] ? 0 : slack / req[r];
        rf = k < rf ? k : rf;
      } else if (slack < 0) rf = 0;
    }
    if (f == 0) inexact_ok = rf > 0;
    best = rf > best ? rf : best;
  }
  if (!(fl & kFlExact)) return inexact_ok ? kRoomSlow : 0;  // per-resource maxima only: a necessary test
  return (unsigned)best;
}
__device__ __noinline__ unsigned run_room(const HotSmem* hs, int a, const long long* req, uint32_t res, int RH) {
  long long q[kHotRes], b1[kHotRes], b2[kHotRes];
#pragma unroll
  for (int r = 0; r < kHotRes; ++r) { q[r] = hs->q[r][a]; b1[r] = hs->bound[r][a]; b2[r] = hs->bound2[r][a]; }
  return room_of(hs->flags[a], q, b1, b2, req, res, RH);
}
// A fresh node's room word for the class: its room, dead when one of its hostname relations refuses the node's count
// after its first pod (the relation's times)
__device__ __forceinline__ uint32_t fresh_room_word(unsigned room, int n_host, const uint8_t* times, const int* lim) {
  for (int j = 0; j < n_host; ++j) if ((int)times[j] > lim[j]) room |= kRpDead;
  return room;
}
// A commit's Topology.Record for the class's hostname groups: t more pods on the node at slot a (counters saturate at
// 0xFFFF). Returns the room word rp with t pods moved from room to placed, dead once a group no longer admits the node.
__device__ __forceinline__ uint32_t run_record_host(const RunCtx& rc, uint16_t* hc, int n_host, int a, uint32_t rp, int t) {
  uint32_t rp2 = rp - (uint32_t)t + ((uint32_t)t << 16);
#pragma unroll
  for (int j = 0; j < kRunHost; ++j) {
    if (j >= n_host) break;
    const int times = rc.rec.h_times[j];
    const int old = hc[j * kTopoCap + a];
    const int now = old + t * times > 0xFFFF ? 0xFFFF : old + t * times;
    if (times) hc[j * kTopoCap + a] = (uint16_t)now;
    if (now > rc.rec.h_lim[j]) rp2 |= kRpDead;
  }
  return rp2;
}
// A commit left the node at slot a no room for the class (room word rp, room 0): true when no pod of the batch fits it
// any more either (node_closed on the run's start requests plus the placed pods) - the node leaves the active set. The
// callers test the room first, in their own condition: a bool merged from an early return here costs the one-warp
// level / fill loop a branch and a convergence barrier per commit.
__device__ __forceinline__ bool run_closes(const HotSmem* hs, int a, uint32_t rp, const long long* p_req, const long long* min_req, int RH) {
  const int placed = (rp >> 16) & 0x7FFF;
  long long nq[kHotRes], b1[kHotRes], b2[kHotRes];
#pragma unroll
  for (int r = 0; r < kHotRes; ++r) { nq[r] = hs->q[r][a] + placed * p_req[r]; b1[r] = hs->bound[r][a]; b2[r] = hs->bound2[r][a]; }
  return node_closed(nq, min_req, RH, b1, b2, hs->flags[a]);
}

// A slot's domain word for one mask relation, from the node's requirement r on key k (dictionary mask dict): bits 0..15
// the domains r admits, kZvExact when r is an In, kZvPresent when the node has a requirement on the key
constexpr uint32_t kZvExact = 1u << 16, kZvPresent = 1u << 17;
__device__ __forceinline__ uint32_t zv_word(const Req& r, uint32_t dict, int k) {
  KS_K2
  const uint32_t allowed = r.present ? (uint32_t)ksched::req_allowed(r, dict, key_meta(c, k)) : dict;
  return allowed | ((r.present && !r.complement) ? kZvExact : 0) | (r.present ? kZvPresent : 0);
}
// the word of a node pinned to domain d (requirements.Add(In{d})): a node is pinned to one domain exactly when its word
// has this form
__device__ __forceinline__ uint32_t zv_pinned(int d) { return (1u << d) | kZvExact | kZvPresent; }

// The class run's constants for one call, shared by its steps (all inlined into class_run)
struct RunEnv {
  HotSmem* hs;
  uint32_t* zv;   // [kRunMask][kTopoCap] domain words (zv_word)
  uint32_t* rpv;  // [kActCap] room | placed << 16 | dead
  uint16_t* hc;   // [kRunHost][kTopoCap] the hostname groups' counts
  int NE, MAXN, W32, RH, hstride, n_host, n_mask;
  unsigned cls;
  bool topo, simple;
  long long p_req[kHotRes], min_req[kHotRes];
  // relation constants of the commit
  uint32_t m_reg0, m_reg1;
  int m_bias0, m_bias1;
  bool m_rec0, m_rec1;
  // mask run: its lists live in the second mask relation's plane, which is unused (n_mask == 1)
  __device__ __forceinline__ uint16_t* m1_arr() const { return reinterpret_cast<uint16_t*>(zv + kTopoCap); }
  __device__ __forceinline__ uint16_t* m1_nxt() const { return m1_arr() + kTopoCap; }
};

// A commit settles the node at slot a with room word rp2 and order (count, tb): the new order key, or - once the class no
// longer fits anywhere on it (run_closes) - the tombstone key ~0 with the order kept in nn_last. Returns whether the node
// closed; the caller counts the tombstone.
__device__ __forceinline__ bool run_settle(const RunEnv& e, int a, uint32_t rp2, int count, int tb) {
  unsigned long long key = order_key(count, tb);
  bool closed = false;
  if ((rp2 & 0xFFFF) == 0 && run_closes(e.hs, a, rp2, e.p_req, e.min_req, e.RH)) {
    key = ~0ull;
    e.hs->nn_last[a] = ((unsigned long long)(unsigned)count << 32) | (unsigned)tb;
    closed = true;
  }
  e.hs->key[a] = key;
  e.rpv[a] = rp2;
  return closed;
}
// NewNode + Add replayed from variant v on the fresh slot a (node n) with order (1, tb): hot state, room word and the
// hostname counts of its one pod (grp_host now; the run's write-back stores the counts of later pods)
__device__ __forceinline__ void run_fresh(const RunEnv& e, const RunVariant& v, int a, int n, int tb) {
  KS_K2
  const RunCtx& rc = g_rc;
  HotSmem* hs = e.hs;
  for (int j = 0; j < e.n_host; ++j) {
    const int times = rc.rec.h_times[j];
    e.hc[j * kTopoCap + a] = (uint16_t)times;
    if (times) s.grp_host[(size_t)rc.rec.h_row[j] * e.hstride + e.NE + n] = (uint16_t)times;
  }
  hs->key[a] = order_key(1, tb);
#pragma unroll
  for (int r = 0; r < kHotRes; ++r) { hs->q[r][a] = v.q[r]; hs->bound[r][a] = v.b1[r]; hs->bound2[r][a] = v.b2[r]; }
  hs->node[a] = n;
  hs->flags[a] = v.fl;
  hs->absorbed[a] = e.simple ? e.cls : KSCHED_NONE;
  hs->rejected[a] = KSCHED_NONE;
  e.rpv[a] = v.rp;
}
// requirements.Add(In{d}) of spread relation j on the node at slot a. Two reductions instead of a read-modify-write of
// nn_meta: the load would stall the commit for an L2 round trip (a node has one writer, and nothing in the run reads it).
__device__ __forceinline__ void run_pin(const RunEnv& e, int j, int a, int d) {
  KS_K2
  const int n = e.hs->node[a], k = g_rc.rec.m_key[j];
  e.zv[j * kTopoCap + a] = zv_pinned(d);
  s.nn_vals[(size_t)k * e.MAXN + n] = 1ull << d;
  atomicOr(reinterpret_cast<unsigned long long*>(&s.nn_meta[n]), 1ull << (KSCHED_META_PRESENT_SHIFT + k));
  atomicAnd(reinterpret_cast<unsigned long long*>(&s.nn_meta[n]), ~(1ull << (KSCHED_META_COMPLEMENT_SHIFT + k)));
}
// the ring slot of the variant whose spread relations pinned domain d0 (and d1), or -1
__device__ __forceinline__ int run_ring_find(const RunCtx& rc, int n_mask, int d0, int d1) {
  int vi = -1;
  for (int v2 = 0; v2 < rc.n_var && vi < 0; ++v2)
    if ((n_mask < 1 || rc.var[v2].dom[0] == d0) && (n_mask < 2 || rc.var[v2].dom[1] == d1)) vi = v2;
  return vi;
}
// fill step: the pods the node at slot a takes before it refuses - its room `cap`, cut by the hostname limits
__device__ __forceinline__ int run_fill_cap(const RunEnv& e, int a, int cap) {
  const RunCtx& rc = g_rc;
  for (int j = 0; j < e.n_host; ++j) {
    const int times = rc.rec.h_times[j], lim = rc.rec.h_lim[j];
    if (!times || lim >= 0x10000) continue;
    if (lim >= 0xFFF0) { cap = 1; continue; }  // saturating counters nearby: one pod at a time
    const int td = (lim - (int)e.hc[j * kTopoCap + a]) / times + 1;
    cap = td < cap ? td : cap;
  }
  return cap;
}
// the assignments of staged entries 0 .. n - 1 of buffer buf, placed from sequence number seq on
__device__ __forceinline__ void run_store_chunk(const RunEnv& e, int buf, int n, int seq) {
  KS_K2
  const int tid = threadIdx.x;
  if (tid < n) {
    const uint32_t pd = g_rc.q_pod[buf][tid];
    int nd = g_rc.q_node[buf][tid];
    if (nd < -1) nd = e.NE + e.hs->node[-nd - 2];  // the mask run stores the slot
    s.assign[pd] = nd;
    s.place_seq[pd] = seq + tid;
  }
}

// ---- mask run, list build (block, once per call): sorts the accepting nodes into the lists of M1Ctx. Nothing of this
// call has been committed yet, so nn_last is free as scratch. False: a node the lists cannot represent (per-pod loop).
__device__ __forceinline__ bool m1_build(const RunEnv& e, int n_active) {
  M1Ctx& m1 = g_m1;
  const HotSmem* hs = e.hs;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5;
  uint16_t* m1_arr = e.m1_arr();
  uint16_t* m1_nxt = e.m1_nxt();
  uint8_t* t_b = reinterpret_cast<uint8_t*>(e.hs->nn_last);            // bucket of slot a (0xFF: not a member)
  uint16_t* t_pos = reinterpret_cast<uint16_t*>(t_b + kTopoCap);        // its arrival order inside the bucket
  uint16_t* t_slot = t_pos + kTopoCap;                                  // members, bucket by bucket, unsorted
  uint32_t* t_tie = reinterpret_cast<uint32_t*>(t_slot + kTopoCap);     // their tie-breaks
  for (int b = tid; b < kM1Lv * kM1Lists; b += T) m1.bcnt[b] = 0;
  if (tid == 0) m1.bad = 0;
  __syncthreads();
  for (int a = tid; a < n_active; a += T) {
    const uint32_t rp = e.rpv[a];
    int b = 0xFF;
    if ((rp & 0xFFFF) != 0 && !(rp & kRpDead)) {
      const uint32_t z = e.zv[a], adm = z & 0xFFFF;
      const unsigned cn = (unsigned)(hs->key[a] >> 32);
      int list = -1;
      if (adm && !(adm & (adm - 1)) && (z & kZvExact)) {  // pinned to one domain
        if (adm & e.m_reg0) list = __ffs(adm) - 1;           // (a domain that is not registered never admits a pod)
      } else if ((adm & e.m_reg0) == e.m_reg0) list = kM1Dom;  // admits every registered domain
      else if (adm & e.m_reg0) m1.bad = 1;                    // some of them: per-pod loop
      if (list >= 0) {
        if (cn >= (unsigned)kM1Lv) m1.bad = 1;
        else { b = list * kM1Lv + (int)cn; t_pos[a] = (uint16_t)atomicAdd(&m1.bcnt[b], 1); }
      }
    }
    t_b[a] = (uint8_t)b;
  }
  __syncthreads();
  if (warp == 0) {  // exclusive scan of the bucket sizes -> arr segments
    int run = 0;
    for (int b0 = 0; b0 < kM1Lv * kM1Lists; b0 += 32) {
      const int b = b0 + lane;
      const int v = b < kM1Lv * kM1Lists ? m1.bcnt[b] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      if (b < kM1Lv * kM1Lists) {
        const int list = b / kM1Lv, lv = b - list * kM1Lv;
        m1.ap[lv][list] = (uint16_t)(run + inc - v);
        m1.ae[lv][list] = (uint16_t)(run + inc);
      }
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  __syncthreads();
  const bool bad = m1.bad != 0;
  if (!bad) {
    for (int a = tid; a < n_active; a += T) {
      const int b = t_b[a];
      if (b == 0xFF) continue;
      const int list = b / kM1Lv, lv = b - list * kM1Lv;
      const int j = m1.ap[lv][list] + t_pos[a];
      t_slot[j] = (uint16_t)a;
      t_tie[j] = (uint32_t)hs->key[a];
    }
  }
  __syncthreads();
  if (!bad) {
    for (int a = tid; a < n_active; a += T) {
      const int b = t_b[a];
      if (b == 0xFF) continue;
      const int list = b / kM1Lv, lv = b - list * kM1Lv;
      const int p0 = m1.ap[lv][list], p1 = m1.ae[lv][list];
      const uint32_t tie = (uint32_t)hs->key[a];
      int rank = 0;
      for (int j = p0; j < p1; ++j) rank += t_tie[j] < tie;
      m1_arr[p0 + rank] = (uint16_t)a;
      t_pos[a] = (uint16_t)(p0 + rank);
    }
  }
  __syncthreads();
  if (!bad) {  // link every list (its buckets are contiguous in arr), tails and heads
    for (int a = tid; a < n_active; a += T) {
      const int b = t_b[a];
      if (b == 0xFF) continue;
      const int list = b / kM1Lv, gp = t_pos[a];
      m1_nxt[a] = gp + 1 < (int)m1.ae[kM1Lv - 1][list] ? m1_arr[gp + 1] : kM1None;
    }
    for (int b = tid; b < kM1Lv * kM1Lists; b += T) {
      const int list = b / kM1Lv, lv = b - list * kM1Lv;
      m1.tl[lv][list] = m1.ae[lv][list] > m1.ap[lv][list] ? m1_arr[m1.ae[lv][list] - 1] : kM1None;
    }
    if (tid < kM1Lists) m1.head[tid] = m1.ae[kM1Lv - 1][tid] > m1.ap[0][tid] ? m1_arr[m1.ap[0][tid]] : kM1None;
    if (tid == 0) m1.upos = m1.ap[0][kM1Dom];
  }
  __syncthreads();
  return !bad;
}

// ---- mask run, warp 0: lane L < kM1Lists holds list L - its head (slot, key, room word), the node after it, the tail of
// the head's bucket, the first node behind that bucket and its pod count
struct M1Lane {
  int L;
  int h = -1, n1 = -1, tcur = -1, bn = -1, bnc = 0;
  unsigned long long hk = ~0ull, nk = ~0ull;
  uint32_t hr = 0, nr = 0;

  __device__ __forceinline__ int nxt_of(const RunEnv& e, int sl) const { const uint16_t v = e.m1_nxt()[sl]; return v == kM1None ? -1 : (int)v; }
  __device__ __forceinline__ void level_state(const RunEnv& e) {
    if (h < 0) { tcur = -1; bn = -1; bnc = 0; return; }
    tcur = g_m1.tl[(int)(hk >> 32)][L];
    bn = nxt_of(e, tcur);
    bnc = bn >= 0 ? (int)(e.hs->key[bn] >> 32) : 0;
  }
  // the list's head is slot a (-1: empty): it and the node behind it are read
  __device__ __forceinline__ void set_head(const RunEnv& e, int a) {
    h = a; hk = ~0ull; hr = 0; n1 = -1; nk = ~0ull; nr = 0;
    if (h >= 0) {
      hk = e.hs->key[h]; hr = e.rpv[h]; n1 = nxt_of(e, h);
      if (n1 >= 0) { nk = e.hs->key[n1]; nr = e.rpv[n1]; }
    }
  }
  // the head has left the bucket of count c: when that bucket is exhausted, its tail goes and the next bucket is read
  __device__ __forceinline__ void bucket_left(const RunEnv& e, int c) {
    if (h < 0 || (int)(hk >> 32) != c) { g_m1.tl[c][L] = kM1None; level_state(e); }
  }
  // node a (key ak, room word ar) enters this lane's list at the FRONT of the block of count La
  __device__ __forceinline__ void insert_front(const RunEnv& e, int a, int La, unsigned long long ak, uint32_t ar) {
    M1Ctx& m1 = g_m1;
    uint16_t* m1_nxt = e.m1_nxt();
    const int hl = h >= 0 ? (int)(hk >> 32) : 0x7fffffff;
    if (hl >= La) {  // nothing lies below: the new head
      m1_nxt[a] = h >= 0 ? (uint16_t)h : kM1None;
      if (hl > La) { m1.tl[La][L] = (uint16_t)a; tcur = a; bn = h; bnc = hl; }
      n1 = h; nk = hk; nr = hr;
      h = a; hk = ak; hr = ar;
    } else if (bn < 0 || bnc >= La) {  // right behind the head's bucket
      m1_nxt[a] = bn >= 0 ? (uint16_t)bn : kM1None;
      m1_nxt[tcur] = (uint16_t)a;
      if (bn < 0 || bnc > La) m1.tl[La][L] = (uint16_t)a;
      if (tcur == h) { n1 = a; nk = ak; nr = ar; }
      bn = a; bnc = La;
    } else {  // behind the last bucket below La (the head's level is not the one)
      int lv = La - 1;
      while (m1.tl[lv][L] == kM1None) --lv;
      const int pred = m1.tl[lv][L];
      m1_nxt[a] = m1_nxt[pred];
      m1_nxt[pred] = (uint16_t)a;
      if (m1.tl[La][L] == kM1None) m1.tl[La][L] = (uint16_t)a;
      if (pred == h) { n1 = a; nk = ak; nr = ar; }
      if (pred == tcur) { bn = a; bnc = La; }
    }
  }
  // a fresh node (count 1, the largest tie-break so far) enters at the END of the block of count 1
  __device__ __forceinline__ void insert_back1(const RunEnv& e, int a, unsigned long long ak, uint32_t ar) {
    M1Ctx& m1 = g_m1;
    uint16_t* m1_nxt = e.m1_nxt();
    const int hl = h >= 0 ? (int)(hk >> 32) : 0x7fffffff;
    if (hl > 1) {
      m1_nxt[a] = h >= 0 ? (uint16_t)h : kM1None;
      m1.tl[1][L] = (uint16_t)a;
      tcur = a; bn = h; bnc = hl;
      n1 = h; nk = hk; nr = hr;
      h = a; hk = ak; hr = ar;
    } else if (hl == 1) {
      m1_nxt[a] = bn >= 0 ? (uint16_t)bn : kM1None;
      m1_nxt[tcur] = (uint16_t)a;
      m1.tl[1][L] = (uint16_t)a;
      if (tcur == h) { n1 = a; nk = ak; nr = ar; }
      tcur = a;
    } else {  // nodes without pods in front (not produced by the scheduler, kept exact anyway)
      int lv = 1;
      while (m1.tl[lv][L] == kM1None) --lv;
      const int pred = m1.tl[lv][L];
      m1_nxt[a] = m1_nxt[pred];
      m1_nxt[pred] = (uint16_t)a;
      m1.tl[1][L] = (uint16_t)a;
      if (pred == h) { n1 = a; nk = ak; nr = ar; }
      if (pred == tcur) { bn = a; bnc = 1; }
    }
  }
  // the head (pod count c) leaves this lane's list: the node behind it moves up, the one behind that is fetched (it is used
  // at this list's next pop)
  __device__ __forceinline__ void pop_head(const RunEnv& e, int c) {
    h = n1; hk = nk; hr = nr;
    n1 = -1; nk = ~0ull; nr = 0;
    if (h >= 0) {
      n1 = nxt_of(e, h);
      if (n1 >= 0) { nk = e.hs->key[n1]; nr = e.rpv[n1]; }
    }
    bucket_left(e, c);
  }
};
// warp 0's place in the mask run: staged entry, tick, new nodes and slots, fr entries, ring slots the nodes created in this
// entry replay (a store fetch must not overwrite them), and the spread count of this lane's domain
struct M1Walk { int li, ltick, lnew, lact, nfr, cnt_d; unsigned fr_used; };

// a mask-run commit of one pod on the pinned node a (pod count c, room word rp) with tick `tick`, staged entry q:
// Topology.Record, the node's new key and room word (returned); closed: the class no longer fits anywhere on it
__device__ __forceinline__ uint32_t m1_commit(const RunEnv& e, int buf, int a, uint32_t rp, int c, int tick, int q, bool& closed) {
  RunCtx& rc = g_rc;
  const uint32_t rp2 = run_record_host(rc, e.hc, e.n_host, a, rp, 1);
  rc.q_node[buf][q] = -(a + 2);  // the slot: translated to the node when the chunk is stored
  closed = run_settle(e, a, rp2, c + 1, -(tick + 1));
  return rp2;
}
// a mask-run fresh node from ring slot vi on slot a (node n) with order (1, tb) for staged entry q, pinned to domain d;
// its global state is stored by the CTA after the walk (fr entry f)
__device__ __forceinline__ void m1_fresh(const RunEnv& e, int buf, int vi, int a, int n, int tb, int q, int d, int f) {
  run_fresh(e, g_rc.var[vi], a, n, tb);
  g_rc.q_node[buf][q] = e.NE + n;
  e.zv[a] = zv_pinned(d);
  g_m1.fr[f] = (uint32_t)a | ((uint32_t)vi << 16);
}

// ---- fill stretch (DESIGN.md section 4): every domain of an all-equal round has a head that is alone in its bucket (pod
// count c). The round sends it to the FRONT of block c + 1, where nothing of its list lies before it, so while it accepts,
// stays below the unpinned head and does not pass the node behind it, the next rounds take the same node per domain. The
// order inside a round is known: heads of lower count first, and keys of equal count break ties on the previous round's
// ticks (later first), so inside a group of equal head count every round reverses the order of the one before. The pod of
// round r on this lane's node is pod r * na + m1_fill_pos(r, fp) of the step, fp = its place in the even rounds | its place
// in the odd rounds << 8.
__device__ __forceinline__ int m1_fill_pos(int r, int fp) { return (r & 1) ? fp >> 8 : fp & 0xFF; }
// warp-wide: this lane's bound on the rounds (32 outside the round) and its places fp
__device__ __forceinline__ int m1_fill_len(const RunEnv& e, const M1Lane& l, bool act, unsigned okm, int na, int cap,
                                           unsigned long long ukey, int ltick, int& fp) {
  const int c = (int)(l.hk >> 32);
  int rank0 = 0, lo = 0, gs = 0;  // the head's place in round 0; heads of the round with a lower / the same pod count
  for (unsigned m = okm; m; m &= m - 1) {
    const unsigned long long k2 = __shfl_sync(kFull, l.hk, __ffs(m) - 1);
    rank0 += k2 < l.hk;
    lo += (int)(k2 >> 32) < c;
    gs += (int)(k2 >> 32) == c;
  }
  fp = rank0 | (2 * lo + gs - 1 - rank0) << 8;
  if (!act) return 32;
  const int c1 = l.n1 >= 0 ? (int)(l.nk >> 32) : 0x7fffffff;  // pod count of the node behind the head
  if (c1 == c || (l.hr & 0xFFFF) == kRoomSlow || l.hk >= ukey) return 0;
  int rd = run_fill_cap(e, l.h, (int)(l.hr & 0xFFFF));  // room and hostname limits
  if (kM1Lv - 1 - c < rd) rd = kM1Lv - 1 - c;            // round r commits at count c + r + 1 < kM1Lv
  if (c1 != 0x7fffffff && c1 - c + 1 < rd) rd = c1 - c + 1;  // at count c + r > c1 the node behind comes first
  if (cap < rd) rd = cap;
  if (ukey != ~0ull)  // round r's key: count c + r, tie-break from the tick of round r - 1
    for (int r = 1; r < rd; ++r)
      if (order_key(c + r, -(ltick + (r - 1) * na + m1_fill_pos(r - 1, fp) + 1)) >= ukey) rd = r;
  return rd;
}

// ---- round / round stretch. Skew 1 with a self-matching selector: only the domains with the fewest pods admit a pod, so
// once every one of them has a pinned node at hand and the unpinned nodes come later in the order, the next pods go one to
// each of these domains, smallest head key first - a whole round is committed at once, every lane its own domain. Returns
// the pods placed (0: no round applies).
__device__ __forceinline__ int m1_round(const RunEnv& e, int buf, M1Lane& l, M1Walk& w, int i_end, bool allowed, unsigned okm) {
  KS_K2
  RunCtx& rc = g_rc;
  M1Ctx& m1 = g_m1;
  HotSmem* hs = e.hs;
  const int L = l.L;
  const int na = __popc(okm);
  if (na <= 1 || i_end - w.li < na) return 0;
  const bool act = L < kM1Dom && allowed;
  const bool hd = act && l.h >= 0;                       // this domain's pod goes to the head of its list
  const unsigned hv = __ballot_sync(kFull, hd), fv = okm & ~hv;  // fv: domains that get a fresh node (no pinned node at hand)
  const bool bad_l = hd && ((l.hr & 0xFFFF) == kRoomSlow || (int)(l.hk >> 32) + 1 >= kM1Lv);
  const unsigned long long ukey = __shfl_sync(kFull, l.hk, kM1Dom);
  // ---- round stretch: when every registered domain admits a pod (all counts are equal), each round gives every domain
  // one pod, so the counts stay equal and the round's shape repeats. R rounds are placed in one step while R single rounds
  // would take the same nodes (DESIGN.md section 4): pinned, the r-th members of each head's bucket; fresh, R fresh nodes
  // per domain that take no second pod.
  int R = 0, vi_s = -1, Rf = 0, fp = 0;  // Rf: rounds of a fill stretch, fp: its places (m1_fill_pos)
  const bool pinned = hv == okm;
  const int jd = __popc(okm & ((1u << L) - 1u));  // act: this domain's place among the round's domains
#ifdef KSCHED_PROFILE_PACK
  if (okm == e.m_reg0 && 2 * na <= i_end - w.li && 2 * na <= 32) {
#else
  if (s.use_round_stretch && okm == e.m_reg0 && 2 * na <= i_end - w.li && 2 * na <= 32) {
#endif
    const int cap = (i_end - w.li) / na < 32 / na ? (i_end - w.li) / na : 32 / na;
    if (pinned) {  // the bucket's keys ascend; nodes re-entering at count + 1 lie behind it
      int rd = 0;
      if (act) {
        const int c = (int)(l.hk >> 32);
        int a = l.h;
        unsigned long long k = l.hk;
        uint32_t rp = l.hr;
        while (rd < cap && (int)(k >> 32) == c && k < ukey && (rp & 0xFFFF) != kRoomSlow && c + 1 < kM1Lv) {
          m1.ps[rd * na + jd] = (uint16_t)a;
          m1.rk[rd * na + jd] = k;
          ++rd;
          a = l.nxt_of(e, a);
          if (a < 0) break;
          k = hs->key[a];
          rp = e.rpv[a];
        }
      }
      R = __reduce_min_sync(kFull, act ? rd : 32);
#ifdef KSCHED_PROFILE_PACK
      if (R < 2) {  // why the bucket stretch stopped, on the first lane that stopped it
        int why = 3;  // (a second member with an inexact room word)
        if (act && rd < 2) {
          const int c = (int)(l.hk >> 32);
          if ((l.hr & 0xFFFF) == kRoomSlow) why = 3;
          else if (c + 1 >= kM1Lv) why = 4;
          else if (l.hk >= ukey) why = 2;
          else if (l.n1 < 0 || (int)(l.nk >> 32) != c) why = run_fill_cap(e, l.h, (int)(l.hr & 0xFFFF)) >= 2 ? 0 : 1;
          else if (l.nk >= ukey) why = 2;
        }
        why = __shfl_sync(kFull, why, __ffs(__ballot_sync(kFull, act && rd < 2)) - 1);
        if (L == 0) s.counters[kCtrBucketEnd + why] += 1;
      }
      if (R < 2)
#else
      if (R < 2 && s.use_fill_stretch)
#endif
        Rf = __reduce_min_sync(kFull, m1_fill_len(e, l, act, okm, na, cap, ukey, w.ltick, fp));
    } else if (hv == 0 && ukey == ~0ull && (okm & ~rc.rec.m_tallow[0]) == 0) {  // fresh nodes that never re-enter a list
      if (act) vi_s = run_ring_find(rc, 1, L, 0);
      const bool shut = vi_s >= 0 && ((rc.var[vi_s].rp & 0xFFFF) == 0 || (rc.var[vi_s].rp & kRpDead));
      bool ok = !__any_sync(kFull, act && !shut);
      for (int j = 0; j < e.n_host; ++j) ok = ok && rc.rec.h_lim[j] >= 0;
      int room = e.MAXN - w.lnew;
      if (kActCap - w.lact < room) room = kActCap - w.lact;
      if (kTopoCap - w.lact < room) room = kTopoCap - w.lact;
      R = !ok ? 0 : room / na < cap ? room / na : cap;
    }
#ifdef KSCHED_PROFILE_PACK
    if (L == 0 && R > 0) s.counters[(pinned ? kCtrStretchPinned : kCtrStretchFresh) + (R > 16 ? 16 : R) - 1] += 1;
    if (L == 0 && Rf > 0) s.counters[kCtrFillLen + (Rf > 16 ? 16 : Rf) - 1] += 1;
    if (!s.use_round_stretch) R = 0;
    if (!s.use_fill_stretch) Rf = 0;
#endif
    if (Rf >= 2) R = Rf;
  }
#ifdef KSCHED_PROFILE_PACK
  else if (L == 0 && pinned && okm == e.m_reg0) s.counters[kCtrBucketEnd + 5] += 1;
#endif
  if (R >= 2) {
    const int np = R * na;
    if (Rf >= 2) {  // each domain's lane commits its head once for its R pods: no pop or insert per round
      bool closed_l = false;
      if (act) {
        const int a = l.h, c = (int)(l.hk >> 32);
        const uint32_t rp = l.hr;
        l.pop_head(e, c);
        for (int r = 0; r < R; ++r) rc.q_node[buf][w.li + r * na + m1_fill_pos(r, fp)] = -(a + 2);
        const int tl = w.ltick + (R - 1) * na + m1_fill_pos(R - 1, fp);  // tick of its last pod
        const uint32_t rp2 = run_record_host(rc, e.hc, e.n_host, a, rp, R);
        closed_l = run_settle(e, a, rp2, c + R, -(tl + 1));
        if ((rp2 & 0xFFFF) != 0 && !(rp2 & kRpDead)) l.insert_front(e, a, c + R, order_key(c + R, -(tl + 1)), rp2);
        w.cnt_d += R;
      }
      const unsigned tb = __ballot_sync(kFull, closed_l);
      if (L == 0 && tb) rc.tomb = rc.tomb + __popc(tb);
    } else if (pinned) {
      const int c = (int)(l.hk >> 32);
      if (act) for (int r = 0; r < R; ++r) l.pop_head(e, c);  // (reads the keys of the bucket before they change)
      __syncwarp();
      bool closed_l = false;
      if (L < np) {  // pod L: round L / na, the node whose key has rank L % na in that round
        const int r = L / na, a = m1.ps[L];
        const unsigned long long k = m1.rk[L];
        int p = r * na;
        for (int j = 0; j < na; ++j) p += m1.rk[r * na + j] < k;
        m1_commit(e, buf, a, e.rpv[a], (int)(k >> 32), w.ltick + p, w.li + p, closed_l);
      }
      const unsigned tb = __ballot_sync(kFull, closed_l);
      if (L == 0 && tb) rc.tomb = rc.tomb + __popc(tb);
      __syncwarp();  // key and room words
      if (act) {  // the nodes that still accept enter the front of block c + 1, round by round
        for (int r = 0; r < R; ++r) {
          const int a = m1.ps[r * na + jd];
          const uint32_t rp2 = e.rpv[a];
          if ((rp2 & 0xFFFF) != 0 && !(rp2 & kRpDead)) l.insert_front(e, a, c + 1, hs->key[a], rp2);
        }
        w.cnt_d += R;
      }
    } else {
      w.fr_used |= __reduce_or_sync(kFull, act ? 1u << vi_s : 0u);
      unsigned m = okm;  // pod L: round L / na, the (L % na)-th domain in id order
      for (int j = L % na; j > 0; --j) m &= m - 1;
      const int d = __ffs(m) - 1;
      const int vi = __shfl_sync(kFull, vi_s, d);
      if (L < np) m1_fresh(e, buf, vi, w.lact + L, w.lnew + L, w.ltick + L + 1, w.li + L, d, w.nfr + L);
      if (L < e.n_host && rc.rec.h_times[L]) rc.h_inc[L] = rc.h_inc[L] + np;
      if (act) w.cnt_d += R;
      w.lnew += np;
      w.lact += np;
      w.nfr += np;
    }
    return np;
  }
  const unsigned hi = hd ? (unsigned)(l.hk >> 32) : 0u;
  const unsigned mhi = __reduce_max_sync(kFull, hi);
  const unsigned mlo = __reduce_max_sync(kFull, (hd && hi == mhi) ? (unsigned)l.hk : 0u);
  const unsigned long long mx = ((unsigned long long)mhi << 32) | mlo;  // largest head key of the round
  // fresh nodes come last in a round, lowest domain id first (every admissible domain has the same count: run_pick takes
  // the lowest id), and only when no unpinned node is left (it would be taken first)
  int vi_l = -1;
  const int nf = __popc(fv);
  bool fresh_ok = true;
  if (fv) {
    const bool fl = act && l.h < 0;
    if (fl) vi_l = run_ring_find(rc, 1, L, 0);
    fresh_ok = ukey == ~0ull && (fv & ~rc.rec.m_tallow[0]) == 0 && !__any_sync(kFull, fl && vi_l < 0) && w.lnew + nf <= e.MAXN &&
               w.lact + nf <= kActCap && w.lact + nf <= kTopoCap;
    for (int j = 0; j < e.n_host; ++j) fresh_ok = fresh_ok && rc.rec.h_lim[j] >= 0;
  }
  if (!fresh_ok || __any_sync(kFull, bad_l) || (hv != 0 && ukey <= mx)) return 0;
  w.fr_used |= __reduce_or_sync(kFull, (act && !hd) ? 1u << vi_l : 0u);
  int rank = 0;  // position of this lane's node in the round
  for (unsigned m = hv; m; m &= m - 1) {
    const unsigned long long k2 = __shfl_sync(kFull, l.hk, __ffs(m) - 1);
    rank += k2 < l.hk;
  }
  bool closed_l = false;
  if (hd) {
    const int a = l.h;
    const uint32_t rp = l.hr;
    const int c = (int)(l.hk >> 32);
    const int mytick = w.ltick + rank;
    l.pop_head(e, c);
    const uint32_t rp2 = m1_commit(e, buf, a, rp, c, mytick, w.li + rank, closed_l);
    if ((rp2 & 0xFFFF) != 0 && !(rp2 & kRpDead)) l.insert_front(e, a, c + 1, order_key(c + 1, -(mytick + 1)), rp2);
    ++w.cnt_d;
  } else if (act) {  // NewNode + Add replayed from the variant of this lane's domain
    const RunVariant& v = rc.var[vi_l];
    const int idx = __popc(fv & ((1u << L) - 1u));
    const int mytick = w.ltick + __popc(hv) + idx;
    m1_fresh(e, buf, vi_l, w.lact + idx, w.lnew + idx, mytick + 1, w.li + __popc(hv) + idx, L, w.nfr + idx);
    if ((v.rp & 0xFFFF) != 0 && !(v.rp & kRpDead)) l.insert_back1(e, w.lact + idx, order_key(1, mytick + 1), v.rp);
    ++w.cnt_d;
  }
  if (nf && L < e.n_host && rc.rec.h_times[L]) rc.h_inc[L] = rc.h_inc[L] + nf;
  const unsigned tb = __ballot_sync(kFull, closed_l);
  if (L == 0 && tb) rc.tomb = rc.tomb + __popc(tb);
#ifdef KSCHED_PROFILE_PACK
  if (L == 0 && okm != e.m_reg0) s.counters[kCtrRoundsUnequal] += 1;
#endif
  w.lnew += nf;
  w.lact += nf;
  w.nfr += nf;
  return na;
}

// ---- pin step: the unpinned head (key wkey) wins, so the next pods take the next unpinned nodes one each, in list order
// (lane t: pod t), as long as no node of a domain list can come first: every member of the stretch has the first one's pod
// count c and a key below every pinned head (a node pinned by the stretch re-enters at c + 1). Pod t's domain is the t-th
// pick of run_pick's (count, id) order while the counts advance. Returns the pods placed.
__device__ __forceinline__ int m1_pin_step(const RunEnv& e, int buf, M1Lane& l, M1Walk& w, int i_end, unsigned long long wkey, int mn, bool valid) {
  const PackState& s = g_k2.st; (void)s;  // (c: the pod count below)
  RunCtx& rc = g_rc;
  M1Ctx& m1 = g_m1;
  const int L = l.L;
  const uint16_t* m1_arr = e.m1_arr();
  const int c = (int)(wkey >> 32);
  const int upos = m1.upos;
  int lim = i_end - w.li < 32 ? i_end - w.li : 32;
  if (m1.ae[kM1Lv - 1][kM1Dom] - upos < lim) lim = m1.ae[kM1Lv - 1][kM1Dom] - upos;
  const unsigned long long pmin = warp_min_u64(L < kM1Dom ? l.hk : ~0ull);
  const bool in = L < lim;
  const int a_t = in ? (int)m1_arr[upos + L] : 0;
  const unsigned long long k_t = in ? e.hs->key[a_t] : ~0ull;
  const uint32_t rp_t = in ? e.rpv[a_t] : 0u;
  const uint32_t z_t = in ? e.zv[a_t] : 0u;
  int d_t;
  {
    // domain e has a slot on every level >= its count; pod t takes the t-th slot in (level, id) order (without Record the
    // counts stay, and every pod takes the first pick). Levels are counted from mn: pod t's level is at most t, so a domain
    // more than 31 pods above mn never gets one. Byte e of dw: domain e's level.
    const unsigned dl = !valid ? 0xFFu : (unsigned)(w.cnt_d - mn < 32 ? w.cnt_d - mn : 32);
    const unsigned dw0 = __reduce_or_sync(kFull, L < 4 ? dl << (8 * L) : 0u);
    const unsigned dw1 = __reduce_or_sync(kFull, L >= 4 && L < kM1Dom ? dl << (8 * (L - 4)) : 0u);
    unsigned y = 0, r = e.m_rec0 ? L : 0, am;
    while (true) {
      const unsigned yy = y * 0x01010101u;  // bit 0 of every byte of the compares -> bits 24..27 (no carries)
      am = (((__vcmpleu4(dw0, yy) & 0x01010101u) * 0x01020408u) >> 24) & 0xFu;
      am |= (((__vcmpleu4(dw1, yy) & 0x01010101u) * 0x01020408u) >> 20) & 0xF0u;
      const unsigned k = __popc(am);
      if (am == e.m_reg0) { r %= k; break; }  // every domain has a slot on every level from here on
      if (r < k) break;
      r -= k;
      ++y;
    }
    for (; r > 0; --r) am &= am - 1;
    d_t = __ffs(am) - 1;
  }
  const bool same_c = (int)(k_t >> 32) == c, below = k_t < pmin;
  const bool ok_t = in && same_c && below && (rp_t & 0xFFFF) != kRoomSlow && c + 1 < kM1Lv &&
                    ((rc.rec.m_neutral[0] >> d_t) & 1) && ((z_t & kZvPresent) || rc.rec.m_wk[0]);
  const unsigned okb = __ballot_sync(kFull, ok_t);
  const int J = okb == kFull ? 32 : __ffs(~okb) - 1;
#ifdef KSCHED_PROFILE_PACK
  if (J > 0 && L == J)
    s.counters[!in ? (lim == i_end - w.li ? kCtrPinEndStaged : kCtrPinEndList) : !same_c ? kCtrPinEndCount : !below ? kCtrPinEndKey : kCtrPinEndRefused] += 1;
  if (J == 32 && L == 0) s.counters[kCtrPinEndList] += 1;
  if (J > 0 && L == 0) { s.counters[kCtrPinSteps] += 1; s.counters[kCtrPinPods] += J; }
#endif
  if (J == 0) return 0;
  bool closed_l = false;
  if (L < J) {  // the single step's commit for pod L on node a_t, pinned to d_t
    run_pin(e, 0, a_t, d_t);
    m1_commit(e, buf, a_t, rp_t, c, w.ltick + L, w.li + L, closed_l);
    m1.ps[L] = (uint16_t)a_t;
  }
  const unsigned tb = __ballot_sync(kFull, closed_l);
  if (L == 0 && tb) rc.tomb = rc.tomb + __popc(tb);
  unsigned mine = 0;  // the pods of this lane's domain
#pragma unroll
  for (int d = 0; d < kM1Dom; ++d) {
    const unsigned b = __ballot_sync(kFull, L < J && d_t == d);
    if (L == d) mine = b;
  }
  __syncwarp();  // ps, key and room words
  // the nodes that still accept enter their domain's list at the front of block c + 1, in pod order: the last one ends up
  // first (the smallest tie-break)
  for (unsigned m = mine; m; m &= m - 1) {
    const int t = __ffs(m) - 1, a = m1.ps[t];
    const uint32_t rp2 = e.rpv[a];
    if ((rp2 & 0xFFFF) != 0 && !(rp2 & kRpDead)) l.insert_front(e, a, c + 1, order_key(c + 1, -(w.ltick + t + 1)), rp2);
  }
  if (e.m_rec0) w.cnt_d += __popc(mine);
  if (L == 0) m1.upos = upos + J;
  if (L == kM1Dom) {  // the unpinned list's new head and the node behind it
    l.set_head(e, upos + J < (int)m1.ae[kM1Lv - 1][kM1Dom] ? (int)m1_arr[upos + J] : -1);
    l.bucket_left(e, c);
  }
  return J;
}

// ---- single step: the pod goes to the head of list wl (key wkey); the per-pod loop's commit, relation by relation on the
// first lanes. Returns 0, or the reason the walk ends: 1 the pod needs generic_step (why: StopCause), 2 per-pod loop from the
// next pod on.
__device__ __forceinline__ int m1_single(const RunEnv& e, int buf, M1Lane& l, M1Walk& w, unsigned long long wkey, int wl, bool allowed,
                                         int& why) {
  const PackState& s = g_k2.st; (void)s;  // (c: the pod count below)
  RunCtx& rc = g_rc;
  const int L = l.L;
  const int a = __shfl_sync(kFull, l.h, wl);
  const uint32_t rp = __shfl_sync(kFull, l.hr, wl);
  if ((rp & 0xFFFF) == kRoomSlow) { why = kStopRoomSlow; return 1; }  // the winner needs the full evaluation
  int d = wl;
  const bool pin = wl == kM1Dom;
  if (pin) {  // the placement pins the node's domain: fewest pods, lowest id among the admissible ones (run_pick)
    d = warp_pick(allowed, w.cnt_d);
    if (!((rc.rec.m_neutral[0] >> d) & 1) || !((e.zv[a] & kZvPresent) || rc.rec.m_wk[0])) { why = kStopOther; return 1; }
#ifdef KSCHED_PROFILE_PACK
    if (L == 0) s.counters[kCtrMaskUnpinnedSingle] += 1;
#endif
  }
  const int c = (int)(wkey >> 32);
  if (L == wl) l.pop_head(e, c);
  if (pin && L == 0) g_m1.upos = g_m1.upos + 1;  // (read by the next pin step after the __syncwarp below)
  uint32_t rp2 = rp - 1 + (1u << 16);
  bool dead_l = false;
  if (L < e.n_host) {  // Topology.Record, hostname groups
    const int times = rc.rec.h_times[L];
    const int old = e.hc[L * kTopoCap + a];
    const int now = old + times > 0xFFFF ? 0xFFFF : old + times;
    if (times) e.hc[L * kTopoCap + a] = (uint16_t)now;
    dead_l = now > rc.rec.h_lim[L];
  }
  if (e.n_host > 0 && __any_sync(kFull, dead_l)) rp2 |= kRpDead;
  if (L == 0) {
    if (pin) run_pin(e, 0, a, d);
    rc.q_node[buf][w.li] = -(a + 2);  // the slot: translated to the node when the chunk is stored
    if (run_settle(e, a, rp2, c + 1, -(w.ltick + 1))) rc.tomb = rc.tomb + 1;
  }
  int reason = 0;
  if ((rp2 & 0xFFFF) != 0 && !(rp2 & kRpDead)) {  // still accepts the class: front of the block of count + 1
    if (c + 1 >= kM1Lv) reason = 2;
    else if (L == d) l.insert_front(e, a, c + 1, order_key(c + 1, -(w.ltick + 1)), rp2);
  }
  if (e.m_rec0 && L == d) ++w.cnt_d;
  ++w.ltick;
  ++w.li;
  __syncwarp();  // lane 0's key / room words before a later pop fetches them
  return reason;
}

// ---- single step when nobody accepts: NewNode + Add replayed from the variant of the domain a fresh node gets. Returns 0,
// or 1 when the pod needs generic_step (why: StopCause).
__device__ __forceinline__ int m1_single_fresh(const RunEnv& e, int buf, M1Lane& l, M1Walk& w, unsigned okm, int& why) {
  RunCtx& rc = g_rc;
  const int L = l.L;
  if (w.lnew >= e.MAXN || w.lact >= kActCap || w.lact >= kTopoCap) { why = kStopCapacity; return 1; }
  bool ok = true;
  for (int j = 0; j < e.n_host; ++j) ok = ok && rc.rec.h_lim[j] >= 0;
  const unsigned cand = rc.rec.m_tallow[0] & okm;
  if (!ok || !cand) { why = kStopOther; return 1; }
  const int fd = warp_pick((cand >> L) & 1, w.cnt_d);  // (cand is a subset of okm: lanes below kM1Dom)
  int vi = run_ring_find(rc, 1, fd, 0);
  if (vi < 0 && !((w.fr_used >> rc.var_next) & 1)) vi = vt_fetch(rc, e.cls, 1, fd, L);
  if (vi < 0) { why = kStopNoVariant; return 1; }
  const RunVariant& v = rc.var[vi];
  w.fr_used |= 1u << vi;
  if (L < e.n_host && rc.rec.h_times[L]) rc.h_inc[L] = rc.h_inc[L] + 1;
  if (L == 0) m1_fresh(e, buf, vi, w.lact, w.lnew, w.ltick + 1, w.li, fd, w.nfr);  // nothing in this loop reads the node's global state
  ++w.nfr;
  if (L == fd) {
    if ((v.rp & 0xFFFF) != 0 && !(v.rp & kRpDead)) l.insert_back1(e, w.lact, order_key(1, w.ltick + 1), v.rp);  // accepts further pods of the class
    if (e.m_rec0) ++w.cnt_d;
  }
  ++w.ltick; ++w.lnew; ++w.lact; ++w.li;
  __syncwarp();
  return 0;
}

// ---- mask run, warp 0's steps from staged entry i on: each pod's node is the smallest head key over the lists of the
// admissible domains. The outcome goes to g_m1.out_*.
__device__ __forceinline__ void m1_walk(const RunEnv& e, int buf, int i, int qlen, int tick, int n_new, int n_active, int& why) {
  KS_K2
  RunCtx& rc = g_rc;
  M1Ctx& m1 = g_m1;
  const int L = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const bool valid = L < kM1Dom && ((e.m_reg0 >> L) & 1);
  M1Lane l;
  l.L = L;
  if (L < kM1Lists) {
    l.set_head(e, m1.head[L] == kM1None ? -1 : (int)m1.head[L]);
    l.level_state(e);
  }
  M1Walk w{i, tick, n_new, n_active, 0, L < kM1Dom ? rc.cnt[0][0][L] : 0, 0u};
  const bool rounds = e.m_rec0 && e.m_bias0 == 0;
  int i_end = rc.q_end[buf];
  if (i + qlen < i_end) i_end = i + qlen;
  int reason = 0;  // 0: the staged entries of the class are consumed; 1: the pod at li needs generic_step; 2: per-pod loop from li on
  // count + self - min <= maxSkew as count - min <= slack in 32 bits: counts are pod counts (< 2^30), so a slack of 2^30 or
  // more admits every domain exactly like the 64-bit form of the per-pod loop
  const int slack = e.m_bias0 < -(1 << 30) ? (1 << 30) : -e.m_bias0;
  while (w.li < i_end) {
#ifdef KSCHED_PROFILE_PACK
    const long long it0 = clock64();
#endif
    const int mn = __reduce_min_sync(kFull, valid ? w.cnt_d : INT32_MAX);
    const bool allowed = valid && w.cnt_d - mn <= slack;
    const unsigned okm = __ballot_sync(kFull, allowed);
    const bool cand_ok = L < kM1Dom ? allowed : (L == kM1Dom && okm != 0);  // an empty list keeps hk = ~0
    const unsigned long long key = cand_ok ? l.hk : ~0ull;
    const unsigned long long wkey = warp_min_u64(key);
#ifdef KSCHED_PROFILE_PACK
    {  // how often a whole round (one pod per admissible domain, all from pinned lists) could be placed at once
      const unsigned have = __ballot_sync(kFull, L < kM1Dom && allowed && l.h >= 0);
      const unsigned long long ukey = __shfl_sync(kFull, l.hk, kM1Dom);
      unsigned long long mx = (L < kM1Dom && allowed && l.h >= 0) ? l.hk : 0ull;
      for (int o = 16; o; o >>= 1) { const unsigned long long t = __shfl_xor_sync(kFull, mx, o); mx = t > mx ? t : mx; }
      const int na = __popc(okm);
      if (L == 0 && na > 1 && have == okm && ukey > mx && i_end - w.li >= na) s.counters[kCtrMaskRoundable] += 1;
      if (L == 0) s.counters[kCtrMaskSteps] += 1;
      if (L == 0 && na > 1) s.counters[kCtrMaskMultiDomain] += 1;
    }
#endif
    if (rounds) {
      const int np = m1_round(e, buf, l, w, i_end, allowed, okm);
      if (np > 0) {
#ifdef KSCHED_PROFILE_PACK
        if (L == 0) { s.counters[kCtrRoundCycles] += clock64() - it0; s.counters[kCtrRounds] += 1; s.counters[kCtrRoundPods] += np; }
#endif
        w.ltick += np;
        w.li += np;
        __syncwarp();
        continue;
      }
    }
    if (wkey != ~0ull) {
      const int wl = __ffs(__ballot_sync(kFull, key == wkey)) - 1;
      if (wl == kM1Dom) {
        const int J = m1_pin_step(e, buf, l, w, i_end, wkey, mn, valid);
        if (J > 0) {
          w.ltick += J;
          w.li += J;
          __syncwarp();
          continue;
        }
      }
      reason = m1_single(e, buf, l, w, wkey, wl, allowed, why);
    } else reason = m1_single_fresh(e, buf, l, w, okm, why);
    if (reason) break;
  }
  __syncwarp();
  // every warp's copy of the spread counters follows (the per-pod loop and the write-back read them)
  if (L < kM1Dom) for (int wi = 0; wi < nwarps; ++wi) rc.cnt[wi][0][L] = w.cnt_d;
  if (L < kM1Lists) m1.head[L] = l.h >= 0 ? (uint16_t)l.h : kM1None;
  if (L == 0) { m1.out_adv = w.li - i; m1.out_reason = reason; m1.out_tick = w.ltick; m1.out_n_new = w.lnew; m1.out_n_active = w.lact; m1.n_fresh = w.nfr; m1.out_why = why; }
}

// ---- mask run, fresh-node store (block): the global state of the nodes the walk created, 64 words per node across the CTA
__device__ __forceinline__ void m1_store_fresh(const RunEnv& e) {
  KS_K2
  const int tid = threadIdx.x, T = blockDim.x;
  const int nfr = g_m1.n_fresh;
  for (int x = tid; x < nfr * 64; x += T) {
    const uint32_t rec = g_m1.fr[x >> 6];
    const int a = (int)(rec & 0xFFFF), w = x & 63;
    const RunVariant& v = g_rc.var[rec >> 16];
    const int n = e.hs->node[a];
    if (w < e.W32) s.nn_opts[(size_t)w * e.MAXN + n] = v.opts[w];
    if (w < c.n_keys) s.nn_vals[(size_t)w * e.MAXN + n] = v.vals[w];
    if (w < KSCHED_MAX_RES) s.nn_req[(size_t)w * e.MAXN + n] = v.q[w];
    // the class run takes no instance-type class while the slot state is kept; the pod count and tie-break are (1, creation
    // tick) while the node has no further pod, otherwise the run's write-back stores them
    if (w == 0)
      open_node(s, n, v.fl >> 8, v.meta, v.qp, 0, false, 0, KSCHED_NONE, ((e.rpv[a] >> 16) & 0x7FFF) == 0,
                (int)((unsigned)e.hs->key[a] ^ 0x80000000u));
  }
}

// ---- warp level / fill: at most 32 open nodes, the level / fill steps of run_level_block with ONE node per lane of warp 0
// and no block barrier (slot a belongs to thread a, as in the block-wide form). Fresh nodes and winners that need the full
// evaluation go to the block-wide steps. The outcome goes to g_m1.out_*.
__device__ __forceinline__ void run_level_warp(const RunEnv& e, int buf, int i, int qlen, int tick, int n_active) {
  RunCtx& rc = g_rc;
  HotSmem* hs = e.hs;
  const int lane = threadIdx.x & 31;
  const int a = lane;
  const bool mine = a < n_active;
  int li = i, ltick = tick, reason = 0;
  int i_end = rc.q_end[buf];
  if (i + qlen < i_end) i_end = i + qlen;
  while (li < i_end) {
    const uint32_t rp = mine ? e.rpv[a] : 0u;
    const unsigned long long key = mine ? hs->key[a] : ~0ull;
    const bool el = mine && (rp & 0xFFFF) != 0 && !(rp & kRpDead);
    const unsigned elm = __ballot_sync(kFull, el);
    if (!elm || __any_sync(kFull, el && (rp & 0xFFFF) == kRoomSlow)) { reason = 1; break; }
    const unsigned cn = el ? (unsigned)(key >> 32) : 0xFFFFFFFFu;
    const unsigned c_min = __reduce_min_sync(kFull, cn);
    const bool mem = el && cn == c_min;
    const unsigned memm = __ballot_sync(kFull, mem);
    const int k_av = i_end - li;
    int t = 1, rank = 0, adv_w;
    if (!(elm & (elm - 1))) {  // fill: the only accepting node takes pods until it refuses
      int cap = (int)(rp & 0xFFFF);
      if (mem) cap = run_fill_cap(e, a, cap);
      t = __shfl_sync(kFull, cap, __ffs(memm) - 1);
      t = t < k_av ? t : k_av;
      adv_w = t;
    } else {  // level: the accepting nodes with the fewest pods, one pod each in tie order
      const unsigned tie = (unsigned)key;
      for (unsigned m = memm; m; m &= m - 1) {
        const unsigned tm = __shfl_sync(kFull, tie, __ffs(m) - 1);
        rank += tm < tie;
      }
      const int n_s = __popc(memm);
      adv_w = n_s < k_av ? n_s : k_av;
    }
    if (mem && rank < adv_w) {  // (fill: rank 0 < t)
      const uint32_t rp2 = run_record_host(rc, e.hc, e.n_host, a, rp, t);
      const int nd = e.NE + hs->node[a];
      for (int x = 0; x < t; ++x) rc.q_node[buf][li + rank + x] = nd;
      if (run_settle(e, a, rp2, (int)c_min + t, -(ltick + rank + t))) atomicAdd(&rc.tomb, 1);
    }
    ltick += adv_w;
    li += adv_w;
  }
  if (lane == 0) { g_m1.out_adv = li - i; g_m1.out_reason = reason; g_m1.out_tick = ltick; }
}

// ---- block level / fill, for classes without mask-key spread: a node's verdict depends on the node alone, so
//  * level step: the n accepting nodes with the fewest pods take the next n pods one each, in tie order (each leaves for the
//    block of count + 1, behind every node of the level);
//  * fill step: the only accepting node takes pods until it refuses (resources / hostname limits);
//  * a fresh node is filled the same way in the step that creates it (run_fresh_step).
// Returns 0 when a node needs the full evaluation (per-pod argmin step), 1 when `adv` pods are placed (fill: by a fill
// step), 2 when nobody accepts.
__device__ __forceinline__ int run_level_block(const RunEnv& e, int buf, int i, int k_avail, int n_active, int& tick, int& parity, int& lvp,
                                               int& adv, bool& fill) {
  RunCtx& rc = g_rc;
  HotSmem* hs = e.hs;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = T >> 5;
  uint32_t* lvt = e.zv;  // tie-breaks of the level's members (the zone words are unused when n_mask == 0)
  unsigned cmin = 0xFFFFFFFFu;
  int ne = 0;
  bool slow = false;
  for (int a = tid; a < n_active; a += T) {
    const uint32_t rp = e.rpv[a];
    if ((rp & 0xFFFF) != 0 && !(rp & kRpDead)) {  // tombstones have no room
      const unsigned cn = (unsigned)(hs->key[a] >> 32);
      cmin = cn < cmin ? cn : cmin;
      ++ne;
      slow = slow || (rp & 0xFFFF) == kRoomSlow;
    }
  }
  const unsigned wc = __reduce_min_sync(0xffffffffu, cmin);
  const unsigned wn = __reduce_add_sync(0xffffffffu, (unsigned)ne) | (__any_sync(0xffffffffu, slow) ? 0x80000000u : 0u);
  if (lane == 0) rc.red_key[parity][warp] = ((unsigned long long)wc << 32) | wn;
  __syncthreads();
  const unsigned long long rr = lane < nwarps ? rc.red_key[parity][lane] : 0xFFFFFFFF00000000ull;
  parity ^= 1;
  const unsigned c_min = __reduce_min_sync(0xffffffffu, (unsigned)(rr >> 32));
  const int n_el = (int)__reduce_add_sync(0xffffffffu, (unsigned)rr & 0x7FFFFFFFu);
  const bool any_slow = __any_sync(0xffffffffu, ((unsigned)rr >> 31) != 0);
  if (any_slow) return 0;
  if (n_el == 0) return 2;
  const int lp = lvp;
  lvp ^= 1;
  if (tid == 0) rc.lv_cnt[lp ^ 1] = 0;  // last read before this step's first barrier
  // the level's members append their tie-breaks to the list (any order)
  for (int base = 0; base < n_active; base += T) {
    const int a = base + tid;
    bool mem = false;
    unsigned tie = 0;
    if (a < n_active) {
      const uint32_t rp = e.rpv[a];
      const unsigned long long key = hs->key[a];
      mem = (rp & 0xFFFF) != 0 && !(rp & kRpDead) && (unsigned)(key >> 32) == c_min;
      tie = (unsigned)key;
      if (mem && n_el == 1) {  // fill: how many pods this node takes before it refuses
        const int cap = run_fill_cap(e, a, (int)(rp & 0xFFFF));
        rc.lv_fill[lp] = cap < k_avail ? cap : k_avail;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, mem);
    if (bal) {
      const int src = __ffs(bal) - 1;
      int pos0 = 0;
      if (lane == src) pos0 = atomicAdd(&rc.lv_cnt[lp], __popc(bal));
      pos0 = __shfl_sync(0xffffffffu, pos0, src);
      if (mem) lvt[pos0 + __popc(bal & ((1u << lane) - 1u))] = tie;
    }
  }
  __syncthreads();
  const int n_s = rc.lv_cnt[lp];
  const int t_fill = n_el == 1 ? rc.lv_fill[lp] : 1;
  const int k_lvl = n_el == 1 ? 1 : (n_s < k_avail ? n_s : k_avail);
  fill = n_el == 1;
  adv = n_el == 1 ? t_fill : k_lvl;
  for (int a = tid; a < n_active; a += T) {
    const uint32_t rp = e.rpv[a];
    const unsigned long long key = hs->key[a];
    if (!((rp & 0xFFFF) != 0 && !(rp & kRpDead) && (unsigned)(key >> 32) == c_min)) continue;
    const unsigned tie = (unsigned)key;
    int rank = 0;
    if (n_el != 1) {
      int j = 0;
      for (; j + 4 <= n_s; j += 4) {
        const uint4 v = *reinterpret_cast<const uint4*>(lvt + j);
        rank += (v.x < tie) + (v.y < tie) + (v.z < tie) + (v.w < tie);
      }
      for (; j < n_s; ++j) rank += lvt[j] < tie;
      if (rank >= k_lvl) continue;
    }
    // the owner commits: pods i + rank .. i + rank + t - 1 of the chunk
    const int t = t_fill;
    const uint32_t rp2 = run_record_host(rc, e.hc, e.n_host, a, rp, t);
    const int nd = e.NE + hs->node[a];
    for (int x = 0; x < t; ++x) rc.q_node[buf][i + rank + x] = nd;
    if (run_settle(e, a, rp2, (int)c_min + t, -(tick + rank + t))) atomicAdd(&rc.tomb, 1);
  }
  tick += adv;
  return 1;
}

// ---- per-pod argmin step: the node the reference's scan takes, by a block argmin on the order key over the accepting
// nodes (their admissible domains included), committed by its owner. Returns 0 when the pod is placed, 1 when the winner
// needs the full evaluation (why: StopCause), 2 when nobody accepts; okm0 / okm1: the admissible domains of each spread relation.
__device__ __forceinline__ int run_argmin_step(const RunEnv& e, int buf, int i, int n_active, int& tick, int& parity, uint32_t& okm0, uint32_t& okm1,
                                               int& why) {
  RunCtx& rc = g_rc;
  HotSmem* hs = e.hs;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = T >> 5;
  const int n_mask = e.n_mask;
  // node-independent half of nextDomainTopologySpread, one domain per lane: min count over the pod's domains, the
  // domains within max-skew (count + self - min <= maxSkew)
#pragma unroll
  for (int j = 0; j < kRunMask; ++j) {
    if (j >= n_mask) break;
    const bool valid = ((j ? e.m_reg1 : e.m_reg0) >> lane) & 1;  // registered domains have ids < kRunDom
    const int cn = rc.cnt[warp][j][lane & (kRunDom - 1)];
    const int mn = __reduce_min_sync(0xffffffffu, valid ? cn : INT32_MAX);
    (j ? okm1 : okm0) = __ballot_sync(0xffffffffu, valid && (long long)cn + (j ? e.m_bias1 : e.m_bias0) <= (long long)mn);
  }
  // ---- scan the slots this thread owns: key, rp and (topology classes) the admissible domains
  unsigned long long mine = ~0ull;
  int best_a = 0;
  uint32_t best_rp = 0, best_z0 = 0, best_z1 = 0;
  for (int a = tid; a < n_active; a += T) {
    const unsigned long long key = hs->key[a];
    const uint32_t rp = e.rpv[a];
    uint32_t z0 = 0, z1 = 0;
    bool ok = key < mine && (rp & 0xFFFF) != 0 && !(rp & kRpDead);  // tombstones carry key = ~0
    if (n_mask > 0) { z0 = e.zv[a]; ok = ok && (z0 & okm0) != 0; }
    if (n_mask > 1) { z1 = e.zv[kTopoCap + a]; ok = ok && (z1 & okm1) != 0; }
    if (ok) { mine = key; best_a = a; best_rp = rp; best_z0 = z0; best_z1 = z1; }
  }
  // payload of this thread's candidate: slot | slow << 11 | inexact room << 12 | pin bits << 13 | domains << 15 / 19
  unsigned pay = (unsigned)best_a;
  if (mine != ~0ull) {
    if ((best_rp & 0xFFFF) == kRoomSlow) pay |= 3u << 11;
#pragma unroll
    for (int j = 0; j < kRunMask; ++j) {
      if (j >= n_mask) break;
      const uint32_t z = j ? best_z1 : best_z0, cand = z & (j ? okm1 : okm0);
      int d;
      if (!(z & 0xFFFF & ((z & 0xFFFF) - 1)) && (z & kZvExact)) d = __ffs(cand) - 1;  // pinned already
      else {  // the placement pins the node's domain
        d = run_pick(cand, rc.cnt[warp][j]);
        pay |= 1u << (13 + j);
        if (!((rc.rec.m_neutral[j] >> d) & 1) || !((z & kZvPresent) || rc.rec.m_wk[j])) pay |= 1u << 11;
      }
      pay |= (unsigned)d << (15 + 4 * j);
    }
  }
  // ---- block argmin with payload: ONE barrier (double-buffered scratch)
  const unsigned long long wmin = warp_min_u64(mine);
  if (mine == wmin && mine != ~0ull) { rc.red_key[parity][warp] = wmin; rc.red_pay[parity][warp] = pay; }
  else if (lane == 0 && wmin == ~0ull) rc.red_key[parity][warp] = ~0ull;
  __syncthreads();
  const unsigned long long rk = lane < nwarps ? rc.red_key[parity][lane] : ~0ull;
  const unsigned rp_l = lane < nwarps ? rc.red_pay[parity][lane] : 0;
  parity ^= 1;
  const unsigned long long wkey = warp_min_u64(rk);
  if (wkey == ~0ull) return 2;
  const unsigned src = __ballot_sync(0xffffffffu, rk == wkey);
  const unsigned wp = __shfl_sync(0xffffffffu, rp_l, __ffs(src) - 1);
  if (wp & (1u << 11)) { why = (wp >> 12) & 1 ? kStopRoomSlow : kStopOther; return 1; }  // the winner needs the full evaluation
  const int fd0 = (wp >> 15) & 0xF, fd1 = (wp >> 19) & 0xF;
  if (mine == wkey) {  // the owner commits its node: a handful of shared-memory stores
    const int a = best_a;
    const uint32_t rp = run_record_host(rc, e.hc, e.n_host, a, best_rp, 1);
    for (int j = 0; j < n_mask; ++j)  // requirements.Add(In{d}) on the node: once per node and key
      if ((pay >> (13 + j)) & 1) run_pin(e, j, a, j ? fd1 : fd0);
    rc.q_node[buf][i] = e.NE + hs->node[a];
    if (run_settle(e, a, rp, (int)(wkey >> 32) + 1, -(tick + 1))) rc.tomb = rc.tomb + 1;  // tombstone, compacted when the run ends
  }
  if (n_mask > 0) {  // every warp keeps its copy of the spread counters in step (the node's domain is the single value d)
    if (lane == 0) {
      if (e.m_rec0) rc.cnt[warp][0][fd0]++;
      if (e.m_rec1) rc.cnt[warp][1][fd1]++;
    }
    __syncwarp();
  }
  ++tick;
  return 0;
}

// ---- fresh-node step: nobody accepts, so NewNode + Add is replayed from a variant (templates: the one the variant was
// created from). Fill step on the fresh node: it takes `cap` further pods of the class while it is the only accepting node
// and then refuses (room 0 or a hostname limit reached). With an exact cap the run needs F such nodes in a row, m = 1 + cap
// pods each: all of them are created in this step, one per thread (slot a belongs to thread a % T as everywhere). Returns
// false when the pod needs generic_step (why: StopCause); else `adv` pods are placed.
__device__ __forceinline__ bool run_fresh_step(const RunEnv& e, int buf, int i, int k_avail, bool lvl, uint32_t okm0, uint32_t okm1,
                                               int& tick, int& n_new, int& n_active, int& adv, int& why) {
  KS_K2
  RunCtx& rc = g_rc;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int n_mask = e.n_mask, MAXN = e.MAXN;
  if (n_new >= MAXN || n_active >= kActCap || (e.topo && n_active >= kTopoCap)) { why = kStopCapacity; return false; }
  bool ok = true;
#pragma unroll
  for (int j = 0; j < kRunHost; ++j) ok = ok && (j >= e.n_host || rc.rec.h_lim[j] >= 0);  // a fresh hostname has count 0
  int fd0 = 0, fd1 = 0;
  if (n_mask > 0 && ok) {
    const uint32_t cand = rc.rec.m_tallow[0] & okm0;
    if (!cand) ok = false; else fd0 = run_pick(cand, rc.cnt[warp][0]);
  }
  if (n_mask > 1 && ok) {
    const uint32_t cand = rc.rec.m_tallow[1] & okm1;
    if (!cand) ok = false; else fd1 = run_pick(cand, rc.cnt[warp][1]);
  }
  int vi = ok ? run_ring_find(rc, n_mask, fd0, fd1) : -1;
  if (vi < 0 && ok && vt_has(s, e.cls, n_mask, fd0)) {  // (every warp finds the same answer)
    __syncthreads();  // every warp has scanned the ring
    if (warp == 0) {
      const int got = vt_fetch(rc, e.cls, n_mask, fd0, lane);
      if (lane == 0) rc.vt_got = got;
    }
    __syncthreads();
    vi = rc.vt_got;
  }
  if (vi < 0) { why = ok ? kStopNoVariant : kStopOther; return false; }
  const RunVariant& v = rc.var[vi];
  int cap = 0, F = 1;
  bool cap_exact = false;
  if (lvl && (v.rp & 0xFFFF) != kRoomSlow) {
    cap_exact = true;
    if (!(v.rp & kRpDead)) {
      cap = (int)(v.rp & 0xFFFF);
      for (int j = 0; j < e.n_host; ++j) {
        const int times = rc.rec.h_times[j], lim = rc.rec.h_lim[j];
        if (!times || lim >= 0x10000) continue;
        if (lim >= 0xFFF0) { cap = 0; cap_exact = false; continue; }  // saturating counters nearby: one pod at a time
        const int td = (lim - times) / times + 1;  // the count is `times` after the first pod
        cap = td < cap ? td : cap;
      }
    }
  }
  const int m = 1 + cap;
  if (cap_exact) {
    F = (k_avail + m - 1) / m;
    if (F > MAXN - n_new) F = MAXN - n_new;
    if (F > kActCap - n_active) F = kActCap - n_active;
    if (e.topo && F > kTopoCap - n_active) F = kTopoCap - n_active;
  }
  const int K = k_avail < F * m ? k_avail : F * m;  // pods consumed (k_avail is 1 outside level mode: F = m = K = 1)
  for (int idx = tid; idx < e.W32 * F; idx += T) { const int w = idx / F, j = idx - w * F; s.nn_opts[(size_t)w * MAXN + n_new + j] = v.opts[w]; }
  for (int idx = tid; idx < c.n_keys * F; idx += T) { const int k = idx / F, j = idx - k * F; s.nn_vals[(size_t)k * MAXN + n_new + j] = v.vals[k]; }
  for (int idx = tid; idx < KSCHED_MAX_RES * F; idx += T) { const int r = idx / F, j = idx - r * F; s.nn_req[(size_t)r * MAXN + n_new + j] = v.q[r]; }
  for (int x = tid; x < K; x += T) rc.q_node[buf][i + x] = e.NE + n_new + x / m;
  if (tid == 0) for (int j = 0; j < e.n_host; ++j) if (rc.rec.h_times[j]) rc.h_inc[j] = rc.h_inc[j] + F;
  for (int j = (tid + T - n_active % T) % T; j < F; j += T) {  // the new slots this thread owns
    const int a = n_active + j, n = n_new + j;
    const int t = (K - j * m < m ? K - j * m : m) - 1;  // further pods on this node (the last one may get fewer)
    const int tk = tick + j * m;                          // tick of its first pod
    run_fresh(e, v, a, n, tk + 1);
    open_node(s, n, v.fl >> 8, v.meta, v.qp, 0, false, 0, KSCHED_NONE, true, tk + 1);
    if (n_mask > 0) e.zv[a] = zv_pinned(fd0);
    if (n_mask > 1) e.zv[kTopoCap + a] = zv_pinned(fd1);
    // the fill's t further pods (the slot holds the variant's requests and front, and v.rp carries no placed pod)
    if (t > 0 && run_settle(e, a, run_record_host(rc, e.hc, e.n_host, a, v.rp, t), 1 + t, -(tk + 1 + t))) atomicAdd(&rc.tomb, 1);
  }
  if (n_mask > 0) {
    if (lane == 0) {
      if (e.m_rec0) rc.cnt[warp][0][fd0]++;
      if (e.m_rec1) rc.cnt[warp][1][fd1]++;
    }
    __syncwarp();
  }
  adv = K;
  tick += K;
  n_new += F;
  n_active += F;
  return true;
}

// ---- capture node slot a (node hs->node[a]), which the generic step opened for the run's class with one pod, as a
// fresh-node variant into the ring. zv / rpv hold the slot's per-run inputs.
// Returns the ring slot, or -1 when the node does not pin one exact domain per mask relation or the ring already holds a
// variant of its template and domains. Block-wide.
__device__ __forceinline__ int run_capture(const HotSmem* hs, const uint32_t* zv, const uint32_t* rpv, int a, int n_mask) {
  KS_K2
  RunCtx& rc = g_rc;
  const int tid = threadIdx.x, T = blockDim.x;
  const int MAXN = s.max_new, W32 = c.W32, n = hs->node[a];
  int dom[kRunMask] = {0, 0};
  bool ok = true;
#pragma unroll
  for (int j = 0; j < kRunMask; ++j) {
    if (j >= n_mask) continue;
    const uint32_t z = zv[j * kTopoCap + a], v = z & 0xFFFF;
    if (!v || (v & (v - 1)) || !(z & kZvExact)) ok = false;
    else dom[j] = __ffs(v) - 1;
  }
  for (int i = 0; i < rc.n_var && ok; ++i) {
    bool same = (rc.var[i].fl >> 8) == (hs->flags[a] >> 8);
#pragma unroll
    for (int j = 0; j < kRunMask; ++j) same = same && (j >= n_mask || rc.var[i].dom[j] == dom[j]);
    if (same) ok = false;  // already known
  }
  const int slot = rc.var_next;  // read BEFORE the barrier: thread 0 moves it while the others still copy (racecheck warning, round 2)
  __syncthreads();  // rc.n_var / var_next read by everybody before thread 0 moves them
  if (!ok) return -1;
  RunVariant& v = rc.var[slot];
  for (int w = tid; w < W32; w += T) v.opts[w] = s.nn_opts[(size_t)w * MAXN + n];
  if (tid < KSCHED_MAX_KEYS) v.vals[tid] = tid < c.n_keys ? s.nn_vals[(size_t)tid * MAXN + n] : 0;
  if (tid == 0) {
    v.meta = s.nn_meta[n];
    for (int r = 0; r < KSCHED_MAX_RES; ++r) v.q[r] = r < kHotRes ? hs->q[r][a] : s.nn_req[(size_t)r * MAXN + n];
    for (int r = 0; r < kHotRes; ++r) { v.b1[r] = hs->bound[r][a]; v.b2[r] = hs->bound2[r][a]; }
    v.qp = s.nn_req_present[n];
    v.fl = hs->flags[a];
    v.rp = rpv[a] & (kRpDead | 0xFFFF);
    for (int j = 0; j < kRunMask; ++j) v.dom[j] = (uint8_t)dom[j];
    rc.var_next = (slot + 1) % kRunVariants;
    if (rc.n_var < kRunVariants) rc.n_var++;
  }
  __syncthreads();  // the ring slot is complete
  return slot;
}

// ---- derive the variant a run is missing for the fresh node of the pod at FFD position fpos: the generic step's
// NewNode + Add (generic_step, derive mode) opens node n_new at slot n_active as the step would open it for this pod, from
// the topology counts as they stand (the run's counts of its mask relations are stored first, as its write-back stores
// them), and the node is captured (run_capture). Its slot and node stay unused: the run replays the variant into them.
// Returns the ring slot, or -1 (the pod fails, or the node closes at once, pins no single domain or is known already).
// Block-wide; the guards of a capture (no provisioner limit, W32 <= kRunW32) and the run's capacity guards hold.
__device__ __noinline__ int run_derive(const PodRegs& first_in, int fpos, int n_new, int n_active, int tick, int seq, int parity) {
  KS_K2
  RunCtx& rc = g_rc;
  HotSmem* hs = reinterpret_cast<HotSmem*>(dyn_smem);
  uint32_t* zv = reinterpret_cast<uint32_t*>(dyn_smem + sizeof(HotSmem) + s.run_off);
  uint32_t* rpv = zv + (size_t)kRunMask * kTopoCap;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_mask = rc.rec.n_mask, n_host = rc.rec.n_host, MAXN = s.max_new;
  for (int j = 0; j < n_mask; ++j)
    if (rc.rec.m_rec[j] && warp == 0 && lane < kRunDom && ((rc.m_registered[j] >> lane) & 1)) s.grp_cnt[(size_t)rc.rec.m_group[j] * 64 + lane] = rc.cnt[0][j][lane];
  if (tid == 0) g_rio.staged = 1;
  int fatal = 0;
  uint32_t epoch = 0;
  bool pt_nonempty = true;  // g_pt is built for the class whatever it holds now
  long long nodes_visited = 0;
  LoopVars L{0, 0, n_new, n_active, tick, seq, parity, fatal, epoch, pt_nonempty, nodes_visited, KSCHED_NONE, KSCHED_NONE, 0, 0, KSCHED_NONE, 0, 1};
  generic_step<false>(first_in, true, fpos, L);  // (run classes request no ext resource)
  if (L.n_new != n_new + 1 || L.n_active != n_active + 1) return -1;  // no node, or one that closed at once
  const int a = n_active, n = n_new;
  if (tid == 0) {  // the slot's per-run inputs as class_run's entry computes them (its hostname counts: the relations' times)
    long long p_req[kHotRes];
    for (int r = 0; r < kHotRes; ++r) p_req[r] = first_in.req[r];
    rpv[a] = fresh_room_word(run_room(hs, a, p_req, first_in.res, c.n_res < kHotRes ? c.n_res : kHotRes), n_host, rc.rec.h_times, rc.rec.h_lim);
    const uint64_t meta = s.nn_meta[n];
    for (int j = 0; j < n_mask; ++j) {
      const int k = rc.rec.m_key[j];
      zv[j * kTopoCap + a] = zv_word(load_soa(s.nn_vals, meta, MAXN, n, k), (uint32_t)c.keys[k].dict_mask, k);
    }
  }
  __syncthreads();
  return run_capture(hs, zv, rpv, a, n_mask);
}

// run_derive for class_run's loop: true when the variant is in the ring (counts derivations; profile: their cycles, refusals)
__device__ __forceinline__ bool run_derive_at(const PodRegs& first_in, int fpos, int n_new, int n_active, int tick, int seq, int parity) {
#ifdef KSCHED_PROFILE_PACK
  const long long t0 = clock64();
#endif
  const int vi = run_derive(first_in, fpos, n_new, n_active, tick, seq, parity);
  KS_K2
  if (threadIdx.x == 0) s.counters[kCtrRunDerives] += 1;
#ifdef KSCHED_PROFILE_PACK
  if (threadIdx.x == 0) { s.counters[kCtrRunDeriveCycles] += clock64() - t0; s.counters[kCtrRunDeriveRefused] += vi < 0; }
#endif
  return vi >= 0;
}

// ---- run records: class cls's relation tables for class_run, from the class's topology relations and the catalog alone.
// A class is eligible (ok) when every relation constrains, none records through a TopologyNodeFilter, a topology class has
// one template, and the relations fit the tables: at most kRunHost hostname relations (spread or anti-affinity), at most
// kRunMask spread relations over distinct mask keys with fewer than kRunDom domains and no inverse record. Whether each
// relation's group exists and counts every slot (relaxation) changes during a Solve: class_run checks it at entry.
// An ineligible class's record is all 0. first_mask: the class_topo entry of its first mask relation (when n_mask > 0).
__device__ __forceinline__ RunRec run_rec_of(unsigned cls, int& first_mask) {
  KS_K2
  const ksched_pod_row& row = s.classes[cls];
  RunRec r = {};
  first_mask = -1;
  int ok = row.topo_begin == row.topo_end || c.n_templates == 1;
  for (uint32_t e = row.topo_begin; e < row.topo_end && ok; ++e) {
    const RelX x = s.relx[e];
    if (!(x.flags & KSCHED_TOPO_CONSTRAINS)) { ok = 0; break; }            // record-only relations: generic step
    if ((x.flags & KSCHED_TOPO_RECORDS) && x.has_filter) { ok = 0; break; }  // TopologyNodeFilter: generic step
    const int times = ((x.flags & KSCHED_TOPO_RECORDS) ? 1 : 0) + ((x.flags & KSCHED_TOPO_RECORDS_INVERSE) ? 1 : 0);
    const int self = (x.flags & KSCHED_TOPO_SELECTS) ? 1 : 0;
    if (x.key == KSCHED_KEY_HOSTNAME) {
      if (x.type == 1 || r.n_host == kRunHost) { ok = 0; break; }
      const int j = r.n_host++;
      r.h_row[j] = x.host_row; r.h_group[j] = (int)x.group; r.h_times[j] = (uint8_t)times;
      // spread: count + self <= maxSkew (min is 0 for hostnames, topologygroup.go:186-188); anti-affinity: count == 0
      const long long lim = x.type == 0 ? (long long)x.max_skew - self : 0;
      r.h_lim[j] = lim > 0x10000 ? 0x10000 : (lim < -1 ? -1 : (int)lim);
    } else {
      const int k = x.key;
      const uint64_t dict = c.keys[k].dict_mask;
      if (x.type != 0 || r.n_mask == kRunMask || (x.flags & KSCHED_TOPO_RECORDS_INVERSE) || (dict >> kRunDom)) { ok = 0; break; }
      static_assert(kRunMask == 2, "one earlier mask key to compare");
      if (r.n_mask == 1 && r.m_key[0] == k) { ok = 0; break; }
      if (r.n_mask == 0) first_mask = (int)e;
      const int j = r.n_mask++;
      r.m_group[j] = (int)x.group; r.m_skew[j] = x.max_skew; r.m_key[j] = (uint8_t)k;
      r.m_self[j] = (uint8_t)self; r.m_rec[j] = (x.flags & KSCHED_TOPO_RECORDS) ? 1 : 0;
      r.m_wk[j] = c.keys[k].well_known != 0; r.m_neutral[j] = (uint32_t)c.pin_neutral[k]; r.m_dict[j] = (uint32_t)dict;
      const Req tr = ksched::req_load(c.templates[0].reqs, nullptr, k);
      r.m_tallow[j] = (uint32_t)(tr.present ? ksched::req_allowed(tr, dict, key_meta(c, k)) : dict);
    }
  }
  if (!ok) r = RunRec{};
  r.ok = ok;
  return r;
}

// ---- variant table, entry (cls, d): the generic step's NewNode + Add for the class's fresh node with its mask relation
// pinned to domain d (templates in weight order, the first that opens a node), captured as run_capture captures it.
// Block-wide, in a launch before the pack kernel; reads only what is fixed for the Solve. Covered: an eligible run record
// (run_rec_of) with at most one mask relation, whose group registers d (d == 0 without one), and no hostname limit below 0
// (no pod goes on a fresh node then), plus the table's guards: no provisioner limit, W32 <= kRunW32, no instance-type or
// hostname requirement, no volumes, no ext resource. The entry is none when no template opens a node, the node closes at
// once or it is not pinned to exactly d (the pod's own requirement excludes d).
__device__ void vt_build_entry(unsigned cls, int d) {
  KS_K2
  KS_PT
  StepShared& sh = g_sh;
  Touched& fresh_t = g_fresh_t;
  TypeCtx& fresh_x = g_fresh_x;
  const int tid = threadIdx.x, W32 = c.W32, V = c.n_templates, NE = s.n_existing;
  const int RH = c.n_res < kHotRes ? c.n_res : kHotRes;
  const ksched_pod_row* src = s.classes + cls;
  __shared__ int vt_go;
  __shared__ RunRec vt_rec;
  if (tid < 32) reinterpret_cast<uint64_t*>(&g_row)[tid] = reinterpret_cast<const uint64_t*>(src)[tid];
  if (tid == 0) {
    int e_mask;
    vt_rec = run_rec_of(cls, e_mask);
    bool ok = vt_rec.ok && vt_rec.n_mask <= 1 && !s.any_limits && W32 <= kRunW32 && src->itype_req == KSCHED_NONE &&
              src->hostname_req == KSCHED_NONE && !class_has_volumes(s, cls) && !class_ext(s, cls);
    for (int j = 0; j < vt_rec.n_host; ++j) ok = ok && vt_rec.h_lim[j] >= 0;
    if (vt_rec.n_mask) {
      const uint64_t reg = s.grp_registered[vt_rec.m_group[0]];
      ok = ok && ((reg >> d) & 1);
      // the pin: d is the one admissible domain in (count, id) order, so the node gets d exactly when it admits d
      fill_pod_topo_static(s.relx[e_mask], pt, 0);
      pt.registered[0] = reg;
      pt.n_sorted[0] = 1;
      pt.sorted[0][0] = (uint8_t)d;
      pt.min_slot[0] = 0;
    } else ok = ok && d == 0;
    pt.n = vt_rec.n_mask;
    pt.overflow = 0;
    vt_go = ok;
  }
  __syncthreads();
  const size_t idx = vt_index(cls, d);
  if (!vt_go) {
    if (tid == 0) s.vt_ok[idx] = 0;
    return;
  }
  RunVariant& out = s.vtable[idx];
  const ksched_pod_row& row = g_row;
  const uint64_t p_tol = row.tolerated_taintsets;
  const uint32_t p_res = row.res_present;
  const bool plain = ((row.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF) == 0 && row.topo_begin == row.topo_end;
  int parity = 0;
  bool built = false;
  for (int v = 0; v < V && !built; ++v) {
    const ksched_template& tm = c.templates[v];
    __syncthreads();  // every reader of the previous template's g_sh / fresh_t / fresh_x is done
    if (tid == 0) {
      const bool ok = fresh_node_reqs(tm, p_tol, plain, p_res, NE, fresh_t);
      if (ok) build_type_ctx(fresh_t, sh.q, sh.qp, tm.reqs.values, tm.reqs.meta & 0xFFFFFFFFull, 1, 0, true, c.alloc_sorted, fresh_x);
      sh.path = ok ? 1 : 0;
    }
    __syncthreads();
    if (!sh.path) continue;
    bool any = false;
    for (int w = tid; w < W32; w += blockDim.x) {
      const uint32_t base = c.member[(size_t)v * W32 + w];
      const uint32_t sw = base ? type_word(c, s, fresh_x, base, w) : 0u;
      out.opts[w] = sw;
      any = any || sw;
    }
    if (tid < KSCHED_MAX_KEYS) out.vals[tid] = tid < c.n_keys ? (((fresh_t.keys >> tid) & 1) ? fresh_t.fin[tid] : tm.reqs.values[tid]) : 0;
    if (!__syncthreads_or(any)) continue;  // Node.Add fails on this template: the next one
    built = true;
    compute_front_block(out.opts, 1, 0, sh.bound, sh.bound2, &sh.front_bits, g_red, parity);
    __syncthreads();
    if (tid == 0) {
      bool ok = !node_closed(sh.q, s.min_req, RH, sh.bound, sh.bound2, sh.front_bits);
      const uint64_t meta = sh.meta;
      if (ok && vt_rec.n_mask) {
        const int k = vt_rec.m_key[0];
        ok = zv_word(load_soa(out.vals, meta, 1, 0, k), vt_rec.m_dict[0], k) == zv_pinned(d);
      }
      if (ok) {
        const unsigned short fl = (unsigned short)(sh.front_bits | ((sh.qp & 0xF) << 1) | (v << 8));
        long long p_req[kHotRes];
        for (int r = 0; r < kHotRes; ++r) p_req[r] = row.requests[r];
        out.meta = meta;
        for (int r = 0; r < KSCHED_MAX_RES; ++r) out.q[r] = sh.q[r];
        for (int r = 0; r < kHotRes; ++r) { out.b1[r] = sh.bound[r]; out.b2[r] = sh.bound2[r]; }
        out.qp = sh.qp;
        out.fl = fl;
        out.rp = fresh_room_word(room_of(fl, sh.q, sh.bound, sh.bound2, p_req, p_res, RH), vt_rec.n_host, vt_rec.h_times, vt_rec.h_lim);
        out.dom[0] = (uint8_t)d;
        out.dom[1] = 0;
      }
      s.vt_ok[idx] = ok ? 1 : 0;
#ifdef KSCHED_PROFILE_PACK
      if (ok) atomicAdd(reinterpret_cast<unsigned long long*>(&s.counters[kCtrVtEntries]), 1ull);
#endif
    }
  }
  if (!built && tid == 0) s.vt_ok[idx] = 0;
}
// block b of the table build: entry (b / vt_ndom, b % vt_ndom); the build's first start and last end (globaltimer, ns) go
// to the Solve's counters
__device__ void vt_build_block(int b) {
  KS_K2
  unsigned long long t;
  if (threadIdx.x == 0) {
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    atomicMax(reinterpret_cast<unsigned long long*>(&s.counters[kCtrVtStart]), ~t);
  }
  vt_build_entry((unsigned)(b / s.vt_ndom), b % s.vt_ndom);
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    atomicMax(reinterpret_cast<unsigned long long*>(&s.counters[kCtrVtEnd]), t);
  }
}

// the run records' build in the row gather's launch: one thread per class
__device__ __noinline__ void run_rec_build(unsigned cls) {
  KS_K2
  int first_mask;
  s.run_rec[cls] = run_rec_of(cls, first_mask);
}

// block b of the row gather's launch past the gather itself: the variant table's entries first, then the run records
__device__ void k0_extra_block(int b) {
  KS_K2
  const int vt_blocks = s.vt_classes * s.vt_ndom;
  if (b < vt_blocks) {
    vt_build_block(b);
    return;
  }
  const int cls = (b - vt_blocks) * blockDim.x + threadIdx.x;
  if (cls < s.rec_classes) run_rec_build((unsigned)cls);
}

__device__ __noinline__ void class_run(const PodRegs& first_in) {
  KS_K2
  RunCtx& rc = g_rc;
  RunIO& io = g_rio;
#ifdef KSCHED_PROFILE_PACK
  const long long cr_e0 = clock64();
  if (threadIdx.x == 0) s.counters[kCtrRunActiveSum] += io.n_active;
#endif
  HotSmem* hs = reinterpret_cast<HotSmem*>(dyn_smem);
  uint32_t* zv = reinterpret_cast<uint32_t*>(dyn_smem + sizeof(HotSmem) + s.run_off);  // [kRunMask][kTopoCap] domain words (zv_word)
  uint32_t* rpv = zv + (size_t)kRunMask * kTopoCap;                                      // [kActCap] room | placed << 16 | dead
  uint16_t* hc = reinterpret_cast<uint16_t*>(rpv + kActCap);                             // [kRunHost][kTopoCap]
  const uint32_t* tmpl_taintset = g_tmpl_taintset;
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int NE = s.n_existing, MAXN = s.max_new, W32 = c.W32;
  const int RH = c.n_res < kHotRes ? c.n_res : kHotRes;
  const int hstride = s.n_existing + s.max_new;
  // the pod row's words, in registers (identical for every pod of the run)
  const unsigned cls = (unsigned)first_in.cls64;
  const uint32_t p_res = first_in.res;
  const uint64_t p_tol = first_in.tol;
  long long p_req[kHotRes];
#pragma unroll
  for (int r = 0; r < kHotRes; ++r) p_req[r] = first_in.req[r];
  const bool topo = first_in.topo_begin != first_in.topo_end;
  const bool plain = plain_pod_regs(first_in);
  const bool simple = !topo;
  const bool resume = io.resume;
  const int qi0 = resume ? io.r_qi0 : io.qi, seq0 = resume ? io.r_seq0 : io.seq;
  int qi = io.qi, qlen = io.qlen, tick = io.tick, n_active = io.n_active, n_new = io.n_new, parity = io.parity;
  const int fresh_valid = io.fresh_valid && io.fresh_cls == cls, fresh_a = io.fresh_a;
  const int CH = T < kRunChunk ? T : kRunChunk;  // queue entries staged at a time: one per thread
  if (tid == 0 && !resume) { rc.q_end[0] = CH; rc.q_end[1] = CH; rc.lv_cnt[0] = 0; rc.lv_cnt[1] = 0; }  // (nobody reads these outside class_run)
  const bool new_cls = rc.cls != cls;  // read BEFORE the barrier: thread 0 rewrites rc.cls right after it (racecheck, round 2)
  __syncthreads();  // everybody has read g_rio; earlier readers of g_rc are done

  // ---- queue staging: the next CH (pod, class) entries; the chunk after them is fetched into registers meanwhile. Issued
  // first: its loads do not depend on the class's record.
  const ksched_pod_row* ffd_rows = reinterpret_cast<const ksched_pod_row*>(s.rows);
  int cb = resume ? io.r_cb : qi, buf = resume ? io.r_buf : 0;
  uint32_t nx_pod = 0, nx_cls = KSCHED_NONE;
  auto stage = [&](int b, uint32_t pd, uint32_t pc) {  // thread tid < CH: entry cb + tid into buffer b, entry cb + CH + tid into registers
    rc.q_pod[b][tid] = pd; rc.q_cls[b][tid] = pc;
    const unsigned mm = __ballot_sync(0xffffffffu, pc != cls);  // CH is a multiple of 32: whole warps
    if (lane == 0 && mm) atomicMin(&rc.q_end[b], (tid & ~31) + __ffs(mm) - 1);
    const int idx2 = cb + CH + tid;
    nx_cls = KSCHED_NONE;
    if (idx2 < s.n_pods) { nx_pod = s.order[idx2]; nx_cls = (uint32_t)ffd_rows[idx2].reserved; }
  };
  if (tid < CH && resume) {  // the staged chunk is in place: the one after it into registers
    const int idx2 = cb + CH + tid;
    if (idx2 < s.n_pods) { nx_pod = s.order[idx2]; nx_cls = (uint32_t)ffd_rows[idx2].reserved; }
  } else if (tid < CH) {
    const int idx = cb + tid;
    const bool in = idx < s.n_pods;
    stage(0, in ? s.order[idx] : 0, in ? (uint32_t)ffd_rows[idx].reserved : KSCHED_NONE);
  }
  // ---- relation tables: the class's record (run_rec_build) and the group state it is checked against. Every warp loads the
  // record, one word per lane, so that its copy of the spread counters needs no barrier; warp 0 keeps it in rc.rec and
  // decides eligibility from its lanes' loads of the groups: a relaxation-created group that does not exist yet, or that
  // never registered some slots, sends the class to the generic step. A run that resumes has all of it as it left it.
  constexpr int kWHGroup = offsetof(RunRec, h_group) / 4, kWMGroup = offsetof(RunRec, m_group) / 4;
  static_assert(offsetof(RunRec, ok) == 0 && offsetof(RunRec, n_host) == 4 && offsetof(RunRec, n_mask) == 8, "RunRec's first words");
  if (!resume) {
    const uint32_t rw = reinterpret_cast<const uint32_t*>(s.run_rec + cls)[lane];
    const int r_ok = __shfl_sync(0xffffffffu, rw, 0), r_nh = __shfl_sync(0xffffffffu, rw, 1), r_nm = __shfl_sync(0xffffffffu, rw, 2);
    const int hg = (int)__shfl_sync(0xffffffffu, rw, kWHGroup + (lane & 3)), mg = (int)__shfl_sync(0xffffffffu, rw, kWMGroup + (lane & 1));
    for (int j = 0; j < r_nm; ++j) {
      const int g = __shfl_sync(0xffffffffu, mg, j);
      if (lane < kRunDom) rc.cnt[warp][j][lane] = s.grp_cnt[(size_t)g * 64 + lane];
    }
    if (warp == 0) {
      reinterpret_cast<uint32_t*>(&rc.rec)[lane] = rw;
      const bool host = lane < kRunHost && lane < r_nh, mask = lane >= kRunHost && lane - kRunHost < r_nm;  // lane 4 + j: mask relation j
      const int g = host ? hg : mg;
      bool bad = false, zero = false;
      if (host || mask) {
        const uint8_t act = s.grp_active[g];
        const int32_t ms = s.grp_min_slot[g];
        const int32_t tot = host ? s.grp_host_total[g] : 1;
        const uint64_t reg = mask ? s.grp_registered[g] : 0;
        bad = !act || ms != 0;
        zero = host && tot == 0;
        if (mask) rc.m_registered[lane - kRunHost] = (uint32_t)reg;
      }
      const unsigned nbad = __ballot_sync(0xffffffffu, bad), nzero = __ballot_sync(0xffffffffu, zero);
      if (lane == 0) {
        rc.eligible = r_ok && !nbad;
        rc.h_zero = (int)nzero;
        if (new_cls) { rc.cls = cls; rc.n_var = 0; rc.var_next = 0; }
      }
    }
  }

  if (tid == 0 && !resume) rc.tomb = 0;
  if (tid < kRunHost && !resume) rc.h_inc[tid] = 0;
  __syncthreads();  // rc.rec, rc.eligible, rc.h_zero, rc.m_registered and the spread counters are in place
  if (!rc.eligible || (topo && n_active > kTopoCap)) {
    if (tid == 0) { io.status = rc.eligible ? 1 : 2; io.placed = 0; io.parity = parity; }
#ifdef KSCHED_PROFILE_PACK
    if (tid == 0 && rc.eligible) s.counters[kCtrStopCapacity] += 1;
#endif
    __syncthreads();
    return;
  }
  const int n_host = rc.rec.n_host, n_mask = rc.rec.n_mask;

  // ---- per-node inputs (each thread fills the slots it owns), every global load of a slot issued at once: the mask keys'
  // values are loaded whatever nn_meta says and masked afterwards, a hostname relation whose group counted no slot at entry
  // (grp_host_total 0) has the count 0 on every slot. A run that resumes has them in shared memory as it left them.
#ifdef KSCHED_PROFILE_PACK
  const long long cr_in0 = clock64();
#endif
  const int h_zero = rc.h_zero;
  for (int a = tid; a < (resume ? 0 : n_active); a += T) {
    const unsigned short fl = hs->flags[a];
    unsigned rm;
    if (!((p_tol >> tmpl_taintset[fl >> 8]) & 1)) rm = 0;                        // Taints.Tolerates
    else if (simple && hs->rejected[a] == cls) rm = 0;                           // memo: refused this class, untouched since
    else if (simple && !plain && hs->absorbed[a] != cls) rm = kRoomSlow;         // requirement verdict unknown for this class
    else rm = run_room(hs, a, p_req, p_res, RH);
    if (topo) {
      const int n = hs->node[a];
      const uint64_t meta = s.nn_meta[n];
      uint64_t mval[kRunMask];
#pragma unroll
      for (int j = 0; j < kRunMask; ++j) mval[j] = j < n_mask ? s.nn_vals[(size_t)rc.rec.m_key[j] * MAXN + n] : 0;
      for (int j = 0; j < n_host; ++j) {
        const uint16_t v = ((h_zero >> j) & 1) ? 0 : s.grp_host[(size_t)rc.rec.h_row[j] * hstride + NE + n];
        hc[j * kTopoCap + a] = v;
        if ((int)v > rc.rec.h_lim[j]) rm |= kRpDead;
      }
#pragma unroll
      for (int j = 0; j < kRunMask; ++j) {
        if (j >= n_mask) break;
        const int k = rc.rec.m_key[j];
        zv[j * kTopoCap + a] = zv_word(soa_req(mval[j], meta, k), rc.rec.m_dict[j], k);
      }
    }
    rpv[a] = rm;
  }
  __syncthreads();
#ifdef KSCHED_PROFILE_PACK
  if (tid == 0) s.counters[kCtrRunInputCycles] += clock64() - cr_in0;
#endif
  // ---- capture the node generic_step has just created for this class as a fresh-node variant
  if (fresh_valid && !s.any_limits && W32 <= kRunW32 && fresh_a == n_active - 1 && fresh_a >= 0) {
    const int slot = run_capture(hs, zv, rpv, fresh_a, n_mask);
#ifdef KSCHED_PROFILE_PACK
    if (tid == 0 && slot >= 0) s.counters[kCtrRunCaptures] += 1;
#endif
    (void)slot;
  }

  RunEnv e{hs, zv, rpv, hc, NE, MAXN, W32, RH, hstride, n_host, n_mask, cls, topo, simple};
#pragma unroll
  for (int r = 0; r < kHotRes; ++r) { e.p_req[r] = p_req[r]; e.min_req[r] = r < RH ? s.min_req[r] : 0; }
  e.m_reg0 = n_mask > 0 ? rc.m_registered[0] : 0; e.m_reg1 = n_mask > 1 ? rc.m_registered[1] : 0;
  e.m_bias0 = n_mask > 0 ? (int)rc.rec.m_self[0] - rc.rec.m_skew[0] : 0; e.m_bias1 = n_mask > 1 ? (int)rc.rec.m_self[1] - rc.rec.m_skew[1] : 0;
  e.m_rec0 = n_mask > 0 && rc.rec.m_rec[0]; e.m_rec1 = n_mask > 1 && rc.rec.m_rec[1];
  int status = 0;
  int why = kStopNone;  // StopCause of a status-1 stop
  // a stop for want of a variant ends the call with status 3 (the variant is derived and the run resumes, see RunIO::resume),
  // once per pod: a pod whose step still finds no variant (the derived node pinned another domain) stops the run
  const bool derive_ok = s.use_run_derive && !s.any_limits && W32 <= kRunW32;
  int derived_at = resume ? io.r_derived : -1;
  const bool lvl = s.use_level_run && n_mask == 0;
  // mask run (see M1Ctx): one mask-key spread relation, domains and counts small enough for the lists
  bool m1_ok = resume ? (io.r_m1 & 1) != 0 : s.use_mask_run && n_mask == 1 && (e.m_reg0 >> kM1Dom) == 0;
  bool m1_built = resume && (io.r_m1 & 2);
  int lvp = resume ? io.r_lvp : 0;
#ifdef KSCHED_PROFILE_PACK
  const long long cr_t0 = clock64();
  int cr_it[4] = {0, 0, 0, 0};  // iterations: level, fill, fresh, per-pod argmin
#define CR_IT(k) { ++cr_it[k]; }
#else
#define CR_IT(k)
#endif

  while (true) {
    int i = qi - cb;
    if (i == CH) {  // chunk consumed: store its assignments, registers -> the other buffer, fetch the chunk after
      __syncthreads();  // the last commit's q_node entry is visible
      run_store_chunk(e, buf, CH, seq0 + (cb - qi0));
      buf ^= 1;
      cb += CH;
      i = 0;
      if (tid < CH) stage(buf, nx_pod, nx_cls);
      __syncthreads();
      if (tid == 0) rc.q_end[buf ^ 1] = CH;  // the consumed buffer: its next atomicMin comes after the next chunk's first barrier
    }
    if (rc.q_cls[buf][i] != cls) break;  // class change or end of the first pass
    if (m1_ok && !m1_built) {
#ifdef KSCHED_PROFILE_PACK
      const long long m1_t0 = clock64();
#endif
      m1_built = true;
      m1_ok = m1_build(e, n_active);
#ifdef KSCHED_PROFILE_PACK
      if (tid == 0) { s.counters[kCtrMaskBuildCycles] += clock64() - m1_t0; s.counters[kCtrMaskBuildRefused] += m1_ok ? 0 : 1; }
#endif
    }
    if (m1_ok) {
#ifdef KSCHED_PROFILE_PACK
      const long long m1_t1 = clock64();
#endif
      if (warp == 0) m1_walk(e, buf, i, qlen, tick, n_new, n_active, why);
      __syncthreads();
      m1_store_fresh(e);
      const int m_adv = g_m1.out_adv, m_reason = g_m1.out_reason;
      tick = g_m1.out_tick; n_new = g_m1.out_n_new; n_active = g_m1.out_n_active;
      why = g_m1.out_why;  // (warp 0's: the status below is the same in every warp)
      qi += m_adv;
      qlen -= m_adv;
      __syncthreads();  // out_* are rewritten by the next entry
#ifdef KSCHED_PROFILE_PACK
      if (tid == 0) { s.counters[kCtrMaskCycles] += clock64() - m1_t1; s.counters[kCtrMaskPods] += m_adv; s.counters[kCtrMaskEntries] += 1; }
#endif
      if (m_reason == 1) { status = why == kStopNoVariant && derive_ok && qi != derived_at ? 3 : 1; break; }
      if (qlen == 0) break;
      if (m_reason == 2) m1_ok = false;
      continue;
    }
    if (lvl && n_active > 0 && n_active <= 32 && s.use_level_warp) {
      if (warp == 0) run_level_warp(e, buf, i, qlen, tick, n_active);
      __syncthreads();
      const int w_adv = g_m1.out_adv, w_reason = g_m1.out_reason;
      tick = g_m1.out_tick;
      qi += w_adv;
      qlen -= w_adv;
      i += w_adv;
      __syncthreads();  // out_* are rewritten by the next entry
      if (qlen == 0) break;
      if (w_reason == 0) continue;  // the staged entries of the class are consumed
      // w_reason == 1: the pod at i takes the block-wide steps (fresh nodes / full evaluation)
    }
    int adv = 1;       // pods this iteration consumes
    int mode = 0;      // 0: per-pod argmin step; 1: placed by a level / fill step; 2: nobody accepts (fresh node)
    int k_avail = 1;   // pods of the class that may be consumed now: staged, same class, still queued
    if (lvl) {
      k_avail = rc.q_end[buf] - i;
      k_avail = k_avail < qlen ? k_avail : qlen;
      bool fill = false;
      mode = run_level_block(e, buf, i, k_avail, n_active, tick, parity, lvp, adv, fill);
      if (mode == 1) { CR_IT(fill ? 1 : 0) }
    }
    uint32_t okm0 = 0, okm1 = 0;
    if (mode == 0) {
      CR_IT(3)
      const int r = run_argmin_step(e, buf, i, n_active, tick, parity, okm0, okm1, why);
      if (r == 1) { status = 1; break; }
      if (r == 2) mode = 2;
    }
    if (mode == 2) {
      if (!run_fresh_step(e, buf, i, k_avail, lvl, okm0, okm1, tick, n_new, n_active, adv, why)) {
        status = why == kStopNoVariant && derive_ok && qi != derived_at ? 3 : 1;
        break;
      }
      CR_IT(2)
    }
    // ---- the pods are placed: pop them
    qi += adv;
    qlen -= adv;
    if (qlen == 0) break;
  }
  __syncthreads();
  if (status == 3) {  // (see RunIO::resume)
    if (tid == 0) {
      io.qi = qi; io.qlen = qlen; io.tick = tick; io.n_active = n_active; io.n_new = n_new; io.parity = parity; io.placed = 0; io.status = 3;
      io.r_qi0 = qi0; io.r_seq0 = seq0; io.r_cb = cb; io.r_buf = buf; io.r_lvp = lvp; io.r_m1 = (m1_ok ? 1 : 0) | (m1_built ? 2 : 0); io.r_derived = qi;
    }
    __syncthreads();
    return;
  }
#ifdef KSCHED_PROFILE_PACK
  const long long cr_t1 = clock64();
#endif
  // ---- the run is over: write back what the commits deferred
  const int placed_total = qi - qi0;
  run_store_chunk(e, buf, qi - cb < CH ? qi - cb : CH, seq0 + (cb - qi0));  // assignments of the partly consumed chunk
  for (int a = tid; a < n_active; a += T) {  // requests, order statistics, hostname counters of the nodes that took pods
    const uint32_t rp = rpv[a];
    const int placed = (rp >> 16) & 0x7FFF;
    if (!placed) continue;
    const int n = hs->node[a];
    unsigned long long key = hs->key[a];
    const bool tomb = key == ~0ull;
    if (tomb) key = hs->nn_last[a];
#pragma unroll
    for (int r = 0; r < kHotRes; ++r) {
      const long long nq = hs->q[r][a] + placed * p_req[r];
      hs->q[r][a] = nq;
      if (tomb && r < RH) s.nn_req[(size_t)r * MAXN + n] = nq;
    }
    hs->rejected[a] = KSCHED_NONE;
    const unsigned short fl = hs->flags[a];
    if ((p_res & 0xF) & ~((fl >> 1) & 0xF)) {  // a request key new to the node
      s.nn_req_present[n] |= p_res;
      hs->flags[a] = fl | (unsigned short)((p_res & 0xF) << 1);
    }
    s.nn_count[n] = (int)(key >> 32);
    s.nn_tb[n] = (int)((unsigned)key ^ 0x80000000u);
    for (int j = 0; j < n_host; ++j) {
      const int times = rc.rec.h_times[j];
      if (!times) continue;
      const int now = hc[j * kTopoCap + a];
      s.grp_host[(size_t)rc.rec.h_row[j] * hstride + NE + n] = (uint16_t)now;
      if (now - placed * times == 0) atomicAdd(&rc.h_inc[j], 1);  // the hostname's first matching pod (not saturated: counts <= pods per node)
    }
  }
  for (int j = 0; j < n_mask; ++j)
    if (rc.rec.m_rec[j] && warp == 0 && lane < kRunDom && ((rc.m_registered[j] >> lane) & 1)) s.grp_cnt[(size_t)rc.rec.m_group[j] * 64 + lane] = rc.cnt[0][j][lane];
  __syncthreads();
  if (tid < n_host && rc.h_inc[tid]) s.grp_host_total[rc.rec.h_group[tid]] += rc.h_inc[tid];
#ifdef KSCHED_PROFILE_PACK
  const long long cr_t2 = clock64();
  const int cr_slots = rc.tomb > 0 ? n_active : 0;  // slots the compaction scans
#endif
  // ---- compact the active list (tombstones out); ownership ends with the run. The k-th tombstone below n_live (ascending)
  // takes the k-th live slot at or above n_live (descending), the order of the two-pointer scan the slots always had.
  if (rc.tomb > 0) {
    const int n_live = n_active - rc.tomb;
    const int per = (n_active + T - 1) / T, a0 = tid * per, a1 = min(a0 + per, n_active);  // each thread: one stretch of slots
    int live = 0;
    for (int a = a0; a < a1; ++a) live += hs->key[a] != ~0ull;
    int total, xpar = 0;
    int lb = block_scan_incl(live, &total, xpar) - live;  // live slots below a0, then below the slot at hand
    uint32_t* hole = rpv;  // hole rank -> slot (rpv is dead after the write-back)
    int a = a0;
    for (; a < a1 && a < n_live; ++a) {
      if (hs->key[a] == ~0ull) hole[a - lb] = a;  // rank: tombstones below a
      else ++lb;
    }
    __syncthreads();
    for (; a < a1; ++a) {  // slots at or above n_live: only their owner touches them
      if (hs->key[a] == ~0ull) continue;
      const int i = hole[n_live - 1 - lb];  // rank: live slots above a
      hs->key[i] = hs->key[a];
#pragma unroll
      for (int r = 0; r < kHotRes; ++r) { hs->q[r][i] = hs->q[r][a]; hs->bound[r][i] = hs->bound[r][a]; hs->bound2[r][i] = hs->bound2[r][a]; }
      hs->node[i] = hs->node[a]; hs->flags[i] = hs->flags[a]; hs->absorbed[i] = hs->absorbed[a]; hs->rejected[i] = hs->rejected[a];
      hs->key[a] = ~0ull;
      ++lb;
    }
    n_active = n_live;
  }
#ifdef KSCHED_PROFILE_PACK
  if (tid == 0) {
    const long long cr_t3 = clock64();
    s.counters[kCtrRunEntryCycles] += cr_t0 - cr_e0; s.counters[kCtrRunWbCycles] += cr_t2 - cr_t1;
    if (cr_slots) { s.counters[kCtrRunCompacts] += 1; s.counters[kCtrRunCompactSlots] += cr_slots; s.counters[kCtrRunCompactCycles] += cr_t3 - cr_t2; }
    if (lvl) {
      s.counters[kCtrRunLvCycles] += clock64() - cr_t0; s.counters[kCtrRunLvPods] += placed_total;
      s.counters[kCtrRunLvSteps] += cr_it[0] + cr_it[1]; s.counters[kCtrRunLvFresh] += cr_it[2]; s.counters[kCtrRunLvPerPod] += cr_it[3];
    } else {
      s.counters[kCtrRunCycles] += clock64() - cr_t0; s.counters[kCtrRunPods] += placed_total;
      s.counters[kCtrRunFresh] += cr_it[2]; s.counters[kCtrRunPerPod] += cr_it[3];
    }
    s.counters[kCtrRunLvFills] += cr_it[1];
    if (status == 1 && why != kStopNone) s.counters[kCtrNoVariantStops + why - 1] += 1;
  }
#endif
  // the pack loop's next steps load the next entry's pod row and, for the next class run, its record: into L2 now (the
  // entry's class is staged, or thread 0 holds it when the staged chunk is consumed)
  if (qlen > 0 && qi < s.n_pods && tid < 3) {
    if (tid == 0) {
      const int i = qi - cb;
      const uint32_t nc = i < CH ? rc.q_cls[buf][i] : (i == CH ? nx_cls : KSCHED_NONE);
      if (nc < (uint32_t)s.rec_classes) prefetch_l2(s.run_rec + nc);
    } else {
      prefetch_l2(reinterpret_cast<const char*>(ffd_rows + qi) + (tid - 1) * 128);
    }
  }
  if (tid == 0) {
    const int qcap = s.n_pods + 1;
    io.qi = qi; io.head = (io.head + placed_total) % qcap; io.qlen = qlen; io.tick = tick; io.seq = seq0 + placed_total; io.n_active = n_active; io.n_new = n_new; io.parity = parity;
    io.add_calls += placed_total; io.placed = placed_total; io.status = status;
  }
  __syncthreads();
}


// kExt: the problem has ext resources (DESIGN.md §3). Without them the kernel is compiled without any ext gate.
// kMaxThreads: the largest block the instantiation is launched with. Its register budget is 64 K / kMaxThreads (capped at
// 255): 128 registers at 512 threads spill in class_run and the generic step, 222 at 256 threads do not (run_pack picks the instantiation).
template <bool kExt, int kMaxThreads>
__global__ void __launch_bounds__(kMaxThreads, 1) pack_kernel() {
  static_assert(kMaxThreads % 32 == 0 && kMaxThreads <= kPackThreads, "pack_kernel: whole warps, at most kPackThreads");
#ifdef KSCHED_PROFILE_PACK
  long long pk_acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  long long pk_last = clock64();
  long long pk_bail = -1;  // when the last class_run call stopped with status 1 (-1: none since the last one that placed pods)
  bool pk_bail_novar = false;
#endif
  KS_K2
  const int tid = threadIdx.x;
  if (tid == 0) {  // the launch's start (ksched_timings::pack_interval_ns)
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    s.counters[kCtrPackStart] = (long long)t;
  }
  const int NE = s.n_existing, MAXN = s.max_new;
  const int R = c.n_res, RH = R < kHotRes ? R : kHotRes;

  int64_t* sm_alloc = reinterpret_cast<int64_t*>(dyn_smem + sizeof(HotSmem));
  const Hot H = make_hot(s);
  if (s.alloc_in_smem)
    for (int i = tid; i < R * c.n_types; i += blockDim.x) sm_alloc[i] = c.alloc_sorted[i];

  PodTopo& pt = g_pt;
  uint32_t* tmpl_taintset = g_tmpl_taintset;
  for (int v = tid; v < c.n_templates; v += blockDim.x) tmpl_taintset[v] = c.templates[v].taintset;
  if (tid == 0) { pt.n = 0; g_rc.cls = KSCHED_NONE; g_rc.eligible = 0; }

  int head = 0, qlen = s.n_pods;
  const int qcap = s.n_pods + 1;
  int n_new = 0, n_active = 0, tick = 0, seq = 0, parity = 0;
  uint32_t epoch = 1;
  long long nodes_visited = 0, add_calls = 0;
  int fatal = 0;
  bool pt_nonempty = false;
  uint32_t pt_class = KSCHED_NONE, row_class = KSCHED_NONE;
  int fresh_valid = 0, fresh_a = 0;
  uint32_t fresh_cls = KSCHED_NONE;
  // class-run bookkeeping: classes found ineligible are not tried again; a run that places nothing backs off
  uint32_t run_block_cls = KSCHED_NONE;
  int run_skip = 0, run_fail = 0;
  uint32_t xrun_block_cls = KSCHED_NONE;  // existing-node run: class the existing nodes have no room left for
  // failure memo: the class whose Scheduler.add has just failed, valid while nothing is placed (seq) or relaxed (epoch)
  uint32_t fail_cls = KSCHED_NONE, fail_epoch = 0;
  int fail_seq = 0;

  for (int i = tid; i < s.n_pods; i += blockDim.x) {
    s.queue[i] = s.order[i];
    s.pod_pos[s.order[i]] = (uint32_t)i;
    s.assign[i] = -1;
    s.place_seq[i] = -1;
    s.last_epoch[i] = 0;
  }
  __syncthreads();

  // First pass over the queue = FFD order: row qi of the dense pod-row matrix (K0) belongs to pod order[qi], so the
  // next pod's words are fetched one iteration ahead with addresses that depend on no earlier load.
  int qi = 0;
  const ksched_pod_row* ffd_rows = reinterpret_cast<const ksched_pod_row*>(s.rows);
  PodRegs nxt{};
  if (s.n_pods > 0) nxt = load_pod_regs(ffd_rows, s.order[0]);
  const bool fast_allowed = NE == 0 && !s.count_visited;

  while (qlen > 0) {
    // ---- failure memo: pods at the head of the queue of the class that has just failed fail again (same class, same state:
    // scheduler.go:117-123 pushes them back unchanged, queue.go:61-68) - requeued in one step, up to one per thread
    if (fast_allowed && fail_cls != KSCHED_NONE && seq == fail_seq && epoch == fail_epoch) {
      const int T = blockDim.x;
      int lim = qlen < T ? qlen : T;
      if (qi < s.n_pods && s.n_pods - qi < lim) lim = s.n_pods - qi;  // the first pass ends with its last pod
      uint32_t pj = 0;
      bool stop = true;
      if (tid < lim) {
        int pos = head + tid;
        if (pos >= qcap) pos -= qcap;
        pj = s.queue[pos];
        stop = s.pod_class[pj] != fail_cls || (s.last_epoch[pj] == epoch && s.last_len[pj] == qlen);  // Pop() would stop here
      }
      unsigned first, unused;
      block_min2_u32_db(stop ? (unsigned)tid : 0xFFFFFFFFu, 0u, g_red, parity, &first, &unused);
      const int k = first < (unsigned)lim ? (int)first : lim;
      if (k > 0) {
        if (tid < k) {
          s.queue[(head + qlen + tid) % qcap] = pj;  // (every read of the old entries happened before the barrier above)
          s.last_len[pj] = qlen;
          s.last_epoch[pj] = epoch;
        }
        if (qi < s.n_pods) qi += k;
        head = (head + k) % qcap;
        add_calls += k;
        __syncthreads();
        if (qi < s.n_pods) nxt = load_pod_regs(ffd_rows + qi, s.order[qi]);
        continue;
      }
    }
    PK_T(0)
    // ---- class-run mode (see class_run): first-pass pods of a class whose accept test is exact from shared memory
    bool skip_run = true;
    if (fast_allowed && s.use_class_run && s.rec_classes > 0 && qi < s.n_pods && n_active <= kActCap) {  // (a run reads the class's record)
      const bool topo_cls = nxt.topo_begin != nxt.topo_end;
      // (host-port classes never get here)
      // (with the instance-type slot state, PackState::nn_it, only the generic step writes it: instance-type classes stay there)
      const bool shape_ok = !has_host_ports(s, nxt) && (nxt.res >> kHotRes) == 0 && !(kExt && class_ext(s, (unsigned)nxt.cls64)) &&
                            (nxt.itype == KSCHED_NONE || !s.nn_it) &&
                            (!topo_cls || (((nxt.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF) == 0 && nxt.itype == KSCHED_NONE && nxt.hostname == KSCHED_NONE));
      if (shape_ok && (unsigned)nxt.cls64 != run_block_cls) {
        if (fresh_valid && fresh_cls == (unsigned)nxt.cls64) skip_run = false;  // a fresh node of this class to capture
        else if (run_skip > 0) --run_skip;
        else skip_run = false;
      }
    }
    if (!skip_run) {
      __syncthreads();
      if (tid == 0) {
        RunIO& io = g_rio;
        io.qi = qi; io.head = head; io.qlen = qlen; io.tick = tick; io.seq = seq; io.n_active = n_active; io.n_new = n_new; io.parity = parity;
        io.add_calls = add_calls; io.placed = 0; io.status = 0;
        io.fresh_valid = fresh_valid; io.fresh_a = fresh_a; io.fresh_cls = fresh_cls; io.staged = 0; io.resume = 0;
      }
      __syncthreads();
#ifdef KSCHED_PROFILE_PACK
      const long long pk_entry = clock64();
      const long long pk_novar0 = tid == 0 ? s.counters[kCtrNoVariantStops] : 0;
#endif
      class_run(nxt);
      while (g_rio.status == 3) {  // derive the variant the run needs, then resume it
        run_derive_at(nxt, g_rio.qi, g_rio.n_new, g_rio.n_active, g_rio.tick, g_rio.seq, g_rio.parity);
        if (tid == 0) { g_rio.resume = 1; g_rio.fresh_valid = 0; }
        __syncthreads();
        class_run(nxt);
      }
      const RunIO& io = g_rio;
      const int placed = io.placed, status = io.status;
      qi = io.qi; head = io.head; qlen = io.qlen; tick = io.tick; seq = io.seq; n_active = io.n_active; n_new = io.n_new; parity = io.parity;
      add_calls = io.add_calls;
      fresh_valid = 0;
      if (io.staged) { row_class = KSCHED_NONE; pt_class = KSCHED_NONE; pt_nonempty = true; }  // (rebuilt by the next generic step)
#ifdef KSCHED_PROFILE_PACK
      if (tid == 0) {
        s.counters[kCtrRunCalls] += 1; s.counters[kCtrRunPlaced] += placed; s.counters[kCtrRunBails] += status == 1; s.counters[kCtrRunIneligible] += status == 2;
        // round trips: from a call that stopped with status 1 to the entry of the next call that places pods
        if (placed > 0 && pk_bail >= 0) {
          s.counters[kCtrRoundTripCycles] += pk_entry - pk_bail;
          if (pk_bail_novar) s.counters[kCtrNoVariantTripCycles] += pk_entry - pk_bail;
          pk_bail = -1;
        }
        if (status == 1 && pk_bail < 0) { pk_bail = clock64(); pk_bail_novar = s.counters[kCtrNoVariantStops] != pk_novar0; }
      }
#endif
      if (status == 2) run_block_cls = (unsigned)nxt.cls64;
      if (placed == 0 && status == 1) { run_fail = run_fail < 6 ? run_fail + 1 : 6; run_skip = (1 << run_fail) - 1; }
      else if (placed > 0) run_fail = 0;
      PK_T(1)
      if (qlen == 0) break;
      if (placed > 0) {
        if (qi < s.n_pods) nxt = load_pod_regs(ffd_rows + qi, s.order[qi]);
        if (status == 0) continue;  // class change / end of the first pass: pick the mode for the next pod
      }
      // status 1 / 2: the pod at qi takes the generic step
    }
    // ---- existing-node run (see existing_run): identical plain pods take the existing nodes in one prefix-sum pass
    if (NE > 0 && !s.count_visited && qi < s.n_pods && (unsigned)nxt.cls64 != xrun_block_cls &&
        ((nxt.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF) == 0 && nxt.topo_begin == nxt.topo_end && nxt.itype == KSCHED_NONE &&
        !has_host_ports(s, nxt) && (nxt.res >> kHotRes) == 0 && !class_has_volumes(s, (unsigned)nxt.cls64) &&
        !(kExt && class_ext(s, (unsigned)nxt.cls64))) {
      __syncthreads();
      if (tid == 0) { ExRunIO& io = g_xio; io.qi = qi; io.head = head; io.qlen = qlen; io.seq = seq; io.parity = parity; io.add_calls = add_calls; io.placed = 0; }
      __syncthreads();
      existing_run(nxt);
      const ExRunIO& io = g_xio;
      const int placed = io.placed;
      qi = io.qi; head = io.head; qlen = io.qlen; seq = io.seq; parity = io.parity; add_calls = io.add_calls;
      __syncthreads();  // g_xio is rewritten by the next run
      if (placed == 0) xrun_block_cls = (unsigned)nxt.cls64;  // no existing node takes this class: the generic step does the rest of it
      if (placed > 0) {
        fresh_valid = 0;
        if (qlen == 0) break;
        if (qi < s.n_pods) nxt = load_pod_regs(ffd_rows + qi, s.order[qi]);
        if ((unsigned)nxt.cls64 == (unsigned)ffd_rows[qi - 1].reserved) xrun_block_cls = (unsigned)nxt.cls64;  // the existing nodes are full for this class
        continue;
      }
    }
    if (s.stop_new_nodes > 0 && n_new >= s.stop_new_nodes) break;  // simulation: the verdict no longer depends on the rest (cluster.cuh)
    PodRegs cur;
    const bool first_pass = qi < s.n_pods;
    if (first_pass) {
      cur = nxt;
      if (qi + 1 < s.n_pods) nxt = load_pod_regs(ffd_rows + qi + 1, s.order[qi + 1]);
      if (tid < 2 && qi + 24 < s.n_pods) prefetch_l2(reinterpret_cast<const char*>(ffd_rows + qi + 24) + tid * 128);
      if (tid == 2 && (qi & 31) == 0 && qi + 96 < s.n_pods) prefetch_l2(s.order + qi + 96);
    } else {
      const uint32_t qpod = s.queue[head];
      if (s.last_epoch[qpod] == epoch && s.last_len[qpod] == qlen) break;  // Pop(): no progress in a whole cycle (queue.go:52)
      cur = load_pod_regs(s.classes + s.pod_class[qpod], qpod);
    }
    const int fpos_first = qi;
    ++qi;
    head = head + 1 == qcap ? 0 : head + 1;
    --qlen;
    ++add_calls;
#ifdef KSCHED_PROFILE_PACK
    if (tid == 0) s.counters[kCtrGenSteps] += 1;
#endif
    LoopVars L{head, qlen, n_new, n_active, tick, seq, parity, fatal, epoch, pt_nonempty, nodes_visited, pt_class, row_class, 0, 0, KSCHED_NONE, 0};
    generic_step<kExt>(cur, first_pass, fpos_first, L);
    if (L.fail_memo) { fail_cls = (unsigned)cur.cls64; fail_seq = L.seq; fail_epoch = L.epoch; } else fail_cls = KSCHED_NONE;
    head = L.head; qlen = L.qlen; n_new = L.n_new; n_active = L.n_active; tick = L.tick; seq = L.seq; parity = L.parity; fatal = L.fatal;
    epoch = L.epoch; pt_nonempty = L.pt_nonempty; nodes_visited = L.nodes_visited; pt_class = L.pt_class; row_class = L.row_class;
    fresh_valid = L.fresh_valid; fresh_a = L.fresh_a; fresh_cls = L.fresh_cls;
    if (fatal) break;
    PK_T(5)
  }
  __syncthreads();
  for (int a = tid; a < n_active; a += blockDim.x) {
    const int n = H.node(a);
    for (int r = 0; r < RH; ++r) s.nn_req[(size_t)r * MAXN + n] = H.q(r, a);
  }
  if (tid == 0) {
    s.counters[kCtrNewNodes] = n_new;
    s.counters[kCtrUnscheduled] = qlen;
    s.counters[kCtrNodesVisited] = nodes_visited;
    s.counters[kCtrAddCalls] = add_calls;
    s.counters[kCtrError] = fatal;
    s.counters[kCtrSteps] = add_calls;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    s.counters[kCtrPackEnd] = (long long)t;
#ifdef KSCHED_PROFILE_PACK
    s.counters[kCtrRunCallCycles] = pk_acc[1];
    s.counters[kCtrGenCallCycles] = pk_acc[5];  // (incl. the call)
#endif
  }
}
