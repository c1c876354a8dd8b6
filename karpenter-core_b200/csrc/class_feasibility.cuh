// class_feasibility.cuh - the kernels that read the K1 class pass's constant parameters (g_k1) or, through the variant
// table's build, the pack kernel's (g_k2): class_feasibility_kernel and the row gather.
// Part of the single translation unit ksched.cu, which includes it once per parameter slot (namespaces slot0, slot1, each
// followed by topology.cuh and pack_kernel.cuh); not a standalone header.

__device__ void k0_extra_block(int b);  // pack_kernel.cuh
// FFD-ordered dense pod-row matrix: row j = class row of the j-th pod of the queue. One warp per row,
// 256-byte coalesced loads and stores. kTable: the blocks from `blocks` on build the pack kernel's variant table and run
// records (k0_extra_block), which depend on nothing this launch writes; the launches without them keep the gather's small
// register and shared-memory footprint.
template <bool kTable>
__global__ void gather_rows_kernel(int n, const ksched_pod_row* __restrict__ classes, const uint32_t* __restrict__ pod_class,
                                   const uint32_t* __restrict__ order, uint64_t* __restrict__ rows, int blocks) {
  if (kTable && (int)blockIdx.x >= blocks) {
    k0_extra_block((int)blockIdx.x - blocks);
    return;
  }
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nwarps = (blocks * blockDim.x) >> 5;
  for (int j = warp; j < n; j += nwarps) {
    const uint64_t* src = reinterpret_cast<const uint64_t*>(&classes[pod_class[order[j]]]);
    rows[(size_t)j * KSCHED_ROW_WORDS + lane] = src[lane];
  }
}

// Parameters in constant memory and the CTA's catalog view (table pointers redirected to the staged shared-memory
// copies) in shared memory: the out-of-line row evaluation reads both with immediate addresses instead of through
// references to a kernel parameter / a stack copy (see g_k2 in topology.cuh for what that costs).
// One copy per parameter slot, like g_k2.
__constant__ K1Params g_k1;
__shared__ DevCatalog g_k1cat;

// One row's feasibility against every (template, column): the rarely taken path of feasibility_kernel (rows that differ
// from their predecessor), kept out of line so that the batched streaming loop stays small.
__device__ __noinline__ unsigned long long k1_compute_row(int j, uint64_t word, uint32_t* cache, bool cacheable) {
  const DevCatalog& c = g_k1cat;
  const K1Params& p = g_k1;
  const int lane = threadIdx.x & 31;
  const int V = c.n_templates, W32 = c.W32, NK = c.n_keys, R = c.n_res, T = c.n_types;
  const int wpl = (W32 + 31) >> 5;
    const uint64_t meta = __shfl_sync(0xffffffffu, word, 24);
    const uint64_t tolerated = __shfl_sync(0xffffffffu, word, 25);
    const uint32_t pod_res_present = (uint32_t)__shfl_sync(0xffffffffu, word, 28);
    const uint32_t itype_req = (uint32_t)__shfl_sync(0xffffffffu, word, 29);
    unsigned long long best = kNoBest;
    for (int v = 0; v < V; ++v) {
      const ksched_template& tm = c.templates[v];
      uint32_t* out = p.F + ((size_t)j * V + v) * W32;
      bool ok = (tolerated >> tm.taintset) & 1;  // Taints.Tolerates
      // lanes 8..23 own one requirement key each: Compatible + merge (node.go:73-81 on a fresh node)
      uint64_t allowed = 0;
      bool neg = false, present = false, compat = true;
      const int k = lane - 8;
      if (k >= 0 && k < NK) {
        Req pod;
        pod.present = (meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1;
        pod.complement = (meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1;
        pod.has_gt = pod.has_lt = false; pod.gt = pod.lt = 0;
        pod.values = word;
        Req node = ksched::req_load(tm.reqs, nullptr, k);
        KeyMeta km = key_meta(c, k);
        compat = ksched::key_compatible(node, pod, c.keys[k].well_known != 0, km);
        Req merged = ksched::key_add(node, pod, km);
        present = merged.present;
        if (present) {
          allowed = ksched::req_allowed(merged, c.keys[k].dict_mask, km);
          neg = ksched::req_op_negative(merged, km);
        }
      }
      ok = ok && (__ballot_sync(0xffffffffu, !compat) == 0);
      const uint32_t present_keys = (__ballot_sync(0xffffffffu, present) >> 8) & c.type_relevant;
      // resources: lanes 0..7 own one resource each (Fits, resources.go:138-145)
      int rank = 0;
      bool res_used = false;
      if (lane < R) {
        uint32_t pres = pod_res_present | tm.daemon_res_present;
        res_used = (pres >> lane) & 1;
        if (res_used) rank = fit_rank(c.alloc_sorted, T, lane, (int64_t)word + tm.daemon_requests[lane]);
      }
      const uint32_t res_mask = __ballot_sync(0xffffffffu, res_used);
      uint64_t zallowed = ~0ull, callowed = ~0ull;
      bool zc_unconstrained = true;
      if (c.zone_key >= 0) {
        bool zp = __shfl_sync(0xffffffffu, (int)present, 8 + c.zone_key);
        uint64_t za = __shfl_sync(0xffffffffu, allowed, 8 + c.zone_key);
        if (zp) { zallowed = za; zc_unconstrained = false; }
      }
      if (c.ct_key >= 0) {
        bool cp = __shfl_sync(0xffffffffu, (int)present, 8 + c.ct_key);
        uint64_t ca = __shfl_sync(0xffffffffu, allowed, 8 + c.ct_key);
        if (cp) { callowed = ca; zc_unconstrained = false; }
      }
      const uint64_t slots = zc_unconstrained ? ~0ull : node_slots(c, zallowed, callowed);
      bool any = false;
      int first_word = -1;
      uint32_t first_bits = 0;
      for (int wi = 0; wi < wpl; ++wi) {
        const int w = wi * 32 + lane;
        const bool mine = w < W32 && w >= p.word_begin && w < p.word_end;
        uint32_t s = 0;
        if (ok && mine) s = c.member[(size_t)v * W32 + w];
        uint32_t pk = present_keys;
        while (pk) {  // uniform loop: every lane walks the same keys
          int kk = __ffs(pk) - 1;
          pk &= pk - 1;
          uint64_t a = __shfl_sync(0xffffffffu, allowed, 8 + kk);
          bool ng = __shfl_sync(0xffffffffu, (int)neg, 8 + kk);
          if (s) s &= key_typeset_word(c, kk, a, ng, w);
        }
        if (s) s &= offer_word(c, slots, zc_unconstrained, w);
        uint32_t rm = res_mask, fit = 0xFFFFFFFFu;
        while (rm) {  // the loads do not depend on each other (nor on s): one memory round trip for all resources
          int r = __ffs(rm) - 1;
          rm &= rm - 1;
          int rk = __shfl_sync(0xffffffffu, rank, r);
          if (w < W32) fit &= c.fitset[((size_t)r * (T + 1) + rk) * W32 + w];
        }
        s &= fit;
        if (s && p.cls_ext_present) {  // the rows are the class table: row j is class j
          const uint32_t xp = p.cls_ext_present[j];
          if (xp) s = ext_fit_word(c, nullptr, p.cls_req_ext + (size_t)j * c.n_res_ext, xp, s, w);
        }
        if (s && itype_req != KSCHED_NONE) s &= p.itype_sets[(size_t)itype_req * W32 + w];
        if (mine) out[w] = s;
        if (cacheable) cache[v * wpl + wi] = s;
        uint32_t nz = __ballot_sync(0xffffffffu, s != 0);
        if (nz && !any) {
          any = true;
          int src = __ffs(nz) - 1;
          first_word = wi * 32 + src;
          first_bits = __shfl_sync(0xffffffffu, s, src);
        }
      }
      if (any) {
        int t = first_word * 32 + __ffs(first_bits) - 1;  // columns are in price order: first set bit = cheapest
        unsigned long long key = ((unsigned long long)__float_as_uint(c.price32[t]) << 32) | ((unsigned long long)v << 24) | (unsigned)t;
        best = key < best ? key : best;
      }
    }
  return best;
}


// class_feasibility_kernel: the row evaluation, run over the n_classes DISTINCT pod rows (K1Params::rows = the class table):
// pods of one class are indistinguishable to the scheduler, so their feasibility rows are identical and each is computed
// once. feasibility_kernel (below) then materialises the dense pods x (template, instance type) matrix from them.
// Shared-memory staging: the small tables every row evaluation walks with DEPENDENT loads (templates, key info, the
// value->row maps, the sorted allocatable arrays of the Fits binary search) are copied once per CTA; the wide column
// bitsets (valset / fitset / member / offset) stay in global memory and are read one coalesced word per lane.
// Each warp owns a CONTIGUOUS chunk of the FFD-ordered pod-row matrix: consecutive rows are very often identical in
// every field that matters to feasibility (same deployment), and then the previous result is written out again.
__global__ void __launch_bounds__(kK1Threads, 1) class_feasibility_kernel() {
  extern __shared__ __align__(16) unsigned char k1_smem[];
#ifdef KSCHED_PROFILE_K1
  long long t_start = clock64(), t_stage = 0, t_compute = 0, n_compute = 0;
#endif
  const K1Params& p = g_k1;
  DevCatalog c = p.cat;
  const int V = c.n_templates, W32 = c.W32, NK = c.n_keys, R = c.n_res, T = c.n_types;
  {
    unsigned char* ptr = k1_smem;
    ksched_template* s_tmpl = reinterpret_cast<ksched_template*>(ptr); ptr += sizeof(ksched_template) * V;
    ksched_keyinfo* s_keys = reinterpret_cast<ksched_keyinfo*>(ptr); ptr += sizeof(ksched_keyinfo) * KSCHED_MAX_KEYS;
    int64_t* s_alloc = reinterpret_cast<int64_t*>(ptr); ptr += p.alloc_in_smem ? sizeof(int64_t) * R * T : 0;
    int16_t* s_valrow = reinterpret_cast<int16_t*>(ptr); ptr += sizeof(int16_t) * KSCHED_MAX_KEYS * 64;
    int16_t* s_offrow = reinterpret_cast<int16_t*>(ptr); ptr += sizeof(int16_t) * 64;
    uint64_t* s_slots = reinterpret_cast<uint64_t*>(ptr);
    // cp.async (LDGSTS): every 4-byte element of every table is requested before anything is waited on, so the whole
    // staging costs about one memory round trip instead of one per table.
    auto stage4 = [&](void* dst, const void* src, int n_words) {
      const uint32_t* g = reinterpret_cast<const uint32_t*>(src);
      int done = 0;
      if ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) {  // 16-byte copies for the aligned bulk (4x fewer requests)
        const int n16 = n_words >> 2;
        for (int i = threadIdx.x; i < n16; i += blockDim.x) {
          const unsigned d = (unsigned)__cvta_generic_to_shared(reinterpret_cast<uint32_t*>(dst) + 4 * i);
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(g + 4 * i));
        }
        done = n16 << 2;
      }
      for (int i = done + threadIdx.x; i < n_words; i += blockDim.x) {
        const unsigned d = (unsigned)__cvta_generic_to_shared(reinterpret_cast<uint32_t*>(dst) + i);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(g + i));
      }
    };
    stage4(s_tmpl, c.templates, (int)(sizeof(ksched_template) * V / 4));
    stage4(s_keys, c.keys, (int)(sizeof(ksched_keyinfo) * NK / 4));
    if (p.alloc_in_smem) stage4(s_alloc, c.alloc_sorted, R * T * 2);
    stage4(s_valrow, c.valrow, NK * 64 / 2);
    stage4(s_offrow, c.offrow, 32);
    stage4(s_slots, c.slots, 128 * 2);
    if (p.tables_in_smem) {
      // the narrow column bitsets: one 4*W32-byte row per (key,value) / key / offering / template
      uint32_t* sp = reinterpret_cast<uint32_t*>(s_slots + 128);
      auto stage = [&](const uint32_t*& tbl, int rows) {
        stage4(sp, tbl, rows * W32);
        tbl = sp;
        sp += rows * W32;
      };
      stage(c.valset, p.n_valrows);
      stage(c.absent, NK);
      stage(c.negempty, NK);
      stage(c.offset, p.n_offrows);
      stage(c.anyoffer, 1);
      stage(c.member, V);
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    c.templates = s_tmpl;
    c.keys = s_keys;
    if (p.alloc_in_smem) c.alloc_sorted = s_alloc;
    c.valrow = s_valrow;
    c.offrow = s_offrow;
    c.slots = s_slots;
    if (threadIdx.x == 0) g_k1cat = c;
  }
  __syncthreads();
#ifdef KSCHED_PROFILE_K1
  t_stage = clock64() - t_start;
#endif

  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int chunk = k1_chunk(p.n_pods, nwarps);
  const int j0 = warp * chunk, j1 = min(p.n_pods, j0 + chunk);
  const int wpl = (W32 + 31) >> 5;  // column words per lane
  const bool cacheable = k1_cacheable(V, W32);
  // fields of the row that feasibility depends on (requests, requirement masks, meta, tolerations, res_present, itype_req)
  // With ext resources the class index (word 31) as well: two classes may differ in an ext request only.
  const uint64_t cmp_mask = lane <= 25 ? ~0ull : ((lane == 28 || lane == 29) ? 0xFFFFFFFFull : ((lane == 31 && p.cls_ext_present) ? ~0ull : 0ull));
  uint32_t cache[kK1Cache];
  unsigned long long best_prev = kNoBest;
  uint64_t prev_word = 0;
  bool have_prev = false;

  // rows are fetched kBatch at a time (kBatch independent 256-byte loads in flight per warp), then consumed in order
  constexpr int kBatch = 16;
  uint64_t wbuf[kBatch];
  for (int jb = j0; jb < j1; jb += kBatch) {
#pragma unroll
    for (int b = 0; b < kBatch; ++b) wbuf[b] = jb + b < j1 ? __ldg(p.rows + (size_t)(jb + b) * KSCHED_ROW_WORDS + lane) : 0;
    if (have_prev && cacheable) {
      // the usual case: the whole batch repeats the cached row (same deployment) -> one vote, then nothing but stores
      uint64_t diff = 0;
#pragma unroll
      for (int b = 0; b < kBatch; ++b) diff |= jb + b < j1 ? ((wbuf[b] ^ prev_word) & cmp_mask) : 0;
      if (__all_sync(0xffffffffu, diff == 0)) {
        const int nb = min(kBatch, j1 - jb);
        const size_t row_stride = (size_t)V * W32;
        for (int v = 0; v < V; ++v)
          for (int wi = 0; wi < wpl; ++wi) {
            const int w = wi * 32 + lane;
            if (w < W32 && w >= p.word_begin && w < p.word_end) {
              const uint32_t val = cache[v * wpl + wi];
              uint32_t* dst = p.F + ((size_t)jb * V + v) * W32 + w;
              for (int b = 0; b < nb; ++b, dst += row_stride) *dst = val;
            }
          }
        if (lane < nb) p.best[jb + lane] = best_prev;
        continue;
      }
    }
#pragma unroll
    for (int b = 0; b < kBatch; ++b) {
    const int j = jb + b;
    if (j >= j1) break;
    const uint64_t word = wbuf[b];  // lane l holds u64 word l of the 256-byte row
    const bool same = have_prev && cacheable && __all_sync(0xffffffffu, ((word ^ prev_word) & cmp_mask) == 0);
    if (same) {
      for (int v = 0; v < V; ++v)
        for (int wi = 0; wi < wpl; ++wi) {
          const int w = wi * 32 + lane;
          if (w < W32 && w >= p.word_begin && w < p.word_end) p.F[((size_t)j * V + v) * W32 + w] = cache[v * wpl + wi];
        }
      if (lane == 0) p.best[j] = best_prev;
      continue;
    }
    prev_word = word;
    have_prev = true;
#ifdef KSCHED_PROFILE_K1
    long long tc0 = clock64();
#endif
    const unsigned long long best = k1_compute_row(j, word, cache, cacheable);
#ifdef KSCHED_PROFILE_K1
    t_compute += clock64() - tc0; ++n_compute;
#endif
    best_prev = best;
    if (lane == 0) p.best[j] = best;
    }
  }
#ifdef KSCHED_PROFILE_K1
  if (p.dbg && lane == 0) {
    atomicMax((unsigned long long*)&p.dbg[0], (unsigned long long)t_stage);
    atomicMax((unsigned long long*)&p.dbg[1], (unsigned long long)t_compute);
    atomicMax((unsigned long long*)&p.dbg[2], (unsigned long long)(clock64() - t_start));
    atomicMax((unsigned long long*)&p.dbg[3], (unsigned long long)n_compute);
    atomicAdd((unsigned long long*)&p.dbg[4], (unsigned long long)n_compute);
    atomicAdd((unsigned long long*)&p.dbg[5], (unsigned long long)t_compute);
  }
#endif
}
