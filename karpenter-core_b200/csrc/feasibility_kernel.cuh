// feasibility_kernel.cuh - K0 (queue order, dense pod-row matrix) and K1 (dense pods x instance-types feasibility bitmask).
// Part of the single translation unit ksched.cu (included inside its anonymous namespace, in this order: catalog.cuh,
// feasibility_kernel.cuh, topology.cuh, pack_kernel.cuh); not a standalone header.
#pragma once

// ------------------------------------------------------------------------------------------------
// K0: queue order
// ------------------------------------------------------------------------------------------------
// queue.go:82-108 (cpu desc, memory desc, timestamp asc, UID asc) as ONE packed key: (rank of the class's (cpu, memory)
// pair among all classes, timestamp - ts_min or the timestamp's dense rank, UID rank). cls_rank and the timestamp field are
// chosen on the host at upload (bind_problem).
__global__ void sort_key1_kernel(int n, const uint32_t* __restrict__ cls_rank, const uint32_t* __restrict__ pod_class, const int64_t* __restrict__ ts,
                                 const uint32_t* __restrict__ uid_rank, long long ts_min, int ts_bits, int uid_bits, uint64_t* key, uint32_t* idx) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = ((uint64_t)cls_rank[pod_class[i]] << (ts_bits + uid_bits)) | ((uint64_t)(ts[i] - ts_min) << uid_bits) | (uint64_t)uid_rank[i];
  idx[i] = (uint32_t)i;
}

// ------------------------------------------------------------------------------------------------
// K1: feasibility. One warp per pod row; lane l owns column words l, l+32, ...
// ------------------------------------------------------------------------------------------------
struct K1Params {
  DevCatalog cat;
  const uint64_t* rows;  // [n_pods][32] FFD order
  int n_pods;
  const uint32_t* itype_sets;  // [n][W32]
  uint32_t* F;                 // [n_pods][n_templates][W32]
  unsigned long long* best;    // [n_pods]
  int word_begin, word_end;    // column shard (u32 words) this device computes
  int alloc_in_smem;           // the sorted allocatable arrays fit in the CTA's shared memory
  long long* dbg;              // optional cycle counters (KSCHED_PROFILE_K1)
  int tables_in_smem;          // valset / absent / negempty / offset / anyoffer / member are staged too
  int n_valrows, n_offrows;
  const int64_t* cls_req_ext;        // [n_pods = classes][n_res_ext] or nullptr (ksched.h: ksched_problem.class_requests_ext)
  const uint32_t* cls_ext_present;   // [classes] or nullptr
};


constexpr int kK1Threads = 512;
constexpr int kK1Cache = 16;  // per-lane words of the previous row's result kept for identical consecutive rows

// The class pass's work split and cache rule, shared by the kernel and the host's record of its launch (ksched_k1_plan):
// each warp owns a contiguous chunk of rows, and the consecutive-row cache holds V * wpl words per lane.
__host__ __device__ constexpr int k1_chunk(int n_rows, int n_warps) { return (n_rows + n_warps - 1) / n_warps; }
__host__ __device__ constexpr bool k1_cacheable(int n_templates, int W32) { return n_templates * ((W32 + 31) >> 5) <= kK1Cache; }




// ------------------------------------------------------------------------------------------------
// K1 proper: the dense P x (templates x instance types) feasibility bitmask F and the per-pod best column, in FFD order.
// Row j of F is the row of pod j's class (class_feasibility_kernel): this kernel is a pure stream - per 32 pod rows one
// coalesced load of their class words (the `reserved` word of the 256-byte FFD rows K0 wrote), then 16-byte stores of the
// class rows (read through L1: consecutive pods share a class, the n_classes x RW table stays cache-resident).
// Algorithmic bytes (SURVEY 8d): P*256 + C*256 + P*C/8; physical: the class word's 32-byte sector of every row + the
// matrix + the best vector.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) feasibility_kernel(const uint64_t* __restrict__ rows, int n_pods, int n_classes, int RW,
                                                          const uint32_t* __restrict__ Fclass, const unsigned long long* __restrict__ best_class,
                                                          uint32_t* __restrict__ F, unsigned long long* __restrict__ best) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const int nblk = (n_pods + 31) >> 5;
  const int Q = RW >> 2;  // 16-byte chunks per row (RW = templates x column words is a multiple of 4: W32 is even, see below)
  for (int blk = warp; blk < nblk; blk += nwarps) {
    const int j = (blk << 5) + lane;
    uint32_t cls = 0;
    if (j < n_pods) {
      cls = (uint32_t)__ldg(rows + (size_t)j * KSCHED_ROW_WORDS + 31);  // ksched_pod_row::reserved = the row's class
      if (cls >= (uint32_t)n_classes) cls = 0;
      best[j] = __ldg(best_class + cls);
    }
    const int rows_here = min(32, n_pods - (blk << 5));
    uint4* dst = reinterpret_cast<uint4*>(F + (size_t)(blk << 5) * RW);
    const int total = rows_here * Q;
    if ((RW & 3) == 0) {
      for (int q0 = 0; q0 < total; q0 += 32) {  // uniform trip count: every lane takes part in the shuffle
        const int q = q0 + lane, qc = q < total ? q : total - 1;
        const int r = qc / Q, part = qc - r * Q;
        const uint32_t c2 = __shfl_sync(0xffffffffu, cls, r);
        if (q < total) dst[q] = __ldg(reinterpret_cast<const uint4*>(Fclass + (size_t)c2 * RW) + part);
      }
    } else {
      for (int r = 0; r < rows_here; ++r) {
        const uint32_t c2 = __shfl_sync(0xffffffffu, cls, r);
        for (int w = lane; w < RW; w += 32) F[((size_t)(blk << 5) + r) * RW + w] = __ldg(Fclass + (size_t)c2 * RW + w);
      }
    }
  }
}
