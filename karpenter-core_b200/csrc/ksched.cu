// ksched.cu — sm_90a kernels and the C-ABI of include/ksched.h.
//
//  K0  sort_keys / gather_rows   FFD order of the queue (queue.go:35-110) and the dense, FFD-ordered
//                                P x 256 B pod-row matrix the feasibility kernel streams.
//  K1  class_feasibility_kernel + feasibility_kernel: dense pods x (template, instance type) bitmask F, bit-sliced over columns:
//                                Requirements.Compatible/Intersects (requirements.go:123-206), fits /
//                                hasOffering (node.go:143-159), Taints.Tolerates (taints.go:28) as AND/OR of
//                                precomputed column bitsets; warp ballot/ffs gives the per-pod best column.
//  K2  pack_kernel               the sequential first-fit of Scheduler.add (scheduler.go:174-219) with
//                                Node.Add / ExistingNode.Add (node.go:62-107, existingnode.go:77-130),
//                                topology domains (topology.go:120-167, topologygroup.go:88-243), queue
//                                requeue / relaxation (scheduler.go:104-124, queue.go:44-68) in ONE persistent
//                                CTA: candidate nodes are examined in parallel, the reference's scan order is
//                                recovered with a block-wide argmin on (pod count, stable tie-break).
// Integer / bitmask work only — no tensor cores by design (BASELINE.json north_star).
#include <cuda_runtime.h>
#include <nccl.h>
#include <stdint.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cub/cub.cuh>
#include <string>
#include <mutex>
#include <vector>

#include "ksched.h"
#include "reqmask.cuh"
#include "launch.cuh"

using ksched::KeyMeta;
using ksched::Req;

#define CUDA_TRY(h, expr)                                                                         \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      (h)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                              \
      return KSCHED_ERR_CUDA;                                                                     \
    }                                                                                             \
  } while (0)

namespace {

constexpr int kMaxCG = 8;        // topology groups that may constrain one pod class
constexpr int kMaxTouched = 8;   // requirement keys one Add may touch (pod keys + topology keys)
constexpr int kPackThreads = 512;
constexpr int kPackThreadsSmall = 256;  // blocks up to this size launch the pack_kernel instantiation with twice the registers
constexpr int kFreshMemoSlots = 8192;  // PackState::fd_*
// PackState::counters: the results of a Solve, then the KSCHED_PROFILE_PACK profile (print_pack_profile)
enum Counter : int {
  kCtrNewNodes, kCtrUnscheduled, kCtrNodesVisited, kCtrAddCalls, kCtrError, kCtrSteps,
  kCtrMaskCycles, kCtrMaskPods,  // mask run: cycles of its walks and stores, pods
  // generic_step (GK_T / GK_C): cycles per phase, then counts
  kCtrGenTopo, kCtrGenExisting, kCtrGenEval, kCtrGenCommit, kCtrGenFresh, kCtrGenFail,
  kCtrRunCallCycles, kCtrGenCallCycles,  // cycles inside class_run / generic_step calls
  kCtrMaskEntries,
  kCtrGenSteps, kCtrGenInflightPlaced, kCtrGenFreshSteps, kCtrGenFailures,
  kCtrGenPath,  // 5 paths: rejected, cached, row, dyn, cached empty
  kCtrGenFreshDecide = kCtrGenPath + 5, kCtrGenFreshWords, kCtrGenFreshCommit, kCtrGenInflightVerify,
  kCtrGenInflightWinner, kCtrGenInflightRecord,
  // class_run, classes without mask-key spread in level mode (RunLv) and all others (Run)
  kCtrRunLvCycles, kCtrRunLvPods, kCtrRunLvSteps, kCtrRunLvFresh, kCtrRunCycles, kCtrRunPods,
  kCtrMaskBuildCycles,
  kCtrRunFresh, kCtrRunCalls, kCtrRunPlaced, kCtrRunBails, kCtrRunIneligible, kCtrRunLvPerPod, kCtrRunPerPod, kCtrRunLvFills,
  kCtrMaskBuildRefused, kCtrMaskUnpinnedSingle,
  kCtrPinSteps, kCtrPinPods, kCtrPinEndStaged, kCtrPinEndCount, kCtrPinEndKey, kCtrPinEndRefused, kCtrPinEndList,
  kCtrRoundTripCycles, kCtrNoVariantStops, kCtrNoVariantTripCycles, kCtrVarStoreHits, kCtrVarStoreEntries,
  kCtrRoundCycles, kCtrRounds, kCtrRoundPods,
  kCtrStretchPinned, kCtrStretchFresh = kCtrStretchPinned + 16,  // round stretches by length 1..16
  kCtrMaskSteps = kCtrStretchFresh + 16, kCtrMaskMultiDomain, kCtrMaskRoundable,
  // pinned rounds with equal counts whose bucket stretch stopped before a second round, by the first lane's reason: singleton
  // bucket whose head accepts again, singleton bucket whose head is done, unpinned key, inexact room word, kM1Lv, staged end
  kCtrBucketEnd,
  kCtrFillLen = kCtrBucketEnd + 6,   // fill stretches by length 1..16 (rounds that keep every zone's head)
  kCtrRoundsUnequal = kCtrFillLen + 16,  // single rounds whose counts are not all equal
  // class_run's fixed cost per call: open nodes at entry (summed), cycles from entry to the first loop iteration of the
  // eligible calls (of which the per-node inputs), write-back cycles, and the compactions with the slots they scanned and their cycles
  kCtrRunActiveSum, kCtrRunEntryCycles, kCtrRunInputCycles, kCtrRunWbCycles, kCtrRunCompacts, kCtrRunCompactSlots, kCtrRunCompactCycles,
  kNumCounters
};
constexpr uint64_t kNoBest = ~0ull;

#include "catalog.cuh"
#include "feasibility_kernel.cuh"
#include "topology.cuh"

}  // namespace

#include "pack_kernel.cuh"
#include "cluster.cuh"

namespace {

// Launch choice per finished new node (launch.cuh): one warp per node, lanes over the words of its final option set.
__global__ void launch_choice_kernel(DevCatalog c, const long long* counters, const uint64_t* nn_vals, const uint64_t* nn_meta,
                                     const uint32_t* nn_opts, int max_new, ksched_launch_choice* out) {
  const int n_new = (int)counters[kCtrNewNodes];
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int n = warp; n < n_new; n += nwarps) {
    // offering slots the node's requirements admit (Offerings.Requirements, types.go:120-126)
    uint64_t zallowed = ~0ull, callowed = ~0ull;
    const uint64_t meta = nn_meta[n];
    if (c.zone_key >= 0) {
      const Req z = load_soa(nn_vals, meta, max_new, n, c.zone_key);
      if (z.present) zallowed = ksched::req_allowed(z, c.keys[c.zone_key].dict_mask, key_meta(c, c.zone_key));
    }
    if (c.ct_key >= 0) {
      const Req ct = load_soa(nn_vals, meta, max_new, n, c.ct_key);
      if (ct.present) callowed = ksched::req_allowed(ct, c.keys[c.ct_key].dict_mask, key_meta(c, c.ct_key));
    }
    const uint64_t slots = node_slots(c, zallowed, callowed) & c.offer_used;
    unsigned long long best = ~0ull, best_off = ksched::kNoOffering;
    int best_col = -1;
    for (int w = lane; w < c.W32; w += 32) {
      uint32_t m = nn_opts[(size_t)w * max_new + n];
      while (m) {
        const int t = w * 32 + __ffs(m) - 1;
        m &= m - 1;
        const uint64_t ok = ksched::offering_min_key(c.offer_keys + (size_t)t * 64, slots);
        if (ok == ksched::kNoOffering) continue;
        const unsigned long long key = ksched::option_key(ok, c.input_index[t]);
        if (key < best) { best = key; best_off = ok; best_col = t; }
      }
    }
    const unsigned long long wbest = warp_min_u64(best);
    const unsigned owner = __ballot_sync(0xffffffffu, best == wbest && best != ~0ull);  // keys are unique per option
    if (owner) {
      const int src = __ffs(owner) - 1;
      best_col = __shfl_sync(0xffffffffu, best_col, src);
      best_off = __shfl_sync(0xffffffffu, best_off, src);
    } else {
      best_col = -1;
    }
    if (lane == 0) {
      ksched_launch_choice o;
      o.type_column = best_col;
      o.offering_slot = best_col >= 0 ? (int32_t)(best_off & 0xFF) : -1;
      o.price_rank = best_col >= 0 ? (uint32_t)(best_off >> 16) : 0;
      o.offering_index = best_col >= 0 ? (uint32_t)((best_off >> 8) & 0xFF) : 0;
      out[n] = o;
    }
  }
}

// L2 flush helper: write a buffer larger than L2 between timed iterations
__global__ void flush_kernel(uint32_t* buf, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) buf[i] = (uint32_t)i;
}

template <class T>
struct DevBuf {
  T* ptr = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n) {
    if (n <= cap && ptr) return cudaSuccess;
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    cap = 0;
    size_t want = n ? n : 1;
    cudaError_t e = cudaMalloc(&ptr, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (ptr) cudaFree(ptr); ptr = nullptr; cap = 0; }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
};

}  // namespace

// Every array a Solve mutates goes back to its pristine copy (or to zero) in ONE launch: a table of (dst, src, bytes)
// segments passed by value (reset_kernel). (Round 1 issued ~20 cudaMemcpyAsync / cudaMemsetAsync calls per Solve; a
// consolidation simulation is so short that those launches were most of it.)
struct ResetSeg { void* dst; const void* src; unsigned long long bytes; };
struct ResetTable { int n; ResetSeg seg[30]; };

struct ksched_handle {
  K1Params k1_host;  // staging copies of the kernels' constant-memory parameters (must outlive the async copies)
  K2Params k2_host;  // staging copy of the pack kernel's constant-memory parameters (must outlive the async copy)
  int device = 0;
  int n_sm = 132;  // streaming multiprocessors of `device` (grid sizes of the grid-stride kernels)
  cudaStream_t stream = nullptr;
  std::string err;
  // ---- catalog (ksched_load_catalog): `cat` points into the buffers of this group
  bool have_catalog = false;
  DevCatalog cat{};
  int n_valrows = 1, n_offrows = 1;  // rows of cat.valset / cat.offset
  std::vector<ksched_template> h_templates;
  std::vector<unsigned char> catalog_blob;  // host copy of the resident catalog's inputs (ksched_load_catalog early-out)
  DevBuf<ksched_keyinfo> d_keys;
  DevBuf<ksched_key_regions> d_key_regions;
  DevBuf<ksched_template> d_templates;
  DevBuf<ksched_type_row> d_types;
  DevBuf<int64_t> d_key_int, d_capacity, d_alloc_sorted, d_alloc_rt, d_alloc_ext;
  DevBuf<float> d_price32;
  DevBuf<int16_t> d_valrow, d_offrow;
  DevBuf<int32_t> d_perm_desc;
  DevBuf<uint32_t> d_valset, d_absent, d_negempty, d_offset, d_anyoffer, d_member, d_fitset, d_domset, d_input_index;
  DevBuf<uint64_t> d_offer_keys, d_slots;
  // ---- problem (ksched_upload): `st` points into the buffers of this group; reset_state restores the `resets` segments
  bool uploaded = false;
  bool sorted = false;  // the FFD-ordered pod-row matrix of the uploaded problem exists
  PackState st{};
  ResetTable resets{};
  // queue order (feasibility_kernel.cuh: sort_key1_kernel): total key bits and the timestamp field's width and origin
  int sort1_bits = 0, sort1_ts_bits = 0, sort1_uid_bits = 0;
  long long sort1_ts_min = 0;
  std::vector<int64_t> ts_dense;  // each pod's rank among the distinct timestamps when the offset is too wide, else empty
  size_t cub_tmp_bytes = 0;
  // inputs
  DevBuf<ksched_pod_row> d_classes;
  DevBuf<ksched_topo_group> d_groups;
  DevBuf<ksched_class_topo> d_class_topo;
  DevBuf<RelX> d_relx;
  DevBuf<ksched_reqset> d_filter_terms;
  DevBuf<ksched_class_volumes> d_cls_vol;
  DevBuf<int32_t> d_hostname_reqs, d_grp_host_row;
  DevBuf<int64_t> d_ts, d_ex_avail, d_cls_req_ext, d_ex_avail_ext;
  DevBuf<uint8_t> d_itype_comp, d_cls_hp_ext, d_cls_has_vol;
  DevBuf<uint32_t> d_pod_class0, d_uid_rank, d_itype_sets, d_filter_hostname, d_cls_rank, d_cls_ext_present, d_ex_avail_present, d_ex_taintset,
      d_ex_itype;
  DevBuf<uint64_t> d_hostname_slots, d_cls_tol_ext, d_cls_hpc_ext, d_cls_hpe_ext, d_cls_vol_ext, d_vol_mask_ext;
  DevBuf<uint32_t> d_filter_itype, d_tmpl_itype, d_ex_it0, d_ex_it, d_nn_it;  // instance-type filter tables and slot state
  // pristine copies of what a Solve mutates
  DevBuf<ksched_node_volumes> d_ex_vol0;
  DevBuf<int32_t> d_grp_cnt0, d_grp_host_total0;
  DevBuf<int64_t> d_ex_req0;
  DevBuf<uint8_t> d_grp_active0;
  DevBuf<uint16_t> d_grp_host0;
  DevBuf<uint32_t> d_ex_req_present0;
  DevBuf<uint64_t> d_ex_vals0, d_ex_meta0, d_ex_hp0, d_ex_hp_ext0, d_ex_vol_ext0, d_grp_registered0;
  // working state
  DevBuf<ksched_node_volumes> d_ex_vol;
  DevBuf<int32_t> d_relax, d_assign, d_place_seq, d_last_len, d_cls_cursor, d_grp_cnt, d_grp_host_total, d_grp_min_slot;
  DevBuf<int64_t> d_ex_req, d_ex_req_ext, d_remaining;
  DevBuf<uint8_t> d_ex_closed, d_grp_active;
  DevBuf<uint16_t> d_grp_host;
  DevBuf<uint32_t> d_pod_class, d_queue, d_last_epoch, d_ex_req_present;
  DevBuf<uint64_t> d_ex_vals, d_ex_meta, d_ex_hp, d_ex_hp_ext, d_ex_vol_ext, d_grp_registered;
  DevBuf<long long> d_counters;  // kNumCounters entries (Counter)
  // K0 / K1
  DevBuf<uint32_t> d_order, d_idx_tmp, d_pod_pos, d_F, d_Fclass;
  DevBuf<uint64_t> d_k_tie, d_k_tmp, d_rows;
  DevBuf<unsigned long long> d_best, d_best_class;
  DevBuf<uint8_t> d_cub_tmp;
  // new nodes, open-node overflow and the fresh-node memos (PackState)
  DevBuf<int32_t> d_nn_count, d_nn_tb, d_ov_node;
  DevBuf<int64_t> d_nn_req, d_nn_req_ext;
  DevBuf<uint8_t> d_nn_tmpl, d_fc_state, d_fc_dom, d_fc_front_state, d_fd_state, d_fd_dom;
  DevBuf<uint32_t> d_nn_req_present, d_nn_opts, d_nn_ext_present, d_ov_absorbed, d_ov_rejected, d_fc_opts, d_fc_qp, d_fd_fc, d_fd_opts;
  DevBuf<uint64_t> d_nn_vals, d_nn_meta, d_nn_hp, d_nn_hp_ext, d_fc_vals, d_fc_meta, d_fd_meta, d_fd_vals;
  DevBuf<unsigned long long> d_ov_key;
  DevBuf<unsigned short> d_ov_flags;
  DevBuf<long long> d_ov_q, d_ov_bound, d_ov_bound2, d_fc_bound, d_fc_bound2, d_fc_q, d_fd_bound, d_fd_bound2;
  DevBuf<VarStoreEntry> d_vstore;
  // ---- device-resident cluster snapshot (ksched_load_cluster)
  bool have_cluster = false;
  int sup_pods = 0, sup_pending = 0;
  std::vector<int32_t> h_node_first, h_node_count;   // per existing slot: first superset pod bound to it, how many
  DevBuf<int32_t> d_sup_pod_node, d_node_first, d_node_dst, d_set_nodes, d_pod_src;
  DevBuf<uint32_t> d_sup_class, d_sup_uid, d_sim_types;
  DevBuf<int64_t> d_sup_ts, d_sim_remaining;
  DevBuf<uint8_t> d_in_set;
  DevBuf<SimResultDev> d_sim_results;
  bool cluster_topology = false;
  int filt_words = 0;
  DevBuf<uint32_t> d_cc_begin, d_filt;
  DevBuf<ksched_count_rel> d_cc;
  DevBuf<int8_t> d_node_dom;
  DevBuf<uint8_t> d_node_hostlabel;
  // ---- candidate ranking (ksched_rank_candidates)
  DevBuf<int32_t> d_rk_off, d_rk_prio, d_rk_order, d_rk_n;
  DevBuf<double> d_rk_dc, d_rk_age, d_rk_ttl, d_rk_cost_in, d_rk_cost, d_rk_cost_out;
  DevBuf<uint8_t> d_rk_flags, d_rk_elig_in, d_rk_elig;
  // ---- launch choices, all-gather, L2 flush, K1 profile
  DevBuf<ksched_launch_choice> d_launch;
  DevBuf<uint8_t> d_gather_send, d_gather_recv;
  DevBuf<uint32_t> d_flush;
  DevBuf<long long> d_k1dbg;
  // sharding / nccl
  int rank = 0, world = 1;
  ncclComm_t comm = nullptr;
  // timings
  ksched_timings tm{};
  cudaEvent_t ev[8] = {nullptr};
};

template <class T>
static cudaError_t upload(ksched_handle* h, DevBuf<T>& buf, const T* src, size_t n) {
  cudaError_t e = buf.ensure(n);
  if (e != cudaSuccess) return e;
  if (n == 0) return cudaSuccess;
  h->tm.h2d_bytes += (int64_t)(n * sizeof(T));
  return cudaMemcpyAsync(buf.ptr, src, n * sizeof(T), cudaMemcpyHostToDevice, h->stream);
}
template <class T>
static cudaError_t upload_vec(ksched_handle* h, DevBuf<T>& buf, const std::vector<T>& v) { return upload(h, buf, v.data(), v.size()); }

template <class T>
static cudaError_t download(ksched_handle* h, T* dst, const T* src, size_t n) {
  h->tm.d2h_bytes += (int64_t)(n * sizeof(T));
  return cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, h->stream);
}
// The first n columns of a device SoA array [rows][pitch] (new nodes), packed to [rows][n] on the host.
template <class T>
static cudaError_t download_soa(ksched_handle* h, std::vector<T>& dst, const T* src, int rows, size_t pitch, int n) {
  dst.resize((size_t)rows * n);
  h->tm.d2h_bytes += (int64_t)(dst.size() * sizeof(T));
  return cudaMemcpy2DAsync(dst.data(), (size_t)n * sizeof(T), src, pitch * sizeof(T), (size_t)n * sizeof(T), rows, cudaMemcpyDeviceToHost, h->stream);
}
// Node i's entries of a host copy [rows][n] of a SoA array, to row_of(i)[0 .. rows).
template <class T, class RowOf>
static void soa_to_rows(const std::vector<T>& soa, int rows, int n, RowOf row_of) {
  for (int i = 0; i < n; ++i) {
    T* row = row_of(i);
    for (int r = 0; r < rows; ++r) row[r] = soa[(size_t)r * n + i];
  }
}

static cudaError_t record_reset(ResetTable& t, void* dst, const void* src, size_t bytes) {
  if (!bytes) return cudaSuccess;
  if (t.n == (int)(sizeof t.seg / sizeof t.seg[0])) return cudaErrorInvalidValue;  // ResetTable::seg is too small
  t.seg[t.n++] = ResetSeg{dst, src, (unsigned long long)bytes};
  return cudaSuccess;
}

// One device array of the catalog or the problem: sized for n elements, `src` uploaded when given, and `field` (a DevCatalog
// or PackState pointer) bound to it.
template <class T, class F>
static cudaError_t bind(ksched_handle* h, DevBuf<T>& buf, F*& field, size_t n, const T* src = nullptr) {
  const cudaError_t e = src ? upload(h, buf, src, n) : buf.ensure(n);
  field = buf.ptr;
  return e;
}
// An array the pack kernel mutates: bound like bind(), with its pristine copy in `init` (uploaded from `src` when given,
// otherwise filled by the caller) and restored from it by reset_state before every run.
template <class T, class F>
static cudaError_t bind_restored(ksched_handle* h, DevBuf<T>& buf, F*& field, DevBuf<T>& init, size_t n, const T* src = nullptr) {
  cudaError_t e = src ? upload(h, init, src, n) : init.ensure(n);
  if (e == cudaSuccess) e = bind(h, buf, field, n);
  return e == cudaSuccess ? record_reset(h->resets, buf.ptr, init.ptr, n * sizeof(T)) : e;
}
// An array the pack kernel mutates that reset_state clears before every run.
template <class T, class F>
static cudaError_t bind_zeroed(ksched_handle* h, DevBuf<T>& buf, F*& field, size_t n) {
  const cudaError_t e = bind(h, buf, field, n);
  return e == cudaSuccess ? record_reset(h->resets, buf.ptr, nullptr, n * sizeof(T)) : e;
}

static int type_words64(int n_types) { int w = (n_types + 63) / 64; return w ? w : 1; }

extern "C" {

int ksched_abi_version(void) { return KSCHED_ABI_VERSION; }
int ksched_type_words(int n_types) { return type_words64(n_types); }

int ksched_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) return KSCHED_ERR_NO_DEVICE;
  return n;
}

int ksched_create(int device_ordinal, ksched_handle** out) {
  if (!out) return KSCHED_ERR_INVALID;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0 || device_ordinal >= n) return KSCHED_ERR_NO_DEVICE;
  ksched_handle* h = new ksched_handle();
  h->device = device_ordinal;
  if (cudaSetDevice(device_ordinal) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device_ordinal) != cudaSuccess) {
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return KSCHED_ERR_CUDA;
  }
  for (auto& e : h->ev) cudaEventCreate(&e);
  {
    // CUDA loads kernels lazily on first launch: pull ours in here, not inside the first Solve
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, pack_kernel<false, kPackThreadsSmall>);
    cudaFuncGetAttributes(&fa, pack_kernel<true, kPackThreadsSmall>);
    cudaFuncGetAttributes(&fa, pack_kernel<false, kPackThreads>);
    cudaFuncGetAttributes(&fa, pack_kernel<true, kPackThreads>);
    cudaFuncGetAttributes(&fa, feasibility_kernel);
    cudaFuncGetAttributes(&fa, class_feasibility_kernel);
    cudaFuncGetAttributes(&fa, finalize_options_kernel);
    cudaFuncGetAttributes(&fa, gather_rows_kernel);
    cudaFuncGetAttributes(&fa, sort_key1_kernel);
  }
  *out = h;
  return KSCHED_OK;
}

void ksched_destroy(ksched_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->comm) ncclCommDestroy(h->comm);
  for (auto& e : h->ev) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;  // every DevBuf frees its allocation
}

const char* ksched_last_error(const ksched_handle* h) { return h ? h->err.c_str() : "null handle"; }


// Every refusal of ksched_load_catalog, before it touches the handle (h->err aside).
static int check_catalog(ksched_handle* h, const ksched_catalog* cat) {
  if (cat->n_keys > KSCHED_MAX_KEYS || cat->n_res > KSCHED_MAX_RES || cat->n_templates > KSCHED_MAX_TEMPLATES || cat->n_templates < 1 ||
      cat->n_types < 0) { h->err = "catalog dimensions out of range"; return KSCHED_ERR_INVALID; }
  if (cat->n_res_ext < 0 || cat->n_res_ext > KSCHED_MAX_RES_EXT || (cat->n_res_ext > 0 && (cat->n_res != KSCHED_MAX_RES || !cat->type_alloc_ext))) {
    h->err = "inconsistent ext resources: n_res_ext in [0, 24], and with ext resources n_res == 8 and type_alloc_ext set";
    return KSCHED_ERR_INVALID;
  }
  // Gt/Lt cross the ABI in region form (ksched_key_regions): a requirement set that still carries gt / lt is a caller bug
  if (cat->type_bounds || cat->template_bounds) { h->err = "bounds arrays must be NULL: Gt/Lt requirements are passed in region form (ksched_key_regions)"; return KSCHED_ERR_INVALID; }
  for (int v = 0; v < cat->n_templates; ++v) {
    if (cat->templates[v].reqs.meta >> KSCHED_META_HASGT_SHIFT) { h->err = "template requirement with HASGT/HASLT set: pass Gt/Lt in region form"; return KSCHED_ERR_INVALID; }
    if (cat->templates[v].taintset >= 64) { h->err = "template taint set id beyond 63: ids from 64 on belong to existing nodes only"; return KSCHED_ERR_INVALID; }
  }
  for (int t = 0; t < cat->n_types; ++t)
    if (cat->types[t].meta >> KSCHED_META_HASGT_SHIFT) { h->err = "instance-type requirement with HASGT/HASLT set: pass Gt/Lt in region form"; return KSCHED_ERR_INVALID; }
  if (cat->key_regions)
    for (int k = 0; k < cat->n_keys; ++k) {
      const ksched_key_regions& g = cat->key_regions[k];
      if (!g.region_mask) continue;
      const uint64_t want = (g.n_thresholds + 1 >= 64 ? ~0ull : ((1ull << (g.n_thresholds + 1)) - 1)) << g.region_shift;
      if (g.n_thresholds < 0 || g.n_thresholds > KSCHED_MAX_THRESHOLDS || g.region_shift < 0 || g.region_shift + g.n_thresholds + 1 > 63 ||
          g.region_mask != want || (g.region_mask & cat->keys[k].dict_mask)) { h->err = "inconsistent ksched_key_regions"; return KSCHED_ERR_INVALID; }
    }
  for (int t = 0; t < cat->n_types; ++t) {
    const ksched_type_row& row = cat->types[t];
    if (t > 0 && row.min_price < cat->types[t - 1].min_price) { h->err = "instance types must be in ascending price order"; return KSCHED_ERR_INVALID; }
    for (int k = 0; k < cat->n_keys; ++k) {
      const bool complement = (row.meta >> (KSCHED_META_PRESENT_SHIFT + k)) & (row.meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1;
      if (complement && !(cat->key_regions && cat->key_regions[k].region_mask)) {
        h->err = "instance type with a complement requirement on a key without region bits";
        return KSCHED_ERR_INVALID;
      }
    }
  }
  // offering slot tables (read only here, after every check of the fields that precede them)
  if (!cat->zone_slots != !cat->ct_slots) { h->err = "zone_slots and ct_slots must both be set or both be NULL"; return KSCHED_ERR_INVALID; }
  if (cat->zone_slots) {
    uint64_t zones = 0, cts = 0;
    bool overlap = false;
    for (int v = 0; v < 64; ++v) {
      overlap = overlap || (zones & cat->zone_slots[v]) || (cts & cat->ct_slots[v]);
      zones |= cat->zone_slots[v];
      cts |= cat->ct_slots[v];
    }
    uint64_t offered = 0;
    for (int t = 0; t < cat->n_types; ++t) offered |= cat->types[t].offerings;
    if (overlap || zones != cts || (offered & ~zones)) {
      h->err = "inconsistent offering slot tables: every slot belongs to exactly one zone and one capacity type, and every offering is a slot";
      return KSCHED_ERR_INVALID;
    }
  }
  return KSCHED_OK;
}

// The catalog's inputs byte for byte: a catalog equal to the resident one needs no rebuild (ksched_load_catalog).
static std::vector<unsigned char> catalog_key(const ksched_catalog* cat) {
  const int NK = cat->n_keys, T = cat->n_types;
  std::vector<unsigned char> blob;
  auto put = [&](const void* p, size_t n) { const unsigned char* b = (const unsigned char*)p; blob.insert(blob.end(), b, b + n); };
  int dims[4] = {NK, cat->n_res, T, cat->n_templates};
  put(dims, sizeof dims);
  put(cat->keys, sizeof(ksched_keyinfo) * (size_t)NK);
  unsigned char has_int = cat->key_int_values != nullptr, has_off = cat->offering_keys != nullptr, has_reg = cat->key_regions != nullptr;
  put(&has_int, 1); put(&has_off, 1); put(&has_reg, 1);
  if (has_reg) put(cat->key_regions, sizeof(ksched_key_regions) * (size_t)NK);
  if (has_int) put(cat->key_int_values, sizeof(int64_t) * (size_t)NK * 64);
  put(cat->types, sizeof(ksched_type_row) * (size_t)T);
  put(cat->type_capacity, sizeof(int64_t) * (size_t)T * KSCHED_MAX_RES);
  if (has_off) put(cat->offering_keys, sizeof(uint64_t) * (size_t)T * 64);
  put(&cat->n_res_ext, sizeof cat->n_res_ext);
  if (cat->n_res_ext) put(cat->type_alloc_ext, sizeof(int64_t) * (size_t)T * cat->n_res_ext);
  const unsigned char has_slots = cat->zone_slots != nullptr;
  put(&has_slots, 1);
  if (has_slots) { put(cat->zone_slots, sizeof(uint64_t) * 64); put(cat->ct_slots, sizeof(uint64_t) * 64); }
  return blob;
}

// DevCatalog's bit-sliced tables, built on the host (amortised: instance types change rarely).
struct CatalogTables {
  std::vector<ksched_keyinfo> keys;
  std::vector<int16_t> valrow, offrow;
  std::vector<uint32_t> valset, absent, negempty, offset, anyoffer, member, fitset, domset, input_index;
  std::vector<int32_t> perm_desc;
  std::vector<int64_t> alloc_rt, alloc_sorted;
  std::vector<float> price32;
  uint32_t type_relevant = 0;
  int zone_key = -1, ct_key = -1;
  uint64_t pin_neutral[KSCHED_MAX_KEYS] = {};
  std::vector<uint64_t> slots;  // [128] zone value -> its slots, capacity-type value -> its slots (the tables or the formula)
  uint64_t zone_used = 0, ct_used = 0, all_slots = 0, offer_used = 0;
};

static void build_catalog(const ksched_catalog* cat, CatalogTables& b) {
  const int T = cat->n_types, NK = cat->n_keys, V = cat->n_templates, R = cat->n_res;
  const int W32 = type_words64(T) * 2;
  // the device's dict_mask includes the region bits: "every admissible value" of a complement requirement then covers the
  // regions a complement instance type shares with it (catalog.cuh: key_typeset_word walks the admitted bits)
  b.keys.assign(cat->keys, cat->keys + NK);
  if (cat->key_regions) for (int k = 0; k < NK; ++k) b.keys[k].dict_mask |= cat->key_regions[k].region_mask;
  b.valrow.assign((size_t)NK * 64, -1);
  b.offrow.assign(64, -1);
  b.slots.assign(128, 0);
  if (cat->zone_slots) {
    std::copy(cat->zone_slots, cat->zone_slots + 64, b.slots.begin());
    std::copy(cat->ct_slots, cat->ct_slots + 64, b.slots.begin() + 64);
  } else {
    ksched::formula_slot_tables(b.slots.data(), b.slots.data() + 64);
  }
  for (int v = 0; v < 64; ++v) {
    if (b.slots[v]) b.zone_used |= 1ull << v;
    if (b.slots[64 + v]) b.ct_used |= 1ull << v;
    b.all_slots |= b.slots[v];
  }
  b.absent.assign((size_t)std::max(NK, 1) * W32, 0);
  b.negempty.assign((size_t)std::max(NK, 1) * W32, 0);
  b.anyoffer.assign(W32, 0);
  b.member.assign((size_t)V * W32, 0);
  for (int k = 0; k < NK; ++k) {
    if (cat->keys[k].is_zone) b.zone_key = k;
    if (cat->keys[k].is_capacity_type) b.ct_key = k;
  }
  b.price32.assign(std::max(T, 1), 0.f);
  for (int t = 0; t < T; ++t) {
    const ksched_type_row& row = cat->types[t];
    b.price32[t] = (float)row.min_price;
    const int w = t >> 5;
    const uint32_t bit = 1u << (t & 31);
    for (int k = 0; k < NK; ++k) {
      bool present = (row.meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1;
      if (!present) { b.absent[(size_t)k * W32 + w] |= bit; continue; }
      b.type_relevant |= 1u << k;
      uint64_t v = row.values[k];
      if ((row.meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1) {
        // complement requirement (NotIn / Exists / Gt / Lt, region form): the type admits every value and region it does not
        // exclude; its operator is negative (NotIn) when it really excludes a value (requirement.go:186-197)
        const uint64_t region_mask = cat->key_regions[k].region_mask;  // check_catalog: set
        ksched::Req r{v, 0, 0, true, true, false, false};
        if (ksched::req_excluded(r, KeyMeta{0, nullptr, cat->key_regions + k}) != 0) b.negempty[(size_t)k * W32 + w] |= bit;
        v = ~v & (cat->keys[k].dict_mask | region_mask);
      } else if (!v) { b.negempty[(size_t)k * W32 + w] |= bit; continue; }
      while (v) {
        int vb = __builtin_ctzll(v);
        v &= v - 1;
        int16_t& r = b.valrow[(size_t)k * 64 + vb];
        if (r < 0) { r = (int16_t)(b.valset.size() / W32); b.valset.resize(b.valset.size() + W32, 0); }
        b.valset[(size_t)r * W32 + w] |= bit;
      }
    }
    uint64_t o = row.offerings;
    if (o) b.anyoffer[w] |= bit;
    while (o) {
      int ob = __builtin_ctzll(o);
      o &= o - 1;
      int16_t& r = b.offrow[ob];
      if (r < 0) { r = (int16_t)(b.offset.size() / W32); b.offset.resize(b.offset.size() + W32, 0); b.offer_used |= 1ull << ob; }
      b.offset[(size_t)r * W32 + w] |= bit;
    }
    for (int v = 0; v < V; ++v) if ((row.template_members >> v) & 1) b.member[(size_t)v * W32 + w] |= bit;
  }
  if (b.valset.empty()) b.valset.resize(W32, 0);
  if (b.offset.empty()) b.offset.resize(W32, 0);
  b.perm_desc.assign((size_t)std::max(R, 1) * std::max(T, 1), 0);
  b.alloc_rt.assign((size_t)std::max(R, 1) * std::max(T, 1), 0);
  b.alloc_sorted.assign((size_t)std::max(R, 1) * std::max(T, 1), 0);
  b.fitset.assign((size_t)std::max(R, 1) * (T + 1) * W32, 0);
  {
    std::vector<int> perm(T);
    for (int r = 0; r < R; ++r) {
      for (int t = 0; t < T; ++t) perm[t] = t;
      std::stable_sort(perm.begin(), perm.end(), [&](int a, int c) { return cat->types[a].allocatable[r] < cat->types[c].allocatable[r]; });
      for (int i = 0; i < T; ++i) {
        b.alloc_sorted[(size_t)r * T + i] = cat->types[perm[i]].allocatable[r];
        b.perm_desc[(size_t)r * T + (T - 1 - i)] = perm[i];
        b.alloc_rt[(size_t)r * T + i] = cat->types[i].allocatable[r];
      }
      uint32_t* base = &b.fitset[(size_t)r * (T + 1) * W32];
      for (int i = T - 1; i >= 0; --i) {
        uint32_t* cur = base + (size_t)i * W32;
        std::memcpy(cur, base + (size_t)(i + 1) * W32, W32 * sizeof(uint32_t));
        cur[perm[i] >> 5] |= 1u << (perm[i] & 31);
      }
    }
  }
  {
    // dominance bitsets over the first min(R,4) resources (pack kernel: Pareto front of a node's options)
    const int RH = std::min(R, 4);
    b.domset.assign((size_t)std::max(T, 1) * W32, 0);
    for (int a = 0; a < T; ++a)
      for (int c = 0; c < T; ++c) {
        bool dom = true;
        for (int r = 0; r < RH && dom; ++r) dom = cat->types[a].allocatable[r] >= cat->types[c].allocatable[r];
        if (dom) b.domset[(size_t)a * W32 + (c >> 5)] |= 1u << (c & 31);
      }
  }
  if (cat->offering_keys)
    for (int t = 0; t < T; ++t) b.input_index.push_back(cat->types[t].input_index);
  {
    // pin_neutral (catalog.cuh): U = union of every template's member types
    const int zone_key = b.zone_key, ct_key = b.ct_key;
    std::vector<uint32_t> U(W32, 0);
    for (int v = 0; v < V; ++v) for (int w = 0; w < W32; ++w) U[w] |= b.member[(size_t)v * W32 + w];
    auto covers = [&](const std::vector<uint32_t>& set) { for (int w = 0; w < W32; ++w) if (U[w] & ~set[w]) return false; return true; };
    // types with an available offering in one of `slots`
    auto offers = [&](uint64_t slots) {
      std::vector<uint32_t> acc(W32, 0);
      for (uint64_t m = slots & b.offer_used; m; m &= m - 1) {
        const int16_t r = b.offrow[__builtin_ctzll(m)];
        for (int w = 0; w < W32; ++w) acc[w] |= b.offset[(size_t)r * W32 + w];
      }
      return acc;
    };
    // pinning value d of one of the two offering keys (own = its value -> slots table) is neutral when d owns a slot and,
    // for every value of the other key (other, other_key), the types offered in the pair's slots cover U
    auto offering_neutral = [&](const uint64_t* own, const uint64_t* other, int other_key, int d) {
      if (!own[d]) return false;
      if (other_key < 0) return covers(offers(own[d]));
      for (uint64_t m = cat->keys[other_key].dict_mask; m; m &= m - 1) {
        const int v = __builtin_ctzll(m);
        if (!other[v] || !covers(offers(own[d] & other[v]))) return false;
      }
      return true;
    };
    for (int k = 0; k < NK; ++k) {
      for (int d = 0; d < 64; ++d) {
        if (!((cat->keys[k].dict_mask >> d) & 1)) continue;
        std::vector<uint32_t> set(W32, 0);
        for (int w = 0; w < W32; ++w) set[w] = b.absent[(size_t)k * W32 + w];
        if (b.valrow[(size_t)k * 64 + d] >= 0) for (int w = 0; w < W32; ++w) set[w] |= b.valset[(size_t)b.valrow[(size_t)k * 64 + d] * W32 + w];
        bool ok = covers(set);
        if (ok && k == zone_key) ok = offering_neutral(b.slots.data(), b.slots.data() + 64, ct_key, d);
        if (ok && k == ct_key) ok = offering_neutral(b.slots.data() + 64, b.slots.data(), zone_key, d);
        if (ok) b.pin_neutral[k] |= 1ull << d;
      }
    }
  }
}

// Uploads the tables and binds every DevCatalog field to them (ksched_load_catalog's commit).
static int bind_catalog(ksched_handle* h, const ksched_catalog* cat, const CatalogTables& b) {
  const int T = cat->n_types, NK = cat->n_keys, V = cat->n_templates;
  DevCatalog& c = h->cat;
  c = DevCatalog{};
  c.n_keys = NK; c.n_res = cat->n_res; c.n_types = T; c.n_templates = V; c.W32 = type_words64(T) * 2;
  c.type_relevant = b.type_relevant;
  c.zone_key = b.zone_key; c.ct_key = b.ct_key;
  std::memcpy(c.pin_neutral, b.pin_neutral, sizeof c.pin_neutral);
  c.zone_used = b.zone_used; c.ct_used = b.ct_used; c.all_slots = b.all_slots; c.offer_used = b.offer_used;
  c.n_res_ext = cat->n_res_ext;
  CUDA_TRY(h, bind(h, h->d_keys, c.keys, b.keys.size(), b.keys.data()));
  if (cat->key_regions) CUDA_TRY(h, bind(h, h->d_key_regions, c.key_regions, (size_t)NK, cat->key_regions));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (cat->key_int_values) CUDA_TRY(h, bind(h, h->d_key_int, c.key_int_values, (size_t)NK * 64, cat->key_int_values));
  CUDA_TRY(h, bind(h, h->d_templates, c.templates, (size_t)V, cat->templates));
  CUDA_TRY(h, bind(h, h->d_types, c.types, (size_t)T, cat->types));
  CUDA_TRY(h, bind(h, h->d_capacity, c.capacity, (size_t)T * KSCHED_MAX_RES, cat->type_capacity));
  CUDA_TRY(h, bind(h, h->d_price32, c.price32, b.price32.size(), b.price32.data()));
  CUDA_TRY(h, bind(h, h->d_valrow, c.valrow, b.valrow.size(), b.valrow.data()));
  CUDA_TRY(h, bind(h, h->d_offrow, c.offrow, b.offrow.size(), b.offrow.data()));
  CUDA_TRY(h, bind(h, h->d_valset, c.valset, b.valset.size(), b.valset.data()));
  CUDA_TRY(h, bind(h, h->d_absent, c.absent, b.absent.size(), b.absent.data()));
  CUDA_TRY(h, bind(h, h->d_negempty, c.negempty, b.negempty.size(), b.negempty.data()));
  CUDA_TRY(h, bind(h, h->d_offset, c.offset, b.offset.size(), b.offset.data()));
  CUDA_TRY(h, bind(h, h->d_anyoffer, c.anyoffer, b.anyoffer.size(), b.anyoffer.data()));
  CUDA_TRY(h, bind(h, h->d_slots, c.slots, b.slots.size(), b.slots.data()));
  CUDA_TRY(h, bind(h, h->d_member, c.member, b.member.size(), b.member.data()));
  CUDA_TRY(h, bind(h, h->d_alloc_sorted, c.alloc_sorted, b.alloc_sorted.size(), b.alloc_sorted.data()));
  CUDA_TRY(h, bind(h, h->d_perm_desc, c.perm_desc, b.perm_desc.size(), b.perm_desc.data()));
  CUDA_TRY(h, bind(h, h->d_alloc_rt, c.alloc_rt, b.alloc_rt.size(), b.alloc_rt.data()));
  CUDA_TRY(h, bind(h, h->d_domset, c.domset, b.domset.size(), b.domset.data()));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, bind(h, h->d_fitset, c.fitset, b.fitset.size(), b.fitset.data()));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (cat->n_res_ext > 0 && T > 0) {
    CUDA_TRY(h, bind(h, h->d_alloc_ext, c.alloc_ext, (size_t)T * cat->n_res_ext, cat->type_alloc_ext));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  if (cat->offering_keys && T > 0) {
    CUDA_TRY(h, bind(h, h->d_offer_keys, c.offer_keys, (size_t)T * 64, cat->offering_keys));
    CUDA_TRY(h, bind(h, h->d_input_index, c.input_index, b.input_index.size(), b.input_index.data()));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  return KSCHED_OK;
}

int ksched_load_catalog(ksched_handle* h, const ksched_catalog* cat) {
  if (!h || !cat) return KSCHED_ERR_INVALID;
  int rc = check_catalog(h, cat);
  if (rc != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaSetDevice(h->device));
  const int V = cat->n_templates;
  // Instance types change rarely: when the byte-identical catalog is already resident there is nothing to do (exact
  // comparison against a host copy; the O(T^2) dominance table alone is milliseconds of host time at T = 1000).
  std::vector<unsigned char> blob = catalog_key(cat);
  if (h->have_catalog && blob == h->catalog_blob) {
    // same instance types: only the templates can differ (remaining provisioner limits move between solves, daemonset
    // overhead with the daemonsets) - they are small, re-upload them when they changed
    if (std::memcmp(h->h_templates.data(), cat->templates, sizeof(ksched_template) * (size_t)V) != 0) {
      const bool uploaded = h->uploaded;
      h->have_catalog = h->uploaded = false;  // until the new templates are on the device
      CUDA_TRY(h, bind(h, h->d_templates, h->cat.templates, (size_t)V, cat->templates));
      CUDA_TRY(h, cudaStreamSynchronize(h->stream));
      h->h_templates.assign(cat->templates, cat->templates + V);
      h->have_catalog = true;
      h->uploaded = uploaded;
    }
    return KSCHED_OK;
  }
  CatalogTables tables;
  build_catalog(cat, tables);
  // a new catalog drops the resident problem; a CUDA error part-way through leaves neither
  h->have_catalog = h->uploaded = false;
  if ((rc = bind_catalog(h, cat, tables)) != KSCHED_OK) return rc;
  h->n_valrows = (int)(tables.valset.size() / h->cat.W32);
  h->n_offrows = (int)(tables.offset.size() / h->cat.W32);
  h->h_templates.assign(cat->templates, cat->templates + V);
  h->catalog_blob.swap(blob);
  h->have_catalog = true;
  return KSCHED_OK;
}

int ksched_set_shard(ksched_handle* h, int rank, int world) {
  if (!h || world < 1 || rank < 0 || rank >= world) return KSCHED_ERR_INVALID;
  h->rank = rank;
  h->world = world;
  return KSCHED_OK;
}

int ksched_shard_range(int n_words32, int rank, int world, int* begin, int* end) {
  if (n_words32 < 0 || world < 1 || rank < 0 || rank >= world || !begin || !end) return KSCHED_ERR_INVALID;
  const int per = (n_words32 + world - 1) / world;
  *begin = std::min(n_words32, rank * per);
  *end = std::min(n_words32, *begin + per);
  return KSCHED_OK;
}

int ksched_nccl_unique_id(void* out128) {
  ncclUniqueId id;
  if (ncclGetUniqueId(&id) != ncclSuccess) return KSCHED_ERR_NCCL;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  std::memcpy(out128, &id, 128);
  return KSCHED_OK;
}
int ksched_nccl_init(ksched_handle* h, const void* id128, int rank, int world) {
  if (!h || !id128) return KSCHED_ERR_INVALID;
  if (cudaSetDevice(h->device) != cudaSuccess) return KSCHED_ERR_CUDA;
  ncclUniqueId id;
  std::memcpy(&id, id128, 128);
  ncclResult_t r = ncclCommInitRank(&h->comm, world, id, rank);
  if (r != ncclSuccess) { h->err = std::string("ncclCommInitRank: ") + ncclGetErrorString(r); return KSCHED_ERR_NCCL; }
  h->rank = rank;
  h->world = world;
  return KSCHED_OK;
}

// One ncclAllGather of `bytes` bytes per rank on the handle's communicator (consolidation: the verdicts of the simulations
// each rank ran, SURVEY.md 8e). Host buffers in and out; recv holds world * bytes.
int ksched_allgather(ksched_handle* h, const void* send, size_t bytes, void* recv) {
  if (!h || !send || !recv) return KSCHED_ERR_INVALID;
  if (!h->comm) { h->err = "ksched_nccl_init must be called first"; return KSCHED_ERR_INVALID; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  int world = 0;
  if (ncclCommCount(h->comm, &world) != ncclSuccess) return KSCHED_ERR_NCCL;
  CUDA_TRY(h, h->d_gather_send.ensure(std::max<size_t>(bytes, 1)));
  CUDA_TRY(h, h->d_gather_recv.ensure(std::max<size_t>(bytes * (size_t)world, 1)));
  CUDA_TRY(h, cudaMemcpyAsync(h->d_gather_send.ptr, send, bytes, cudaMemcpyHostToDevice, h->stream));
  ncclResult_t r = ncclAllGather(h->d_gather_send.ptr, h->d_gather_recv.ptr, bytes, ncclUint8, h->comm, h->stream);
  if (r != ncclSuccess) { h->err = std::string("ncclAllGather: ") + ncclGetErrorString(r); return KSCHED_ERR_NCCL; }
  CUDA_TRY(h, cudaMemcpyAsync(recv, h->d_gather_recv.ptr, bytes * (size_t)world, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return KSCHED_OK;
}

// The tables of one optional input are set exactly when its count is positive. `omittable` may also stay NULL then: a
// per-existing-node table without existing nodes, or a table that only some entries read.
static bool present_iff(bool positive, std::initializer_list<const void*> tables, const void* omittable, bool may_omit) {
  for (const void* t : tables)
    if ((t != nullptr) != positive) return false;
  return omittable ? positive : !positive || may_omit;
}

// Every refusal of ksched_upload, before it touches the handle (h->err aside).
static int check_problem(ksched_handle* h, const ksched_problem* pb) {
  if (!h->have_catalog) { h->err = "ksched_load_catalog must be called first"; return KSCHED_ERR_INVALID; }
  if (pb->class_bounds || pb->existing_bounds) { h->err = "bounds arrays must be NULL: Gt/Lt requirements are passed in region form (ksched_key_regions)"; return KSCHED_ERR_INVALID; }
  bool hasgt = false;
  for (int i = 0; i < pb->n_classes; ++i) hasgt = hasgt || pb->classes[i].meta >> KSCHED_META_HASGT_SHIFT;
  for (int i = 0; i < pb->n_existing; ++i) hasgt = hasgt || pb->existing[i].reqs.meta >> KSCHED_META_HASGT_SHIFT;
  for (int i = 0; i < pb->n_filter_terms; ++i) hasgt = hasgt || pb->filter_terms[i].meta >> KSCHED_META_HASGT_SHIFT;
  if (hasgt) { h->err = "requirement with HASGT/HASLT set: pass Gt/Lt in region form"; return KSCHED_ERR_INVALID; }
  {
    // taint sets from id 64 on: existing nodes only, each covered by the per-class table
    const int tol_words = pb->class_tolerated_ext ? pb->n_tolerated_ext_words : 0;
    if (tol_words < 0) { h->err = "n_tolerated_ext_words out of range"; return KSCHED_ERR_INVALID; }
    for (int i = 0; i < pb->n_existing; ++i)
      if (pb->existing[i].taintset >= 64 && (pb->existing[i].taintset - 64) / 64 >= (uint32_t)tol_words) {
        h->err = "existing node with a taint set id from 64 on that class_tolerated_ext does not cover";
        return KSCHED_ERR_INVALID;
      }
  }
  const int NE = pb->n_existing, HP = pb->n_hostport_ext_words, HW = pb->n_hostname_words, X = h->cat.n_res_ext;
  if (HP < 0 || !present_iff(HP > 0, {pb->class_hostport_conflicts_ext, pb->class_hostport_entries_ext}, pb->existing_hostport_ext, NE == 0)) {
    h->err = "host-port entry tables must be set exactly when n_hostport_ext_words is positive";
    return KSCHED_ERR_INVALID;
  }
  {
    // tracked volume claims from id 64 on: the three tables exist exactly when the count is positive, and only beside the
    // volume tables they extend
    const int VW = pb->n_volume_ext_words;
    const bool vol = pb->class_volumes && pb->existing_volumes && NE > 0;
    if (VW < 0 || !present_iff(VW > 0, {pb->class_volumes_shared_ext, pb->existing_volumes_mounted_ext, pb->volume_driver_mask_ext}, nullptr, true) ||
        (VW > 0 && !vol)) {
      h->err = "volume claim tables must be set exactly when n_volume_ext_words is positive, with class_volumes and existing_volumes";
      return KSCHED_ERR_INVALID;
    }
  }
  {
    // hostname requirement table: wide enough for every existing slot, and present when an entry reads it
    bool ok = HW >= 0 && present_iff(HW > 0, {pb->hostname_slots}, pb->filter_term_hostname, true) && (HW == 0 || (int64_t)HW * 64 >= NE);
    for (int i = 0; ok && i < pb->n_hostname_reqs; ++i) ok = pb->hostname_reqs[2 * i + 1] != KSCHED_HOSTNAME_TABLE || HW > 0;
    for (int f = 0; ok && pb->filter_term_hostname && f < pb->n_filter_terms; ++f)
      ok = pb->filter_term_hostname[f] == KSCHED_NONE || pb->filter_term_hostname[f] < (uint32_t)pb->n_hostname_reqs;
    if (!ok) {
      h->err = "hostname_slots / filter_term_hostname must be set exactly when n_hostname_words is positive and cover the entries";
      return KSCHED_ERR_INVALID;
    }
  }
  {
    // instance-type filter tables: all three or none, every value an itype_req entry or KSCHED_NONE
    const bool on = pb->filter_term_itype != nullptr;
    bool ok = present_iff(on, {pb->template_itype}, pb->existing_itype, NE == 0);
    auto entry = [&](uint32_t v) { return v == KSCHED_NONE || v < (uint32_t)pb->n_itype_reqs; };
    for (int f = 0; ok && on && f < pb->n_filter_terms; ++f) ok = entry(pb->filter_term_itype[f]);
    for (int v = 0; ok && on && v < h->cat.n_templates; ++v) ok = entry(pb->template_itype[v]);
    for (int e = 0; ok && pb->existing_itype && e < NE; ++e) ok = entry(pb->existing_itype[e]) || pb->existing_itype[e] == KSCHED_ITYPE_UNLISTED;
    if (!ok) {
      h->err = "filter_term_itype / template_itype / existing_itype must be set together and name itype_req entries";
      return KSCHED_ERR_INVALID;
    }
  }
  // ext resources: the tables exist exactly when the catalog has ext resources, and name no resource beyond them
  if (!present_iff(X > 0, {pb->class_requests_ext, pb->class_res_ext_present}, pb->existing_available_ext, NE == 0)) {
    h->err = "ext resource tables must be set exactly when the catalog has ext resources";
    return KSCHED_ERR_INVALID;
  }
  for (int c = 0; c < (X > 0 ? pb->n_classes : 0); ++c)
    if (pb->class_res_ext_present[c] >> X) { h->err = "class_res_ext_present names an ext resource beyond n_res_ext"; return KSCHED_ERR_INVALID; }
  const int NC = pb->n_classes, NG = pb->n_groups;
  for (int e = 0; e < pb->n_class_topo; ++e)
    if (pb->class_topo[e].group >= (uint32_t)NG) { h->err = "class_topo group out of range"; return KSCHED_ERR_INVALID; }
  for (int c = 0; c < NC; ++c) {
    const ksched_pod_row& row = pb->classes[c];
    if (row.relax_next != KSCHED_NONE && row.relax_next >= (uint32_t)NC) { h->err = "relax_next out of range"; return KSCHED_ERR_INVALID; }
    if (row.topo_end < row.topo_begin || row.topo_end > (uint32_t)pb->n_class_topo) { h->err = "class_topo range out of bounds"; return KSCHED_ERR_INVALID; }
    int ncg = 0, touched = __builtin_popcountll((row.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF);
    for (uint32_t e = row.topo_begin; e < row.topo_end; ++e)
      if (pb->class_topo[e].flags & KSCHED_TOPO_CONSTRAINS) { ++ncg; if (pb->groups[pb->class_topo[e].group].key != KSCHED_KEY_HOSTNAME) ++touched; }
    if (ncg > kMaxCG || touched > kMaxTouched) { h->err = "a pod class is constrained by more topology groups / label keys than the pack kernel carries"; return KSCHED_ERR_UNSUPPORTED; }
  }
  for (int g = 0; g < NG; ++g)
    if (pb->groups[g].key != KSCHED_KEY_HOSTNAME && pb->groups[g].key >= h->cat.n_keys) { h->err = "topology group key out of range"; return KSCHED_ERR_INVALID; }
  return KSCHED_OK;
}

// the timestamps sort_key1_kernel reads for pb, once bind_problem has chosen the timestamp field
static const int64_t* queue_timestamps(const ksched_handle* h, const ksched_problem* pb) {
  return h->ts_dense.empty() ? pb->pod_timestamp : h->ts_dense.data();
}

// Uploads one checked problem and binds every PackState field to it (ksched_upload's commit). Arrays the pack kernel mutates
// get a pristine copy that reset_state restores before every run.
static int bind_problem(ksched_handle* h, const ksched_problem* pb) {
  h->tm.h2d_bytes = 0;
  const DevCatalog& c = h->cat;
  PackState& s = h->st;
  s = PackState{};
  h->resets.n = 0;
  const int P = pb->n_pods, NC = pb->n_classes, NE = pb->n_existing, NG = pb->n_groups, W32 = c.W32, V = c.n_templates;
  const int MAXN = std::max(1, std::min(pb->max_new_nodes > 0 ? pb->max_new_nodes : P, std::max(P, 1)));
  const size_t p1 = (size_t)std::max(P, 1), ne = (size_t)std::max(NE, 1), nc = (size_t)std::max(NC, 1), ng = (size_t)std::max(NG, 1), mn = (size_t)MAXN;
  s.n_pods = P; s.n_classes = NC; s.n_existing = NE; s.n_groups = NG; s.max_new = MAXN;
  s.count_visited = pb->count_nodes_visited;
  // min request per resource over all classes (node closing rule)
  for (int r = 0; r < KSCHED_MAX_RES; ++r) {
    int64_t m = INT64_MAX;
    for (int i = 0; i < NC; ++i) m = std::min(m, ((pb->classes[i].res_present >> r) & 1) ? pb->classes[i].requests[r] : (int64_t)0);
    s.min_req[r] = (NC == 0 || m == INT64_MAX || m < 0) ? 0 : m;
  }
  CUDA_TRY(h, bind(h, h->d_classes, s.classes, (size_t)NC, pb->classes));
  s.tol_ext_words = pb->class_tolerated_ext ? pb->n_tolerated_ext_words : 0;
  if (s.tol_ext_words > 0) CUDA_TRY(h, bind(h, h->d_cls_tol_ext, s.cls_tol_ext, (size_t)NC * s.tol_ext_words, pb->class_tolerated_ext));
  if (const int X = c.n_res_ext) {
    CUDA_TRY(h, bind(h, h->d_cls_req_ext, s.cls_req_ext, (size_t)NC * X, pb->class_requests_ext));
    CUDA_TRY(h, bind(h, h->d_cls_ext_present, s.cls_ext_present, (size_t)NC, pb->class_res_ext_present));
    // existing nodes: [x][n_existing] (the scan reads one resource of consecutive nodes)
    std::vector<int64_t> avail((size_t)X * ne, 0);
    for (int e = 0; e < NE; ++e)
      for (int x = 0; x < X; ++x) avail[(size_t)x * NE + e] = pb->existing_available_ext[(size_t)e * X + x];
    CUDA_TRY(h, bind(h, h->d_ex_avail_ext, s.ex_avail_ext, avail.size(), avail.data()));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    // ext sums of existing and new nodes: every mode that opens a node relies on zeros here
    CUDA_TRY(h, bind_zeroed(h, h->d_ex_req_ext, s.ex_req_ext, (size_t)X * ne));
    CUDA_TRY(h, bind_zeroed(h, h->d_nn_req_ext, s.nn_req_ext, (size_t)X * mn));
    CUDA_TRY(h, bind_zeroed(h, h->d_nn_ext_present, s.nn_ext_present, mn));
  }
  {
    // queue.go:82-108 orders by cpu desc, memory desc, timestamp asc, UID asc. (cpu, memory) is a property of the class: rank
    // the classes once here, and the whole order is one packed key of class rank, timestamp field and UID rank.
    std::vector<uint32_t> by((size_t)NC), rank(nc, 0);
    for (int i = 0; i < NC; ++i) by[(size_t)i] = (uint32_t)i;
    auto cpu = [&](uint32_t i) { return pb->classes[i].requests[0]; };
    auto mem = [&](uint32_t i) { return pb->classes[i].requests[1]; };
    std::sort(by.begin(), by.end(), [&](uint32_t a, uint32_t b) { return cpu(a) != cpu(b) ? cpu(a) > cpu(b) : mem(a) > mem(b); });
    uint32_t r = 0;
    for (int i = 0; i < NC; ++i) {
      if (i > 0 && (cpu(by[(size_t)i]) != cpu(by[(size_t)i - 1]) || mem(by[(size_t)i]) != mem(by[(size_t)i - 1]))) ++r;
      rank[by[(size_t)i]] = r;
    }
    auto bits = [](unsigned long long v) { int b = 0; while (v) { ++b; v >>= 1; } return std::max(b, 1); };
    long long ts_min = 0, ts_max = 0;
    uint32_t uid_max = 0;
    for (int i = 0; i < P; ++i) {
      const long long t = pb->pod_timestamp[i];
      if (i == 0 || t < ts_min) ts_min = t;
      if (i == 0 || t > ts_max) ts_max = t;
      uid_max = std::max(uid_max, pb->pod_uid_rank[i]);
    }
    // the timestamp field: the offset from the earliest timestamp, or, when that is too wide, the timestamp's rank among
    // the batch's distinct timestamps (the same order). Every field is then at most bits(P - 1) wide, so the key always
    // fits for batches of up to 2^21 pods.
    const unsigned long long span = (unsigned long long)ts_max - (unsigned long long)ts_min;
    h->ts_dense.clear();
    h->sort1_ts_bits = bits(span);
    h->sort1_uid_bits = bits(uid_max);
    h->sort1_ts_min = ts_min;
    if (span >= (1ull << 62) || bits(r) + h->sort1_ts_bits + h->sort1_uid_bits > 64) {
      std::vector<int64_t> distinct(pb->pod_timestamp, pb->pod_timestamp + P);
      std::sort(distinct.begin(), distinct.end());
      distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
      h->ts_dense.resize((size_t)P);
      for (int i = 0; i < P; ++i)
        h->ts_dense[(size_t)i] = std::lower_bound(distinct.begin(), distinct.end(), pb->pod_timestamp[i]) - distinct.begin();
      h->sort1_ts_bits = bits(distinct.size() - 1);
      h->sort1_ts_min = 0;
    }
    h->sort1_bits = bits(r) + h->sort1_ts_bits + h->sort1_uid_bits;
    if (h->sort1_bits > 64) {
      h->err = "unsupported: the queue order key of " + std::to_string(P) + " pods needs " + std::to_string(h->sort1_bits) +
               " bits (class, timestamp and UID ranks; at most 64)";
      return KSCHED_ERR_UNSUPPORTED;
    }
    CUDA_TRY(h, upload_vec(h, h->d_cls_rank, rank));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));  // rank is a stack vector
  }
  CUDA_TRY(h, bind_restored(h, h->d_pod_class, s.pod_class, h->d_pod_class0, (size_t)P, pb->pod_class));
  CUDA_TRY(h, upload(h, h->d_ts, queue_timestamps(h, pb), (size_t)P));
  CUDA_TRY(h, upload(h, h->d_uid_rank, pb->pod_uid_rank, (size_t)P));
  CUDA_TRY(h, bind(h, h->d_groups, s.groups, (size_t)NG, pb->groups));
  CUDA_TRY(h, bind(h, h->d_class_topo, s.class_topo, (size_t)pb->n_class_topo, pb->class_topo));
  CUDA_TRY(h, bind(h, h->d_filter_terms, s.filter_terms, (size_t)pb->n_filter_terms, pb->filter_terms));
  CUDA_TRY(h, bind(h, h->d_hostname_reqs, s.hostname_reqs, (size_t)pb->n_hostname_reqs * 2, pb->hostname_reqs));
  s.hostname_words = pb->n_hostname_words;
  if (s.hostname_words) CUDA_TRY(h, bind(h, h->d_hostname_slots, s.hostname_slots, (size_t)pb->n_hostname_reqs * s.hostname_words, pb->hostname_slots));
  if (pb->filter_term_hostname) CUDA_TRY(h, bind(h, h->d_filter_hostname, s.filter_hostname, (size_t)pb->n_filter_terms, pb->filter_term_hostname));
  CUDA_TRY(h, bind(h, h->d_itype_comp, s.itype_complement, (size_t)pb->n_itype_reqs, pb->itype_req_complement));
  CUDA_TRY(h, bind(h, h->d_itype_sets, s.itype_sets, (size_t)pb->n_itype_reqs * W32, reinterpret_cast<const uint32_t*>(pb->itype_req_sets)));
  // existing nodes -> SoA
  {
    std::vector<int64_t> req(8 * ne, 0), avail(8 * ne, 0);
    std::vector<uint32_t> reqp(ne, 0), availp(ne, 0), ts(ne, 0), it(ne, 0);
    std::vector<uint64_t> vals(16 * ne, 0), meta(ne, 0), hp(ne, 0);
    for (int e = 0; e < NE; ++e) {
      const ksched_existing_node& n = pb->existing[e];
      for (int r = 0; r < 8; ++r) { req[(size_t)r * NE + e] = n.requests[r]; avail[(size_t)r * NE + e] = n.available[r]; }
      for (int k = 0; k < 16; ++k) vals[(size_t)k * NE + e] = n.reqs.values[k];
      meta[e] = n.reqs.meta & 0xFFFFFFFFull;
      reqp[e] = n.requests_present; availp[e] = n.available_present; ts[e] = n.taintset; it[e] = n.itype; hp[e] = n.hostport_entries;
    }
    CUDA_TRY(h, bind_restored(h, h->d_ex_req, s.ex_req, h->d_ex_req0, req.size(), req.data()));
    CUDA_TRY(h, bind(h, h->d_ex_avail, s.ex_avail, avail.size(), avail.data()));
    CUDA_TRY(h, bind_restored(h, h->d_ex_req_present, s.ex_req_present, h->d_ex_req_present0, reqp.size(), reqp.data()));
    CUDA_TRY(h, bind(h, h->d_ex_avail_present, s.ex_avail_present, availp.size(), availp.data()));
    CUDA_TRY(h, bind(h, h->d_ex_taintset, s.ex_taintset, ts.size(), ts.data()));
    CUDA_TRY(h, bind(h, h->d_ex_itype, s.ex_itype, it.size(), it.data()));
    CUDA_TRY(h, bind_restored(h, h->d_ex_vals, s.ex_vals, h->d_ex_vals0, vals.size(), vals.data()));
    CUDA_TRY(h, bind_restored(h, h->d_ex_meta, s.ex_meta, h->d_ex_meta0, meta.size(), meta.data()));
    CUDA_TRY(h, bind_restored(h, h->d_ex_hp, s.ex_hp, h->d_ex_hp0, hp.size(), hp.data()));
    // host-port entries from id 64 on: per-class tables as given, the existing nodes' words as [word][node] like ex_hp
    const int HW = pb->n_hostport_ext_words;
    s.hp_ext_words = HW;
    std::vector<uint64_t> hp_ext(HW > 0 ? (size_t)HW * ne : 0, 0);
    std::vector<uint8_t> cls_hp(HW > 0 ? nc : 0, 0);
    if (HW > 0) {
      for (int e = 0; e < NE; ++e)
        for (int w = 0; w < HW; ++w) hp_ext[(size_t)w * NE + e] = pb->existing_hostport_ext[(size_t)e * HW + w];
      for (int i = 0; i < NC; ++i)
        for (int w = 0; w < HW; ++w)
          if (pb->class_hostport_conflicts_ext[(size_t)i * HW + w] | pb->class_hostport_entries_ext[(size_t)i * HW + w]) cls_hp[i] = 1;
      CUDA_TRY(h, bind(h, h->d_cls_hpc_ext, s.cls_hpc_ext, (size_t)NC * HW, pb->class_hostport_conflicts_ext));
      CUDA_TRY(h, bind(h, h->d_cls_hpe_ext, s.cls_hpe_ext, (size_t)NC * HW, pb->class_hostport_entries_ext));
      CUDA_TRY(h, bind(h, h->d_cls_hp_ext, s.cls_hp_ext, cls_hp.size(), cls_hp.data()));
      CUDA_TRY(h, bind_restored(h, h->d_ex_hp_ext, s.ex_hp_ext, h->d_ex_hp_ext0, hp_ext.size(), hp_ext.data()));  // new nodes: set at creation
      CUDA_TRY(h, bind(h, h->d_nn_hp_ext, s.nn_hp_ext, (size_t)HW * mn));
    }
    if (pb->class_volumes && pb->existing_volumes && NE > 0) {
      CUDA_TRY(h, bind(h, h->d_cls_vol, s.cls_vol, (size_t)NC, pb->class_volumes));
      CUDA_TRY(h, bind_restored(h, h->d_ex_vol, s.ex_vol, h->d_ex_vol0, (size_t)NE, pb->existing_volumes));
      std::memcpy(s.vol_mask, pb->volume_driver_mask, sizeof s.vol_mask);
      // tracked claims from id 64 on: per-class table and driver masks as given, the existing nodes' words as [word][node];
      // and per class whether it mounts a claim at all (its row or its table words)
      const int VW = pb->n_volume_ext_words;
      s.vol_ext_words = VW;
      std::vector<uint8_t> has_vol(nc, 0);
      for (int i = 0; i < NC; ++i) {
        const ksched_class_volumes& v = pb->class_volumes[i];
        has_vol[i] = (v.shared | v.priv[0] | v.priv[1] | v.priv[2] | v.priv[3]) != 0;
        for (int w = 0; w < VW; ++w) has_vol[i] |= pb->class_volumes_shared_ext[(size_t)i * VW + w] != 0;
      }
      CUDA_TRY(h, bind(h, h->d_cls_has_vol, s.cls_has_vol, has_vol.size(), has_vol.data()));
      std::vector<uint64_t> vol_ext(VW > 0 ? (size_t)VW * ne : 0, 0);
      if (VW > 0) {
        for (int e = 0; e < NE; ++e)
          for (int w = 0; w < VW; ++w) vol_ext[(size_t)w * NE + e] = pb->existing_volumes_mounted_ext[(size_t)e * VW + w];
        CUDA_TRY(h, bind(h, h->d_cls_vol_ext, s.cls_vol_ext, (size_t)NC * VW, pb->class_volumes_shared_ext));
        CUDA_TRY(h, bind(h, h->d_vol_mask_ext, s.vol_mask_ext, (size_t)KSCHED_MAX_VOLUME_DRIVERS * VW, pb->volume_driver_mask_ext));
        CUDA_TRY(h, bind_restored(h, h->d_ex_vol_ext, s.ex_vol_ext, h->d_ex_vol_ext0, vol_ext.size(), vol_ext.data()));
      }
      CUDA_TRY(h, cudaStreamSynchronize(h->stream));  // host vectors go out of scope
    }
    // instance-type requirement of every slot (topology.cuh: itype_state_add), only when a filter term names the key
    std::vector<uint32_t> ex_it;
    if (pb->filter_term_itype) {
      const size_t IW = 1 + (size_t)W32;
      const uint32_t* sets = reinterpret_cast<const uint32_t*>(pb->itype_req_sets);
      ex_it.assign(ne * IW, 0);
      for (int e = 0; e < NE; ++e) {
        const uint32_t v = pb->existing_itype[e];
        uint32_t* row = &ex_it[(size_t)e * IW];
        if (v == KSCHED_ITYPE_UNLISTED) row[0] = kItPresent | kItOwn;
        if (v == KSCHED_NONE || v == KSCHED_ITYPE_UNLISTED) continue;
        row[0] = kItPresent | (pb->itype_req_complement[v] ? kItComp : 0u);
        std::memcpy(row + 1, sets + (size_t)v * W32, (size_t)W32 * sizeof(uint32_t));
      }
      CUDA_TRY(h, bind(h, h->d_filter_itype, s.filter_itype, (size_t)pb->n_filter_terms, pb->filter_term_itype));
      CUDA_TRY(h, bind(h, h->d_tmpl_itype, s.tmpl_itype, (size_t)V, pb->template_itype));
      CUDA_TRY(h, bind_restored(h, h->d_ex_it, s.ex_it, h->d_ex_it0, ex_it.size(), ex_it.data()));
      CUDA_TRY(h, bind(h, h->d_nn_it, s.nn_it, mn * IW));  // new nodes: set when they open
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));  // host vectors go out of scope
    CUDA_TRY(h, bind_zeroed(h, h->d_ex_closed, s.ex_closed, ne));
  }
  // topology counters
  {
    std::vector<int32_t> host_row(ng, -1), host_total(ng, 0), cnt(ng * 64, 0);
    std::vector<uint64_t> registered(ng, 0);
    std::vector<uint8_t> active(ng, 1);
    int nh = 0;
    for (int g = 0; g < NG; ++g) {
      if (pb->groups[g].key == KSCHED_KEY_HOSTNAME) host_row[g] = nh++;
      registered[g] = pb->groups[g].registered;
      active[g] = pb->groups[g].dormant ? 0 : 1;
      for (int d = 0; d < 64; ++d) cnt[(size_t)g * 64 + d] = pb->group_domain_counts[(size_t)g * 64 + d];
    }
    const size_t stride = (size_t)NE + MAXN;
    // [hostname group][existing node | new node slot] counters: only the existing-node columns carry initial values, the
    // rest of the (up to 40 MB) matrix is zeroed on the device instead of being built and shipped from the host
    std::vector<uint16_t> host((size_t)std::max(nh, 1) * ne, 0);
    for (int g = 0; g < NG; ++g) {
      if (host_row[g] < 0) continue;
      int total = pb->groups[g].extra_nonzero_domains;
      for (int e = 0; e < NE; ++e) {
        int32_t v = pb->group_existing_counts[(size_t)g * ne + e];
        host[(size_t)host_row[g] * NE + e] = (uint16_t)std::min(v, 0xFFFF);
        if (v > 0) ++total;
      }
      host_total[g] = total;
    }
    std::vector<RelX> relx((size_t)std::max(pb->n_class_topo, 1));
    for (int e = 0; e < pb->n_class_topo; ++e) {
      const ksched_class_topo& ct = pb->class_topo[e];
      const ksched_topo_group& g = pb->groups[ct.group];
      RelX x{};
      x.group = ct.group; x.flags = ct.flags; x.key = g.key; x.type = g.type; x.has_filter = g.filter_begin != g.filter_end;
      // a term without any requirement is Compatible with every node (topologynodefilter.go:57-70): such a filter always matches
      for (uint32_t f = g.filter_begin; f < g.filter_end && f < (uint32_t)pb->n_filter_terms; ++f)
        if (((pb->filter_terms[f].meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF) == 0 &&
            (!pb->filter_term_hostname || pb->filter_term_hostname[f] == KSCHED_NONE) &&
            (!pb->filter_term_itype || pb->filter_term_itype[f] == KSCHED_NONE))
          x.has_filter = 0;
      x.max_skew = g.max_skew; x.host_row = host_row[ct.group];
      relx[e] = x;
    }
    CUDA_TRY(h, bind_restored(h, h->d_grp_active, s.grp_active, h->d_grp_active0, active.size(), active.data()));
    CUDA_TRY(h, bind_zeroed(h, h->d_grp_min_slot, s.grp_min_slot, ng));
    CUDA_TRY(h, bind(h, h->d_grp_host_row, s.grp_host_row, host_row.size(), host_row.data()));
    CUDA_TRY(h, bind(h, h->d_relx, s.relx, relx.size(), relx.data()));
    CUDA_TRY(h, bind_restored(h, h->d_grp_host_total, s.grp_host_total, h->d_grp_host_total0, host_total.size(), host_total.data()));
    CUDA_TRY(h, bind_restored(h, h->d_grp_cnt, s.grp_cnt, h->d_grp_cnt0, cnt.size(), cnt.data()));
    CUDA_TRY(h, bind_restored(h, h->d_grp_registered, s.grp_registered, h->d_grp_registered0, registered.size(), registered.data()));
    CUDA_TRY(h, bind_restored(h, h->d_grp_host, s.grp_host, h->d_grp_host0, (size_t)std::max(nh, 1) * stride));
    CUDA_TRY(h, cudaMemsetAsync(h->d_grp_host0.ptr, 0, (size_t)std::max(nh, 1) * stride * sizeof(uint16_t), h->stream));
    if (NE > 0 && nh > 0) {
      CUDA_TRY(h, cudaMemcpy2DAsync(h->d_grp_host0.ptr, stride * sizeof(uint16_t), host.data(), (size_t)NE * sizeof(uint16_t), (size_t)NE * sizeof(uint16_t),
                                    (size_t)nh, cudaMemcpyHostToDevice, h->stream));
      h->tm.h2d_bytes += (int64_t)nh * NE * 2;
    }
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  // scratch / state
  CUDA_TRY(h, bind(h, h->d_order, s.order, p1));
  CUDA_TRY(h, h->d_idx_tmp.ensure(p1));
  CUDA_TRY(h, bind(h, h->d_pod_pos, s.pod_pos, p1));
  CUDA_TRY(h, h->d_k_tie.ensure(p1));
  CUDA_TRY(h, h->d_k_tmp.ensure(p1));
  CUDA_TRY(h, bind(h, h->d_rows, s.rows, p1 * KSCHED_ROW_WORDS));
  CUDA_TRY(h, bind(h, h->d_F, s.F, p1 * V * W32));
  CUDA_TRY(h, bind(h, h->d_best, s.best, p1));
  CUDA_TRY(h, h->d_Fclass.ensure(nc * V * W32));
  CUDA_TRY(h, h->d_best_class.ensure(nc));
  CUDA_TRY(h, bind_zeroed(h, h->d_relax, s.relax_level, p1));
  CUDA_TRY(h, bind(h, h->d_assign, s.assign, p1));
  CUDA_TRY(h, bind(h, h->d_place_seq, s.place_seq, p1));
  CUDA_TRY(h, bind(h, h->d_queue, s.queue, p1 + 1));
  CUDA_TRY(h, bind(h, h->d_last_len, s.last_len, p1));
  CUDA_TRY(h, bind(h, h->d_last_epoch, s.last_epoch, p1));
  CUDA_TRY(h, bind_zeroed(h, h->d_cls_cursor, s.cls_cursor, nc));
  CUDA_TRY(h, bind(h, h->d_nn_tmpl, s.nn_tmpl, mn));
  CUDA_TRY(h, bind(h, h->d_nn_count, s.nn_count, mn));
  CUDA_TRY(h, bind(h, h->d_nn_tb, s.nn_tb, mn));
  CUDA_TRY(h, bind(h, h->d_nn_req, s.nn_req, 8 * mn));
  CUDA_TRY(h, bind(h, h->d_nn_req_present, s.nn_req_present, mn));
  CUDA_TRY(h, bind(h, h->d_nn_vals, s.nn_vals, 16 * mn));
  CUDA_TRY(h, bind(h, h->d_nn_meta, s.nn_meta, mn));
  CUDA_TRY(h, bind(h, h->d_nn_opts, s.nn_opts, (size_t)W32 * mn));
  CUDA_TRY(h, bind(h, h->d_nn_hp, s.nn_hp, mn));
  CUDA_TRY(h, bind(h, h->d_ov_key, s.ov_key, mn));
  CUDA_TRY(h, bind(h, h->d_ov_q, s.ov_q, 4 * mn));
  CUDA_TRY(h, bind(h, h->d_ov_bound, s.ov_bound, 4 * mn));
  CUDA_TRY(h, bind(h, h->d_ov_bound2, s.ov_bound2, 4 * mn));
  CUDA_TRY(h, bind(h, h->d_ov_node, s.ov_node, mn));
  CUDA_TRY(h, bind(h, h->d_ov_flags, s.ov_flags, mn));
  CUDA_TRY(h, bind(h, h->d_ov_absorbed, s.ov_absorbed, mn));
  CUDA_TRY(h, bind(h, h->d_ov_rejected, s.ov_rejected, mn));
  const size_t nfc = nc * V;
  CUDA_TRY(h, bind_zeroed(h, h->d_fc_state, s.fc_state, nfc));
  CUDA_TRY(h, bind(h, h->d_fc_dom, s.fc_dom, nfc));
  CUDA_TRY(h, bind_zeroed(h, h->d_fc_front_state, s.fc_front_state, nfc));
  CUDA_TRY(h, bind(h, h->d_fc_bound, s.fc_bound, nfc * 4));
  CUDA_TRY(h, bind(h, h->d_fc_bound2, s.fc_bound2, nfc * 4));
  CUDA_TRY(h, bind(h, h->d_fc_opts, s.fc_opts, nfc * W32));
  CUDA_TRY(h, bind(h, h->d_fc_vals, s.fc_vals, nfc * KSCHED_MAX_KEYS));
  CUDA_TRY(h, bind(h, h->d_fc_meta, s.fc_meta, nfc));
  CUDA_TRY(h, bind(h, h->d_fc_q, s.fc_q, nfc * KSCHED_MAX_RES));
  CUDA_TRY(h, bind(h, h->d_fc_qp, s.fc_qp, nfc));
  s.fd_cap = kFreshMemoSlots;
  CUDA_TRY(h, bind_zeroed(h, h->d_fd_state, s.fd_state, kFreshMemoSlots));
  CUDA_TRY(h, bind(h, h->d_fd_dom, s.fd_dom, kFreshMemoSlots));
  CUDA_TRY(h, bind(h, h->d_fd_fc, s.fd_fc, kFreshMemoSlots));
  CUDA_TRY(h, bind(h, h->d_fd_meta, s.fd_meta, kFreshMemoSlots));
  CUDA_TRY(h, bind(h, h->d_fd_vals, s.fd_vals, (size_t)kFreshMemoSlots * KSCHED_MAX_KEYS));
  CUDA_TRY(h, bind(h, h->d_fd_opts, s.fd_opts, (size_t)kFreshMemoSlots * W32));
  CUDA_TRY(h, bind(h, h->d_fd_bound, s.fd_bound, (size_t)kFreshMemoSlots * 4));
  CUDA_TRY(h, bind(h, h->d_fd_bound2, s.fd_bound2, (size_t)kFreshMemoSlots * 4));
  CUDA_TRY(h, bind(h, h->d_remaining, s.remaining, (size_t)V * KSCHED_MAX_RES));  // reset_state: limits per call
  CUDA_TRY(h, bind_zeroed(h, h->d_counters, s.counters, kNumCounters));
  CUDA_TRY(h, bind(h, h->d_vstore, s.vstore, kVarStore));
  {
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)p1, 0, 64, h->stream);
    CUDA_TRY(h, h->d_cub_tmp.ensure(need + 256));
    h->cub_tmp_bytes = need + 256;
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return KSCHED_OK;
}

// ---- upload one problem (pods / nodes / topology) and keep pristine copies of everything the pack kernel mutates
int ksched_upload(ksched_handle* h, const ksched_problem* pb) {
  if (!h || !pb) return KSCHED_ERR_INVALID;
  int rc = check_problem(h, pb);
  if (rc != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaSetDevice(h->device));
  // the resident problem is replaced from here on: a CUDA error part-way through leaves none
  h->uploaded = false;
  // the superset buffers ksched_load_cluster filled are about to be overwritten: simulations need a new ksched_load_cluster
  h->have_cluster = false;
  if ((rc = bind_problem(h, pb)) != KSCHED_OK) return rc;
  h->uploaded = true;
  h->sorted = false;
  return KSCHED_OK;
}

// K0 over the first P pods (a simulation's batch, otherwise the whole problem); so are run_class_feasibility and run_feasibility.
static int run_sort(ksched_handle* h, int P) {
  if (P == 0) return KSCHED_OK;
  const int threads = 256, blocks = (P + threads - 1) / threads;
  // one packed key (bind_problem), only its significant bits sorted
  sort_key1_kernel<<<blocks, threads, 0, h->stream>>>(P, h->d_cls_rank.ptr, h->d_pod_class.ptr, h->d_ts.ptr, h->d_uid_rank.ptr, h->sort1_ts_min,
                                                      h->sort1_ts_bits, h->sort1_uid_bits, h->d_k_tie.ptr, h->d_idx_tmp.ptr);
  size_t tmp = h->cub_tmp_bytes;
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(h->d_cub_tmp.ptr, tmp, h->d_k_tie.ptr, h->d_k_tmp.ptr, h->d_idx_tmp.ptr, h->d_order.ptr, P, 0, h->sort1_bits,
                                              h->stream));
  const int gblocks = std::min((P + 7) / 8, h->n_sm * 8);
  gather_rows_kernel<<<gblocks, 256, 0, h->stream>>>(P, h->d_classes.ptr, h->d_pod_class.ptr, h->d_order.ptr, h->d_rows.ptr);
  h->tm.sort_launches = 3;
  h->sorted = true;
  return KSCHED_OK;
}

static void fill_k1(ksched_handle* h, K1Params& k1) {
  // the row evaluation runs over the class table (every class once); feasibility_kernel replicates the rows per pod
  k1.cat = h->cat;
  k1.rows = reinterpret_cast<const uint64_t*>(h->st.classes);
  k1.n_pods = h->st.n_classes;
  k1.itype_sets = h->st.itype_sets;
  k1.F = h->d_Fclass.ptr;
  k1.best = h->d_best_class.ptr;
  k1.cls_req_ext = h->st.cls_req_ext;  // nullptr without ext resources
  k1.cls_ext_present = h->st.cls_ext_present;
  const int W32 = h->cat.W32;
  if (h->world > 1) {
    ksched_shard_range(W32, h->rank, h->world, &k1.word_begin, &k1.word_end);
  } else {
    k1.word_begin = 0;
    k1.word_end = W32;
  }
}

static std::mutex g_k1_mu;
static cudaEvent_t g_k1_done[64] = {};

// K1, class pass: every distinct pod row evaluated once (class_feasibility_kernel over the class table).
static int run_class_feasibility(ksched_handle* h, int P) {
  const int NC = h->st.n_classes;
  if (P == 0 || NC == 0) return KSCHED_OK;
  K1Params k1;
  fill_k1(h, k1);
  const DevCatalog& c = h->cat;
  const size_t alloc_bytes = (size_t)c.n_res * c.n_types * sizeof(int64_t);
  k1.alloc_in_smem = alloc_bytes <= (size_t)(128 << 10) ? 1 : 0;
  size_t smem = sizeof(ksched_template) * c.n_templates + sizeof(ksched_keyinfo) * KSCHED_MAX_KEYS + (k1.alloc_in_smem ? alloc_bytes : 0) +
                sizeof(int16_t) * KSCHED_MAX_KEYS * 64 + sizeof(int16_t) * 64 + sizeof(uint64_t) * 128;
  k1.n_valrows = h->n_valrows;
  k1.n_offrows = h->n_offrows;
  const size_t table_bytes = (size_t)(h->n_valrows + 2 * c.n_keys + h->n_offrows + 1 + c.n_templates) * c.W32 * sizeof(uint32_t);
  k1.tables_in_smem = smem + table_bytes <= (size_t)(160 << 10) ? 1 : 0;
  if (k1.tables_in_smem) smem += table_bytes;
  // one warp per class row (a row evaluation is thousands of cycles of dependent work: no chunking)
  const int warps_per_block = kK1Threads / 32;
  const int blocks = std::max(1, std::min(h->n_sm * 2, (NC + warps_per_block - 1) / warps_per_block));
  k1.dbg = nullptr;
#ifdef KSCHED_PROFILE_K1
  CUDA_TRY(h, h->d_k1dbg.ensure(8));
  CUDA_TRY(h, cudaMemsetAsync(h->d_k1dbg.ptr, 0, 8 * sizeof(long long), h->stream));
  k1.dbg = h->d_k1dbg.ptr;
#endif
  {
    std::lock_guard<std::mutex> lock(g_k1_mu);  // one __constant__ parameter block per device: see run_pack
    if (h->device < 0 || h->device >= 64) { h->err = "device ordinal out of range"; return KSCHED_ERR_INVALID; }
    cudaEvent_t& done = g_k1_done[h->device];
    if (!done) CUDA_TRY(h, cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    CUDA_TRY(h, cudaStreamWaitEvent(h->stream, done, 0));
    h->k1_host = k1;
    CUDA_TRY(h, cudaMemcpyToSymbolAsync(g_k1, &h->k1_host, sizeof(K1Params), 0, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaFuncSetAttribute(class_feasibility_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));  // per function: under the launch lock
    if (h->world > 1)  // column words of the other shards read as 0
      CUDA_TRY(h, cudaMemsetAsync(h->d_Fclass.ptr, 0, (size_t)NC * c.n_templates * c.W32 * 4, h->stream));
    class_feasibility_kernel<<<blocks, kK1Threads, smem, h->stream>>>();
    CUDA_TRY(h, cudaGetLastError());
    CUDA_TRY(h, cudaEventRecord(done, h->stream));
  }
#ifdef KSCHED_PROFILE_K1
  {
    long long dbg[8];
    cudaMemcpyAsync(dbg, h->d_k1dbg.ptr, sizeof dbg, cudaMemcpyDeviceToHost, h->stream);
    cudaStreamSynchronize(h->stream);
    fprintf(stderr, "[k1 profile] blocks=%d max cycles: stage=%lld compute=%lld total=%lld max_computes_per_warp=%lld | total computes=%lld avg compute cycles=%lld\n",
            blocks, dbg[0], dbg[1], dbg[2], dbg[3], dbg[4], dbg[4] ? dbg[5] / dbg[4] : 0);
  }
#endif
  return KSCHED_OK;
}

// K1 proper: the dense pods x (template, instance type) matrix and the per-pod best column, streamed from the class rows.
static int run_feasibility(ksched_handle* h, int P) {
  if (P == 0) return KSCHED_OK;
  const int RW = h->cat.n_templates * h->cat.W32;
  const int nblk = (P + 31) / 32;
  const int blocks = std::max(1, std::min(h->n_sm * 8, (nblk + 7) / 8));  // 8 warps per CTA, one 32-row block per warp and iteration
  feasibility_kernel<<<blocks, 256, 0, h->stream>>>(h->d_rows.ptr, P, h->st.n_classes, RW, h->d_Fclass.ptr, h->d_best_class.ptr, h->d_F.ptr,
                                                    h->d_best.ptr);
  CUDA_TRY(h, cudaGetLastError());
  h->tm.feasibility_launches = 2;
  const long long C = (long long)h->cat.n_templates * h->cat.n_types;
  h->tm.feasibility_bytes = (long long)P * 256 + C * 256 + (long long)P * C / 8;
  return KSCHED_OK;
}

__global__ void reset_kernel(ResetTable t) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  for (int q = 0; q < t.n; ++q) {
    const ResetSeg sg = t.seg[q];
    const size_t n16 = sg.bytes / 16;
    uint4* d = static_cast<uint4*>(sg.dst);
    const uint4* sv = static_cast<const uint4*>(sg.src);
    for (size_t i = tid; i < n16; i += nth) d[i] = sv ? sv[i] : make_uint4(0, 0, 0, 0);
    unsigned char* db = static_cast<unsigned char*>(sg.dst);
    const unsigned char* sb = static_cast<const unsigned char*>(sg.src);
    for (size_t i = n16 * 16 + tid; i < sg.bytes; i += nth) db[i] = sb ? sb[i] : 0;
  }
}

// The segments ksched_upload recorded, and the provisioner limits: a simulation's (already on the device, with the removed
// nodes' capacity given back; its candidate marks are cleared too) or the templates'.
static int reset_state(ksched_handle* h, const int64_t* sim_remaining = nullptr) {
  ResetTable t = h->resets;
  const size_t rem_bytes = (size_t)h->cat.n_templates * KSCHED_MAX_RES * 8;
  if (sim_remaining) {
    CUDA_TRY(h, record_reset(t, h->st.remaining, sim_remaining, rem_bytes));
    CUDA_TRY(h, record_reset(t, h->d_in_set.ptr, nullptr, (size_t)std::max(h->st.n_existing, 1)));
  } else {
    std::vector<int64_t> rem((size_t)h->cat.n_templates * KSCHED_MAX_RES);
    for (int v = 0; v < h->cat.n_templates; ++v)
      for (int r = 0; r < KSCHED_MAX_RES; ++r) rem[(size_t)v * KSCHED_MAX_RES + r] = h->h_templates[v].remaining[r];
    CUDA_TRY(h, cudaMemcpyAsync(h->st.remaining, rem.data(), rem_bytes, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));  // rem is a stack vector
  }
  reset_kernel<<<h->n_sm * 2, 256, 0, h->stream>>>(t);
  CUDA_TRY(h, cudaGetLastError());
  return KSCHED_OK;
}

// g_k2 is one __constant__ object per device: a launch may only overwrite it after the previous pack kernel on that
// device (possibly of another handle, on another stream) has finished. Ordered on the device, never on the host.
static std::mutex g_k2_mu;
static cudaEvent_t g_k2_done[64] = {};

// The pack kernel over the first n_pods pods of the queue (a simulation's batch, otherwise the whole problem).
static int run_pack(ksched_handle* h, int n_pods, int stop_new_nodes) {
  K2Params& k2 = h->k2_host;
  k2.cat = h->cat;
  k2.st = h->st;
  // what may change between launches of one upload: the batch, the column sharding (ksched_set_shard / ksched_nccl_init
  // may follow the upload), the templates (ksched_load_catalog's early-out), the mode switches and the smem layout
  PackState& s = k2.st;
  s.n_pods = n_pods;
  s.stop_new_nodes = stop_new_nodes;
  s.use_F = h->world == 1 ? 1 : 0;
  const size_t alloc_bytes = (size_t)h->cat.n_res * h->cat.n_types * sizeof(int64_t);
  // 227 KB per CTA on sm_90a: the hot node window + ~4 KB of static shared memory come first
  const size_t static_smem = (size_t)(14 << 10);  // file-scope __shared__ objects (pod row, PodTopo, RunCtx with its variants, scratch)
  const size_t smem_left = (size_t)(227 << 10) - sizeof(HotSmem) - kRunArrayBytes - static_smem;
  s.alloc_in_smem = alloc_bytes <= smem_left ? 1 : 0;
  s.run_off = s.alloc_in_smem ? (int)((alloc_bytes + 15) & ~(size_t)15) : 0;
  const size_t smem = sizeof(HotSmem) + (size_t)s.run_off + kRunArrayBytes;
  s.any_limits = 0;
  for (const ksched_template& tm : h->h_templates) if (tm.has_limits && tm.limit_present) s.any_limits = 1;
  s.use_class_run = getenv("KSCHED_NO_CLASSRUN") ? 0 : 1;
  s.use_level_run = std::getenv("KSCHED_NO_LEVELRUN") ? 0 : 1;
  s.use_mask_run = std::getenv("KSCHED_NO_MASKRUN") ? 0 : 1;
  s.use_level_warp = std::getenv("KSCHED_NO_LEVELWARP") ? 0 : 1;
  s.use_varstore = std::getenv("KSCHED_NO_VARSTORE") ? 0 : 1;
  s.use_round_stretch = std::getenv("KSCHED_NO_ROUNDSTRETCH") ? 0 : 1;
  s.use_fill_stretch = s.use_round_stretch && !std::getenv("KSCHED_NO_FILLSTRETCH") ? 1 : 0;
  // block size: the chain is latency-bound on ONE thread's commit; more warps only help when there are many candidate
  // nodes to examine per pod (existing nodes, large in-flight sets)
  int threads = s.n_existing >= 2048 ? kPackThreads : (s.n_existing >= 256 ? 256 : 128);
  if (const char* e = getenv("KSCHED_PACK_THREADS")) { int v = atoi(e); if (v >= 32 && v <= kPackThreads && v % 32 == 0) threads = v; }
  {
    std::lock_guard<std::mutex> lock(g_k2_mu);
    if (h->device < 0 || h->device >= 64) { h->err = "device ordinal out of range"; return KSCHED_ERR_INVALID; }
    cudaEvent_t& done = g_k2_done[h->device];
    if (!done) CUDA_TRY(h, cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    CUDA_TRY(h, cudaStreamWaitEvent(h->stream, done, 0));  // no-op for an event that was never recorded
    CUDA_TRY(h, cudaMemcpyToSymbolAsync(g_k2, &k2, sizeof(K2Params), 0, cudaMemcpyHostToDevice, h->stream));
    // the attribute belongs to the function, not to the handle: set it under the same lock as the launch
    const bool ext = h->cat.n_res_ext > 0, small = threads <= kPackThreadsSmall;
    void (*kern)() = small ? (ext ? pack_kernel<true, kPackThreadsSmall> : pack_kernel<false, kPackThreadsSmall>)
                           : (ext ? pack_kernel<true, kPackThreads> : pack_kernel<false, kPackThreads>);
    cudaFuncAttributes fa;
    CUDA_TRY(h, cudaFuncGetAttributes(&fa, kern));
    if (threads > fa.maxThreadsPerBlock) {  // the instantiation's register budget does not fit this block
      h->err = "pack_kernel: " + std::to_string(threads) + " threads exceed the instantiation's limit of " + std::to_string(fa.maxThreadsPerBlock);
      return KSCHED_ERR_INVALID;
    }
    CUDA_TRY(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<1, threads, smem, h->stream>>>();
    CUDA_TRY(h, cudaGetLastError());
    CUDA_TRY(h, cudaEventRecord(done, h->stream));
  }
  finalize_options_kernel<<<h->n_sm, 256, 0, h->stream>>>(h->cat, s.counters, s.nn_req, s.nn_req_present, s.nn_opts, s.max_new);
  h->tm.pack_launches = 2;
  return KSCHED_OK;
}

static int flush_l2(ksched_handle* h) {
  const size_t n = (size_t)64 << 20;  // 256 MiB of u32, five times the 50 MB L2 of an H100
  CUDA_TRY(h, h->d_flush.ensure(n));
  flush_kernel<<<h->n_sm * 4, 512, 0, h->stream>>>(h->d_flush.ptr, n);
  return KSCHED_OK;
}

static float ev_us(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  return ms * 1000.f;
}

int ksched_run_resident(ksched_handle* h, int do_flush) {
  if (!h || !h->uploaded) return KSCHED_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  const int P = h->st.n_pods;
  int rc;
  if ((rc = reset_state(h)) != KSCHED_OK) return rc;
  if (do_flush && (rc = flush_l2(h)) != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[0], h->stream));
  if ((rc = run_sort(h, P)) != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[1], h->stream));
  if ((rc = run_class_feasibility(h, P)) != KSCHED_OK) return rc;
  if ((rc = run_feasibility(h, P)) != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[2], h->stream));
  h->tm.allreduce_us = 0;
  if (h->world > 1 && h->comm) {
    ncclResult_t r = ncclAllReduce(h->d_best.ptr, h->d_best.ptr, (size_t)P, ncclUint64, ncclMin, h->comm, h->stream);
    if (r != ncclSuccess) { h->err = std::string("ncclAllReduce: ") + ncclGetErrorString(r); return KSCHED_ERR_NCCL; }
  }
  CUDA_TRY(h, cudaEventRecord(h->ev[3], h->stream));
  if ((rc = run_pack(h, P, 0)) != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[4], h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  h->tm.sort_us = ev_us(h->ev[0], h->ev[1]);
  h->tm.feasibility_us = ev_us(h->ev[1], h->ev[2]);
  h->tm.allreduce_us = ev_us(h->ev[2], h->ev[3]);
  h->tm.pack_us = ev_us(h->ev[3], h->ev[4]);
  h->tm.total_us = ev_us(h->ev[0], h->ev[4]);
  return KSCHED_OK;
}

int ksched_run_feasibility_only(ksched_handle* h, int do_flush, float* elapsed_us) {
  if (!h || !h->uploaded) return KSCHED_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  const int P = h->st.n_pods;
  int rc;
  if (!h->sorted) {  // K0 first: the kernel streams the FFD-ordered pod-row matrix
    CUDA_TRY(h, cudaMemcpyAsync(h->d_pod_class.ptr, h->d_pod_class0.ptr, (size_t)P * 4, cudaMemcpyDeviceToDevice, h->stream));
    if ((rc = run_sort(h, P)) != KSCHED_OK) return rc;
  }
  CUDA_TRY(h, cudaEventRecord(h->ev[7], h->stream));
  if ((rc = run_class_feasibility(h, P)) != KSCHED_OK) return rc;  // n_classes row evaluations (timed on their own)
  if (do_flush && (rc = flush_l2(h)) != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[5], h->stream));
  if ((rc = run_feasibility(h, P)) != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[6], h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  if (elapsed_us) *elapsed_us = ev_us(h->ev[5], h->ev[6]);
  h->tm.feasibility_us = ev_us(h->ev[5], h->ev[6]);
  h->tm.class_feasibility_us = ev_us(h->ev[7], h->ev[5]);  // includes the L2 flush when one was asked for
  return KSCHED_OK;
}

#ifdef KSCHED_PROFILE_PACK
static void print_pack_profile(const long long* counters) {
  const long long* c = counters;
  fprintf(stderr, "[pack profile] generic: topo=%lld existing=%lld eval=%lld commit=%lld fresh=%lld fail=%lld | fastblock=%lld genericcall=%lld | "
                  "n_generic=%lld inflight_placed=%lld fresh_steps=%lld failures=%lld paths[rej,cached,row,dyn,cachedempty]=%lld,%lld,%lld,%lld,%lld steps=%lld\n",
          c[kCtrGenTopo], c[kCtrGenExisting], c[kCtrGenEval], c[kCtrGenCommit], c[kCtrGenFresh], c[kCtrGenFail], c[kCtrRunCallCycles],
          c[kCtrGenCallCycles], c[kCtrGenSteps], c[kCtrGenInflightPlaced], c[kCtrGenFreshSteps], c[kCtrGenFailures], c[kCtrGenPath],
          c[kCtrGenPath + 1], c[kCtrGenPath + 2], c[kCtrGenPath + 3], c[kCtrGenPath + 4], c[kCtrSteps]);
  fprintf(stderr, "[pack profile] fresh: decide=%lld words=%lld commit=%lld rest=%lld | in-flight verify=%lld\n", c[kCtrGenFreshDecide],
          c[kCtrGenFreshWords], c[kCtrGenFreshCommit], c[kCtrGenFresh], c[kCtrGenInflightVerify]);
  fprintf(stderr, "[pack profile] in-flight commit: winner+barrier=%lld record=%lld rest=%lld\n", c[kCtrGenInflightWinner], c[kCtrGenInflightRecord],
          c[kCtrGenCommit]);
  fprintf(stderr, "[pack profile] class_run: calls=%lld pods=%lld bails=%lld ineligible=%lld cycles=%lld\n", c[kCtrRunCalls], c[kCtrRunPlaced],
          c[kCtrRunBails], c[kCtrRunIneligible], c[kCtrRunCallCycles]);
  fprintf(stderr, "[pack profile] class_run fixed cost: open nodes at entry (sum)=%lld entry cycles=%lld (per-node inputs %lld) "
                  "write-back cycles=%lld | compactions=%lld slots=%lld cycles=%lld\n", c[kCtrRunActiveSum], c[kCtrRunEntryCycles],
          c[kCtrRunInputCycles], c[kCtrRunWbCycles], c[kCtrRunCompacts], c[kCtrRunCompactSlots], c[kCtrRunCompactCycles]);
  fprintf(stderr, "[pack profile] class_run round trips (status-1 stop -> entry of the next call that places pods): cycles=%lld | "
                  "stops for want of a variant=%lld, their round trips' cycles=%lld | variant store: hits=%lld entries=%lld\n",
          c[kCtrRoundTripCycles], c[kCtrNoVariantStops], c[kCtrNoVariantTripCycles], c[kCtrVarStoreHits], c[kCtrVarStoreEntries]);
  fprintf(stderr, "[pack profile] mask run steps=%lld with >1 admissible domain=%lld round-able=%lld\n", c[kCtrMaskSteps], c[kCtrMaskMultiDomain],
          c[kCtrMaskRoundable]);
  fprintf(stderr, "[pack profile] mask run: build cycles=%lld (refused %lld) loop cycles=%lld pods=%lld entries=%lld\n", c[kCtrMaskBuildCycles],
          c[kCtrMaskBuildRefused], c[kCtrMaskCycles], c[kCtrMaskPods], c[kCtrMaskEntries]);
  fprintf(stderr, "[pack profile] mask run: single steps on the unpinned head=%lld | pin steps=%lld pods=%lld ended by "
                  "[staged entries,count,key,refused,end of list or 32 pods]=%lld,%lld,%lld,%lld,%lld\n",
          c[kCtrMaskUnpinnedSingle], c[kCtrPinSteps], c[kCtrPinPods], c[kCtrPinEndStaged], c[kCtrPinEndCount], c[kCtrPinEndKey],
          c[kCtrPinEndRefused], c[kCtrPinEndList]);
  fprintf(stderr, "[pack profile] mask run rounds: iterations=%lld pods=%lld cycles=%lld | stretch length R (rounds a step could place, "
                  "1..16) [pinned] [fresh]:", c[kCtrRounds], c[kCtrRoundPods], c[kCtrRoundCycles]);
  for (const int k : {kCtrStretchPinned, kCtrStretchFresh}) {
    fprintf(stderr, " [");
    for (int r = 0; r < 16; ++r) fprintf(stderr, r ? ",%lld" : "%lld", c[k + r]);
    fprintf(stderr, "]");
  }
  fprintf(stderr, "\n");
  fprintf(stderr, "[pack profile] mask run rounds: bucket stretch below 2 rounds ended by [singleton bucket, head accepts again; "
                  "singleton bucket, head done; unpinned key; inexact room; kM1Lv; staged end]=%lld,%lld,%lld,%lld,%lld,%lld | "
                  "single rounds with unequal counts=%lld | fill stretch length (1..16):",
          c[kCtrBucketEnd], c[kCtrBucketEnd + 1], c[kCtrBucketEnd + 2], c[kCtrBucketEnd + 3], c[kCtrBucketEnd + 4],
          c[kCtrBucketEnd + 5], c[kCtrRoundsUnequal]);
  for (int r = 0; r < 16; ++r) fprintf(stderr, r ? ",%lld" : " %lld", c[kCtrFillLen + r]);
  fprintf(stderr, "\n");
  fprintf(stderr, "[pack profile] class_run without mask-key spread: cycles=%lld pods=%lld level+fill iterations=%lld (fill %lld) fresh=%lld per-pod=%lld | with: cycles=%lld pods=%lld fresh=%lld per-pod=%lld\n",
          c[kCtrRunLvCycles], c[kCtrRunLvPods], c[kCtrRunLvSteps], c[kCtrRunLvFills], c[kCtrRunLvFresh], c[kCtrRunLvPerPod], c[kCtrRunCycles],
          c[kCtrRunPods], c[kCtrRunFresh], c[kCtrRunPerPod]);
}
#endif

int ksched_download(ksched_handle* h, const ksched_problem* pb, ksched_result* res) {
  if (!h || !pb || !res || !h->uploaded) return KSCHED_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  const PackState& s = h->st;
  const int P = s.n_pods, NE = s.n_existing, W32 = h->cat.W32, W64 = W32 / 2, V = h->cat.n_templates;
  long long counters[kNumCounters];
  h->tm.d2h_bytes = 0;
  CUDA_TRY(h, download(h, counters, s.counters, kNumCounters));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
#ifdef KSCHED_PROFILE_PACK
  print_pack_profile(counters);
#endif
  if (counters[kCtrError] != 0) {
    h->err = counters[kCtrError] == KSCHED_ERR_OVERFLOW ? "new-node capacity exceeded" : "a pod is constrained by more topology groups than the kernel supports";
    return (int)counters[kCtrError];
  }
  const int n_new = (int)counters[kCtrNewNodes];
  res->n_new_nodes = n_new;
  res->n_unscheduled = (int)counters[kCtrUnscheduled];
  res->nodes_visited = counters[kCtrNodesVisited];
  res->add_calls = counters[kCtrAddCalls];
  h->tm.pack_steps = counters[kCtrSteps];
  if (res->assign) CUDA_TRY(h, download(h, res->assign, s.assign, (size_t)P));
  if (res->relax_level) CUDA_TRY(h, download(h, res->relax_level, s.relax_level, (size_t)P));
  if (res->place_seq) CUDA_TRY(h, download(h, res->place_seq, s.place_seq, (size_t)P));
  if (n_new > 0 && res->new_nodes && res->new_node_types) {
    std::vector<uint8_t> tmpl(n_new);
    std::vector<int32_t> count(n_new);
    std::vector<uint32_t> reqp(n_new), opts;
    std::vector<uint64_t> meta(n_new), vals;
    std::vector<int64_t> req;
    CUDA_TRY(h, download(h, tmpl.data(), s.nn_tmpl, (size_t)n_new));
    CUDA_TRY(h, download(h, count.data(), s.nn_count, (size_t)n_new));
    CUDA_TRY(h, download(h, reqp.data(), s.nn_req_present, (size_t)n_new));
    CUDA_TRY(h, download(h, meta.data(), s.nn_meta, (size_t)n_new));
    CUDA_TRY(h, download_soa(h, req, s.nn_req, 8, (size_t)s.max_new, n_new));
    CUDA_TRY(h, download_soa(h, vals, s.nn_vals, 16, (size_t)s.max_new, n_new));
    CUDA_TRY(h, download_soa(h, opts, s.nn_opts, W32, (size_t)s.max_new, n_new));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    auto types_of = [&](int n) { return reinterpret_cast<uint32_t*>(res->new_node_types + (size_t)n * W64); };
    for (int n = 0; n < n_new; ++n) {
      ksched_new_node& o = res->new_nodes[n];
      std::memset(&o, 0, sizeof o);
      o.template_index = tmpl[n];
      o.pod_count = count[n];
      o.requests_present = reqp[n];
      o.reqs.meta = meta[n];
      if (W32 & 1) types_of(n)[W32] = 0;  // the row is W64 64-bit words: the caller's buffer need not be cleared
    }
    soa_to_rows(req, 8, n_new, [&](int n) { return res->new_nodes[n].requests; });
    soa_to_rows(vals, 16, n_new, [&](int n) { return res->new_nodes[n].reqs.values; });
    soa_to_rows(opts, W32, n_new, types_of);
    if (const int X = h->cat.n_res_ext) {
      if (res->new_node_requests_ext) CUDA_TRY(h, download(h, res->new_node_requests_ext, s.nn_req_ext, (size_t)n_new * X));
      if (res->new_node_requests_ext_present) CUDA_TRY(h, download(h, res->new_node_requests_ext_present, s.nn_ext_present, (size_t)n_new));
      CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    }
  }
  if (res->launch && n_new > 0) {
    if (!h->cat.offer_keys) { h->err = "ksched_result.launch needs ksched_catalog.offering_keys"; return KSCHED_ERR_INVALID; }
    CUDA_TRY(h, h->d_launch.ensure((size_t)n_new));
    launch_choice_kernel<<<h->n_sm, 256, 0, h->stream>>>(h->cat, s.counters, s.nn_vals, s.nn_meta, s.nn_opts, s.max_new, h->d_launch.ptr);
    CUDA_TRY(h, download(h, res->launch, h->d_launch.ptr, (size_t)n_new));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  if (res->existing_reqs && NE > 0) {
    std::vector<uint64_t> vals((size_t)16 * NE), meta(NE);
    CUDA_TRY(h, download(h, vals.data(), s.ex_vals, vals.size()));
    CUDA_TRY(h, download(h, meta.data(), s.ex_meta, meta.size()));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    soa_to_rows(vals, 16, NE, [&](int e) { return res->existing_reqs[e].values; });
    for (int e = 0; e < NE; ++e) res->existing_reqs[e].meta = meta[e];
  }
  if (res->feasibility) {
    // device rows are in FFD (queue) order; the caller gets them in its own pod order
    std::vector<uint32_t> order(P), F((size_t)P * V * W32);
    CUDA_TRY(h, download(h, order.data(), s.order, order.size()));
    CUDA_TRY(h, download(h, F.data(), s.F, F.size()));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    const size_t rowb = (size_t)V * W32;
    for (int j = 0; j < P; ++j) std::memcpy(reinterpret_cast<uint32_t*>(res->feasibility) + (size_t)order[j] * rowb, &F[(size_t)j * rowb], rowb * 4);
  }
  if (res->best_column) {
    std::vector<uint32_t> order(P);
    std::vector<unsigned long long> best(P);
    CUDA_TRY(h, download(h, order.data(), s.order, order.size()));
    CUDA_TRY(h, download(h, best.data(), s.best, best.size()));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    for (int j = 0; j < P; ++j) res->best_column[order[j]] = best[j];
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return KSCHED_OK;
}

int ksched_solve(ksched_handle* h, const ksched_problem* pb, ksched_result* res) {
  if (!h || !pb || !res) return KSCHED_ERR_INVALID;
  auto t0 = std::chrono::steady_clock::now();
  int rc = ksched_upload(h, pb);
  if (rc != KSCHED_OK) return rc;
  auto t1 = std::chrono::steady_clock::now();
  rc = ksched_run_resident(h, 0);
  if (rc != KSCHED_OK) return rc;
  auto t2 = std::chrono::steady_clock::now();
  rc = ksched_download(h, pb, res);
  auto t3 = std::chrono::steady_clock::now();
  h->tm.upload_us = std::chrono::duration<double, std::micro>(t1 - t0).count();
  h->tm.download_us = std::chrono::duration<double, std::micro>(t3 - t2).count();
  return rc;
}

// ---- consolidation simulator on a device-resident cluster snapshot (cluster.cuh)
int ksched_load_cluster(ksched_handle* h, const ksched_cluster* cl) {
  if (!h || !cl || !cl->problem || (!cl->pod_node && cl->problem->n_pods > 0)) return KSCHED_ERR_INVALID;
  const ksched_problem* pb = cl->problem;
  h->have_cluster = false;
  const bool topo = pb->n_groups != 0;
  if (topo && (!cl->class_count_begin || !cl->node_domain || !cl->node_has_hostname_label || !cl->group_filter_match)) {
    h->err = "unsupported: a cluster with topology groups needs the counting tables of ksched_cluster";
    return KSCHED_ERR_UNSUPPORTED;
  }
  const int P = pb->n_pods, NE = pb->n_existing;
  // pods: the pending ones first, then node by node (every node's pods contiguous)
  std::vector<int32_t> first((size_t)std::max(NE, 1), -1), count((size_t)std::max(NE, 1), 0);
  int pending = 0;
  for (int i = 0; i < P; ++i) {
    const int nd = cl->pod_node[i];
    if (nd >= NE) { h->err = "pod_node out of range"; return KSCHED_ERR_INVALID; }
    if (nd < 0) { if (i != pending) { h->err = "pending pods must come first"; return KSCHED_ERR_INVALID; } ++pending; continue; }
    if (first[nd] < 0) first[nd] = i;
    else if (cl->pod_node[i - 1] != nd) { h->err = "the pods of one node must be contiguous"; return KSCHED_ERR_INVALID; }
    ++count[nd];
  }
  int rc = ksched_upload(h, pb);  // the superset problem: buffers sized for the largest batch, existing-node state, class tables
  if (rc != KSCHED_OK) return rc;
  CUDA_TRY(h, upload(h, h->d_sup_pod_node, cl->pod_node, (size_t)P));
  CUDA_TRY(h, upload(h, h->d_sup_class, pb->pod_class, (size_t)P));
  CUDA_TRY(h, upload(h, h->d_sup_ts, queue_timestamps(h, pb), (size_t)P));
  CUDA_TRY(h, upload(h, h->d_sup_uid, pb->pod_uid_rank, (size_t)P));
  CUDA_TRY(h, upload_vec(h, h->d_node_first, first));
  CUDA_TRY(h, h->d_node_dst.ensure((size_t)std::max(NE, 1)));
  CUDA_TRY(h, h->d_in_set.ensure((size_t)std::max(NE, 1)));
  CUDA_TRY(h, h->d_pod_src.ensure((size_t)std::max(P, 1)));
  h->cluster_topology = topo;
  if (topo) {
    const int NC = pb->n_classes, NK = h->cat.n_keys;
    h->filt_words = (NE + 31) / 32;
    const uint32_t n_rel = cl->class_count_begin[NC];
    for (uint32_t q = 0; q < n_rel; ++q)
      if (cl->class_count[q].group >= (uint32_t)pb->n_groups) { h->err = "class_count group out of range"; return KSCHED_ERR_INVALID; }
    CUDA_TRY(h, upload(h, h->d_cc_begin, cl->class_count_begin, (size_t)NC + 1));
    CUDA_TRY(h, upload(h, h->d_cc, cl->class_count, (size_t)std::max<uint32_t>(n_rel, 1)));
    CUDA_TRY(h, upload(h, h->d_node_dom, cl->node_domain, (size_t)std::max(NK, 1) * std::max(NE, 1)));
    CUDA_TRY(h, upload(h, h->d_node_hostlabel, cl->node_has_hostname_label, (size_t)std::max(NE, 1)));
    CUDA_TRY(h, upload(h, h->d_filt, cl->group_filter_match, (size_t)pb->n_groups * std::max(h->filt_words, 1)));
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->h_node_first.swap(first);
  h->h_node_count.swap(count);
  h->sup_pods = P;
  h->sup_pending = pending;
  h->have_cluster = true;
  return KSCHED_OK;
}

int ksched_simulate_batch(ksched_handle* h, const ksched_candidate_set* sets, int n_sets, ksched_sim_result* results, uint64_t* node0_types) {
  if (!h || !sets || n_sets < 0 || (n_sets > 0 && !results)) return KSCHED_ERR_INVALID;
  if (!h->have_cluster) { h->err = "ksched_load_cluster must be called first"; return KSCHED_ERR_INVALID; }
  if (n_sets == 0) return KSCHED_OK;
  CUDA_TRY(h, cudaSetDevice(h->device));
  const int NE = h->st.n_existing, V = h->cat.n_templates, W32 = h->cat.W32, W64 = W32 / 2;
  // stage every set's node list, per-node batch offsets and limits in one upload each
  std::vector<int32_t> all_nodes, all_dst((size_t)n_sets * std::max(NE, 1), 0), batch((size_t)n_sets, 0), node_off((size_t)n_sets + 1, 0);
  std::vector<int64_t> all_rem((size_t)n_sets * V * KSCHED_MAX_RES, 0);
  for (int q = 0; q < n_sets; ++q) {
    const ksched_candidate_set& cs = sets[q];
    if (cs.n_nodes < 0 || (cs.n_nodes > 0 && !cs.nodes)) { h->err = "bad candidate set"; return KSCHED_ERR_INVALID; }
    std::vector<int32_t> nodes(cs.nodes, cs.nodes + cs.n_nodes);
    std::sort(nodes.begin(), nodes.end());  // the batch lists the removed nodes' pods in slot order (the queue sorts them anyway, queue.go:35-110)
    int pos = h->sup_pending;
    for (size_t i = 0; i < nodes.size(); ++i) {
      const int nd = nodes[i];
      if (nd < 0 || nd >= NE || (i > 0 && nodes[i - 1] == nd)) { h->err = "candidate set: existing slot out of range or repeated"; return KSCHED_ERR_INVALID; }
      all_dst[(size_t)q * NE + nd] = pos;
      pos += h->h_node_count[(size_t)nd];
    }
    batch[(size_t)q] = pos;
    all_nodes.insert(all_nodes.end(), nodes.begin(), nodes.end());
    node_off[(size_t)q + 1] = (int32_t)all_nodes.size();
    for (int v = 0; v < V; ++v)
      for (int r = 0; r < KSCHED_MAX_RES; ++r)
        all_rem[((size_t)q * V + v) * KSCHED_MAX_RES + r] = cs.remaining ? cs.remaining[(size_t)v * KSCHED_MAX_RES + r] : h->h_templates[(size_t)v].remaining[r];
  }
  if (all_nodes.empty()) all_nodes.push_back(0);
  CUDA_TRY(h, upload_vec(h, h->d_set_nodes, all_nodes));
  CUDA_TRY(h, upload_vec(h, h->d_node_dst, all_dst));
  CUDA_TRY(h, upload_vec(h, h->d_sim_remaining, all_rem));
  CUDA_TRY(h, h->d_sim_results.ensure((size_t)n_sets));
  CUDA_TRY(h, h->d_sim_types.ensure((size_t)n_sets * W32));
  CUDA_TRY(h, cudaEventRecord(h->ev[0], h->stream));
  int rc = KSCHED_OK;
  // nothing computeConsolidation can return depends on what happens after a second new node is opened
  // (consolidation.go:214-224: len(newNodes) != 1 -> do nothing): the simulation stops there
  const int stop_new_nodes = 2;
  for (int q = 0; q < n_sets && rc == KSCHED_OK; ++q) {
    const int n_nodes = node_off[(size_t)q + 1] - node_off[(size_t)q], P = batch[(size_t)q];
    rc = reset_state(h, h->d_sim_remaining.ptr + (size_t)q * V * KSCHED_MAX_RES);
    if (rc != KSCHED_OK) break;
    if (n_nodes > 0)
      cluster_mark_kernel<<<(n_nodes + 255) / 256, 256, 0, h->stream>>>(h->d_set_nodes.ptr + node_off[(size_t)q], n_nodes, h->d_in_set.ptr, h->d_ex_closed.ptr);
    if (h->sup_pods > 0)
      cluster_select_kernel<<<(h->sup_pods + 255) / 256, 256, 0, h->stream>>>(h->sup_pods, h->d_sup_pod_node.ptr, h->d_in_set.ptr, h->d_node_dst.ptr + (size_t)q * NE,
                                                                              h->d_node_first.ptr, h->sup_pending, h->d_sup_class.ptr, h->d_sup_ts.ptr, h->d_sup_uid.ptr,
                                                                              h->d_pod_class0.ptr, h->d_ts.ptr, h->d_uid_rank.ptr, h->d_pod_src.ptr);
    if (h->cluster_topology && h->sup_pods > 0)
      cluster_topology_kernel<<<(h->sup_pods + 255) / 256, 256, 0, h->stream>>>(
          h->sup_pods, h->d_sup_pod_node.ptr, h->d_in_set.ptr, h->d_sup_class.ptr, h->d_cc_begin.ptr, h->d_cc.ptr, h->d_groups.ptr, h->d_node_dom.ptr,
          h->d_node_hostlabel.ptr, h->d_filt.ptr, h->filt_words, NE, NE + h->st.max_new, h->d_grp_host_row.ptr, h->d_grp_cnt.ptr,
          reinterpret_cast<unsigned long long*>(h->d_grp_registered.ptr), h->d_grp_host.ptr, h->d_grp_host_total.ptr);
    // the working copy of the pod classes (reset_state copied the previous batch's): refresh it from the new batch
    if (P > 0) CUDA_TRY(h, cudaMemcpyAsync(h->d_pod_class.ptr, h->d_pod_class0.ptr, (size_t)P * 4, cudaMemcpyDeviceToDevice, h->stream));
    if ((rc = run_sort(h, P)) != KSCHED_OK) break;
    // the class rows of the feasibility matrix depend on the classes and the catalog only: once per batch
    if (q == 0 && (rc = run_class_feasibility(h, P)) != KSCHED_OK) break;
    if ((rc = run_feasibility(h, P)) != KSCHED_OK) break;
    if ((rc = run_pack(h, P, stop_new_nodes)) != KSCHED_OK) break;
    cluster_collect_kernel<<<1, 64, 0, h->stream>>>(h->d_counters.ptr, P, h->d_nn_tmpl.ptr, h->d_nn_count.ptr, h->d_nn_req.ptr, h->d_nn_req_present.ptr,
                                                    h->d_nn_vals.ptr, h->d_nn_meta.ptr, h->d_nn_opts.ptr, h->st.max_new, W32, h->d_sim_results.ptr + q,
                                                    h->d_sim_types.ptr + (size_t)q * W32);
  }
  if (rc != KSCHED_OK) return rc;
  CUDA_TRY(h, cudaEventRecord(h->ev[4], h->stream));
#ifdef KSCHED_PROFILE_PACK
  {
    long long counters[kNumCounters];
    CUDA_TRY(h, cudaMemcpyAsync(counters, h->d_counters.ptr, sizeof counters, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    print_pack_profile(counters);  // the last simulation of the batch
  }
#endif
  std::vector<SimResultDev> dev((size_t)n_sets);
  std::vector<uint32_t> types((size_t)n_sets * W32);
  CUDA_TRY(h, cudaMemcpyAsync(dev.data(), h->d_sim_results.ptr, dev.size() * sizeof(SimResultDev), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(types.data(), h->d_sim_types.ptr, types.size() * 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  h->tm.total_us = ev_us(h->ev[0], h->ev[4]);
  for (int q = 0; q < n_sets; ++q) {
    const SimResultDev& d = dev[(size_t)q];
    ksched_sim_result& o = results[q];
    std::memset(&o, 0, sizeof o);
    o.n_pods = d.n_pods; o.n_unscheduled = d.n_unscheduled; o.n_new_nodes = d.n_new_nodes; o.error = d.error;
    if (d.n_new_nodes >= 1) {
      o.node0.template_index = d.template_index; o.node0.pod_count = d.pod_count; o.node0.requests_present = d.requests_present;
      std::memcpy(o.node0.requests, d.requests, sizeof d.requests);
      std::memcpy(o.node0.reqs.values, d.values, sizeof d.values);
      o.node0.reqs.meta = d.meta;
    }
    if (node0_types) {
      std::memset(node0_types + (size_t)q * W64, 0, (size_t)W64 * 8);
      if (d.n_new_nodes >= 1) std::memcpy(node0_types + (size_t)q * W64, &types[(size_t)q * W32], (size_t)W32 * 4);
    }
  }
  return KSCHED_OK;
}

int ksched_rank_candidates(ksched_handle* h, const ksched_rank_input* in, int32_t* order, double* cost, int32_t* n_candidates) {
  if (!h || !in || !order || !cost || !n_candidates || in->n_nodes < 0 || in->n_pods < 0) return KSCHED_ERR_INVALID;
  *n_candidates = 0;
  const int N = in->n_nodes, NP = in->n_pods;
  if (N == 0) return KSCHED_OK;
  if (!in->node_eligible || (!in->node_cost && (!in->pod_offsets || !in->node_age_seconds || !in->node_ttl_seconds ||
                                                (NP > 0 && (!in->pod_deletion_cost || !in->pod_priority || !in->pod_flags))))) return KSCHED_ERR_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, upload(h, h->d_rk_elig_in, in->node_eligible, (size_t)N));
  if (in->node_cost) {
    CUDA_TRY(h, upload(h, h->d_rk_cost_in, in->node_cost, (size_t)N));
  } else {
    CUDA_TRY(h, upload(h, h->d_rk_off, in->pod_offsets, (size_t)N + 1));
    CUDA_TRY(h, upload(h, h->d_rk_age, in->node_age_seconds, (size_t)N));
    CUDA_TRY(h, upload(h, h->d_rk_ttl, in->node_ttl_seconds, (size_t)N));
    if (NP > 0) {
      CUDA_TRY(h, upload(h, h->d_rk_dc, in->pod_deletion_cost, (size_t)NP));
      CUDA_TRY(h, upload(h, h->d_rk_prio, in->pod_priority, (size_t)NP));
      CUDA_TRY(h, upload(h, h->d_rk_flags, in->pod_flags, (size_t)NP));
    }
  }
  CUDA_TRY(h, h->d_rk_cost.ensure((size_t)N));
  CUDA_TRY(h, h->d_rk_cost_out.ensure((size_t)N));
  CUDA_TRY(h, h->d_rk_elig.ensure((size_t)N));
  CUDA_TRY(h, h->d_rk_order.ensure((size_t)N));
  CUDA_TRY(h, h->d_rk_n.ensure(1));
  const int blocks = (N + 255) / 256;
  rank_cost_kernel<<<blocks, 256, 0, h->stream>>>(N, h->d_rk_off.ptr, h->d_rk_dc.ptr, h->d_rk_prio.ptr, h->d_rk_flags.ptr, h->d_rk_elig_in.ptr, h->d_rk_age.ptr,
                                                  h->d_rk_ttl.ptr, in->node_cost ? h->d_rk_cost_in.ptr : nullptr, h->d_rk_cost.ptr, h->d_rk_elig.ptr);
  rank_position_kernel<<<blocks, 256, 0, h->stream>>>(N, h->d_rk_cost.ptr, h->d_rk_elig.ptr, h->d_rk_order.ptr, h->d_rk_cost_out.ptr, h->d_rk_n.ptr);
  CUDA_TRY(h, cudaGetLastError());
  int32_t n = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&n, h->d_rk_n.ptr, 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (n > 0) {
    CUDA_TRY(h, cudaMemcpyAsync(order, h->d_rk_order.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(cost, h->d_rk_cost_out.ptr, (size_t)n * 8, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  *n_candidates = n;
  return KSCHED_OK;
}

int ksched_get_timings(const ksched_handle* h, ksched_timings* out) {
  if (!h || !out) return KSCHED_ERR_INVALID;
  *out = h->tm;
  return KSCHED_OK;
}

}  // extern "C"
