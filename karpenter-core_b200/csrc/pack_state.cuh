// pack_state.cuh - the pack kernel's parameters (PackState / K2Params): one layout shared by every parameter slot.
// Part of the single translation unit ksched.cu (included inside its anonymous namespace, after catalog.cuh and
// feasibility_kernel.cuh); not a standalone header.
#pragma once

// ------------------------------------------------------------------------------------------------
// K2: pack
// ------------------------------------------------------------------------------------------------
// One (class, group) relation with the group's immutable fields folded in (built at upload): everything
// Topology.Record and the per-step topology build need about the relation arrives with ONE load.
struct RelX {
  uint32_t group, flags;
  uint8_t key, type, has_filter, pad;
  int32_t max_skew;
  int32_t host_row;
  uint32_t pad2[3];
};
static_assert(sizeof(RelX) == 32, "RelX is loaded as two 16-byte vectors");

// a class run's fresh-node variant (pack_kernel.cuh: vt_build_entry), sized by pack_kernel.cuh's constants of the same names
constexpr int kHotRes = 4;
constexpr int kRunMask = 2;
constexpr int kRunW32 = 64;
struct RunVariant {
  uint32_t opts[kRunW32];
  uint64_t vals[KSCHED_MAX_KEYS];
  uint64_t meta;
  long long q[KSCHED_MAX_RES];
  long long b1[kHotRes], b2[kHotRes];
  uint32_t qp;
  uint32_t rp;            // room of the fresh node for further pods of the class (+ dead flag)
  unsigned short fl;      // HotSmem::flags of the fresh node (front bits, request keys, template)
  uint8_t dom[kRunMask];  // domain each spread relation pinned
};

// a class run's relation tables for one class (pack_kernel.cuh: run_rec_build): what class_run's entry needs of the class's
// topology relations that depends on the class and the catalog alone, built before the pack kernel. 128 bytes, one word
// per lane: a warp copies it with one coalesced load.
constexpr int kRunHost = 4;
struct alignas(16) RunRec {
  int32_t ok;                 // the class's relations pass the run's static checks (the group state is checked at entry)
  int32_t n_host, n_mask;
  int32_t h_row[kRunHost], h_group[kRunHost], h_lim[kRunHost];  // h_lim: largest count of the group on a node that still admits the pod
  int32_t m_group[kRunMask], m_skew[kRunMask];
  uint32_t m_neutral[kRunMask], m_tallow[kRunMask], m_dict[kRunMask];  // m_dict: the key's dictionary mask
  uint8_t h_times[kRunHost];
  uint8_t m_key[kRunMask], m_self[kRunMask], m_rec[kRunMask], m_wk[kRunMask];
  uint32_t pad[4];
};
static_assert(sizeof(RunRec) == 128 && offsetof(RunRec, h_times) == 100 && offsetof(RunRec, pad) == 112,
              "RunRec is one word per lane (and karpenter-core_b200/__init__.py: ResidentSolve.RUN_REC_DTYPE)");

struct PackState {
  const RelX* relx;                  // [n_class_topo], parallel to class_topo
  // problem (read-only)
  const ksched_pod_row* classes;
  const ksched_topo_group* groups;
  const ksched_class_topo* class_topo;
  const ksched_reqset* filter_terms;
  const uint32_t* itype_sets;        // [n][W32]
  const uint8_t* itype_complement;
  const int32_t* hostname_reqs;      // [n][2]
  const uint64_t* hostname_slots;    // [n][hostname_words] admitted existing slots of table entries (ksched.h), or nullptr
  const uint32_t* filter_hostname;   // [n_filter_terms] hostname part of a filter term (hostname_reqs entry), or nullptr
  int hostname_words;
  const uint32_t* order;             // FFD order: queue position -> pod
  const uint64_t* rows;              // [n_pods][32] dense pod-row matrix in FFD order (K0)
  uint32_t* pod_pos;                 // pod -> FFD position (row of F / best)
  int use_F;                         // F / best cover every column on this device (not column-sharded)
  const uint32_t* F;                 // [n_pods][V][W32] in FFD order (nullptr: compute fresh-node types dynamically)
  const unsigned long long* best;    // [n_pods] FFD order (after allreduce when sharded) or nullptr
  int n_pods, n_classes, n_existing, n_groups, max_new;
  long long min_req[KSCHED_MAX_RES]; // min over all classes of requests[r] (0 if some class lacks r)
  // mutable
  uint32_t* pod_class;               // [n_pods] current class
  int32_t* relax_level;              // [n_pods]
  int32_t* assign;                   // [n_pods]
  int32_t* place_seq;                // [n_pods]
  uint32_t* queue;                   // [n_pods+1] circular
  int32_t* last_len;                 // [n_pods]
  uint32_t* last_epoch;              // [n_pods]
  // existing nodes (SoA)
  int64_t* ex_req;                   // [8][n_existing]
  const int64_t* ex_avail;           // [8][n_existing]
  uint32_t* ex_req_present;
  const uint32_t* ex_avail_present;
  uint64_t* ex_vals;                 // [16][n_existing]
  uint64_t* ex_meta;
  const uint32_t* ex_taintset;
  const uint32_t* ex_itype;
  uint64_t* ex_hp;
  uint8_t* ex_closed;
  int32_t* cls_cursor;                  // [n_classes] existing nodes below it refuse the class for good (pack_kernel.cuh, generic step 1)
  const ksched_class_volumes* cls_vol;  // [n_classes] or nullptr: CSI volume limits (ksched.h)
  const uint8_t* cls_has_vol;           // [n_classes] 1: the class mounts a claim (row or claim table), nullptr with cls_vol
  ksched_node_volumes* ex_vol;          // [n_existing]
  uint64_t vol_mask[KSCHED_MAX_VOLUME_DRIVERS];
  // new nodes (SoA, capacity max_new)
  uint8_t* nn_tmpl;
  int32_t* nn_count;
  int32_t* nn_tb;
  int64_t* nn_req;                   // [8][max_new]
  uint32_t* nn_req_present;
  uint64_t* nn_vals;                 // [16][max_new]
  uint64_t* nn_meta;
  uint32_t* nn_opts;                 // [W32][max_new]
  uint64_t* nn_hp;
  // hot state of open nodes beyond the shared-memory window (pack_kernel.cuh: Hot)
  unsigned long long* ov_key;
  long long* ov_q;
  long long* ov_bound;
  long long* ov_bound2;
  int* ov_node;
  unsigned short* ov_flags;
  unsigned* ov_absorbed;
  unsigned* ov_rejected;
  // fresh-node outcome memo per (class, template)
  uint8_t* fc_state;                 // 0 unknown, 1 cached, 2 cached: no surviving type
  uint32_t* fc_opts;                 // [n_classes*V][W32]
  long long* fc_bound;               // [n_classes*V][4]
  long long* fc_bound2;
  uint8_t* fc_dom;
  uint8_t* fc_front_state;           // fc_bound / fc_bound2 / fc_dom hold the front of the K1-row option set
  uint64_t* fc_vals;                 // [n_classes*V][16] requirement masks of the fresh node
  uint64_t* fc_meta;
  long long* fc_q;                   // [n_classes*V][8] requests (daemon overhead + pod)
  uint32_t* fc_qp;
  // fresh-node outcome memo for topology-constrained classes: a hash table keyed by (class, template, the new node's
  // requirement masks) -- the option set of NewNode+Add is a function of exactly those (node.go:62-107) when the
  // provisioner has no limits. Direct mapped, full tag compare, so a collision only costs a recomputation.
  int fd_cap;                        // power of two
  uint8_t* fd_state;                 // 0 empty, 1 options cached, 2 cached: no surviving type
  uint32_t* fd_fc;                   // tag: class * V + template
  uint64_t* fd_meta;                 // tag
  uint64_t* fd_vals;                 // tag [fd_cap][16]
  uint32_t* fd_opts;                 // [fd_cap][W32]
  long long* fd_bound;               // [fd_cap][4]
  long long* fd_bound2;
  uint8_t* fd_dom;
  int stop_new_nodes;                // > 0: stop once this many new nodes are open (consolidation simulations, cluster.cuh)
  int count_visited;                 // keep the exact nodes_visited statistic (costs a pass over all in-flight nodes per pod)
  int alloc_in_smem;
  int run_off;                       // byte offset (after HotSmem) of the class-run loop's per-node arrays in dynamic shared memory
  int any_limits;                    // some template has active provisioner limits (fresh nodes are then never replayed from a variant)
  // Mode switches, read from the environment per Solve: the tests turn each step off to compare it with the generic step.
  int use_class_run;                 // class-run loop (KSCHED_NO_CLASSRUN=1: off)
  int use_level_run;                 // class_run: level / fill steps for classes without mask-key spread (KSCHED_NO_LEVELRUN=1: off)
  int use_level_warp;                // class_run: the level / fill steps on one warp while at most 32 nodes are open (KSCHED_NO_LEVELWARP=1: off)
  int use_mask_run;                  // class_run: list-driven loop on warp 0 for one mask-key spread relation (KSCHED_NO_MASKRUN=1: off)
  int use_run_derive;                // class_run: a fresh node's missing variant derived inside the run (KSCHED_NO_RUNDERIVE=1: off)
  int use_round_stretch;             // mask run: several rounds of a zone spread in one step (KSCHED_NO_ROUNDSTRETCH=1: off)
  int use_fill_stretch;              // mask run: rounds that keep the same head per zone in one step (KSCHED_NO_FILLSTRETCH=1 or
                                     // KSCHED_NO_ROUNDSTRETCH=1: off)
  RunVariant* vtable;                // [classes][kM1Dom] fresh-node variants of the class runs (pack_kernel.cuh: vt_build_entry)
  uint32_t* vt_ok;                   // [vt_classes][kM1Dom] 1: the entry holds a variant
  int vt_classes;                    // classes the table covers in this launch (0: no table; KSCHED_NO_VARSTORE=1 turns it off)
  int vt_ndom;                       // domain ids the table covers (below kM1Dom; the build has vt_classes * vt_ndom blocks)
  RunRec* run_rec;                   // [n_classes] class runs' relation tables (pack_kernel.cuh: run_rec_build)
  int rec_classes;                   // classes the row gather's launch builds records for: n_classes when class runs can run, else 0
  // topology counters
  int32_t* grp_cnt;                  // [n_groups][64]
  uint64_t* grp_registered;          // [n_groups]
  uint16_t* grp_host;                // [n_hostgroups][n_existing+max_new]
  const int32_t* grp_host_row;       // [n_groups] row in grp_host or -1
  int32_t* grp_host_total;           // [n_groups] schedulable-slot domains with count > 0 (+ extra_nonzero_domains)
  uint8_t* grp_active;               // [n_groups] 0 while a relaxation-created group does not exist yet (topology.go:86-117)
  int32_t* grp_min_slot;             // [n_groups] hostname slots below this were never Register()ed with the group
  int64_t* remaining;                // [V][8] provisioner limits
  // outputs and profile, indexed by Counter (ksched.cu)
  long long* counters;
  // taint sets from id 64 on, existing nodes only (ksched.h: class_tolerated_ext)
  const uint64_t* cls_tol_ext;       // [n_classes][tol_ext_words], or nullptr
  int tol_ext_words;
  // ext resources (ksched.h: ksched_catalog.n_res_ext; DESIGN.md §3), all nullptr without them
  const int64_t* cls_req_ext;        // [n_classes][n_res_ext]
  const uint32_t* cls_ext_present;   // [n_classes]
  const int64_t* ex_avail_ext;       // [n_res_ext][n_existing]
  int64_t* ex_req_ext;               // [n_res_ext][n_existing] what the batch's pods placed there request
  int64_t* nn_req_ext;               // [max_new][n_res_ext]
  uint32_t* nn_ext_present;          // [max_new]
  // host-port entries from id 64 on (ksched.h: class_hostport_conflicts_ext), all nullptr without them
  const uint64_t* cls_hpc_ext;       // [n_classes][hp_ext_words] conflicts
  const uint64_t* cls_hpe_ext;       // [n_classes][hp_ext_words] entries
  const uint8_t* cls_hp_ext;         // [n_classes] 1: the class has a word of either table that is not 0
  uint64_t* ex_hp_ext;               // [hp_ext_words][n_existing]
  uint64_t* nn_hp_ext;               // [hp_ext_words][max_new]
  int hp_ext_words;
  // tracked volume claims from id 64 on (ksched.h: class_volumes_shared_ext), all nullptr without them
  const uint64_t* cls_vol_ext;       // [n_classes][vol_ext_words]
  const uint64_t* vol_mask_ext;      // [KSCHED_MAX_VOLUME_DRIVERS][vol_ext_words]
  uint64_t* ex_vol_ext;              // [vol_ext_words][n_existing]
  int vol_ext_words;
  // instance-type filter tables (ksched.h: filter_term_itype), all nullptr when no filter term names the key. Each slot's
  // requirement on the key is a row [1 + W32]: word 0 the kIt* flags, then the admitted catalog types (itype_state_add).
  const uint32_t* filter_itype;      // [n_filter_terms] itype_req entry or KSCHED_NONE
  const uint32_t* tmpl_itype;        // [n_templates] itype_req entry a new node starts from, or KSCHED_NONE
  uint32_t* ex_it;                   // [n_existing][1 + W32]
  uint32_t* nn_it;                   // [max_new][1 + W32]
};
// flags of a slot's instance-type row: the node has the key; its complement bit (it admits every name outside the catalog,
// which no requirement names); it admits its own label, a name outside the catalog (an existing node's, KSCHED_ITYPE_UNLISTED)
constexpr uint32_t kItPresent = 1, kItComp = 2, kItOwn = 4;

struct K2Params {
  DevCatalog cat;
  PackState st;
};

__device__ __forceinline__ Req load_soa(const uint64_t* vals, uint64_t meta, int stride, int idx, int k) {
  Req r;
  r.present = (meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1;
  r.complement = (meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1;
  r.has_gt = r.has_lt = false;
  r.gt = r.lt = 0;
  r.values = r.present ? vals[(size_t)k * stride + idx] : 0;
  return r;
}
// load_soa from a value loaded without waiting for meta (vals[k * stride + idx] whatever meta says): the value load need
// not follow the meta load
__device__ __forceinline__ Req soa_req(uint64_t value, uint64_t meta, int k) {
  Req r;
  r.present = (meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1;
  r.complement = (meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1;
  r.has_gt = r.has_lt = false;
  r.gt = r.lt = 0;
  r.values = r.present ? value : 0;
  return r;
}

// 64-bit min over a warp with two 32-bit REDUX operations (hi word first, then lo word among the hi-minimal lanes)
__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
  const unsigned hi = (unsigned)(v >> 32), lo = (unsigned)v;
  const unsigned mhi = __reduce_min_sync(0xffffffffu, hi);
  const unsigned mlo = __reduce_min_sync(0xffffffffu, hi == mhi ? lo : 0xffffffffu);
  return ((unsigned long long)mhi << 32) | mlo;
}
