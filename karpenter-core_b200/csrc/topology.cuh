// topology.cuh - pack-kernel state (PackState / K2Params) and the device side of Requirements / Topology / TopologyGroup.
// Part of the single translation unit ksched.cu (included inside its anonymous namespace, in this order: catalog.cuh,
// feasibility_kernel.cuh, topology.cuh, pack_kernel.cuh); not a standalone header.
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
  int use_varstore;                  // class_run: fresh-node variants shared by classes of one shape (KSCHED_NO_VARSTORE=1: off)
  int use_round_stretch;             // mask run: several rounds of a zone spread in one step (KSCHED_NO_ROUNDSTRETCH=1: off)
  int use_fill_stretch;              // mask run: rounds that keep the same head per zone in one step (KSCHED_NO_FILLSTRETCH=1 or
                                     // KSCHED_NO_ROUNDSTRETCH=1: off)
  struct VarStoreEntry* vstore;      // [kVarStore] (pack_kernel.cuh); valid entries: RunCtx::vs_n, reset per Solve
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
// The pack kernel and every out-of-line device function it calls read their parameters from constant memory with
// immediate offsets (a reference to a __grid_constant__ kernel parameter handed to a __noinline__ function degrades every
// field access to a generic load from the parameter window, on a code path that is one dependent chain).
// One copy per device: run_pack() orders launches of different handles on the same device behind each other.
__constant__ K2Params g_k2;
#define KS_K2 const DevCatalog& c = g_k2.cat; const PackState& s = g_k2.st; (void)c; (void)s;

struct Touched {
  int n;
  int8_t key[kMaxTouched];
  Req merged[kMaxTouched];  // node ∩ pod          (node.go:81)
  Req fin[kMaxTouched];     // ... ∩ topology      (node.go:90)
  bool changed[kMaxTouched];
};

struct PodTopo {  // per (pod step, constraining group): node-independent part of TopologyGroup.Get
  int n;
  int32_t group[kMaxCG];
  uint32_t flags[kMaxCG];
  int32_t min_count[kMaxCG];   // spread: domainMinCount over the pod's domains
  uint64_t options[kMaxCG];    // affinity / anti-affinity: admissible domains (mask keys)
  uint8_t bootstrap[kMaxCG];   // affinity: no domain has a matching pod and the pod selects itself
  uint64_t pod_allowed[kMaxCG]; // pod's own admissible domains for the key
  // the group's own fields, copied once per step so that the per-node checks read shared memory only
  uint8_t gkey[kMaxCG], gtype[kMaxCG];
  int32_t gskew[kMaxCG], host_row[kMaxCG], min_slot[kMaxCG];
  uint64_t registered[kMaxCG];
  // spread over a mask key: the registered domains within max-skew, in (count, domain id) order. The domain the
  // reference picks for a node is the first entry the node's requirement admits (topologygroup.go:157-183).
  uint8_t n_sorted[kMaxCG];
  uint8_t sorted[kMaxCG][64];
  uint64_t ok_mask[kMaxCG];    // the same domains as a set
  int overflow;
};

// Per-CTA working set of the pack kernel's generic step, at file scope so that every out-of-line function reaches it with
// immediate shared-memory addresses instead of pointers handed down the call chain.
__shared__ ksched_pod_row g_row;  // the pod of the current step (copied from its FFD row / class row by warp 0)
__shared__ PodTopo g_pt;          // its topology constraints
#define KS_ROW const ksched_pod_row& row = g_row; (void)row;
#define KS_PT PodTopo& pt = g_pt; (void)pt;

__device__ __forceinline__ Req load_soa(const uint64_t* vals, uint64_t meta, int stride, int idx, int k) {
  Req r;
  r.present = (meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1;
  r.complement = (meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1;
  r.has_gt = r.has_lt = false;
  r.gt = r.lt = 0;
  r.values = r.present ? vals[(size_t)k * stride + idx] : 0;
  return r;
}
__device__ __forceinline__ Req pod_req(const ksched_pod_row& row, int k) {
  Req r;
  r.present = (row.meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1;
  r.complement = (row.meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1;
  r.has_gt = r.has_lt = false;
  r.gt = r.lt = 0;
  r.values = row.values[k];
  return r;
}
__device__ __forceinline__ bool req_equal(const Req& a, const Req& b) {
  return a.present == b.present && a.complement == b.complement && a.values == b.values;
}

// TopologyGroup.Get for a mask-key group (topologygroup.go:88-243). node_dom = the node's requirement for the
// key after the pod's own requirements were merged (topology.go:156-159). Returns false when Len()==0.
__device__ __noinline__ bool topo_domains_mask(int j, const Req& node_dom, uint64_t* out) {
  KS_K2
  KS_PT
  const int k = pt.gkey[j];
  KeyMeta km = key_meta(c, k);
  const uint64_t registered = pt.registered[j];
  const uint64_t node_allowed = node_dom.present ? ksched::req_allowed(node_dom, c.keys[k].dict_mask, km) : c.keys[k].dict_mask;
  if (pt.gtype[j] == 0) {  // nextDomainTopologySpread: min (count, domain id) among the admissible domains of the node
    const int ns = pt.n_sorted[j];
    for (int i = 0; i < ns; ++i) {
      const int d = pt.sorted[j][i];
      if ((node_allowed >> d) & 1) { *out = 1ull << d; return true; }
    }
    return false;
  }
  if (pt.gtype[j] == 1) {  // nextDomainAffinity
    uint64_t opts = pt.options[j];
    if (pt.bootstrap[j]) {
      uint64_t inter = registered & pt.pod_allowed[j] & node_allowed;  // podDomains.Intersection(nodeDomains).Has
      if (inter) opts |= inter & (~inter + 1);
      uint64_t pm = registered & pt.pod_allowed[j];
      if (pm) opts |= pm & (~pm + 1);
    }
    if (!opts) return false;
    *out = opts;
    return true;
  }
  uint64_t opts = pt.options[j];  // nextDomainAntiAffinity
  if (!opts) return false;
  *out = opts;
  return true;
}

// hostname-key groups: the node's hostname domain is its slot.
__device__ __noinline__ bool topo_hostname_ok(int j, int slot, bool pod_allows_slot) {
  KS_K2
  KS_PT
  const int stride = s.n_existing + s.max_new;
  const int32_t cnt = s.grp_host[(size_t)pt.host_row[j] * stride + slot];
  // a group created by a later Topology.Update only knows hostnames registered after that, plus those it counted pods on
  if (slot < pt.min_slot[j] && !(slot < s.n_existing && cnt > 0)) return false;
  const int type = pt.gtype[j];
  if (type == 0) {  // spread, min is 0 for hostname (topologygroup.go:186-188); candidate = the node's own hostname
    int64_t c2 = (int64_t)cnt + ((pt.flags[j] & KSCHED_TOPO_SELECTS) ? 1 : 0);
    return c2 <= (int64_t)pt.gskew[j];
  }
  if (type == 1) {  // affinity
    if (cnt > 0 && pod_allows_slot) return true;
    if (pt.bootstrap[j]) return pod_allows_slot;  // first loop picks the node's own (registered) hostname
    return false;
  }
  return cnt == 0 && pod_allows_slot;  // anti-affinity
}

// Does hostname requirement `req` (an entry of hostname_reqs) admit this slot? The {complement, slot} pair, or a table entry:
// the existing slot's bit, and for a new node (a placeholder hostname) the entry's first word. The table read is out of line:
// the pair test is inlined at every caller, and the kernels' code size decides their speed (DESIGN.md §3).
__device__ __noinline__ bool hostname_table_allows(uint32_t req, int slot, bool is_existing) {
  KS_K2
  if (!is_existing) return s.hostname_reqs[req * 2] != 0;
  return ((s.hostname_slots[(size_t)req * s.hostname_words + (slot >> 6)] >> (slot & 63)) & 1) != 0;
}
__device__ __forceinline__ bool hostname_req_allows(const PackState& s, uint32_t req, int slot, bool is_existing) {
  const int32_t comp = s.hostname_reqs[req * 2], target = s.hostname_reqs[req * 2 + 1];
  if (target == KSCHED_HOSTNAME_TABLE) return hostname_table_allows(req, slot, is_existing);
  const bool same = is_existing && target == slot;
  return comp ? !same : same;
}
// Does the pod's hostname requirement admit this slot? (requirement on kubernetes.io/hostname, never well-known)
__device__ __forceinline__ bool hostname_allows(const PackState& s, const ksched_pod_row& row, int slot, bool is_existing) {
  return row.hostname_req == KSCHED_NONE || hostname_req_allows(s, row.hostname_req, slot, is_existing);
}

// nextDomainAffinity (topologygroup.go:202-231) of hostname group gi for a pod with hostname requirement `req`: does some
// hostname the requirement admits have a matching pod? Existing slots by their own counts; new nodes together, as the
// slots with a count that are neither existing nor extra domains (grp_host_total); extra domains (hostnames that are no slot)
// by the encoder's KSCHED_TOPO_HOST_EXTRA, since their counts never change.
__device__ __noinline__ bool hostname_affinity_options(int gi, int host_row, uint32_t req, uint32_t flags) {
  KS_K2
  if (flags & KSCHED_TOPO_HOST_EXTRA) return true;
  const int NE = s.n_existing;
  const uint16_t* cnt = s.grp_host + (size_t)host_row * (NE + s.max_new);
  int ex_nonzero = 0;
  for (int e = 0; e < NE; ++e) {
    if (!cnt[e]) continue;
    if (hostname_req_allows(s, req, e, true)) return true;
    ++ex_nonzero;
  }
  return s.grp_host_total[gi] - s.groups[gi].extra_nonzero_domains - ex_nonzero > 0 && hostname_req_allows(s, req, NE, false);
}

// Requirement phase of Node.Add / ExistingNode.Add: Compatible(pod) + merge, topology tighten + Compatible + merge.
// vals/meta/stride/idx describe the node's requirement set. Returns false on reject.
__device__ __noinline__ bool requirements_phase(const uint64_t* vals, uint64_t meta, int stride, int idx, int slot, bool is_existing, Touched& t) {
  KS_K2
  KS_ROW KS_PT
  t.n = 0;
  if (!hostname_allows(s, row, slot, is_existing)) return false;
  uint32_t podkeys = (uint32_t)(row.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF;
  while (podkeys) {
    int k = __ffs(podkeys) - 1;
    podkeys &= podkeys - 1;
    Req node = load_soa(vals, meta, stride, idx, k);
    Req pod = pod_req(row, k);
    KeyMeta km = key_meta(c, k);
    if (!ksched::key_compatible(node, pod, c.keys[k].well_known != 0, km)) return false;
    if (t.n >= kMaxTouched) return false;
    Req merged = ksched::key_add(node, pod, km);
    t.key[t.n] = (int8_t)k;
    t.merged[t.n] = merged;
    t.fin[t.n] = merged;
    t.changed[t.n] = !req_equal(merged, node);
    ++t.n;
  }
  for (int j = 0; j < pt.n; ++j) {
    if (pt.gkey[j] == KSCHED_KEY_HOSTNAME) {
      if (!topo_hostname_ok(j, slot, hostname_allows(s, row, slot, is_existing))) return false;
      continue;
    }
    const int k = pt.gkey[j];
    int ti = -1;
    for (int i = 0; i < t.n; ++i) if (t.key[i] == k) ti = i;
    if (ti < 0) {
      if (t.n >= kMaxTouched) return false;
      ti = t.n++;
      Req node = load_soa(vals, meta, stride, idx, k);
      t.key[ti] = (int8_t)k;
      t.merged[ti] = node;
      t.fin[ti] = node;
      t.changed[ti] = false;
    }
    uint64_t dom;
    if (!topo_domains_mask(j, t.merged[ti], &dom)) return false;
    Req d{dom, 0, 0, true, false, false, false};
    KeyMeta km = key_meta(c, k);
    t.fin[ti] = ksched::key_add(t.fin[ti], d, km);  // requirements.Add(domains) topology.go:164
  }
  // nodeRequirements.Compatible(topologyRequirements) node.go:87 — only topology keys can differ
  for (int i = 0; i < t.n; ++i) {
    if (req_equal(t.fin[i], t.merged[i])) continue;
    const int k = t.key[i];
    if (!ksched::key_compatible(t.merged[i], t.fin[i], c.keys[k].well_known != 0, key_meta(c, k))) return false;
    t.fin[i] = ksched::key_add(t.merged[i], t.fin[i], key_meta(c, k));
    t.changed[i] = true;
  }
  return true;
}

// Surviving instance types of a node for one word (filterInstanceTypesByRequirements node.go:137-141):
// previous options ∧ Fits ∧ (keys whose requirement changed) ∧ hasOffering (if zone / capacity-type changed).
struct TypeCtx {
  int rank[KSCHED_MAX_RES];
  uint32_t res_mask;
  int nkeys;
  int8_t key[KSCHED_MAX_KEYS];
  uint64_t allowed[KSCHED_MAX_KEYS];
  uint64_t slots;  // admitted offering slots (offer_word), when offer_needed and not offer_unconstrained
  bool neg[KSCHED_MAX_KEYS];
  bool offer_needed, offer_unconstrained;
  uint32_t itype_req;
};
__device__ __noinline__ void build_type_ctx(const Touched& t, const long long* q,
                               uint32_t q_present, const uint64_t* vals, uint64_t meta, int stride, int idx, bool fresh,
                               const int64_t* alloc_sorted, TypeCtx& x, bool with_ranks = true) {
  KS_K2
  KS_ROW
  x.res_mask = q_present;
  if (with_ranks)
    for (int r = 0; r < c.n_res; ++r) x.rank[r] = ((q_present >> r) & 1) ? fit_rank(alloc_sorted, c.n_types, r, q[r]) : 0;
  x.nkeys = 0;
  x.offer_needed = fresh;
  auto add_key = [&](int k, const Req& f) {
    if (!((c.type_relevant >> k) & 1) || !f.present) return;
    KeyMeta km = key_meta(c, k);
    x.key[x.nkeys] = (int8_t)k;
    x.allowed[x.nkeys] = ksched::req_allowed(f, c.keys[k].dict_mask, km);
    x.neg[x.nkeys] = ksched::req_op_negative(f, km);
    ++x.nkeys;
  };
  if (fresh) {
    // every key of the new node's requirement set is evaluated from scratch
    uint32_t done = 0;
    for (int i = 0; i < t.n; ++i) { add_key(t.key[i], t.fin[i]); done |= 1u << t.key[i]; }
    uint32_t rest = ((uint32_t)(meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF) & ~done;
    while (rest) {
      int k = __ffs(rest) - 1;
      rest &= rest - 1;
      add_key(k, load_soa(vals, meta, stride, idx, k));
    }
  } else {
    for (int i = 0; i < t.n; ++i) {
      if (!t.changed[i]) continue;
      add_key(t.key[i], t.fin[i]);
      if (t.key[i] == c.zone_key || t.key[i] == c.ct_key) x.offer_needed = true;
    }
  }
  x.slots = ~0ull; x.offer_unconstrained = true;
  if (x.offer_needed) {
    uint64_t zallowed = ~0ull, callowed = ~0ull;
    auto final_req = [&](int k) -> Req {
      for (int i = 0; i < t.n; ++i) if (t.key[i] == k) return t.fin[i];
      return load_soa(vals, meta, stride, idx, k);
    };
    if (c.zone_key >= 0) {
      Req z = final_req(c.zone_key);
      if (z.present) { zallowed = ksched::req_allowed(z, c.keys[c.zone_key].dict_mask, key_meta(c, c.zone_key)); x.offer_unconstrained = false; }
    }
    if (c.ct_key >= 0) {
      Req ct = final_req(c.ct_key);
      if (ct.present) { callowed = ksched::req_allowed(ct, c.keys[c.ct_key].dict_mask, key_meta(c, c.ct_key)); x.offer_unconstrained = false; }
    }
    if (!x.offer_unconstrained) x.slots = node_slots(c, zallowed, callowed);
  }
  x.itype_req = row.itype_req;
}
// resource part (Fits) and requirement part (keys / offerings / instance-type requirement) of the per-word filter
__device__ __forceinline__ uint32_t type_word_res(const DevCatalog& c, const TypeCtx& x, uint32_t sw, int w) {
  uint32_t rm = x.res_mask;
  while (sw && rm) {
    int r = __ffs(rm) - 1;
    rm &= rm - 1;
    sw &= c.fitset[((size_t)r * (c.n_types + 1) + x.rank[r]) * c.W32 + w];
  }
  return sw;
}
__device__ __forceinline__ uint32_t type_word_keys(const DevCatalog& c, const PackState& s, const TypeCtx& x, uint32_t sw, int w) {
  for (int i = 0; i < x.nkeys && sw; ++i) sw &= key_typeset_word(c, x.key[i], x.allowed[i], x.neg[i], w);
  if (sw && x.offer_needed) sw &= offer_word(c, x.slots, x.offer_unconstrained, w);
  if (sw && x.itype_req != KSCHED_NONE) sw &= s.itype_sets[(size_t)x.itype_req * c.W32 + w];
  return sw;
}
__device__ __forceinline__ uint32_t type_word(const DevCatalog& c, const PackState& s, const TypeCtx& x, uint32_t base, int w) {
  return type_word_keys(c, s, x, type_word_res(c, x, base, w), w);
}

// Node-independent part of the pod's topology constraints for this step, one constraining (class, group) relation j.
// Static half: what the relation and its group are (a function of the pod class only).
__device__ __forceinline__ void fill_pod_topo_static(const RelX& x, PodTopo& pt, int j) {
  pt.group[j] = (int)x.group;
  pt.flags[j] = x.flags;
  pt.gkey[j] = x.key;
  pt.gtype[j] = x.type;
  pt.gskew[j] = x.max_skew;
  pt.host_row[j] = x.host_row;
}
// Dynamic half: everything derived from the group's counters, re-read every step.
__device__ __noinline__ void fill_pod_topo_dynamic(int j) {
  KS_K2
  KS_ROW KS_PT
  const int gi = pt.group[j];
  const uint32_t flags = pt.flags[j];
  const int gkey = pt.gkey[j], gtype = pt.gtype[j], gskew = pt.gskew[j];
  pt.min_count[j] = 0;
  pt.options[j] = 0;
  pt.bootstrap[j] = 0;
  pt.pod_allowed[j] = 0;
  pt.min_slot[j] = s.grp_min_slot[gi];
  pt.registered[j] = 0;
  pt.n_sorted[j] = 0;
  pt.ok_mask[j] = 0;
  if (gkey == KSCHED_KEY_HOSTNAME) {
    if (gtype == 1) {  // options.Len()==0 <=> no hostname the pod's requirement admits has a matching pod
      const bool any = row.hostname_req == KSCHED_NONE ? s.grp_host_total[gi] != 0
                                                       : hostname_affinity_options(gi, pt.host_row[j], row.hostname_req, flags);
      pt.bootstrap[j] = !any && (flags & KSCHED_TOPO_SELECTS);
    }
    return;
  }
  const int k = gkey;
  KeyMeta km = key_meta(c, k);
  Req pd = pod_req(row, k);
  const uint64_t pod_allowed = pd.present ? ksched::req_allowed(pd, c.keys[k].dict_mask, km) : c.keys[k].dict_mask;
  pt.pod_allowed[j] = pod_allowed;
  const uint64_t registered = s.grp_registered[gi];
  pt.registered[j] = registered;
  uint64_t m = registered & pod_allowed;
  if (gtype == 0) {
    // counts of every registered domain, loaded once (independent loads), ids in ascending order
    int32_t cnts[64];
    uint8_t ids[64];
    int nd = 0;
    for (uint64_t all = registered; all; all &= all - 1) {
      const int d = __ffsll((long long)all) - 1;
      ids[nd] = (uint8_t)d;
      cnts[nd] = s.grp_cnt[(size_t)gi * 64 + d];
      ++nd;
    }
    int32_t mn = INT32_MAX;  // domainMinCount over the pod's own domains (topologygroup.go:186-203)
    for (int i = 0; i < nd; ++i)
      if (((m >> ids[i]) & 1) && cnts[i] < mn) mn = cnts[i];
    pt.min_count[j] = mn;
    // registered domains within the skew bound, insertion-sorted by (count, id)
    const int self = (flags & KSCHED_TOPO_SELECTS) ? 1 : 0;
    int ns = 0;
    int32_t sc[64];
    uint64_t okm = 0;
    for (int i = 0; i < nd; ++i) {
      const int64_t cnt = (int64_t)cnts[i] + self;
      if (cnt - (int64_t)mn > (int64_t)gskew) continue;
      okm |= 1ull << ids[i];
      int q = ns++;
      while (q > 0 && sc[q - 1] > (int32_t)cnt) { sc[q] = sc[q - 1]; pt.sorted[j][q] = pt.sorted[j][q - 1]; --q; }
      sc[q] = (int32_t)cnt;
      pt.sorted[j][q] = ids[i];
    }
    pt.n_sorted[j] = (uint8_t)ns;
    pt.ok_mask[j] = okm;
  } else if (gtype == 1) {
    uint64_t opts = 0;
    while (m) {
      int d = __ffsll((long long)m) - 1;
      m &= m - 1;
      if (s.grp_cnt[(size_t)gi * 64 + d] > 0) opts |= 1ull << d;
    }
    pt.options[j] = opts;
    pt.bootstrap[j] = (opts == 0) && (flags & KSCHED_TOPO_SELECTS);
  } else {
    uint64_t opts = 0;
    while (m) {
      int d = __ffsll((long long)m) - 1;
      m &= m - 1;
      if (s.grp_cnt[(size_t)gi * 64 + d] == 0) opts |= 1ull << d;
    }
    pt.options[j] = opts;
  }
}

// Called by the 32 lanes of warp 0: one (class, group) relation per lane, constraining ones compacted in order.
__device__ void build_pod_topo() {
  KS_K2
  KS_ROW KS_PT
  const int lane = threadIdx.x & 31;
  const uint32_t begin = row.topo_begin, end = row.topo_end;
  int n = 0, overflow = 0;
  for (uint32_t base = begin; base < end; base += 32) {  // uniform trip count
    const uint32_t e = base + lane;
    RelX x{};
    if (e < end) x = s.relx[e];
    const bool cons = e < end && (x.flags & KSCHED_TOPO_CONSTRAINS);
    const unsigned bal = __ballot_sync(0xffffffffu, cons);
    const int j = n + __popc(bal & ((1u << lane) - 1));
    if (cons && j < kMaxCG) {
      fill_pod_topo_static(x, pt, j);
      fill_pod_topo_dynamic(j);
    }
    n += __popc(bal);
    if (n > kMaxCG) { overflow = 1; n = kMaxCG; }
  }
  if (lane == 0) { pt.n = n; pt.overflow = overflow; }
}
// The previous step's pod had the same class: the relations are the same, only the counters moved.
__device__ void refresh_pod_topo() {
  KS_K2
  KS_ROW KS_PT
  const int lane = threadIdx.x & 31;
  if (lane < pt.n) fill_pod_topo_dynamic(lane);
}

// A NECESSARY condition of requirements_phase for an in-flight node, cheap enough to run on every candidate: the
// hostname groups exactly, spread groups over mask keys through the set of admissible domains. The node that wins the
// argmin is then checked in full (and excluded if it fails).
__device__ __forceinline__ bool topo_prefilter(const uint64_t* vals, uint64_t meta,
                                               int stride, int idx, int slot) {
  KS_K2
  KS_PT
  for (int j = 0; j < pt.n; ++j) {
    const int k = pt.gkey[j];
    if (k == KSCHED_KEY_HOSTNAME) {
      if (!topo_hostname_ok(j, slot, true)) return false;
      continue;
    }
    if (pt.gtype[j] != 0) {
      if (!pt.options[j] && !pt.bootstrap[j]) return false;
      continue;
    }
    const Req node = load_soa(vals, meta, stride, idx, k);
    const uint64_t node_allowed = node.present ? ksched::req_allowed(node, c.keys[k].dict_mask, key_meta(c, k)) : c.keys[k].dict_mask;
    if (!(node_allowed & pt.ok_mask[j])) return false;
  }
  return true;
}

// ---- instance-type requirement of a slot (PackState::ex_it / nn_it), kept only when a filter term names the key
__device__ __forceinline__ uint32_t* itype_row(const PackState& s, int W32, int slot) {
  const size_t IW = 1 + (size_t)W32;
  return slot < s.n_existing ? s.ex_it + (size_t)slot * IW : s.nn_it + (size_t)(slot - s.n_existing) * IW;
}
// Requirements.Add of itype_req entry `req` into the slot's requirement (ExistingNode.Add / Node.Add): the first one is
// taken as it is, later ones intersect. A name outside the catalog survives only a complement entry.
__device__ __noinline__ void itype_state_add(int slot, uint32_t req) {
  KS_K2
  uint32_t* r = itype_row(s, c.W32, slot);
  const bool comp = s.itype_complement[req] != 0;
  const uint32_t* set = s.itype_sets + (size_t)req * c.W32;
  const uint32_t f = r[0];
  r[0] = !(f & kItPresent) ? (kItPresent | (comp ? kItComp : 0u)) : (kItPresent | (comp ? (f & (kItComp | kItOwn)) : 0u));
  for (int w = 0; w < c.W32; ++w) r[1 + w] = (f & kItPresent) ? (r[1 + w] & set[w]) : set[w];
}
// New node n of template v starts from its template's requirement (NewMachineTemplate), or without the key; then its first
// pod's entry `req` (or KSCHED_NONE) is added
__device__ __noinline__ void itype_state_open(int n, int v, uint32_t req) {
  KS_K2
  uint32_t* r = s.nn_it + (size_t)n * (1 + c.W32);
  const uint32_t t = s.tmpl_itype[v];
  r[0] = t == KSCHED_NONE ? 0u : (kItPresent | (s.itype_complement[t] ? kItComp : 0u));
  if (t != KSCHED_NONE)
    for (int w = 0; w < c.W32; ++w) r[1 + w] = s.itype_sets[(size_t)t * c.W32 + w];
  if (req != KSCHED_NONE) itype_state_add(s.n_existing + n, req);
}
// Requirements.Intersects on the instance-type key (requirements.go:189-206) of the slot's requirement and filter term part
// `req`: a node without the key passes; otherwise the intersection is not empty, or both operators are NotIn / DoesNotExist.
// Out of line, like hostname_table_allows: problems without the tables do not carry its code in filter_matches.
__device__ __noinline__ bool itype_filter_allows(int slot, uint32_t req) {
  KS_K2
  const uint32_t* r = itype_row(s, c.W32, slot);
  const uint32_t f = r[0];
  if (!(f & kItPresent)) return true;
  const bool tcomp = s.itype_complement[req] != 0;
  if (tcomp && (f & (kItComp | kItOwn))) return true;  // a name outside the catalog that both admit
  const uint32_t* set = s.itype_sets + (size_t)req * c.W32;
  int nn = 0, nt = 0;
  for (int w = 0; w < c.W32; ++w) {
    if (r[1 + w] & set[w]) return true;
    nn += __popc(r[1 + w]);
    nt += __popc(set[w]);
  }
  // Operator(): a complement is NotIn while it excludes a type, Exists otherwise; else In while it admits a name,
  // DoesNotExist otherwise
  const bool node_neg = (f & kItComp) ? nn < c.n_types : (nn == 0 && !(f & kItOwn));
  const bool term_neg = tcomp ? nt < c.n_types : nt == 0;
  return node_neg && term_neg;
}

// TopologyNodeFilter.MatchesRequirements (topologynodefilter.go:57-70): any term Compatible with the node requirements. A
// term's hostname part reads the node's hostname: the slot's bit for an existing node, the placeholder flag for a new one;
// its instance-type part the slot's instance-type requirement.
__device__ __noinline__ bool filter_matches(const ksched_topo_group& g, const uint64_t* vals, uint64_t meta,
                               int stride, int idx, int slot) {
  KS_K2
  if (g.filter_begin == g.filter_end) return true;
  for (uint32_t f = g.filter_begin; f < g.filter_end; ++f) {
    const ksched_reqset& term = s.filter_terms[f];
    const uint32_t host = s.filter_hostname ? s.filter_hostname[f] : KSCHED_NONE;
    bool ok = host == KSCHED_NONE || hostname_req_allows(s, host, slot, slot < s.n_existing);
    const uint32_t it = s.filter_itype ? s.filter_itype[f] : KSCHED_NONE;
    if (ok && it != KSCHED_NONE) ok = itype_filter_allows(slot, it);
    uint32_t keys = (uint32_t)(term.meta >> KSCHED_META_PRESENT_SHIFT) & 0xFFFF;
    while (keys && ok) {
      int k = __ffs(keys) - 1;
      keys &= keys - 1;
      Req node = load_soa(vals, meta, stride, idx, k);
      Req inc = ksched::req_load(term, nullptr, k);
      ok = ksched::key_compatible(node, inc, c.keys[k].well_known != 0, key_meta(c, k));
    }
    if (ok) return true;
  }
  return false;
}

// Topology.Record (topology.go:120-143) for ONE (class, group) relation, after the node's requirements were committed.
// Relations of one class name distinct groups, so different threads may record different relations concurrently.
__device__ __noinline__ void topo_record_entry(uint32_t e, const uint64_t* vals, uint64_t meta, int stride, int idx, int slot) {
  KS_K2
  const int hstride = s.n_existing + s.max_new;
  const RelX x = s.relx[e];
  const int gi = (int)x.group;
  if (!(x.flags & (KSCHED_TOPO_RECORDS | KSCHED_TOPO_RECORDS_INVERSE))) return;
  // the loads the record needs are issued together (one memory round trip, not three)
  const uint8_t active = s.grp_active[gi];
  uint16_t* const host_cell = x.key == KSCHED_KEY_HOSTNAME ? &s.grp_host[(size_t)x.host_row * hstride + slot] : nullptr;
  const uint32_t host_old = host_cell ? *host_cell : 0;
  const int32_t host_total = host_cell ? s.grp_host_total[gi] : 0;
  if (!active) return;  // the group does not exist yet
  bool rec = false, all_values = false;
  if (x.flags & KSCHED_TOPO_RECORDS) {
    if (!x.has_filter || filter_matches(s.groups[gi], vals, meta, stride, idx, slot)) { rec = true; all_values = (x.type == 2); }
  }
  const bool rec_inv = (x.flags & KSCHED_TOPO_RECORDS_INVERSE) != 0;
  if (x.key == KSCHED_KEY_HOSTNAME) {  // the node's hostname requirement is always In [its own hostname]
    const int times = (rec ? 1 : 0) + (rec_inv ? 1 : 0);
    if (!times) return;
    if (host_old == 0) s.grp_host_total[gi] = host_total + 1;
    const uint32_t now = host_old + times;
    *host_cell = (uint16_t)(now > 0xFFFF ? 0xFFFF : now);
    return;
  }
  for (int pass = 0; pass < 2; ++pass) {
    const bool doit = pass == 0 ? rec : rec_inv;
    const bool allv = pass == 0 ? all_values : true;
    if (!doit) continue;
    Req r = load_soa(vals, meta, stride, idx, x.key);
    uint64_t v = 0;
    if (allv) v = r.present ? (r.complement ? ksched::req_excluded(r, key_meta(c, x.key)) : r.values) : 0;  // domains.Values(): members, or the excluded set of a complement
    else if (r.present && ksched::req_len_one(r)) v = r.values;
    while (v) {
      int d = __ffsll((long long)v) - 1;
      v &= v - 1;
      s.grp_cnt[(size_t)gi * 64 + d]++;
      s.grp_registered[gi] |= 1ull << d;
    }
  }
}
// every thread of the CTA: relation tid, tid + blockDim, ... (the commit this records must be visible: call after a barrier)
__device__ __forceinline__ void topo_record_block(const uint64_t* vals, uint64_t meta,
                                                  int stride, int idx, int slot) {
  KS_K2
  KS_ROW
  for (uint32_t e = row.topo_begin + threadIdx.x; e < row.topo_end; e += blockDim.x) topo_record_entry(e, vals, meta, stride, idx, slot);
}

