// cluster.cuh - device-resident cluster snapshot for the consolidation simulator (ksched_load_cluster / ksched_simulate_batch).
// Part of the single translation unit ksched.cu (included after pack_kernel.cuh); not a standalone header.
//
// One consolidation pass simulates many candidate sets against the same cluster (deprovisioning/helpers.go:42-115 is
// re-entered ~13 times by the multi-node binary search and up to once per node by single-node consolidation). The cluster is
// uploaded ONCE as a superset problem - every owned node an existing node with all its pods bound, every reschedulable pod of
// every candidate a pod row - and a simulation only says which existing slots are removed: their pods become the batch, the
// slots are closed, provisioner limits get the removed capacity back. Nothing is re-encoded or re-uploaded per simulation.
#pragma once

// in_set[e] = 1 for the removed existing slots of this simulation
__global__ void cluster_mark_kernel(const int32_t* __restrict__ nodes, int n, uint8_t* __restrict__ in_set, uint8_t* __restrict__ ex_closed) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { in_set[nodes[i]] = 1; ex_closed[nodes[i]] = 1; }
}

// The batch of one simulation: pending pods (pod_node < 0) and the pods bound to a removed slot, compacted in superset order.
// Superset pods are stored node by node, so the compaction is a gather over per-pod destination offsets computed on the host
// from the per-node pod ranges (dst[i] = -1: not in the batch).
__global__ void cluster_select_kernel(int n_sup, const int32_t* __restrict__ pod_node, const uint8_t* __restrict__ in_set,
                                      const int32_t* __restrict__ node_dst,  // [n_existing] first batch position of the node's pods in this simulation
                                      const int32_t* __restrict__ node_first, // [n_existing] first superset pod of the node
                                      int n_pending,                          // pending pods come first, in superset order
                                      const uint32_t* __restrict__ sup_class, const int64_t* __restrict__ sup_ts, const uint32_t* __restrict__ sup_uid,
                                      uint32_t* __restrict__ out_class, int64_t* __restrict__ out_ts, uint32_t* __restrict__ out_uid, int32_t* __restrict__ out_src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_sup) return;
  const int nd = pod_node[i];
  int dst;
  if (nd < 0) dst = i;  // pending pods are the first n_pending superset pods
  else if (in_set[nd]) dst = node_dst[nd] + (i - node_first[nd]);
  else return;
  (void)n_pending;
  out_class[dst] = sup_class[i];
  out_ts[dst] = sup_ts[i];
  out_uid[dst] = sup_uid[i];
  out_src[dst] = i;
}

// Topology counters of one simulation = the superset's (no batch pod counted) + every candidate pod that STAYS on its node:
// countDomains (topology.go:231-276) for the groups that count its class, and the inverse anti-affinity groups it owns
// (topology.go:183-227). One thread per superset pod; the counters are plain integers, so the adds commute.
__global__ void cluster_topology_kernel(int n_sup, const int32_t* __restrict__ pod_node, const uint8_t* __restrict__ in_set,
                                        const uint32_t* __restrict__ sup_class, const uint32_t* __restrict__ cc_begin,
                                        const ksched_count_rel* __restrict__ cc, const ksched_topo_group* __restrict__ groups,
                                        const int8_t* __restrict__ node_dom, const uint8_t* __restrict__ node_hostlabel,
                                        const uint32_t* __restrict__ filt, int filt_words, int n_existing, int hstride,
                                        const int32_t* __restrict__ host_row, int32_t* grp_cnt, unsigned long long* grp_registered, uint16_t* grp_host,
                                        int32_t* grp_host_total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_sup) return;
  const int e = pod_node[i];
  if (e < 0 || in_set[e]) return;  // pending, or part of this simulation's batch
  const uint32_t cls = sup_class[i];
  for (uint32_t q = cc_begin[cls]; q < cc_begin[cls + 1]; ++q) {
    const ksched_count_rel r = cc[q];
    const ksched_topo_group G = groups[r.group];
    if (r.kind == KSCHED_COUNT_DOMAINS && G.filter_begin != G.filter_end &&
        !((filt[(size_t)r.group * filt_words + (e >> 5)] >> (e & 31)) & 1)) continue;      // TopologyNodeFilter.Matches(node)
    if (G.key == KSCHED_KEY_HOSTNAME) {
      if (r.kind == KSCHED_COUNT_INVERSE && !node_hostlabel[e]) continue;                 // node.Labels[key] must exist (topology.go:215)
      const size_t idx = (size_t)host_row[r.group] * hstride + e;
      unsigned* word = reinterpret_cast<unsigned*>(grp_host) + (idx >> 1);
      const int shift = (int)(idx & 1) * 16;
      const unsigned old = atomicAdd(word, (unsigned)r.times << shift);
      if (((old >> shift) & 0xFFFFu) == 0) atomicAdd(&grp_host_total[r.group], 1);
    } else {
      const int d = node_dom[(size_t)G.key * n_existing + e];
      if (d < 0) continue;
      atomicAdd(&grp_cnt[(size_t)r.group * 64 + d], (int)r.times);
      atomicOr(&grp_registered[r.group], 1ull << d);
    }
  }
}

// New node n's row and its W32 option words, gathered from the pack kernel's columns (PackState nn_*) by the threads
// t = 0 .. nt-1 of a group together
__device__ __forceinline__ void gather_new_node(const PackState& s, int W32, int n, int t, int nt, ksched_new_node* row, uint32_t* opts) {
  const size_t mn = (size_t)s.max_new;
  if (t == 0) {
    const int32_t tmpl = s.nn_tmpl[n], count = s.nn_count[n];
    const uint32_t present = s.nn_req_present[n];
    const uint64_t meta = s.nn_meta[n];
    row->template_index = tmpl;
    row->pod_count = count;
    row->requests_present = present;
    row->pad = 0;
    row->reqs.meta = meta;
  }
  for (int r = t; r < KSCHED_MAX_RES; r += nt) row->requests[r] = s.nn_req[r * mn + n];
  for (int k = t; k < KSCHED_MAX_KEYS; k += nt) row->reqs.values[k] = s.nn_vals[k * mn + n];
  for (int w = t; w < W32; w += nt) opts[w] = s.nn_opts[w * mn + n];
}

// What computeConsolidation reads of a simulation (consolidation.go:190-274): how many pods landed, how many nodes were
// opened and, for the price guards, the first new node in full with its option words (W32 / 2 64-bit words), zeros when
// no node was opened. One warp.
__global__ void cluster_collect_kernel(PackState s, int W32, int n_pods, ksched_sim_result* out, uint64_t* node0_types) {
  const int t = threadIdx.x;
  const int n_new = (int)s.counters[kCtrNewNodes];
  uint32_t* opts = reinterpret_cast<uint32_t*>(node0_types);
  if (t == 0) {
    out->n_pods = n_pods;
    out->n_unscheduled = (int32_t)s.counters[kCtrUnscheduled];
    out->n_new_nodes = n_new;
    out->error = (int32_t)s.counters[kCtrError];
  }
  if (n_new >= 1) {
    gather_new_node(s, W32, 0, t, blockDim.x, &out->node0, opts);
    return;
  }
  if (t == 0) out->node0 = ksched_new_node{};
  for (int w = t; w < W32; w += blockDim.x) opts[w] = 0;
}

// The scalars of one full simulation (ksched_simulate_full), copied out with its arrays.
struct SimFullDev {
  long long nodes_visited, add_calls;
  int32_t n_new_nodes, n_unscheduled, error, all_pods_scheduled, uninitialized_existing, pad;
};
// The arrays of one result on the device, laid out as the caller's ksched_result so that each copies out in one piece
// (copy_out): where the collect kernels write, or the pack kernel's own per-pod arrays.
struct ResultArrays {
  int32_t *assign, *relax, *seq;
  ksched_new_node* nodes;
  uint64_t* types;                 // [nodes][W64]
  int64_t* ext;                    // [nodes][X]
  uint32_t* ext_present;           // [nodes]
  ksched_launch_choice* launch;    // [nodes]
  // the same arrays from pod o and new node o on
  ResultArrays at(size_t o, int W64, int X) const {
    return {assign + o, relax + o, seq + o, nodes + o, types + o * W64, ext + o * X, ext_present + o, launch + o};
  }
};

// New node n's row, option words and, with ext resources (X > 0), its ext requests and ext-present word, into row n of
// `out`: the 32 lanes of one warp.
__device__ __forceinline__ void collect_new_node(const PackState& s, int W32, int X, int n, int lane, const ResultArrays& out) {
  gather_new_node(s, W32, n, lane, 32, out.nodes + n, reinterpret_cast<uint32_t*>(out.types + (size_t)n * (W32 / 2)));  // W32 is even
  for (int x = lane; x < X; x += 32) out.ext[(size_t)n * X + x] = s.nn_req_ext[(size_t)n * X + x];
  if (X && lane == 0) out.ext_present[n] = s.nn_ext_present[n];
}

// A Solve's new nodes 0 .. n_new-1 (one warp per node) and, when `ex_rows` is given, the existing nodes' final
// requirements as rows (one thread per node).
__global__ void solve_collect_kernel(PackState s, int W32, int X, int n_new, ResultArrays out, ksched_reqset* ex_rows) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  for (int n = tid >> 5; n < n_new; n += nth >> 5) collect_new_node(s, W32, X, n, threadIdx.x & 31, out);
  if (!ex_rows) return;
  const int NE = s.n_existing;
  for (int e = tid; e < NE; e += nth) {
    ksched_reqset r;
    for (int k = 0; k < KSCHED_MAX_KEYS; ++k) r.values[k] = s.ex_vals[(size_t)k * NE + e];
    r.meta = s.ex_meta[e];
    ex_rows[e] = r;
  }
}

// simulateScheduling's whole answer in the numbering of the problem encoded fresh for this set. The batch holds the
// pending pods (the first n_lead of them lead), then the removed nodes' pods in the set's order (cluster_select_kernel with
// the set's offsets): batch position b goes to pod b, b + n_removed_pods or b - n_pending + n_lead. slot_map[e] = the slot's
// index among the slots that stay, -1 for a removed one. The new nodes are gathered from the pack kernel's columns
// (PackState nn_*) into rows. One block per simulation, a few thousand pods and nodes: microseconds.
__global__ void cluster_full_collect_kernel(PackState s, int W32, int X, int n_pods, int n_pending, int n_lead, int n_removed_pods,
                                            const int32_t* __restrict__ slot_map, const uint8_t* __restrict__ initialized, int n_stay,
                                            ResultArrays out, SimFullDev* scalars) {
  __shared__ int uninit;
  const int tid = threadIdx.x, n_existing = s.n_existing;
  const int n_new = (int)s.counters[kCtrNewNodes];
  if (tid == 0) uninit = 0;
  __syncthreads();
  for (int b = tid; b < n_pods; b += blockDim.x) {
    const int p = b < n_lead ? b : (b < n_pending ? b + n_removed_pods : b - n_pending + n_lead);
    const int a = s.assign[b], relax = s.relax_level[b], seq = s.place_seq[b];
    out.assign[p] = a < 0 ? -1 : (a < n_existing ? slot_map[a] : n_stay + (a - n_existing));
    out.relax[p] = relax;
    out.seq[p] = seq;
  }
  for (int e = tid; e < n_existing; e += blockDim.x)
    if (slot_map[e] >= 0 && initialized && !initialized[e]) uninit = 1;  // helpers.go:104-110 walks every node that stays
  for (int n = tid >> 5; n < n_new; n += blockDim.x >> 5) collect_new_node(s, W32, X, n, tid & 31, out);
  __syncthreads();
  if (tid == 0) {
    SimFullDev d;
    d.nodes_visited = s.counters[kCtrNodesVisited];
    d.add_calls = s.counters[kCtrAddCalls];
    d.n_new_nodes = n_new;
    d.n_unscheduled = (int32_t)s.counters[kCtrUnscheduled];
    d.error = (int32_t)s.counters[kCtrError];
    d.all_pods_scheduled = d.n_unscheduled == 0 ? 1 : 0;
    d.uninitialized_existing = uninit;
    d.pad = 0;
    *scalars = d;
  }
}

// ------------------------------------------------------------------------------------------------
// Candidate ranking for deprovisioning (deprovisioning/helpers.go:125-165,275-287, consolidation.go:85-103)
// ------------------------------------------------------------------------------------------------
// disruptionCost of every node: the pods' eviction costs summed IN POD ORDER (float addition is not associative and the
// reference adds them in list order, helpers.go:159-165), times the node's remaining lifetime. One thread per node.
__global__ void rank_cost_kernel(int n_nodes, const int32_t* __restrict__ pod_off, const double* __restrict__ deletion_cost,
                                 const int32_t* __restrict__ priority, const uint8_t* __restrict__ pod_flags, const uint8_t* __restrict__ eligible_in,
                                 const double* __restrict__ age, const double* __restrict__ ttl, const double* __restrict__ cost_in,
                                 double* __restrict__ cost, uint8_t* __restrict__ eligible) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_nodes) return;
  bool ok = eligible_in[n] != 0;
  double c = 0.0;
  if (cost_in) {
    c = cost_in[n];
  } else {
    for (int p = pod_off[n]; p < pod_off[n + 1]; ++p) {
      const uint8_t f = pod_flags[p];
      double pc = 1.0;                                               // GetPodEvictionCost helpers.go:125-146
      if (f & 1) pc += deletion_cost[p] / 134217728.0;               // / math.Pow(2, 27)
      if (f & 2) pc += (double)priority[p] / 33554432.0;             // / math.Pow(2, 25)
      pc = pc < -10.0 ? -10.0 : (pc > 10.0 ? 10.0 : pc);
      c += pc;
      if (f & 4) ok = false;                                         // a PDB or do-not-evict blocks the node (helpers.go:339-366)
    }
    double remaining = 1.0;                                          // calculateLifetimeRemaining helpers.go:275-287
    if (ttl[n] >= 0.0) {
      const double r = (ttl[n] - age[n]) / ttl[n];
      remaining = r < 0.0 ? 0.0 : (r > 1.0 ? 1.0 : r);
    }
    c = c * remaining;
  }
  cost[n] = c;
  eligible[n] = ok ? 1 : 0;
}
// The disruption order's strict weak order (R8): a NaN cost sorts after every number and ties with another NaN.
__device__ __forceinline__ bool cost_before(double a, double b) { return !isnan(a) && (isnan(b) || a < b); }
// sort.Slice(nodes, disruptionCost <) as a rank computation: position of an eligible node = the number of eligible nodes with
// a smaller cost, or an equal cost and a smaller index (R4: stable, R8: NaN last). O(n^2) compares over shared-memory tiles -
// thousands of nodes, microseconds.
__global__ void rank_position_kernel(int n_nodes, const double* __restrict__ cost, const uint8_t* __restrict__ eligible, int32_t* __restrict__ order,
                                     double* __restrict__ cost_out, int32_t* __restrict__ n_out) {
  __shared__ double t_cost[256];
  __shared__ uint8_t t_ok[256];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool mine = i < n_nodes && eligible[i];
  const double ci = i < n_nodes ? cost[i] : 0.0;
  int rank = 0, total = 0;
  for (int base = 0; base < n_nodes; base += 256) {
    const int j = base + threadIdx.x;
    t_cost[threadIdx.x] = j < n_nodes ? cost[j] : 0.0;
    t_ok[threadIdx.x] = j < n_nodes ? eligible[j] : 0;
    __syncthreads();
    const int lim = min(256, n_nodes - base);
    for (int q = 0; q < lim; ++q) {
      if (!t_ok[q]) continue;
      ++total;
      const double cj = t_cost[q];
      if (cost_before(cj, ci) || (!cost_before(ci, cj) && base + q < i)) ++rank;
    }
    __syncthreads();
  }
  if (mine) { order[rank] = i; cost_out[rank] = ci; }
  if (i == 0) *n_out = total;
}
