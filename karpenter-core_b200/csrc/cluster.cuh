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

// What computeConsolidation reads of a simulation (consolidation.go:190-274): how many pods landed, how many nodes were
// opened and, for the price guards, the first new node in full.
struct SimResultDev {
  int32_t n_pods, n_unscheduled, n_new_nodes, error;
  int32_t template_index, pod_count;
  uint32_t requests_present, pad;
  int64_t requests[KSCHED_MAX_RES];
  uint64_t values[KSCHED_MAX_KEYS];
  uint64_t meta;
};
__global__ void cluster_collect_kernel(const long long* __restrict__ counters, int n_pods, const uint8_t* nn_tmpl, const int32_t* nn_count,
                                       const int64_t* nn_req, const uint32_t* nn_req_present, const uint64_t* nn_vals, const uint64_t* nn_meta,
                                       const uint32_t* nn_opts, int max_new, int W32, SimResultDev* out, uint32_t* out_types) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    out->n_pods = n_pods;
    out->n_new_nodes = (int32_t)counters[kCtrNewNodes];
    out->n_unscheduled = (int32_t)counters[kCtrUnscheduled];
    out->error = (int32_t)counters[kCtrError];
    out->template_index = nn_tmpl[0];
    out->pod_count = nn_count[0];
    out->requests_present = nn_req_present[0];
    out->meta = nn_meta[0];
  }
  if (tid < KSCHED_MAX_RES) out->requests[tid] = nn_req[(size_t)tid * max_new];
  if (tid < KSCHED_MAX_KEYS) out->values[tid] = nn_vals[(size_t)tid * max_new];
  for (int w = tid; w < W32; w += blockDim.x) out_types[w] = nn_opts[(size_t)w * max_new];
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
