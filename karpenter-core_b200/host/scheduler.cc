// Host-side mirror of the reference's entry points for the hot path, on top of the C-ABI:
//   Scheduler.Solve                      pkg/controllers/provisioning/scheduling/scheduler.go:96
//   simulateScheduling                   pkg/controllers/deprovisioning/helpers.go:42-115
//   computeConsolidation / firstNNode... consolidation.go:190-274, multinodeconsolidation.go:74-165
// Everything that decides a placement runs on the GPU through ksched_* (include/ksched.h). There is NO CPU
// fallback: without a CUDA device every call here fails with KSCHED_ERR_NO_DEVICE.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <limits>
#include <map>
#include <stdexcept>
#include <memory>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "encoder.h"
#include "ksched.h"
#include "model.h"
#include "reqmask.cuh"
#include "launch.cuh"

using namespace kmodel;
using khost::Encoded;

namespace {

thread_local std::string g_err;
ksched_handle* g_handle = nullptr;
int g_device = 0;
// g_handle holds one cluster snapshot at a time: the id of the ClusterSession whose snapshot it holds, 0 when anything else
// (a Solve, a fresh-encode simulation, ResidentSolve, another session) has been loaded onto it since
uint64_t g_resident_session = 0;
uint64_t g_last_session = 0;
// The same for ResidentSolve (kh_gpu_*): the encoding kh_gpu_load / kh_gpu_solve_e2e last put on g_handle, and whether
// g_handle still holds it. kh_gpu_run loads it again when something else took the handle since.
const Encoded* g_gpu_encoded = nullptr;
bool g_gpu_current = false;

// something other than the recorded session / ResidentSolve encoding is about to be loaded onto g_handle
void handle_taken() {
  g_resident_session = 0;
  g_gpu_current = false;
}
int g_count_visited = 0;  // exact nodes_visited statistic (opt-in: tests); switches the pack kernel's steady-state paths off

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
int ensure_handle() {
  if (g_handle) return KSCHED_OK;
  int rc = ksched_create(g_device, &g_handle);
  if (rc != KSCHED_OK) return fail(rc, "ksched_create failed: no usable CUDA device (the product has no CPU path)");
  return KSCHED_OK;
}

struct ResultBuffers {
  std::vector<int32_t> assign, relax, seq;
  std::vector<ksched_new_node> nodes;
  std::vector<uint64_t> types;
  std::vector<ksched_reqset> existing_reqs;
  std::vector<uint64_t> feasibility;
  std::vector<uint64_t> best;
  std::vector<ksched_launch_choice> launch;
  ksched_result r{};
  // ksched_solve overwrites every per-pod entry and the rows of the nodes it reports (ksched_download), decode reads nothing
  // else: the buffers are sized, not cleared - kh_scheduler_solve keeps one set per thread, so a 100 000-pod Solve does not
  // fault in and zero ~35 MB per call.
  void prepare(const Encoded& E, bool want_feasibility) {
    const size_t P = E.pods.size(), N = (size_t)std::max(1, E.problem.max_new_nodes);
    assign.resize(P);
    relax.resize(P);
    seq.resize(P);
    nodes.resize(N);
    types.resize(N * E.type_words);
    existing_reqs.resize(std::max<size_t>(1, E.existing.size()));
    std::memset(&r, 0, sizeof r);
    r.assign = assign.data();
    r.relax_level = relax.data();
    r.place_seq = seq.data();
    r.new_nodes = nodes.data();
    r.new_node_types = types.data();
    r.existing_reqs = existing_reqs.data();
    launch.resize(nodes.size());
    r.launch = launch.data();
    r.feasibility = nullptr;
    r.best_column = nullptr;
    if (want_feasibility) {
      feasibility.assign(P * E.templates.size() * E.type_words, 0);
      best.assign(P, 0);
      r.feasibility = feasibility.data();
      r.best_column = best.data();
    }
  }
};

// ksched_result -> the reference's ([]*Node, []*ExistingNode) shape (node.go:34-40, existingnode.go:28-39). The per-node part
// (pods in Add order, requests, rendered requirements, launch choice) is independent node by node and runs on all host cores.
void decode(const Encoded& E, const ResultBuffers& B, Result& out) {
  const size_t P = E.pods.size(), NE = E.existing.size(), NN = (size_t)B.r.n_new_nodes, NA = NE + NN;
  out.assign.assign(B.assign.begin(), B.assign.begin() + (ptrdiff_t)P);
  out.relax_level.assign(B.relax.begin(), B.relax.begin() + (ptrdiff_t)P);
  out.nodes_visited = B.r.nodes_visited;
  out.add_calls = B.r.add_calls;
  out.existing_node_index = E.existing_state_index;
  out.existing_pods.assign(NE, {});
  out.new_nodes.assign(NN, {});
  // pods per node in Add order: place_seq is a permutation of 0..placed-1 over the placed pods. Counting sort by node, then
  // each node orders its few pods by sequence number.
  std::vector<uint32_t> start(NA + 1, 0);
  for (size_t p = 0; p < P; ++p) {
    const int32_t a = B.assign[p];
    if (a >= 0 && (size_t)a < NA && B.seq[p] >= 0) ++start[(size_t)a + 1];
  }
  for (size_t a = 0; a < NA; ++a) start[a + 1] += start[a];
  std::vector<std::pair<int32_t, int32_t>> by_node(start[NA]);  // (sequence, pod)
  {
    std::vector<uint32_t> fill(start.begin(), start.end() - 1);
    for (size_t p = 0; p < P; ++p) {
      const int32_t a = B.assign[p];
      if (a >= 0 && (size_t)a < NA && B.seq[p] >= 0) by_node[fill[(size_t)a]++] = {B.seq[p], (int32_t)p};
    }
  }
  // distinct option bitsets: nodes opened for one deployment end with the same set, each is expanded once and shared.
  // lo.Filter keeps the provider's input order: the surviving columns (price order) are permuted into an input-order bitset.
  const size_t NT = E.type_input_index.size(), TW = (size_t)E.type_words;
  {
    std::unordered_map<std::string, int32_t> set_of;
    std::vector<uint64_t> in_order((NT + 63) / 64);
    for (size_t n = 0; n < NN; ++n) {
      const uint64_t* bits = &B.types[n * TW];
      std::string key(reinterpret_cast<const char*>(bits), TW * 8);
      auto found = set_of.find(key);
      if (found != set_of.end()) { out.new_nodes[n].option_set = found->second; continue; }
      std::fill(in_order.begin(), in_order.end(), 0);
      size_t n_opts = 0;
      for (size_t w = 0; w < TW; ++w) {
        uint64_t m = bits[w];
        while (m) {
          const size_t c = w * 64 + (size_t)__builtin_ctzll(m);
          m &= m - 1;
          if (c >= NT) continue;
          const size_t t = (size_t)E.type_input_index[c];
          in_order[t >> 6] |= 1ull << (t & 63);
          ++n_opts;
        }
      }
      std::vector<int32_t> opts;
      opts.reserve(n_opts);
      for (size_t w = 0; w < in_order.size(); ++w) {
        uint64_t m = in_order[w];
        while (m) { opts.push_back((int32_t)(w * 64 + (size_t)__builtin_ctzll(m))); m &= m - 1; }
      }
      out.new_nodes[n].option_set = (int32_t)out.option_sets.size();
      out.option_sets.push_back(std::move(opts));
      set_of.emplace(std::move(key), out.new_nodes[n].option_set);
    }
  }
  khost::parallel_ranges(NA, 512, [&](size_t a0, size_t a1) {
    // requirement renderings are memoised per (key, masks) - nodes of one deployment share them (one memo per worker)
    std::vector<std::unordered_map<uint64_t, std::string>> rendered(E.key_names.size());
    for (size_t a = a0; a < a1; ++a) {
      auto first = by_node.begin() + start[a], last = by_node.begin() + start[a + 1];
      std::sort(first, last);
      std::vector<int32_t>& pods = a < NE ? out.existing_pods[a] : out.new_nodes[a - NE].pods;
      pods.reserve((size_t)(last - first));
      for (auto it = first; it != last; ++it) pods.push_back(it->second);
      if (a < NE) continue;
      const size_t n = a - NE;
      const ksched_new_node& src = B.nodes[n];
      NewNodeResult& dst = out.new_nodes[n];
      dst.provisioner = src.template_index;
      for (size_t r = 0; r < E.res_names.size(); ++r)
        if ((src.requests_present >> r) & 1) dst.requests[E.res_names[r]] = src.requests[r];
      for (size_t k = 0; k < E.key_names.size(); ++k)
        if ((src.reqs.meta >> (KSCHED_META_PRESENT_SHIFT + k)) & 1) {
          const uint64_t memo_key = src.reqs.values[k] ^ (((src.reqs.meta >> (KSCHED_META_COMPLEMENT_SHIFT + k)) & 1) << 63);  // <= 63 values per key
          auto it = rendered[k].find(memo_key);
          if (it == rendered[k].end()) it = rendered[k].emplace(memo_key, khost::render_requirement(E, src.reqs, (int)k)).first;
          dst.requirements[E.key_names[k]] = it->second;
        }
      // launch choice: column -> the provider's instance type, offering by its position in that type's Offerings list
      if (n < B.launch.size() && B.launch[n].type_column >= 0 && E.problem_ref) {
        const ksched_launch_choice& lc = B.launch[n];
        const int ti = E.type_input_index[(size_t)lc.type_column];
        const kmodel::InstanceType& it = E.problem_ref->instance_types[(size_t)ti];
        dst.launch_type = ti;
        if (lc.offering_index < it.offerings.size()) {
          dst.launch_capacity_type = it.offerings[lc.offering_index].capacity_type;
          dst.launch_zone = it.offerings[lc.offering_index].zone;
        }
        if (lc.price_rank < E.price_by_rank.size()) dst.launch_price = E.price_by_rank[lc.price_rank];
      }
    }
  });
}

int error_code(const std::exception& e) {
  std::string m = e.what();
  return m.rfind("unsupported:", 0) == 0 ? KSCHED_ERR_UNSUPPORTED : KSCHED_ERR_INVALID;
}

// One ksched_solve of E on h (default: the scheduler handle, whose cluster snapshot this displaces).
int solve_encoded(Encoded& E, ResultBuffers& B, bool want_feasibility, ksched_handle* h = nullptr) {
  if (!h) {
    int rc = ensure_handle();
    if (rc != KSCHED_OK) return rc;
    h = g_handle;
  }
  if (h == g_handle) handle_taken();
  int rc = ksched_load_catalog(h, &E.catalog);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(h));
  B.prepare(E, want_feasibility);
  rc = ksched_solve(h, &E.problem, &B.r);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(h));
  return KSCHED_OK;
}

// ---- consolidation price helpers (deprovisioning/helpers.go:148-157,292-315) on the decoded new node
bool req_has(const Encoded& E, const ksched_reqset& rs, const std::string& key, const std::string& value) {
  for (size_t k = 0; k < E.key_names.size(); ++k) {
    if (E.key_names[k] != key) continue;
    static const ksched_bounds zero{};
    ksched::Req r = ksched::req_load(rs, &zero, (int)k);
    if (!r.present) return true;  // Requirements.Get of an undefined key is Exists
    for (size_t b = 0; b < E.key_values[k].size(); ++b)
      if (E.key_values[k][b] == value) return r.complement ? !((r.values >> b) & 1) : ((r.values >> b) & 1);
    return r.complement;  // value outside the dictionary: only a complement set admits it
  }
  return true;
}
// spot_only: the caller has added `capacity-type In [spot]` to the node's requirements (consolidation.go:262-265). The
// flag carries that restriction even when capacity-type is not one of the encoded mask keys (no pod or provisioner
// mentions it), where the reqset cannot.
double worst_launch_price(const Encoded& E, const InstanceType& it, const ksched_reqset& rs, bool spot_only = false) {
  auto worst = [&](const char* ct, double* out) {
    bool any = false;
    double mx = 0;
    for (auto& o : it.offerings) {
      if (!o.available || o.capacity_type != ct) continue;
      if (!req_has(E, rs, "topology.kubernetes.io/zone", o.zone)) continue;
      if (!any || o.price > mx) mx = o.price;
      any = true;
    }
    *out = mx;
    return any;
  };
  double p;
  if (req_has(E, rs, "karpenter.sh/capacity-type", "spot") && worst("spot", &p)) return p;
  if (!spot_only && req_has(E, rs, "karpenter.sh/capacity-type", "on-demand") && worst("on-demand", &p)) return p;
  return std::numeric_limits<double>::max();
}

}  // namespace

extern "C" {

const char* kh_scheduler_error() { return g_err.c_str(); }
int kh_set_device(int ordinal) {
  if (g_handle) { ksched_destroy(g_handle); g_handle = nullptr; }
  handle_taken();
  g_gpu_encoded = nullptr;
  g_device = ordinal;
  return KSCHED_OK;
}
void kh_set_count_visited(int on) { g_count_visited = on; }
ksched_handle* kh_handle() { return ensure_handle() == KSCHED_OK ? g_handle : nullptr; }

// Scheduler.Solve through the C-ABI with host buffers (upload + kernels + download inside the call).
int kh_scheduler_solve(const Problem* P, const int* candidates, int ncand, Result* out) {
  *out = Result();
  try {
    std::vector<int> c(candidates, candidates + ncand);
    auto E = khost::encode(*P, c);
    E->problem.count_nodes_visited = g_count_visited;
    static thread_local ResultBuffers B;
    int rc = solve_encoded(*E, B, false);
    if (rc != KSCHED_OK) { out->error = g_err; return rc; }
    decode(*E, B, *out);
    return KSCHED_OK;
  } catch (const std::exception& e) {
    out->error = e.what();
    return fail(error_code(e), e.what());
  }
}

// The same call with its host phases timed (bench.py's end-to-end leg): phases_us = [encode, catalog, solve, decode, total].
// encode = NewScheduler's marshalling (string-level model -> flat structs); catalog = ksched_load_catalog (a no-op when the
// byte-identical catalog is already resident); solve = ksched_solve (upload + kernels + download); decode = the
// ([]*Node, []*ExistingNode) shape.
int kh_scheduler_solve_timed(const Problem* P, const int* candidates, int ncand, Result* out, double* phases_us) {
  *out = Result();
  try {
    using clk = std::chrono::steady_clock;
    auto us = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
    const auto t0 = clk::now();
    std::vector<int> c(candidates, candidates + ncand);
    auto E = khost::encode(*P, c);
    E->problem.count_nodes_visited = g_count_visited;
    const auto t1 = clk::now();
    int rc = ensure_handle();
    if (rc != KSCHED_OK) return rc;
    handle_taken();
    rc = ksched_load_catalog(g_handle, &E->catalog);
    if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
    const auto t2 = clk::now();
    static thread_local ResultBuffers B;
    B.prepare(*E, false);
    rc = ksched_solve(g_handle, &E->problem, &B.r);
    if (rc != KSCHED_OK) { out->error = ksched_last_error(g_handle); return fail(rc, out->error); }
    const auto t3 = clk::now();
    decode(*E, B, *out);
    const auto t4 = clk::now();
    if (phases_us) { phases_us[0] = us(t0, t1); phases_us[1] = us(t1, t2); phases_us[2] = us(t2, t3); phases_us[3] = us(t3, t4); phases_us[4] = us(t0, t4); }
    return KSCHED_OK;
  } catch (const std::exception& e) {
    out->error = e.what();
    return fail(error_code(e), e.what());
  }
}

// ---- split API for benchmarking / kernel tests: encode once, keep the problem resident, time kernels only
Encoded* kh_encode(const Problem* P, const int* candidates, int ncand) {
  try {
    std::vector<int> c(candidates, candidates + ncand);
    return khost::encode(*P, c).release();
  } catch (const std::exception& e) {
    fail(error_code(e), e.what());
    return nullptr;
  }
}
void kh_encoded_free(Encoded* E) {
  if (E == g_gpu_encoded) { g_gpu_encoded = nullptr; g_gpu_current = false; }
  delete E;
}
// dims: [pods, classes, existing, groups, types, templates, keys, resources, type_words, class_topo]
void kh_encoded_dims(const Encoded* E, long long* out) {
  out[0] = (long long)E->pods.size(); out[1] = (long long)E->classes.size(); out[2] = (long long)E->existing.size();
  out[3] = (long long)E->groups.size(); out[4] = (long long)E->types.size(); out[5] = (long long)E->templates.size();
  out[6] = (long long)E->key_names.size(); out[7] = (long long)E->res_names.size(); out[8] = E->type_words;
  out[9] = (long long)E->class_topo.size();
}
void kh_encoded_set_count_visited(Encoded* E, int on) { E->problem.count_nodes_visited = on; }
const ksched_catalog* kh_encoded_catalog(const Encoded* E) { return &E->catalog; }
const ksched_problem* kh_encoded_problem(const Encoded* E) { return &E->problem; }
int kh_gpu_load(Encoded* E) {
  int rc = ensure_handle();
  if (rc != KSCHED_OK) return rc;
  handle_taken();
  g_gpu_encoded = nullptr;
  rc = ksched_load_catalog(g_handle, &E->catalog);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  rc = ksched_upload(g_handle, &E->problem);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  g_gpu_encoded = E;
  g_gpu_current = true;
  return KSCHED_OK;
}
// the ResidentSolve encoding back on g_handle when a session, a Solve or a fresh-encode simulation took it since its load
int gpu_make_current() {
  if (!g_gpu_encoded || g_gpu_current) return KSCHED_OK;
  return kh_gpu_load(const_cast<Encoded*>(g_gpu_encoded));
}
int kh_gpu_run(int flush_l2) {
  if (!g_handle) return fail(KSCHED_ERR_INVALID, "no handle");
  int rc = gpu_make_current();
  if (rc != KSCHED_OK) return rc;
  g_resident_session = 0;
  rc = ksched_run_resident(g_handle, flush_l2);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  return rc;
}
int kh_gpu_run_feasibility(int flush_l2, float* us) {
  if (!g_handle) return fail(KSCHED_ERR_INVALID, "no handle");
  int rc = gpu_make_current();
  if (rc != KSCHED_OK) return rc;
  g_resident_session = 0;
  rc = ksched_run_feasibility_only(g_handle, flush_l2, us);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  return rc;
}
// download + decode; feasibility_out (optional) receives [pods][templates][type_words] uint64 in caller pod order,
// columns in the caller's instance-type order (bit i of template v = instance_types[i])
int kh_gpu_download(Encoded* E, Result* out, unsigned long long* feasibility_out, unsigned long long* best_out) {
  if (!g_handle) return fail(KSCHED_ERR_INVALID, "no handle");
  *out = Result();
  if (g_gpu_encoded && !g_gpu_current) return fail(KSCHED_ERR_INVALID, "the handle was used for other work since this problem's run: run it again");
  ResultBuffers B;
  B.prepare(*E, feasibility_out != nullptr || best_out != nullptr);
  int rc = ksched_download(g_handle, &E->problem, &B.r);
  if (rc != KSCHED_OK) { out->error = ksched_last_error(g_handle); return fail(rc, out->error); }
  decode(*E, B, *out);
  if (feasibility_out) {
    const size_t P = E->pods.size(), V = E->templates.size(), W = (size_t)E->type_words, T = E->types.size();
    std::memset(feasibility_out, 0, P * V * W * 8);
    for (size_t p = 0; p < P; ++p)
      for (size_t v = 0; v < V; ++v) {
        const uint64_t* src = &B.feasibility[(p * V + v) * W];
        unsigned long long* dst = feasibility_out + (p * V + v) * W;
        for (size_t c = 0; c < T; ++c)
          if ((src[c / 64] >> (c % 64)) & 1) { size_t i = (size_t)E->type_input_index[c]; dst[i / 64] |= 1ull << (i % 64); }
      }
  }
  if (best_out) std::memcpy(best_out, B.best.data(), E->pods.size() * 8);
  return KSCHED_OK;
}
// One Scheduler.Solve through the C-ABI with HOST buffers: pod/node/topology upload, kernels and result download are
// all inside the call (the catalog stays resident, as it would across reconciles). Returns wall-clock microseconds.
int kh_gpu_solve_e2e(Encoded* E, Result* out, double* wall_us) {
  if (!g_handle) return fail(KSCHED_ERR_INVALID, "no handle");
  handle_taken();
  g_gpu_encoded = nullptr;
  ResultBuffers B;
  B.prepare(*E, false);
  auto t0 = std::chrono::steady_clock::now();
  int rc = ksched_solve(g_handle, &E->problem, &B.r);
  auto t1 = std::chrono::steady_clock::now();
  if (wall_us) *wall_us = std::chrono::duration<double, std::micro>(t1 - t0).count();
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  g_gpu_encoded = E;
  g_gpu_current = true;
  if (out) { *out = Result(); decode(*E, B, *out); }
  return KSCHED_OK;
}
int kh_gpu_load_catalog(Encoded* E) {
  int rc = ensure_handle();
  if (rc != KSCHED_OK) return rc;
  g_resident_session = 0;
  rc = ksched_load_catalog(g_handle, &E->catalog);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  return KSCHED_OK;
}
int kh_gpu_timings(ksched_timings* t) { return g_handle ? ksched_get_timings(g_handle, t) : KSCHED_ERR_INVALID; }

}  // extern "C"

// ---- consolidation (deprovisioning/consolidation.go, multinodeconsolidation.go) on the GPU path ------------------
namespace {
struct Cand { int node; const InstanceType* it; std::string ct, zone; double cost; };
struct Cmd { int action = 0; std::vector<int> options; };

// candidateNodes (deprovisioning/helpers.go:171-249) with the ShouldDeprovision predicate consolidation and Validation share
// (consolidation.go:104-118, validation.go:101-107); *prov = the node's provisioner or nullptr
bool candidate_node(const Problem* P, const StateNode& n, const Provisioner** prov_out) {
  const Provisioner* prov = nullptr;
  auto pl = n.labels.find("karpenter.sh/provisioner-name");
  if (pl != n.labels.end())
    for (auto& pr : P->provisioners) if (pr.name == pl->second) prov = &pr;
  *prov_out = prov;
  bool ok = !n.marked_for_deletion && prov != nullptr;                                  // helpers.go:186-192
  if (ok) {
    auto itn = n.labels.find("node.kubernetes.io/instance-type");                       // :194-198
    bool it_ok = false;
    if (itn != n.labels.end())
      for (int idx : prov->instance_types) if (P->instance_types[(size_t)idx].name == itn->second) it_ok = true;
    ok = it_ok;
  }
  ok = ok && n.labels.count("karpenter.sh/capacity-type") && n.labels.count("topology.kubernetes.io/zone");  // :201-208
  if (ok) { auto ini = n.labels.find("karpenter.sh/initialized"); ok = ini != n.labels.end() && ini->second == "true"; }  // :211-213
  ok = ok && !n.nominated;                                                              // :215-217
  if (ok) ok = n.do_not_consolidate != 0 ? n.do_not_consolidate != 1 : prov->consolidation_enabled;  // ShouldDeprovision
  return ok;
}

// candidateNodes + sortAndFilterCandidates (deprovisioning/helpers.go:171-249,339-366, consolidation.go:85-118). The string /
// API-object side (labels, annotations, PDB selectors) is decided here; the disruption costs, their lifetime scaling and the
// order come from the device (ksched_rank_candidates) - there is no host-side sort to fall back to.
void rank_on_device(const Problem* P, std::vector<int>* order, std::vector<double>* cost) {
  const size_t N = P->nodes.size();
  order->clear();
  cost->clear();
  if (N == 0) return;
  if (ensure_handle() != KSCHED_OK) throw std::runtime_error(g_err);
  std::vector<uint8_t> eligible(N, 0), flags;
  std::vector<int32_t> off(N + 1, 0), prio;
  std::vector<double> dc, age(N, 0.0), ttl(N, -1.0), given(N, 0.0);
  for (size_t i = 0; i < N; ++i) {
    const StateNode& n = P->nodes[i];
    off[i] = (int32_t)flags.size();
    if (!P->derive_candidates) {
      eligible[i] = n.candidate ? 1 : 0;
      given[i] = n.disruption_cost;
      continue;
    }
    const Provisioner* prov = nullptr;
    bool ok = candidate_node(P, n, &prov);
    ok = ok && !n.deleting;                                                               // canBeTerminated helpers.go:340
    eligible[i] = ok ? 1 : 0;
    if (prov && prov->has_ttl_until_expired) { ttl[i] = (double)prov->ttl_seconds_until_expired; age[i] = P->now_ts - n.creation_ts; }
    for (auto& p : n.pods) {
      uint8_t f = 0;
      if (p.has_deletion_cost) f |= KSCHED_RANK_HAS_DELETION_COST;
      if (p.has_priority) f |= KSCHED_RANK_HAS_PRIORITY;
      bool blocks = false;
      for (auto& b : P->pdbs)                                                             // CanEvictPods pdblimits.go:55-68
        if (b.ns == p.ns && b.disruptions_allowed == 0 && khost::label_selector_matches(b.selector, p.labels)) blocks = true;
      if (!(p.terminating || p.terminal || p.owned_by_node) && p.do_not_evict) blocks = true;  // PodsPreventEviction helpers.go:354-366
      if (blocks) f |= KSCHED_RANK_BLOCKS_EVICTION;
      flags.push_back(f);
      dc.push_back(p.deletion_cost);
      prio.push_back(p.priority);
    }
  }
  off[N] = (int32_t)flags.size();
  ksched_rank_input in{};
  in.n_nodes = (int32_t)N;
  in.n_pods = (int32_t)flags.size();
  in.pod_offsets = off.data(); in.pod_deletion_cost = dc.data(); in.pod_priority = prio.data(); in.pod_flags = flags.data();
  in.node_eligible = eligible.data(); in.node_age_seconds = age.data(); in.node_ttl_seconds = ttl.data();
  in.node_cost = P->derive_candidates ? nullptr : given.data();
  std::vector<int32_t> ord(N);
  std::vector<double> cst(N);
  int32_t n = 0;
  int rc = ksched_rank_candidates(g_handle, &in, ord.data(), cst.data(), &n);
  if (rc != KSCHED_OK) throw std::runtime_error(ksched_last_error(g_handle));
  order->assign(ord.begin(), ord.begin() + n);
  cost->assign(cst.begin(), cst.begin() + n);
}

std::vector<Cand> sorted_candidates(const Problem* P) {
  std::vector<int> order;
  std::vector<double> cost;
  rank_on_device(P, &order, &cost);
  std::vector<Cand> cands;
  for (size_t q = 0; q < order.size(); ++q) {
    const StateNode& n = P->nodes[(size_t)order[q]];
    Cand c{order[q], nullptr, "", "", cost[q]};
    auto itn = n.labels.find("node.kubernetes.io/instance-type");
    if (itn != n.labels.end())
      for (auto& t : P->instance_types) if (t.name == itn->second) c.it = &t;
    auto ct = n.labels.find("karpenter.sh/capacity-type");
    if (ct != n.labels.end()) c.ct = ct->second;
    auto z = n.labels.find("topology.kubernetes.io/zone");
    if (z != n.labels.end()) c.zone = z->second;
    cands.push_back(c);
  }
  return cands;
}

// computeConsolidation after the simulation (consolidation.go:206-274) + the multi-node caller's filterOutSameType
// (multinodeconsolidation.go:132-165, `multi`): sel = the candidates being removed, node0 / bits = the single new node.
Cmd finish_command(const Problem* P, const Encoded& E, const std::vector<Cand>& sel, bool all_scheduled, int n_new, const ksched_reqset& node0_reqs,
                   const uint64_t* bits, bool multi) {
  Cmd cmd;
  const int count = (int)sel.size();
  if (!all_scheduled) return cmd;
  if (n_new == 0) { cmd.action = 1; return cmd; }
  if (n_new != 1) return cmd;
  double price = 0;  // getNodePrices consolidation.go:277-287
  for (int i = 0; i < count; ++i) {
    const Cand& c = sel[i];
    if (!c.it) throw std::runtime_error("candidate without a known instance type");
    bool ok = false;
    for (auto& o : c.it->offerings) if (o.capacity_type == c.ct && o.zone == c.zone) { price += o.price; ok = true; break; }
    if (!ok) throw std::runtime_error("unable to determine offering");
  }
  ksched_reqset reqs = node0_reqs;
  std::vector<int> opts;
  for (size_t c = 0; c < E.type_input_index.size(); ++c)
    if ((bits[c / 64] >> (c % 64)) & 1) opts.push_back(E.type_input_index[c]);
  std::sort(opts.begin(), opts.end());
  std::vector<int> kept;
  for (int t : opts) if (worst_launch_price(E, P->instance_types[t], reqs) < price) kept.push_back(t);  // filterByPrice
  if (kept.empty()) return cmd;
  bool all_spot = true;
  for (int i = 0; i < count; ++i) if (sel[i].ct != "spot") all_spot = false;
  if (all_spot && req_has(E, reqs, "karpenter.sh/capacity-type", "spot")) return cmd;
  bool spot_only = false;
  if (req_has(E, reqs, "karpenter.sh/capacity-type", "spot") && req_has(E, reqs, "karpenter.sh/capacity-type", "on-demand")) {
    spot_only = true;
    // Requirements.Add(capacity-type In [spot]) (consolidation.go:262-265)
    for (size_t k = 0; k < E.key_names.size(); ++k) {
      if (E.key_names[k] != "karpenter.sh/capacity-type") continue;
      uint64_t spot = 0;
      for (size_t b = 0; b < E.key_values[k].size(); ++b) if (E.key_values[k][b] == "spot") spot = 1ull << b;
      ksched::Req in{spot, 0, 0, true, false, false, false};
      static const ksched_bounds zero{};
      ksched::KeyMeta km{0, nullptr, nullptr};
      ksched_bounds tmp{};
      ksched::req_store(reqs, &tmp, (int)k, ksched::key_add(ksched::req_load(reqs, &zero, (int)k), in, km));
    }
  }
  if (!multi) {  // single-node consolidation takes computeConsolidation's command as it is (singlenodeconsolidation.go:56-76)
    cmd.action = 2;
    cmd.options = kept;
    return cmd;
  }
  std::set<std::string> existing_types;  // filterOutSameType
  std::map<std::string, double> by_type;
  for (int i = 0; i < count; ++i) {
    const Cand& c = sel[i];
    existing_types.insert(c.it->name);
    for (auto& o : c.it->offerings)
      if (o.capacity_type == c.ct && o.zone == c.zone) {
        double ex = by_type.count(c.it->name) ? by_type[c.it->name] : std::numeric_limits<double>::max();
        if (o.price < ex) by_type[c.it->name] = o.price;
        break;
      }
  }
  double max_price = std::numeric_limits<double>::max();
  for (int t : kept) {
    const std::string& name = P->instance_types[t].name;
    if (existing_types.count(name) && by_type[name] < max_price) max_price = by_type[name];
  }
  std::vector<int> kept2;
  for (int t : kept) if (worst_launch_price(E, P->instance_types[t], reqs, spot_only) < max_price) kept2.push_back(t);
  if (kept2.empty()) return cmd;
  cmd.action = 2;
  cmd.options = kept2;
  return cmd;
}

// One simulateScheduling = one ksched_solve of a freshly encoded problem (the path for clusters the snapshot cannot hold).
Cmd compute_consolidation_encoded(const Problem* P, const std::vector<Cand>& sel, bool multi) {
  std::vector<int> nodes;
  for (auto& c : sel) nodes.push_back(c.node);
  auto E = khost::encode(*P, nodes);
  E->problem.count_nodes_visited = g_count_visited;
  ResultBuffers B;
  int rc = solve_encoded(*E, B, false);
  if (rc != KSCHED_OK) throw std::runtime_error(g_err);
  size_t scheduled = 0;
  for (auto a : B.assign) if (a >= 0) ++scheduled;
  // helpers.go:109-113 walks EVERY ExistingNode Solve returns (all owned nodes that are neither candidates nor marked for
  // deletion) and gives up when one of them is not initialised - whether or not a pod landed on it
  for (size_t e = 0; e < E->existing.size(); ++e)
    if (!E->existing_initialized[e]) return Cmd();
  return finish_command(P, *E, sel, scheduled == E->pods.size(), B.r.n_new_nodes, B.nodes[0].reqs, &B.types[0], multi);
}

// ksched_load_catalog + ksched_load_cluster of a superset encoding (khost::encode(..., true)) on h
int load_snapshot(ksched_handle* h, Encoded& E) {
  int rc = ksched_load_catalog(h, &E.catalog);
  if (rc != KSCHED_OK) return rc;
  ksched_cluster cl{};
  cl.problem = &E.problem;
  cl.pod_node = E.pod_node.data();
  if (E.problem.n_groups > 0) {
    cl.class_count_begin = E.class_count_begin.data();
    cl.class_count = E.class_count.data();
    cl.node_domain = E.node_domain.data();
    cl.node_has_hostname_label = E.node_has_hostname_label.data();
    cl.group_filter_match = E.group_filter_match.data();
  }
  return ksched_load_cluster(h, &cl);
}

// One ksched_simulate_batch on the snapshot of E that h holds: simulation q removes the existing slots slot_sets[q].
// skip[q]: an uninitialised node stays, and simulateScheduling gives up on it (helpers.go:109-113).
struct SimBatch {
  std::vector<ksched_sim_result> res;
  std::vector<uint64_t> types;  // [simulation][type_words]: the first new node's InstanceTypeOptions
  std::vector<char> skip;
};
SimBatch simulate_on(ksched_handle* h, const Encoded& E, const std::vector<std::vector<int32_t>>& slot_sets) {
  const size_t n = slot_sets.size(), NE = E.existing.size(), V = E.templates.size();
  SimBatch out;
  out.skip.assign(n, 0);
  std::vector<std::vector<int64_t>> rem(n);
  std::vector<ksched_candidate_set> cs(n);
  std::vector<char> removed(NE);
  for (size_t q = 0; q < n; ++q) {
    std::fill(removed.begin(), removed.end(), 0);
    rem[q].resize(V * KSCHED_MAX_RES);
    for (size_t v = 0; v < V; ++v) for (int r = 0; r < KSCHED_MAX_RES; ++r) rem[q][v * KSCHED_MAX_RES + r] = E.templates[v].remaining[r];
    for (int32_t e : slot_sets[q]) {
      removed[(size_t)e] = 1;
      const int v = E.existing_template[(size_t)e];  // scheduler.go:221-248 only charges the nodes that stay
      if (v >= 0) for (int r = 0; r < KSCHED_MAX_RES; ++r) rem[q][(size_t)v * KSCHED_MAX_RES + r] += E.existing_capacity[(size_t)e * KSCHED_MAX_RES + r];
    }
    for (size_t e = 0; e < NE; ++e) if (!removed[e] && !E.existing_initialized[e]) out.skip[q] = 1;
    cs[q] = ksched_candidate_set{slot_sets[q].data(), (int32_t)slot_sets[q].size(), 0, rem[q].data()};
  }
  out.res.resize(n);
  out.types.resize(n * (size_t)E.type_words);
  int rc = ksched_simulate_batch(h, cs.data(), (int)cs.size(), out.res.data(), out.types.data());
  if (rc != KSCHED_OK) throw std::runtime_error(ksched_last_error(h));
  for (size_t q = 0; q < n; ++q)
    if (!out.skip[q] && out.res[q].error) throw std::runtime_error("simulation failed on the device");
  return out;
}

// A consolidation command as Validation reads it: the names of the nodes it removes, delete (1) or replace (2), and the
// names of the replacement's instance-type options (commands and the cluster after the TTL meet by name).
struct VCmd {
  std::vector<std::string> nodes;
  int action = 0;
  std::vector<std::string> options;
};

// ValidateCommand after its simulateScheduling (validation.go:122-171); bits = the first new node's options (unfiltered)
bool command_valid(const Problem* A, const Encoded& E, const VCmd& c, bool all_scheduled, int n_new, const uint64_t* bits) {
  if (!all_scheduled) return false;
  if (n_new == 0) return c.action == 1;          // :132-140 valid only when no replacement was expected
  if (n_new > 1 || c.action != 2) return false;  // :142-151
  std::set<std::string> rhs;                     // instanceTypesAreSubset (helpers.go:118-122), by name
  for (size_t col = 0; col < E.type_input_index.size(); ++col)
    if ((bits[col / 64] >> (col % 64)) & 1) rhs.insert(A->instance_types[(size_t)E.type_input_index[col]].name);
  for (auto& o : c.options) if (!rhs.count(o)) return false;
  return true;
}

struct HandleDeleter { void operator()(ksched_handle* h) const { ksched_destroy(h); } };

// The cluster after the TTL, resident on a handle of its own (the pass's session keeps the scheduler handle). Every
// validation of one ComputeCommand reads this one snapshot (DESIGN.md §6 R7). The validation candidates are
// candidateNodes(after, Validation.ShouldDeprovision) in node-list order (validation.go:78-83): they do not go through
// sortAndFilterCandidates, so a node that a PDB or a DeletionTimestamp keeps out of the pass is still validated. With
// "deriveCandidates": false they are the nodes marked "candidate" that are not marked for deletion. Clusters the snapshot refuses are validated one freshly
// encoded ksched_solve at a time on the same handle.
struct ValidationSnapshot {
  const Problem* A = nullptr;
  uint64_t problem_id = 0;          // Problem::id of A: never shared with a problem allocated later at the same address
  std::vector<int> cands;           // Problem.nodes indices
  std::set<std::string> nominated;  // Cluster.IsNodeNominated
  std::unique_ptr<ksched_handle, HandleDeleter> h;
  std::unique_ptr<Encoded> E;       // superset encoding (resident == true)
  std::vector<int> slot_of_node;
  bool resident = false;

  explicit ValidationSnapshot(const Problem* a) : A(a), problem_id(a->id) {
    for (size_t i = 0; i < A->nodes.size(); ++i) {
      const StateNode& n = A->nodes[i];
      if (n.nominated) nominated.insert(n.name);
      const Provisioner* prov = nullptr;
      // candidateNodes skips nodes marked for deletion in either mode (helpers.go:185-188)
      if (A->derive_candidates ? candidate_node(A, n, &prov) : n.candidate && !n.marked_for_deletion) cands.push_back((int)i);
    }
    ksched_handle* raw = nullptr;
    if (ksched_create(g_device, &raw) != KSCHED_OK) throw std::runtime_error("ksched_create failed: no usable CUDA device (the product has no CPU path)");
    h.reset(raw);
    auto sup = khost::encode(*A, cands, true);
    sup->problem.count_nodes_visited = 0;
    int rc = load_snapshot(h.get(), *sup);
    if (rc == KSCHED_ERR_UNSUPPORTED) return;  // resident stays false
    if (rc != KSCHED_OK) throw std::runtime_error(ksched_last_error(h.get()));
    E = std::move(sup);
    slot_of_node.assign(A->nodes.size(), -1);
    for (size_t e = 0; e < E->existing_state_index.size(); ++e) slot_of_node[(size_t)E->existing_state_index[e]] = (int)e;
    resident = true;
  }

  // Validation.IsValid for every command: the simulations of all of them in one ksched_simulate_batch call
  std::vector<char> validate(const std::vector<VCmd>& cmds) {
    std::vector<char> ok(cmds.size(), 0);
    std::vector<size_t> run;               // commands that reach simulateScheduling
    std::vector<std::vector<int>> mapped;  // their mapped nodes (Problem.nodes indices)
    for (size_t q = 0; q < cmds.size(); ++q) {
      bool nom = false;
      for (auto& name : cmds[q].nodes) nom = nom || nominated.count(name) > 0;  // validation.go:85-91
      if (nom) continue;
      std::set<std::string> names(cmds[q].nodes.begin(), cmds[q].nodes.end());
      std::vector<int> m;
      for (int i : cands) if (names.count(A->nodes[(size_t)i].name)) m.push_back(i);  // mapNodes helpers.go:328-337
      if (m.empty()) continue;                                                         // validation.go:113-116
      run.push_back(q);
      mapped.push_back(std::move(m));
    }
    if (run.empty()) return ok;
    if (resident) {
      std::vector<std::vector<int32_t>> slots(run.size());
      for (size_t j = 0; j < run.size(); ++j) for (int i : mapped[j]) slots[j].push_back(slot_of_node[(size_t)i]);
      SimBatch sb = simulate_on(h.get(), *E, slots);
      for (size_t j = 0; j < run.size(); ++j)
        if (!sb.skip[j])
          ok[run[j]] = command_valid(A, *E, cmds[run[j]], sb.res[j].n_unscheduled == 0, sb.res[j].n_new_nodes, &sb.types[j * (size_t)E->type_words]);
      return ok;
    }
    for (size_t j = 0; j < run.size(); ++j) {
      auto F = khost::encode(*A, mapped[j]);
      F->problem.count_nodes_visited = 0;
      ResultBuffers B;
      if (solve_encoded(*F, B, false, h.get()) != KSCHED_OK) throw std::runtime_error(g_err);
      bool init = true;
      for (size_t e = 0; e < F->existing.size(); ++e) init = init && F->existing_initialized[e];
      size_t scheduled = 0;
      for (auto a : B.assign) if (a >= 0) ++scheduled;
      ok[run[j]] = init && command_valid(A, *F, cmds[run[j]], scheduled == F->pods.size(), B.r.n_new_nodes, &B.types[0]);
    }
    return ok;
  }
};

// The consolidation pass over one cluster: candidates ranked once, the cluster resident on the device once
// (ksched_load_cluster), every computeConsolidation a ksched_simulate_batch entry. Clusters the snapshot cannot hold
// (topology groups) are simulated one freshly encoded ksched_solve at a time - still on the GPU, never on the CPU.
// Sessions share the scheduler handle: a session whose snapshot something else displaced loads it again before its next
// batch (g_resident_session).
struct ClusterSession {
  const Problem* P = nullptr;
  std::vector<Cand> cands;            // disruption order
  std::unique_ptr<Encoded> E;         // superset encoding (resident == true)
  std::vector<int> slot_of_node;      // Problem.nodes index -> existing slot
  bool resident = false;
  uint64_t id = 0;
  int simulations = 0;
  std::unique_ptr<ValidationSnapshot> validation_snapshot;  // opened at the first command that needs validation

  explicit ClusterSession(const Problem* p) : P(p), cands(sorted_candidates(p)) {
    if (ensure_handle() != KSCHED_OK) throw std::runtime_error(g_err);
    std::vector<int> nodes;
    for (auto& c : cands) nodes.push_back(c.node);
    auto sup = khost::encode(*P, nodes, true);
    sup->problem.count_nodes_visited = 0;
    handle_taken();
    int rc = load_snapshot(g_handle, *sup);
    if (rc == KSCHED_ERR_UNSUPPORTED) return;  // resident stays false
    if (rc != KSCHED_OK) throw std::runtime_error(ksched_last_error(g_handle));
    E = std::move(sup);
    slot_of_node.assign(P->nodes.size(), -1);
    for (size_t e = 0; e < E->existing_state_index.size(); ++e) slot_of_node[(size_t)E->existing_state_index[e]] = (int)e;
    resident = true;
    id = ++g_last_session;
    g_resident_session = id;
  }

  // computeConsolidation for every set (positions in the disruption order), one ksched_simulate_batch call
  std::vector<Cmd> compute_many(const std::vector<std::vector<int>>& sets, bool multi) {
    std::vector<Cmd> out(sets.size());
    simulations += (int)sets.size();
    if (!resident) {
      for (size_t q = 0; q < sets.size(); ++q) {
        std::vector<Cand> sel;
        for (int i : sets[q]) sel.push_back(cands.at((size_t)i));
        out[q] = compute_consolidation_encoded(P, sel, multi);
      }
      return out;
    }
    std::vector<std::vector<int32_t>> slots(sets.size());
    for (size_t q = 0; q < sets.size(); ++q)
      for (int i : sets[q]) {
        const int e = slot_of_node.at((size_t)cands.at((size_t)i).node);
        if (e < 0) throw std::runtime_error("candidate is not an existing node of the snapshot");
        slots[q].push_back(e);
      }
    if (g_resident_session != id) {  // displaced: the time of one reload, the same answers
      if (ensure_handle() != KSCHED_OK) throw std::runtime_error(g_err);
      handle_taken();
      if (load_snapshot(g_handle, *E) != KSCHED_OK) throw std::runtime_error(ksched_last_error(g_handle));
      g_resident_session = id;
    }
    SimBatch sb = simulate_on(g_handle, *E, slots);
    for (size_t q = 0; q < sets.size(); ++q) {
      if (sb.skip[q]) continue;
      std::vector<Cand> sel;
      for (int i : sets[q]) sel.push_back(cands[(size_t)i]);
      out[q] = finish_command(P, *E, sel, sb.res[q].n_unscheduled == 0, sb.res[q].n_new_nodes, sb.res[q].node0.reqs, &sb.types[q * (size_t)E->type_words], multi);
    }
    return out;
  }
  Cmd compute_prefix(int count) {
    std::vector<int> set;
    for (int i = 0; i < count; ++i) set.push_back(i);
    return compute_many({set}, true)[0];
  }

  // the command that removes the candidates at `positions`, in the terms Validation compares (names)
  VCmd command(const std::vector<int>& positions, int action, const std::vector<int>& options) const {
    VCmd c;
    c.action = action;
    for (int i : positions) c.nodes.push_back(P->nodes[(size_t)cands.at((size_t)i).node].name);
    for (int t : options) c.options.push_back(P->instance_types.at((size_t)t).name);
    return c;
  }
  std::vector<char> validate(const Problem* after, const std::vector<VCmd>& cmds) {
    if (!validation_snapshot || validation_snapshot->problem_id != after->id) {
      validation_snapshot.reset();  // one extra device handle at a time
      validation_snapshot = std::make_unique<ValidationSnapshot>(after);
    }
    return validation_snapshot->validate(cmds);
  }
};

// MultiNodeConsolidation.firstNNodeConsolidationOption (multinodeconsolidation.go:74-114): binary search, one probe per step
struct Search {
  Cmd cmd;
  int count = 0, sims = 0;
  std::vector<int> probes, actions;
};
Search first_n_search(ClusterSession& cs) {
  Search s;
  if (cs.cands.size() < 2) return s;
  int mn = 1, mx = (int)cs.cands.size() - 1;
  while (mn <= mx) {
    int mid = (mn + mx) / 2;
    Cmd c = cs.compute_prefix(mid + 1);
    ++s.sims;
    s.probes.push_back(mid + 1);
    s.actions.push_back(c.action);
    if (c.action == 1 || c.action == 2) { s.cmd = c; s.count = mid + 1; mn = mid + 1; }
    else mx = mid - 1;
  }
  return s;
}

// SingleNodeConsolidation.ComputeCommand's loop (singlenodeconsolidation.go:54-84) over positions [first, last), `batch`
// independent simulations per device call. With `after`, the actionable commands of each batch are validated together in
// one more device call and the first valid one wins; the trace holds (position, verdict) of what the sequential loop
// validates - the positions up to and including the winner. Without `after` every command is taken as valid.
struct Sweep {
  Cmd cmd;
  int position = -1, sims = 0;
  bool failed_validation = false;
  std::vector<std::pair<int, int>> trace;
};
Sweep single_sweep(ClusterSession& cs, const Problem* after, int first, int last, int batch) {
  Sweep s;
  const int n = (int)cs.cands.size();
  if (last < 0 || last > n) last = n;
  if (batch < 1) batch = 1;
  for (int b = std::max(first, 0); b < last; b += batch) {
    std::vector<std::vector<int>> sets;
    for (int i = b; i < std::min(last, b + batch); ++i) sets.push_back({i});
    auto cmds = cs.compute_many(sets, false);
    s.sims += (int)sets.size();
    std::vector<int> hits;
    for (size_t q = 0; q < cmds.size(); ++q) if (cmds[q].action == 1 || cmds[q].action == 2) hits.push_back((int)q);
    if (hits.empty()) continue;
    std::vector<char> ok(hits.size(), 1);
    if (after) {
      std::vector<VCmd> vc;
      for (int q : hits) vc.push_back(cs.command({b + q}, cmds[(size_t)q].action, cmds[(size_t)q].options));
      ok = cs.validate(after, vc);
    }
    for (size_t j = 0; j < hits.size(); ++j) {
      if (after) s.trace.push_back({b + hits[j], ok[j] ? 1 : 0});
      if (!ok[j]) { s.failed_validation = true; continue; }
      s.cmd = cmds[(size_t)hits[j]];
      s.position = b + hits[j];
      return s;
    }
  }
  return s;
}
}  // namespace

extern "C" {
// number of consolidation candidates
int kh_consolidate_candidates(const Problem* P) {
  try { return (int)sorted_candidates(P).size(); } catch (const std::exception& e) { return fail(error_code(e), e.what()); }
}
// candidate ranking on the device: order = Problem.nodes indices by disruption cost, cost parallel; returns their number
int kh_rank_candidates(const Problem* P, int* order, double* cost, int cap) {
  try {
    std::vector<int> o;
    std::vector<double> c;
    rank_on_device(P, &o, &c);
    for (size_t i = 0; i < o.size() && (int)i < cap; ++i) { order[i] = o[i]; cost[i] = c[i]; }
    return (int)o.size();
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// A consolidation pass over one cluster (ClusterSession): open once, probe many times, close. The session keeps the
// cluster resident on the device (ksched_load_cluster); `resident` tells whether the snapshot path took it.
ClusterSession* kh_cluster_open(const Problem* P, int* resident, int* n_candidates) {
  try {
    auto* cs = new ClusterSession(P);
    if (resident) *resident = cs->resident ? 1 : 0;
    if (n_candidates) *n_candidates = (int)cs->cands.size();
    return cs;
  } catch (const std::exception& e) {
    fail(error_code(e), e.what());
    return nullptr;
  }
}
void kh_cluster_close(ClusterSession* cs) { delete cs; }
// computeConsolidation for n_sets candidate sets in ONE ksched_simulate_batch call. sets = positions in the disruption order,
// set q = sets[set_off[q] .. set_off[q+1]); multi = apply the multi-node caller's filterOutSameType.
// actions[q] = 0 / 1 / 2; options of set q are written to options[q * options_stride ...], n_options[q] of them.
int kh_cluster_probe_sets(ClusterSession* cs, const int* sets, const int* set_off, int n_sets, int multi, int* actions, int* options, int options_stride,
                          int* n_options) {
  try {
    std::vector<std::vector<int>> v((size_t)n_sets);
    for (int q = 0; q < n_sets; ++q) v[(size_t)q].assign(sets + set_off[q], sets + set_off[q + 1]);
    auto cmds = cs->compute_many(v, multi != 0);
    for (int q = 0; q < n_sets; ++q) {
      actions[q] = cmds[(size_t)q].action;
      n_options[q] = (int)cmds[(size_t)q].options.size();
      for (size_t i = 0; i < cmds[(size_t)q].options.size() && (int)i < options_stride; ++i) options[(size_t)q * options_stride + i] = cmds[(size_t)q].options[i];
    }
    return KSCHED_OK;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}
// disruption order of the session's candidates (Problem.nodes indices)
int kh_cluster_candidates(const ClusterSession* cs, int* nodes, int cap) {
  for (size_t i = 0; i < cs->cands.size() && (int)i < cap; ++i) nodes[i] = cs->cands[i].node;
  return (int)cs->cands.size();
}

// One probe of the multi-node search: computeConsolidation over the `count` cheapest-to-disrupt candidates.
// Returns the action (0 nothing, 1 delete, 2 replace) or a negative error; options = surviving replacement types.
int kh_consolidate_probe(const Problem* P, int count, int* options, int options_cap, int* n_options) {
  try {
    ClusterSession cs(P);
    if (count < 1 || count > (int)cs.cands.size()) return fail(KSCHED_ERR_INVALID, "probe size out of range");
    Cmd c = cs.compute_prefix(count);
    *n_options = (int)c.options.size();
    for (size_t i = 0; i < c.options.size() && (int)i < options_cap; ++i) options[i] = c.options[i];
    return c.action;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// MultiNodeConsolidation.firstNNodeConsolidationOption (multinodeconsolidation.go:74-114): binary search, one probe per step.
// out ints: [action, nodes_removed, simulations, n_options]; options = instance type indices.
int kh_consolidate(const Problem* P, int* out4, int* options, int options_cap, int* probes, int* probe_actions, int probes_cap, int* n_probes) {
  try {
    ClusterSession cs(P);
    const Search s = first_n_search(cs);
    *n_probes = (int)s.probes.size();
    for (int i = 0; i < *n_probes && i < probes_cap; ++i) { probes[i] = s.probes[(size_t)i]; probe_actions[i] = s.actions[(size_t)i]; }
    out4[0] = s.cmd.action;
    out4[1] = s.count;
    out4[2] = s.sims;
    out4[3] = (int)s.cmd.options.size();
    for (size_t i = 0; i < s.cmd.options.size() && (int)i < options_cap; ++i) options[i] = s.cmd.options[i];
    return KSCHED_OK;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// MultiNodeConsolidation.ComputeCommand (multinodeconsolidation.go:41-70): the search on `before`, then Validation.IsValid of
// its command against `after`, the cluster when the TTL ends. out4 and the probes as kh_consolidate; a command that fails
// validation becomes retry (out4 = [3, 0, simulations, 0]). *verdict = 1 valid, 0 invalid, -1 nothing to validate.
int kh_consolidate_validated(const Problem* before, const Problem* after, int* out4, int* options, int options_cap, int* probes, int* probe_actions,
                             int probes_cap, int* n_probes, int* verdict) {
  try {
    ClusterSession cs(before);
    const Search s = first_n_search(cs);
    *n_probes = (int)s.probes.size();
    for (int i = 0; i < *n_probes && i < probes_cap; ++i) { probes[i] = s.probes[(size_t)i]; probe_actions[i] = s.actions[(size_t)i]; }
    Cmd cmd = s.cmd;
    int removed = s.count;
    *verdict = -1;
    if (cmd.action == 1 || cmd.action == 2) {
      std::vector<int> positions;
      for (int i = 0; i < s.count; ++i) positions.push_back(i);
      *verdict = cs.validate(after, {cs.command(positions, cmd.action, cmd.options)})[0] ? 1 : 0;
      if (!*verdict) { cmd = Cmd(); cmd.action = 3; removed = 0; }
    }
    out4[0] = cmd.action;
    out4[1] = removed;
    out4[2] = s.sims;
    out4[3] = (int)cmd.options.size();
    for (size_t i = 0; i < cmd.options.size() && (int)i < options_cap; ++i) options[i] = cmd.options[i];
    return KSCHED_OK;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// Validation.IsValid (validation.go:63-172) of n_sets commands of an open session against `after`, the cluster when the TTL
// ends: command q removes the candidates at positions sets[set_off[q] .. set_off[q+1]) of the session's disruption order,
// actions[q] is 1 (delete) or 2 (replace) and its options are options[q * options_stride ...], n_options[q] of them - what
// kh_cluster_probe_sets returns. valid[q] = 1 / 0. The session keeps the snapshot of `after` until it closes or is handed a
// different problem (Problem::id): every validation of one ComputeCommand passes the same one (DESIGN.md §6 R7).
int kh_cluster_validate(ClusterSession* cs, const Problem* after, const int* sets, const int* set_off, int n_sets, const int* actions, const int* options,
                        int options_stride, const int* n_options, int* valid) {
  try {
    std::vector<VCmd> cmds;
    if (n_sets < 0 || (n_sets > 0 && set_off[0] < 0)) return fail(KSCHED_ERR_INVALID, "n_sets / set_off out of range");
    for (int q = 0; q < n_sets; ++q) {
      if (set_off[q + 1] < set_off[q]) return fail(KSCHED_ERR_INVALID, "set_off must be non-decreasing");
      if (actions[q] != 1 && actions[q] != 2) return fail(KSCHED_ERR_INVALID, "only delete (1) and replace (2) commands are validated");
      if (n_options[q] < 0 || n_options[q] > options_stride) return fail(KSCHED_ERR_INVALID, "n_options out of range");
      std::vector<int> positions(sets + set_off[q], sets + set_off[q + 1]);
      for (int i : positions) if (i < 0 || i >= (int)cs->cands.size()) return fail(KSCHED_ERR_INVALID, "position out of range");
      std::vector<int> opts(options + (size_t)q * options_stride, options + (size_t)q * options_stride + n_options[q]);
      for (int t : opts) if (t < 0 || t >= (int)cs->P->instance_types.size()) return fail(KSCHED_ERR_INVALID, "instance type out of range");
      cmds.push_back(cs->command(positions, actions[q], opts));
    }
    auto ok = cs->validate(after, cmds);
    for (int q = 0; q < n_sets; ++q) valid[q] = ok[(size_t)q] ? 1 : 0;
    return KSCHED_OK;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// ncclAllGather of n ints per rank on the scheduler handle's communicator (kh_nccl_init first)
int kh_allgather_i32(const int* send, int n, int* recv) {
  int rc = ensure_handle();
  if (rc != KSCHED_OK) return rc;
  rc = ksched_allgather(g_handle, send, (size_t)n * sizeof(int), recv);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  return KSCHED_OK;
}
// communicator for the scheduler handle without column sharding (replicas / sharded consolidation)
int kh_nccl_init(const void* id128, int rank, int world) {
  int rc = ensure_handle();
  if (rc != KSCHED_OK) return rc;
  rc = ksched_nccl_init(g_handle, id128, rank, world);
  if (rc == KSCHED_OK) rc = ksched_set_shard(g_handle, 0, 1);
  if (rc != KSCHED_OK) return fail(rc, ksched_last_error(g_handle));
  return KSCHED_OK;
}

// SingleNodeConsolidation.ComputeCommand (singlenodeconsolidation.go:43-84) without validation: the candidates in disruption
// order, the first whose computeConsolidation yields delete / replace wins. The independent simulations go to the device
// `batch` at a time (ksched_simulate_batch). out4: [action, position of the winning candidate in the disruption order or -1,
// simulations, n_options]; *node = its Problem.nodes index. first / last bound the positions tried (a rank's share of the
// sweep); last < 0 = all.
int kh_consolidate_single(const Problem* P, int first, int last, int batch, int* out4, int* node, int* options, int options_cap) {
  try {
    ClusterSession cs(P);
    const Sweep s = single_sweep(cs, nullptr, first, last, batch);
    out4[0] = s.cmd.action;
    out4[1] = s.position;
    out4[2] = s.sims;
    out4[3] = (int)s.cmd.options.size();
    *node = s.position >= 0 ? cs.cands[(size_t)s.position].node : -1;
    for (size_t i = 0; i < s.cmd.options.size() && (int)i < options_cap; ++i) options[i] = s.cmd.options[i];
    return KSCHED_OK;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// SingleNodeConsolidation.ComputeCommand with Validation against `after` (singlenodeconsolidation.go:52-84): the first
// actionable command that validates wins; none, after a failed validation, is retry (action 3). out4, *node and options as
// kh_consolidate_single. trace[i] / trace_valid[i] = the positions validated and their verdicts, in order, *n_trace of them;
// *failed_validation = a validation failed before the winner (or anywhere, without one). Shares [first, last) of one sweep
// merge as: the first share with a winner gives the command; with none, retry when any share failed a validation.
int kh_consolidate_single_validated(const Problem* before, const Problem* after, int first, int last, int batch, int* out4, int* node, int* options,
                                    int options_cap, int* trace, int* trace_valid, int trace_cap, int* n_trace, int* failed_validation) {
  try {
    ClusterSession cs(before);
    const Sweep s = single_sweep(cs, after, first, last, batch);
    out4[0] = s.position >= 0 ? s.cmd.action : s.failed_validation ? 3 : 0;
    out4[1] = s.position;
    out4[2] = s.sims;
    out4[3] = (int)s.cmd.options.size();
    *node = s.position >= 0 ? cs.cands[(size_t)s.position].node : -1;
    for (size_t i = 0; i < s.cmd.options.size() && (int)i < options_cap; ++i) options[i] = s.cmd.options[i];
    *n_trace = (int)s.trace.size();
    for (int i = 0; i < *n_trace && i < trace_cap; ++i) { trace[i] = s.trace[(size_t)i].first; trace_valid[i] = s.trace[(size_t)i].second; }
    *failed_validation = s.failed_validation ? 1 : 0;
    return KSCHED_OK;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// Two handles on one device, one host thread each, solving different problems at the same time. The pack kernel's
// parameter block is one __constant__ object per device, so concurrent handles only stay correct through the device-side
// ordering in run_pack(); this entry point lets the GPU tests prove it. Returns 0 when every repetition of each problem
// reproduced that problem's first result bit for bit, a negative ksched error otherwise, or 1 on a mismatch.
extern "C" int kh_selftest_two_handles(const Problem* A, const Problem* B, int iters) {
  int rc = ensure_handle();
  if (rc != KSCHED_OK) return rc;
  const Problem* probs[2] = {A, B};
  int status[2] = {0, 0};
  std::thread workers[2];
  for (int w = 0; w < 2; ++w) {
    workers[w] = std::thread([&, w]() {
      try {
        ksched_handle* h = nullptr;
        if (ksched_create(g_device, &h) != KSCHED_OK) { status[w] = KSCHED_ERR_CUDA; return; }
        auto E = khost::encode(*probs[w], {});
        E->problem.count_nodes_visited = 0;
        std::vector<int32_t> first;
        for (int it = 0; it < iters && status[w] == 0; ++it) {
          ResultBuffers R;
          int r2 = ksched_load_catalog(h, &E->catalog);
          if (r2 == KSCHED_OK) { R.prepare(*E, false); r2 = ksched_solve(h, &E->problem, &R.r); }
          if (r2 != KSCHED_OK) { status[w] = r2; break; }
          std::vector<int32_t> sig(R.assign.begin(), R.assign.end());
          sig.push_back(R.r.n_new_nodes);
          for (int n = 0; n < R.r.n_new_nodes; ++n)
            for (int k = 0; k < E->type_words; ++k) {
              const uint64_t b = R.types[(size_t)n * E->type_words + k];
              sig.push_back((int32_t)b);
              sig.push_back((int32_t)(b >> 32));
            }
          if (it == 0) first = sig;
          else if (sig != first) status[w] = 1;
        }
        ksched_destroy(h);
      } catch (const std::exception& e) {
        status[w] = error_code(e);
      }
    });
  }
  for (auto& t : workers) t.join();
  return status[0] ? status[0] : status[1];
}

// ---- launch-choice table + shared core (csrc/launch.cuh) checked on the CPU: for every new node of `ref` (a Result of
// the same problem, e.g. the oracle's) recompute the launch choice from the ENCODED offering table exactly as the device
// kernel does, and compare with the fields `ref` carries. Returns the number of nodes that differ, or a negative error.
extern "C" int kh_launch_table_selfcheck(const Problem* P, const Result* ref) {
  try {
    auto E = khost::encode(*P, {});
    int zone_key = -1, ct_key = -1;
    for (size_t k = 0; k < E->key_names.size(); ++k) {
      if (E->key_names[k] == "topology.kubernetes.io/zone") zone_key = (int)k;
      if (E->key_names[k] == "karpenter.sh/capacity-type") ct_key = (int)k;
    }
    // admissible dictionary ids of a rendered requirement ("In [a b]", "NotIn [a]", "Exists", "DoesNotExist")
    auto allowed = [&](int key, const std::map<std::string, std::string>& reqs, uint32_t all) -> uint32_t {
      if (key < 0) return all;
      auto it = reqs.find(E->key_names[(size_t)key]);
      if (it == reqs.end()) return all;
      const std::string& r = it->second;
      std::set<std::string> vals;
      size_t lb = r.find('['), rb = r.rfind(']');
      if (lb != std::string::npos && rb != std::string::npos && rb > lb) {
        std::string body = r.substr(lb + 1, rb - lb - 1), cur;
        for (char ch : body) { if (ch == ' ') { if (!cur.empty()) vals.insert(cur); cur.clear(); } else cur.push_back(ch); }
        if (!cur.empty()) vals.insert(cur);
      }
      const bool is_in = r.rfind("In", 0) == 0, is_notin = r.rfind("NotIn", 0) == 0, exists = r.rfind("Exists", 0) == 0;
      uint32_t m = 0;
      for (size_t b = 0; b < E->key_values[(size_t)key].size(); ++b) {
        const bool has = vals.count(E->key_values[(size_t)key][b]) > 0;
        if (exists || (is_in && has) || (is_notin && !has)) m |= 1u << b;
      }
      return m;
    };
    std::vector<int> col_of(P->instance_types.size(), -1);
    for (size_t c = 0; c < E->type_input_index.size(); ++c) col_of[(size_t)E->type_input_index[c]] = (int)c;
    int bad = 0;
    for (auto& nn : ref->new_nodes) {
      const uint32_t zmask = allowed(zone_key, nn.requirements, 0xFFFF), cmask = allowed(ct_key, nn.requirements, 0xF);
      uint64_t best = ~0ull, best_off = ksched::kNoOffering;
      int best_col = -1;
      for (int ti : kmodel::node_options(*ref, nn)) {
        const int c = col_of[(size_t)ti];
        const uint64_t ok = ksched::offering_min_key(&E->offering_keys[(size_t)c * 64], zmask, cmask);
        if (ok == ksched::kNoOffering) continue;
        const uint64_t key = ksched::option_key(ok, E->types[(size_t)c].input_index);
        if (key < best) { best = key; best_off = ok; best_col = c; }
      }
      int type = -1;
      std::string ct, zone;
      double price = 0;
      if (best_col >= 0) {
        type = E->type_input_index[(size_t)best_col];
        const auto& it = P->instance_types[(size_t)type];
        const size_t oi = (size_t)((best_off >> 8) & 0xFF);
        if (oi < it.offerings.size()) { ct = it.offerings[oi].capacity_type; zone = it.offerings[oi].zone; }
        price = E->price_by_rank[(size_t)(best_off >> 16)];
      }
      if (type != nn.launch_type || ct != nn.launch_capacity_type || zone != nn.launch_zone || price != nn.launch_price) ++bad;
    }
    return bad;
  } catch (const std::exception& e) {
    return fail(error_code(e), e.what());
  }
}

// ---- digest of everything an encoding hands to the C-ABI (tests: a faster encoder must produce the same bytes)
extern "C" unsigned long long kh_encoded_digest(const Encoded* E) {
  unsigned long long h = 1469598103934665603ull;
  auto bytes = [&](const void* p, size_t n) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  };
  auto str = [&](const std::string& x) { size_t n = x.size(); bytes(&n, sizeof n); bytes(x.data(), n); };
  auto vec = [&](const auto& v) { size_t n = v.size(); bytes(&n, sizeof n); if (n) bytes(v.data(), n * sizeof(v[0])); };
  for (auto& k : E->key_names) str(k);
  for (auto& vs : E->key_values) { size_t n = vs.size(); bytes(&n, sizeof n); for (auto& v : vs) str(v); }
  for (auto& r : E->res_names) str(r);
  for (auto* p : E->pods) str(p->uid);
  vec(E->existing_state_index);
  for (bool b : E->existing_initialized) { unsigned char c = b; bytes(&c, 1); }
  vec(E->template_provisioner); vec(E->type_input_index);
  bytes(&E->type_words, sizeof E->type_words);
  vec(E->keys); vec(E->key_int_values);
  if (!E->key_regions.empty()) vec(E->key_regions);  // absent for problems without Gt/Lt: their digests predate the region form
  vec(E->types); vec(E->type_capacity); vec(E->offering_keys); vec(E->price_by_rank);
  vec(E->templates); vec(E->template_bounds); vec(E->classes); vec(E->class_bounds);
  unsigned char flags[2] = {(unsigned char)E->any_class_bounds, (unsigned char)E->any_template_bounds};
  bytes(flags, 2);
  vec(E->pod_class); vec(E->pod_timestamp); vec(E->pod_uid_rank); vec(E->existing); vec(E->groups); vec(E->group_domain_counts);
  vec(E->group_existing_counts); vec(E->class_topo); vec(E->filter_terms); vec(E->itype_req_sets); vec(E->itype_req_complement); vec(E->hostname_reqs);
  if (!E->class_volumes.empty()) { vec(E->class_volumes); vec(E->existing_volumes); bytes(E->volume_driver_mask, sizeof E->volume_driver_mask); }
  const ksched_catalog& c = E->catalog;
  int cat[4] = {c.n_keys, c.n_res, c.n_types, c.n_templates};
  bytes(cat, sizeof cat);
  const ksched_problem& q = E->problem;
  int pr[11] = {q.n_pods, q.n_classes, q.n_existing, q.n_groups, q.n_class_topo, q.n_filter_terms, q.n_itype_reqs, q.n_hostname_reqs, q.max_new_nodes,
                q.write_feasibility, 0};
  bytes(pr, sizeof pr);
  return h;
}

// ---- host-side mask algebra exposed for the CPU golden-vector tests (same code the kernels run)
// spec: op ("In","NotIn","Exists","DoesNotExist","Gt","Lt") + comma separated values; dictionary = A,B,1,2,9
static ksched::Req spec_req(const char* op_c, const char* vals_c, const std::vector<std::string>& dict) {
  std::string op = op_c, vals = vals_c;
  std::vector<std::string> v;
  size_t pos = 0;
  while (pos <= vals.size() && !vals.empty()) {
    size_t c = vals.find(',', pos);
    if (c == std::string::npos) c = vals.size();
    v.push_back(vals.substr(pos, c - pos));
    pos = c + 1;
  }
  ksched::Req r{0, 0, 0, true, true, false, false};
  r.complement = !(op == "In" || op == "DoesNotExist");
  if (op == "In" || op == "NotIn")
    for (auto& x : v)
      for (size_t b = 0; b < dict.size(); ++b) if (dict[b] == x) r.values |= 1ull << b;
  if (op == "Gt") { r.has_gt = true; r.gt = std::stoll(v.at(0)); }
  if (op == "Lt") { r.has_lt = true; r.lt = std::stoll(v.at(0)); }
  return r;
}
struct TestDict {
  std::vector<std::string> dict{"1", "2", "9", "A", "B"};
  int64_t ints[64] = {1, 2, 9};
  ksched::KeyMeta km{0x7, ints, nullptr};
};
// out: [present, complement, values, has_gt, gt, has_lt, lt, len_zero, op_negative]
void kh_mask_intersection(const char* aop, const char* avals, const char* bop, const char* bvals, long long* out) {
  TestDict d;
  ksched::Req a = spec_req(aop, avals, d.dict), b = spec_req(bop, bvals, d.dict);
  ksched::Req r = ksched::req_intersect(a, b, d.km);
  out[0] = r.present; out[1] = r.complement; out[2] = (long long)r.values; out[3] = r.has_gt; out[4] = r.gt; out[5] = r.has_lt; out[6] = r.lt;
  out[7] = ksched::req_len_zero(r); out[8] = ksched::req_op_negative(r, d.km);
}
long long kh_mask_allowed(const char* aop, const char* avals) {
  TestDict d;
  return (long long)ksched::req_allowed(spec_req(aop, avals, d.dict), 0x1F, d.km);
}
int kh_mask_compatible(const char* aop, const char* avals, int a_present, const char* bop, const char* bvals, int b_present, int well_known) {
  TestDict d;
  ksched::Req a = spec_req(aop, avals, d.dict), b = spec_req(bop, bvals, d.dict);
  a.present = a_present;
  b.present = b_present;
  return ksched::key_compatible(a, b, well_known != 0, d.km) ? 1 : 0;
}

// Region form of Gt/Lt (ksched.h: ksched_key_regions) against the host algebra: random requirements over a dictionary with
// integer and non-integer values and random thresholds; for every pair the region-form results must equal the converted
// host results (Intersection, Len()==0, Operator negativity, Has over the dictionary, the excluded set, Compatible).
// Returns the number of mismatches.
int kh_region_selftest(unsigned seed, int iters) {
  uint64_t st = seed * 0x9E3779B97F4A7C15ull + 12345;
  auto rnd = [&](int n) { st = st * 6364136223846793005ull + 1442695040888963407ull; return (int)((st >> 33) % (uint64_t)n); };
  const int64_t pool[8] = {0, 1, 2, 3, 5, 7, 9, 10};
  int bad = 0;
  for (int it = 0; it < iters; ++it) {
    // dictionary: bits 0..3 integers 1,2,5,9; bits 4,5 non-integers
    int64_t ints[64] = {1, 2, 5, 9};
    const uint64_t dict = 0x3F;
    ksched::KeyMeta hk{0xF, ints, nullptr};
    std::set<int64_t> tset;
    const int m = rnd(5);
    while ((int)tset.size() < m) tset.insert(pool[rnd(8)]);
    std::vector<int64_t> ts(tset.begin(), tset.end());
    ksched_key_regions g;
    ksched::regions_build(&g, ts.data(), m, 6, dict, hk);
    ksched::KeyMeta rk{0xF, ints, &g};
    auto atom = [&]() {
      ksched::Req r{0, 0, 0, true, true, false, false};
      const int op = rnd(m > 0 ? 6 : 4);
      if (op == 0) { r.complement = false; r.values = (uint64_t)rnd(64); }
      else if (op == 1) { r.values = (uint64_t)rnd(64); }
      else if (op == 2) {}
      else if (op == 3) { r.complement = false; }
      else if (op == 4) { r.has_gt = true; r.gt = ts[(size_t)rnd(m)]; }
      else { r.has_lt = true; r.lt = ts[(size_t)rnd(m)]; }
      return r;
    };
    auto compound = [&]() { ksched::Req r = atom(); for (int i = rnd(3); i > 0; --i) r = ksched::req_intersect(atom(), r, hk); return r; };
    const ksched::Req a = compound(), b = compound();
    ksched::Req ra, rb;
    if (!ksched::req_to_region_form(a, g, dict, &ra) || !ksched::req_to_region_form(b, g, dict, &rb)) { ++bad; continue; }
    const ksched::Req h = ksched::req_intersect(a, b, hk), r = ksched::req_intersect_regions(ra, rb, rk);
    ksched::Req want;
    if (!ksched::req_to_region_form(h, g, dict, &want)) { ++bad; continue; }
    bool ok = want.complement == r.complement && want.values == r.values;
    ok = ok && ksched::req_len_zero(h) == ksched::req_len_zero(r);
    ok = ok && ksched::req_op_negative(h, hk) == ksched::req_op_negative(r, rk);
    ok = ok && ksched::req_op_negative(a, hk) == ksched::req_op_negative(ra, rk);
    ok = ok && ksched::req_allowed(h, dict, hk) == (ksched::req_allowed(r, dict | g.region_mask, rk) & dict);
    if (h.complement) ok = ok && ksched::req_excluded(r, rk) == h.values;
    for (int wk = 0; wk < 2; ++wk)
      for (int pa = 0; pa < 2; ++pa) {
        ksched::Req na = a, nra = ra;
        na.present = nra.present = pa != 0;
        ok = ok && ksched::key_compatible(na, b, wk != 0, hk) ==
                       [&] {  // key_compatible with the region-form intersection (what the device compiles)
                         if (!rb.present) return true;
                         if (!wk && !nra.present && !ksched::req_op_negative(rb, rk)) return false;
                         if (!nra.present) return true;
                         ksched::Req i = ksched::req_intersect_regions(nra, rb, rk);
                         if (!ksched::req_len_zero(i)) return true;
                         return ksched::req_op_negative(rb, rk) && ksched::req_op_negative(nra, rk);
                       }();
      }
    if (!ok) ++bad;
  }
  return bad;
}

// Value classes (khost::value_classes, DESIGN.md §3) against the exact string algebra (requirement.go:117-204). Each
// iteration draws a wide key: 64-143 integer and non-integer values, some of them named, 0-7 thresholds. Over it, requirements
// of the two kinds a problem carries: the named side (In / NotIn over named values, Exists, DoesNotExist, Gt / Lt: pods,
// provisioners, complement instance types) and the type / node side (In over any values: instance types' In requirements,
// node labels). Every pair is evaluated on the strings and on the collapsed masks, in the host algebra and in region form:
// Len() == 0 of the intersection, Operator(), the excluded set, Intersects and Compatible must agree; Has must agree on every
// named value, and on every value when both requirements are from the named side (no requirement tells a class's members
// apart, which is the point). Also: at most m + 2 representatives. Returns the number of mismatches.
int kh_value_class_selftest(unsigned seed, int iters) {
  uint64_t st = seed * 0x9E3779B97F4A7C15ull + 777;
  auto rnd = [&](int n) { st = st * 6364136223846793005ull + 1442695040888963407ull; return (int)((st >> 33) % (uint64_t)n); };
  struct SReq {
    bool present = true, complement = true, has_gt = false, has_lt = false;
    int64_t gt = 0, lt = 0;
    std::set<std::string> values;
  };
  int bad = 0;
  for (int it = 0; it < iters; ++it) {
    std::set<std::string> all;
    std::map<std::string, int64_t> ival;  // strconv.Atoi of the integer values
    const int n_values = 64 + rnd(80);
    while ((int)all.size() < n_values) {
      if (rnd(10) < 6) {
        const int64_t x = rnd(120) - 10;
        const std::string s = (rnd(8) == 0 && x >= 0 ? "0" : "") + std::to_string(x);
        all.insert(s);
        ival[s] = x;
      } else {
        all.insert(std::string(rnd(2) ? "fam-" : "g") + std::to_string(rnd(1000)));
      }
    }
    const std::vector<std::string> pool(all.begin(), all.end());
    std::set<int64_t> tset;
    const int m = rnd(8);
    while ((int)tset.size() < m) tset.insert(rnd(120) - 10);
    const std::vector<int64_t> ts(tset.begin(), tset.end());
    std::set<std::string> named;
    for (int i = rnd(24); i > 0; --i) named.insert(pool[(size_t)rnd((int)pool.size())]);
    const std::map<std::string, std::string> rep_of = khost::value_classes(all, named, tset);
    // the collapsed dictionary, as the encoder builds it
    std::map<std::string, int> id;
    std::vector<std::string> dict_values;
    int64_t ints[64] = {};
    uint64_t int_mask = 0;
    int n_reps = 0;
    for (auto& v : all) {
      auto r = rep_of.find(v);
      if (r != rep_of.end() && r->second != v) continue;
      n_reps += r != rep_of.end();
      const int b = (int)dict_values.size();
      id[v] = b;
      dict_values.push_back(v);
      auto iv = ival.find(v);
      if (iv != ival.end()) { int_mask |= 1ull << b; ints[b] = iv->second; }
    }
    for (auto& kv : rep_of) id[kv.first] = id.at(kv.second);
    const int nd = (int)dict_values.size();
    if (n_reps > m + 2 || nd + m + 1 > 63) { ++bad; continue; }
    const uint64_t dict = (1ull << nd) - 1;
    const ksched::KeyMeta hk{int_mask, ints, nullptr};
    ksched_key_regions g{};
    const bool regions = m > 0 || rnd(2);
    if (regions) ksched::regions_build(&g, ts.data(), m, nd, dict, hk);
    const ksched::KeyMeta rk{int_mask, ints, regions ? &g : nullptr};

    // ---- the string algebra
    auto s_within = [&](const SReq& r, const std::string& v) {
      if (!r.has_gt && !r.has_lt) return true;
      auto iv = ival.find(v);
      return iv != ival.end() && (!r.has_gt || iv->second > r.gt) && (!r.has_lt || iv->second < r.lt);
    };
    auto s_intersect = [&](const SReq& a, const SReq& b) {
      SReq r;
      r.complement = a.complement && b.complement;
      r.has_gt = a.has_gt || b.has_gt;
      r.has_lt = a.has_lt || b.has_lt;
      r.gt = a.has_gt ? (b.has_gt ? std::max(a.gt, b.gt) : a.gt) : b.gt;
      r.lt = a.has_lt ? (b.has_lt ? std::min(a.lt, b.lt) : a.lt) : b.lt;
      if (r.has_gt && r.has_lt && r.gt >= r.lt) { SReq dne; dne.complement = false; return dne; }
      std::set<std::string> v;
      if (a.complement && b.complement) { v = a.values; v.insert(b.values.begin(), b.values.end()); }
      else if (a.complement) { for (auto& x : b.values) if (!a.values.count(x)) v.insert(x); }
      else if (b.complement) { for (auto& x : a.values) if (!b.values.count(x)) v.insert(x); }
      else { for (auto& x : a.values) if (b.values.count(x)) v.insert(x); }
      for (auto& x : v) if (s_within(r, x)) r.values.insert(x);
      if (!r.complement) { r.has_gt = r.has_lt = false; r.gt = r.lt = 0; }
      return r;
    };
    auto s_has = [&](const SReq& r, const std::string& v) { return s_within(r, v) && (r.complement ? !r.values.count(v) : r.values.count(v) > 0); };
    auto s_len_zero = [](const SReq& r) { return !r.complement && r.values.empty(); };
    auto s_negative = [](const SReq& r) { return r.complement ? !r.values.empty() : r.values.empty(); };
    auto s_intersects = [&](const SReq& e, const SReq& i) {
      if (!e.present || !i.present) return true;
      if (!s_len_zero(s_intersect(e, i))) return true;
      return s_negative(i) && s_negative(e);
    };
    auto s_compatible = [&](const SReq& n, const SReq& i, bool wk) {
      if (!i.present) return true;
      if (!wk && !n.present && !s_negative(i)) return false;
      return s_intersects(n, i);
    };
    auto bits = [&](const std::set<std::string>& vs) { uint64_t b = 0; for (auto& v : vs) b |= 1ull << id.at(v); return b; };
    auto to_mask = [&](const SReq& r) { return ksched::Req{bits(r.values), r.gt, r.lt, r.present, r.complement, r.has_gt, r.has_lt}; };

    // ---- random requirements
    const std::vector<std::string> named_list(named.begin(), named.end());
    auto named_atom = [&]() {
      SReq r;
      const int op = rnd(m > 0 ? 6 : 4);
      if ((op == 0 || op == 1) && !named_list.empty()) {
        r.complement = op == 1;
        for (int i = 1 + rnd(3); i > 0; --i) r.values.insert(named_list[(size_t)rnd((int)named_list.size())]);
      }
      else if (op == 3) r.complement = false;
      else if (op == 4) { r.has_gt = true; r.gt = ts[(size_t)rnd(m)]; }
      else if (op == 5) { r.has_lt = true; r.lt = ts[(size_t)rnd(m)]; }
      return r;
    };
    auto named_compound = [&]() { SReq r = named_atom(); for (int i = rnd(3); i > 0; --i) r = s_intersect(named_atom(), r); return r; };
    auto side_atom = [&]() {  // an instance type's In requirement or a node's label
      SReq r;
      r.complement = false;
      for (int i = 1 + rnd(4); i > 0; --i) r.values.insert(pool[(size_t)rnd((int)pool.size())]);
      return r;
    };
    const SReq a = named_compound();
    const bool b_named = rnd(2) != 0;
    const SReq b = b_named ? named_compound() : side_atom();
    const ksched::Req ha = to_mask(a), hb = to_mask(b);
    const SReq si = s_intersect(a, b);
    bool ok = true;
    // host algebra
    const ksched::Req hi = ksched::req_intersect(ha, hb, hk);
    ok = ok && s_len_zero(si) == ksched::req_len_zero(hi);
    ok = ok && s_negative(si) == ksched::req_op_negative(hi, hk) && s_negative(a) == ksched::req_op_negative(ha, hk) &&
         s_negative(b) == ksched::req_op_negative(hb, hk);
    if (si.complement) ok = ok && bits(si.values) == hi.values;
    const uint64_t allowed_a = ksched::req_allowed(ha, dict, hk), allowed_i = ksched::req_allowed(hi, dict, hk);
    for (auto& v : all) {
      ok = ok && s_has(a, v) == (((allowed_a >> id.at(v)) & 1) != 0);
      if (b_named || !rep_of.count(v)) ok = ok && s_has(si, v) == (((allowed_i >> id.at(v)) & 1) != 0);
    }
    for (int wk = 0; wk < 2; ++wk)
      for (int pa = 0; pa < 2; ++pa)
        for (int pb = 0; pb < 2; ++pb) {
          SReq na = a, nb = b;
          na.present = pa != 0;
          nb.present = pb != 0;
          ok = ok && s_compatible(na, nb, wk != 0) == ksched::key_compatible(to_mask(na), to_mask(nb), wk != 0, hk) &&
               s_compatible(nb, na, wk != 0) == ksched::key_compatible(to_mask(nb), to_mask(na), wk != 0, hk);
        }
    // region form (what crosses the C-ABI and what the device computes)
    if (regions) {
      ksched::Req ra, rb;
      if (!ksched::req_to_region_form(ha, g, dict, &ra) || !ksched::req_to_region_form(hb, g, dict, &rb)) { ++bad; continue; }
      const ksched::Req ri = ksched::req_intersect_regions(ra, rb, rk);
      ok = ok && s_len_zero(si) == ksched::req_len_zero(ri) && s_negative(si) == ksched::req_op_negative(ri, rk) &&
           s_negative(a) == ksched::req_op_negative(ra, rk);
      if (si.complement) ok = ok && bits(si.values) == ksched::req_excluded(ri, rk);
      const uint64_t allowed_r = ksched::req_allowed(ri, dict | g.region_mask, rk) & dict;
      for (auto& v : all)
        if (b_named || !rep_of.count(v)) ok = ok && s_has(si, v) == (((allowed_r >> id.at(v)) & 1) != 0);
      for (int wk = 0; wk < 2; ++wk)
        for (int pa = 0; pa < 2; ++pa) {
          SReq na = a;
          na.present = pa != 0;
          ksched::Req nra = ra;
          nra.present = na.present;
          const bool device = [&] {  // key_compatible with the region-form intersection (what the device compiles)
            if (!rb.present) return true;
            if (!wk && !nra.present && !ksched::req_op_negative(rb, rk)) return false;
            if (!nra.present) return true;
            ksched::Req i = ksched::req_intersect_regions(nra, rb, rk);
            if (!ksched::req_len_zero(i)) return true;
            return ksched::req_op_negative(rb, rk) && ksched::req_op_negative(nra, rk);
          }();
          ok = ok && s_compatible(na, b, wk != 0) == device;
        }
    }
    if (!ok) ++bad;
  }
  return bad;
}

// Dictionary facts of one mask key of an encoding (tests): out = [values, representatives of unnamed value classes,
// Gt/Lt thresholds]. Returns -1 when `key` is not a mask key of the encoding.
int kh_encoded_key_info(const Encoded* E, const char* key, long long* out) {
  for (size_t k = 0; k < E->key_names.size(); ++k) {
    if (E->key_names[k] != key) continue;
    out[0] = (long long)E->key_values[k].size();
    out[1] = E->key_representatives[k];
    out[2] = E->key_regions.empty() ? 0 : E->key_regions[k].n_thresholds;
    return 0;
  }
  return -1;
}
}
