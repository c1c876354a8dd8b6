// ORACLE — TEST INFRASTRUCTURE ONLY (see requirements.h header). Restates, on top of oracle.h:
//   Validation.IsValid / ShouldDeprovision / ValidateCommand   pkg/controllers/deprovisioning/validation.go:63-172
//   candidateNodes / mapNodes / instanceTypesAreSubset          helpers.go:171-249, 328-337, 118-122
//   simulateScheduling's uninitialised-node rule                helpers.go:106-113
//   SingleNodeConsolidation.ComputeCommand                      singlenodeconsolidation.go:43-84
//   MultiNodeConsolidation.ComputeCommand                       multinodeconsolidation.go:41-70
// R7 (DESIGN.md section 6): every validation of one ComputeCommand reads one snapshot, `after`; the TTL wait
// (validation.go:65-76) is the caller's.
#include "validation.h"

#include <algorithm>
#include <cstring>
#include <set>
#include <stdexcept>

namespace oracle {
using namespace kmodel;

std::vector<int> validation_candidates(const Problem& A) {
  std::vector<int> out;
  for (size_t i = 0; i < A.nodes.size(); ++i) {
    const StateNode& n = A.nodes[i];
    if (!A.derive_candidates) {
      if (n.candidate && !n.marked_for_deletion) out.push_back((int)i);
      continue;
    }
    const Provisioner* prov = nullptr;                                     // helpers.go:178-184
    auto pl = n.labels.find(kProvisionerName);
    if (pl != n.labels.end())
      for (auto& pr : A.provisioners) if (pr.name == pl->second) prov = &pr;
    if (n.marked_for_deletion) continue;                                   // :185-188
    if (!prov) continue;                                                   // :189-192
    auto itn = n.labels.find(kInstanceType);                               // :194-198
    bool it_ok = false;
    if (itn != n.labels.end())
      for (int t : prov->instance_types) if (A.instance_types[(size_t)t].name == itn->second) it_ok = true;
    if (!it_ok) continue;
    if (!n.labels.count(kCapacityType) || !n.labels.count(kZone)) continue;  // :200-208
    auto ini = n.labels.find(kInitialized);                                // :210-213
    if (ini == n.labels.end() || ini->second != "true") continue;
    if (n.nominated) continue;                                             // :214-217
    // Validation.ShouldDeprovision (validation.go:102-107): the do-not-consolidate annotation decides when present
    const bool ok = n.do_not_consolidate != 0 ? n.do_not_consolidate != 1 : prov->consolidation_enabled;
    if (ok) out.push_back((int)i);
  }
  return out;
}

Command command_of(const Problem& B, const std::vector<int>& nodes, int action, const std::vector<int>& options) {
  Command c;
  c.action = action;
  for (int i : nodes) c.nodes.push_back(B.nodes.at((size_t)i).name);
  for (int t : options) c.options.push_back(B.instance_types.at((size_t)t).name);
  return c;
}

bool is_valid(const Problem& A, const std::vector<int>& cands, const Command& cmd) {
  const std::set<std::string> names(cmd.nodes.begin(), cmd.nodes.end());
  for (auto& n : A.nodes)                                                  // validation.go:85-91 (IsNodeNominated)
    if (names.count(n.name) && n.nominated) return false;
  std::vector<int> mapped;                                                 // mapNodes helpers.go:328-337
  for (int i : cands) if (names.count(A.nodes[(size_t)i].name)) mapped.push_back(i);
  if (mapped.empty()) return false;                                        // validation.go:112-116
  Result r;                                                                // simulateScheduling helpers.go:42-115
  solve(A, mapped, r);
  if (!r.error.empty()) throw std::runtime_error(r.error);
  for (int e : r.existing_node_index) {                                    // helpers.go:106-113
    auto ini = A.nodes[(size_t)e].labels.find(kInitialized);
    if (ini == A.nodes[(size_t)e].labels.end() || ini->second != "true") return false;
  }
  for (int a : r.assign) if (a < 0) return false;                          // validation.go:122-124
  if (r.new_nodes.empty()) return cmd.action == 1;                         // :132-140
  if (r.new_nodes.size() > 1) return false;                                // :142-145
  if (cmd.action != 2) return false;                                       // :147-151
  std::set<std::string> rhs;                                               // instanceTypesAreSubset helpers.go:118-122
  for (int t : node_options(r, r.new_nodes[0])) rhs.insert(A.instance_types[(size_t)t].name);
  for (auto& o : cmd.options) if (!rhs.count(o)) return false;             // validation.go:164-166
  return true;
}

void single_compute_command(const Problem& B, const Problem& A, int first, int last, ValidatedCommand& out) {
  out = ValidatedCommand();
  std::vector<int> order;
  std::vector<double> cost;
  rank_candidates(B, &order, &cost);                                       // sortAndFilterCandidates :47-50
  const int n = (int)order.size();
  if (last < 0 || last > n) last = n;
  std::vector<int> cands;
  bool have_cands = false;                                                 // built at the first validation (validation.go:78-83)
  for (int pos = std::max(first, 0); pos < last; ++pos) {                  // singlenodeconsolidation.go:54-78
    ConsolidationResult r;
    consolidate_single(B, r, pos);
    if (!r.error.empty()) throw std::runtime_error(r.error);
    if (r.action != 1 && r.action != 2) continue;                          // :61-63
    if (!have_cands) { cands = validation_candidates(A); have_cands = true; }
    const bool ok = is_valid(A, cands, command_of(B, {order[(size_t)pos]}, r.action, r.replacement_options));
    out.validations.push_back({pos, ok});
    if (!ok) { out.failed_validation = true; continue; }                  // :70-73
    out.action = r.action;                                                 // :75-77
    out.position = pos;
    out.node = order[(size_t)pos];
    out.options = r.replacement_options;
    return;
  }
  out.action = out.failed_validation ? kActionRetry : 0;                   // :80-84
}

void multi_compute_command(const Problem& B, const Problem& A, ValidatedCommand& out) {
  out = ValidatedCommand();
  consolidate(B, out.search);                                              // firstNNodeConsolidationOption :50-55
  if (!out.search.error.empty()) throw std::runtime_error(out.search.error);
  out.action = out.search.action;
  if (out.action != 1 && out.action != 2) return;                          // :56-58
  const int k = out.search.nodes_removed;
  std::vector<int> nodes(out.search.candidate_order.begin(), out.search.candidate_order.begin() + k);
  const bool ok = is_valid(A, validation_candidates(A), command_of(B, nodes, out.action, out.search.replacement_options));  // :60-64
  out.validations.push_back({k, ok});
  if (!ok) { out.action = kActionRetry; out.failed_validation = true; return; }  // :66-68
  out.nodes_removed = k;
  out.options = out.search.replacement_options;
}

}  // namespace oracle

using namespace oracle;

static int put_err(const std::exception& e, char* err, int cap) {
  if (err && cap > 0) { std::strncpy(err, e.what(), (size_t)cap - 1); err[cap - 1] = 0; }
  return -1;
}

extern "C" {
// Validation.IsValid of the command removing before.nodes[nodes] (action 1 / 2, options = before.instance_types indices)
// against `after`. Returns 1 valid, 0 invalid, -1 error.
int oracle_is_valid(const Problem* B, const Problem* A, const int* nodes, int n_nodes, int action, const int* options, int n_options, char* err,
                    int err_cap) {
  try {
    Command c = command_of(*B, std::vector<int>(nodes, nodes + n_nodes), action, std::vector<int>(options, options + n_options));
    return is_valid(*A, validation_candidates(*A), c) ? 1 : 0;
  } catch (const std::exception& e) {
    return put_err(e, err, err_cap);
  }
}

// SingleNodeConsolidation.ComputeCommand with validation. out3 = [action, position, node]; trace / trace_valid =
// the validations in order. Returns 0 or -1 (err).
int oracle_single_compute_command(const Problem* B, const Problem* A, int first, int last, int* out3, int* options, int options_cap, int* n_options,
                                  int* trace, int* trace_valid, int trace_cap, int* n_trace, int* failed, char* err, int err_cap) {
  try {
    ValidatedCommand v;
    single_compute_command(*B, *A, first, last, v);
    out3[0] = v.action; out3[1] = v.position; out3[2] = v.node;
    *n_options = (int)v.options.size();
    for (int i = 0; i < *n_options && i < options_cap; ++i) options[i] = v.options[(size_t)i];
    *n_trace = (int)v.validations.size();
    for (int i = 0; i < *n_trace && i < trace_cap; ++i) { trace[i] = v.validations[(size_t)i].first; trace_valid[i] = v.validations[(size_t)i].second; }
    *failed = v.failed_validation ? 1 : 0;
    return 0;
  } catch (const std::exception& e) {
    return put_err(e, err, err_cap);
  }
}

// MultiNodeConsolidation.ComputeCommand. out3 = [action, nodes_removed, simulations]; probes / probe_actions = the search;
// *verdict = 1 valid, 0 invalid, -1 nothing validated. Returns 0 or -1 (err).
int oracle_multi_compute_command(const Problem* B, const Problem* A, int* out3, int* options, int options_cap, int* n_options, int* probes,
                                 int* probe_actions, int probes_cap, int* n_probes, int* verdict, char* err, int err_cap) {
  try {
    ValidatedCommand v;
    multi_compute_command(*B, *A, v);
    out3[0] = v.action; out3[1] = v.nodes_removed; out3[2] = v.search.simulations;
    *n_options = (int)v.options.size();
    for (int i = 0; i < *n_options && i < options_cap; ++i) options[i] = v.options[(size_t)i];
    *n_probes = (int)v.search.probes.size();
    for (int i = 0; i < *n_probes && i < probes_cap; ++i) { probes[i] = v.search.probes[(size_t)i]; probe_actions[i] = v.search.probe_actions[(size_t)i]; }
    *verdict = v.validations.empty() ? -1 : v.validations[0].second ? 1 : 0;
    return 0;
  } catch (const std::exception& e) {
    return put_err(e, err, err_cap);
  }
}
}
