// Host-side marshalling of a string-level kmodel::Problem into the flat C-ABI structures of
// include/ksched.h — what a cgo shim would do from the Go objects handed to
// scheduling.NewScheduler (provisioner.go:237-296, scheduler.go:42-78).
#pragma once
#include <algorithm>
#include <cstdlib>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "ksched.h"
#include "model.h"

namespace khost {

// Split [0, n) over the host's cores; fn(begin, end) must only write what it owns. Small inputs stay on the calling thread.
template <class F>
void parallel_ranges(size_t n, size_t min_per_thread, F fn) {
  static const size_t env_threads = [] { const char* e = std::getenv("KSCHED_HOST_THREADS"); return e ? (size_t)std::max(1, std::atoi(e)) : (size_t)0; }();
  size_t nt = env_threads ? env_threads : std::min<size_t>(std::max(1u, std::thread::hardware_concurrency()), 16);
  nt = std::min(nt, std::max<size_t>(1, n / std::max<size_t>(1, min_per_thread)));
  if (nt <= 1) { fn((size_t)0, n); return; }
  std::vector<std::thread> th;
  const size_t per = (n + nt - 1) / nt;
  for (size_t t = 0; t < nt; ++t) {
    const size_t b = t * per, e = std::min(n, b + per);
    if (b >= e) break;
    th.emplace_back([=] { fn(b, e); });
  }
  for (auto& x : th) x.join();
}

struct Encoded {
  // ---- dictionary
  std::vector<std::string> key_names;                 // mask keys
  std::vector<std::vector<std::string>> key_values;   // per key, ascending string order (canonical domain order)
  std::vector<int32_t> key_representatives;           // per key: dictionary values that stand for a class of unnamed values
                                                      // (value_classes below), 0 = every value of the key is its own
  std::vector<std::string> res_names;                 // resource ids: cpu, memory, pods, then ascending
  // ---- which objects take part (provisioner.go:119-144 / deprovisioning/helpers.go:42-93)
  std::vector<const kmodel::Pod*> pods;               // Solve's pod list
  std::vector<int> existing_state_index;              // existing slot -> Problem.nodes index
  std::vector<int32_t> pod_node;                      // cluster_superset: existing slot a batch pod is bound to, -1 = pending
  std::vector<int64_t> existing_capacity;             // cluster_superset: [n_existing][KSCHED_MAX_RES] node capacity (limits bookkeeping)
  std::vector<int32_t> existing_template;
  // cluster_superset with topology groups: what a bound pod that stays contributes to the counters (ksched.h: ksched_cluster)
  std::vector<uint32_t> class_count_begin;
  std::vector<ksched_count_rel> class_count;
  std::vector<int8_t> node_domain;
  std::vector<uint8_t> node_has_hostname_label;
  std::vector<uint32_t> group_filter_match;             // cluster_superset: template whose limits the node's capacity was charged to, or -1
  std::vector<bool> existing_initialized;
  std::vector<int> template_provisioner;              // template v -> Problem.provisioners index
  std::vector<int> type_input_index;                  // column -> Problem.instance_types index
  int type_words = 0;
  const kmodel::Problem* problem_ref = nullptr;       // the problem this encoding was made from (must outlive it)

  // ---- backing storage of the flat structures
  std::vector<ksched_keyinfo> keys;
  std::vector<int64_t> key_int_values;
  std::vector<ksched_key_regions> key_regions;        // [n_keys] or empty: region form of Gt/Lt (ksched.h)
  std::vector<ksched_type_row> types;
  std::vector<int64_t> type_capacity;
  std::vector<uint64_t> offering_keys;                // [n_types][64] launch-choice table (ksched_catalog.offering_keys)
  std::vector<double> price_by_rank;                  // distinct available offering prices, ascending (rank -> price)
  std::vector<ksched_template> templates;
  std::vector<ksched_bounds> template_bounds;
  std::vector<ksched_pod_row> classes;
  std::vector<ksched_bounds> class_bounds;
  bool any_class_bounds = false, any_template_bounds = false;
  std::vector<uint32_t> pod_class;
  std::vector<int64_t> pod_timestamp;
  std::vector<uint32_t> pod_uid_rank;
  std::vector<ksched_existing_node> existing;
  std::vector<ksched_topo_group> groups;
  std::vector<int32_t> group_domain_counts;
  std::vector<int32_t> group_existing_counts;
  std::vector<ksched_class_topo> class_topo;
  std::vector<ksched_reqset> filter_terms;
  std::vector<uint64_t> itype_req_sets;
  std::vector<uint8_t> itype_req_complement;
  std::vector<int32_t> hostname_reqs;
  std::vector<ksched_class_volumes> class_volumes;    // CSI volume limits (ksched.h); empty when no pod mounts a limited claim
  std::vector<ksched_node_volumes> existing_volumes;
  uint64_t volume_driver_mask[KSCHED_MAX_VOLUME_DRIVERS] = {};

  ksched_catalog catalog{};
  ksched_problem problem{};
};

// Throws std::runtime_error; messages starting with "unsupported:" map to KSCHED_ERR_UNSUPPORTED.
// cluster_superset: the encoding ksched_load_cluster wants (ksched.h: ksched_cluster) - the candidates' pods form the batch as
// usual but the candidate nodes STAY existing nodes, with all their pods bound; Encoded::pod_node says where each pod lives.
std::unique_ptr<Encoded> encode(const kmodel::Problem& P, const std::vector<int>& candidates, bool cluster_superset = false);

// Value classes of one label key (DESIGN.md §3). A value is named when some requirement, label or threshold of the problem
// names it (`named`, plus every value equal to one of `thresholds`); no requirement tells apart two unnamed integers of the
// same region between consecutive thresholds (ksched.h: ksched_key_regions), nor two unnamed non-integers. Returns, for every
// unnamed value, its class's representative: the smallest member in string order (which maps to itself).
std::map<std::string, std::string> value_classes(const std::set<std::string>& values, const std::set<std::string>& named,
                                                 const std::set<int64_t>& thresholds);

// metav1.LabelSelectorAsSelector(sel).Matches(labels); a nil selector matches nothing
bool label_selector_matches(const kmodel::LabelSelector& sel, const kmodel::Labels& labels);

// Render one requirement of a reqset the way the oracle's Requirement::Canonical() does ("In [a b]").
std::string render_requirement(const Encoded& E, const ksched_reqset& rs, int key);

}  // namespace khost
