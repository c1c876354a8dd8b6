// String-level data model for the Scheduler.Solve hot path.
//
// These plain structs mirror the Go objects that cross into
// pkg/controllers/provisioning/scheduling.NewScheduler / Scheduler.Solve in the
// reference (scheduler.go:42-45, :96): v1.Pod (only the fields the solver reads),
// cloudprovider.InstanceType / Offering (pkg/cloudprovider/types.go:72-113),
// v1alpha5.Provisioner (pkg/apis/v1alpha5/provisioner.go), state.Node
// (pkg/controllers/state/node.go). A cgo shim would fill the flat C-ABI
// (include/ksched.h) directly from the Go objects; in this repo the C++ host
// layer (encoder.cc) does that encoding from these structs.
//
// Resource quantities are int64 MILLI-units (k8s resource.Quantity is exact
// decimal; every quantity the reference tests use is a whole number of milli).
#pragma once
#include <atomic>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace kmodel {

using ResourceList = std::map<std::string, int64_t>;  // name -> milli-units
using Labels = std::map<std::string, std::string>;

enum class Op : uint8_t { In, NotIn, Exists, DoesNotExist, Gt, Lt };

// v1.NodeSelectorRequirement
struct NodeSelectorRequirement {
  std::string key;
  Op op = Op::In;
  std::vector<std::string> values;
};
using NodeSelectorTerm = std::vector<NodeSelectorRequirement>;  // MatchExpressions

struct PreferredSchedulingTerm {
  int32_t weight = 0;
  NodeSelectorTerm preference;
};

// metav1.LabelSelector. is_nil mirrors a nil *LabelSelector (selects nothing,
// topologygroup.go:246-252 via LabelSelectorAsSelector(nil) = Nothing()).
struct LabelSelector {
  bool is_nil = true;
  Labels match_labels;
  std::vector<NodeSelectorRequirement> match_expressions;  // In/NotIn/Exists/DoesNotExist
};

struct PodAffinityTerm {
  LabelSelector selector;
  std::vector<std::string> namespaces;
  std::string topology_key;
};
struct WeightedPodAffinityTerm {
  int32_t weight = 0;
  PodAffinityTerm term;
};

struct TopologySpreadConstraint {
  int32_t max_skew = 1;
  std::string topology_key;
  bool schedule_anyway = false;  // WhenUnsatisfiable == ScheduleAnyway
  LabelSelector selector;
};

struct Toleration {
  std::string key;
  std::string op;  // "", "Equal", "Exists"
  std::string value;
  std::string effect;  // "" matches all effects
};
struct Taint {
  std::string key, value, effect;
};

struct HostPort {
  std::string ip;  // "" == 0.0.0.0 (hostportusage.go:125-130)
  int32_t port = 0;
  std::string protocol;
};

struct Container {
  ResourceList requests, limits;
  std::vector<HostPort> ports;
};

// One volume of a pod as the host resolved it (volumeusage.go:133-190 does the API Gets: PVC -> storage class / bound PV ->
// CSI driver name). driver "" = a non-CSI volume, which the reference does not track.
struct PodVolume {
  std::string driver, pvc_id;  // pvc_id = "<namespace>/<claim>" (or the generated ephemeral claim name)
};

struct Pod {
  std::string name, ns = "default", uid;
  int64_t creation_ts = 0;
  Labels labels;
  std::vector<Container> containers, init_containers;
  Labels node_selector;
  bool has_node_affinity = false;
  bool has_required_node_affinity = false;             // Required... != nil
  std::vector<NodeSelectorTerm> required_node_terms;   // OR'd NodeSelectorTerms
  std::vector<PreferredSchedulingTerm> preferred_node_terms;
  std::vector<PodAffinityTerm> pod_affinity_required;
  std::vector<WeightedPodAffinityTerm> pod_affinity_preferred;
  std::vector<PodAffinityTerm> pod_anti_affinity_required;
  std::vector<WeightedPodAffinityTerm> pod_anti_affinity_preferred;
  std::vector<TopologySpreadConstraint> topology_spread;
  std::vector<Toleration> tolerations;
  // only meaningful for pods already bound to a node (cluster state)
  std::string node_name;
  bool is_daemonset = false;
  bool terminal = false, terminating = false;
  std::vector<PodVolume> volumes;           // Spec.Volumes that are PVC / ephemeral claims (existingnode.go:91-96)
  // deprovisioning candidate ranking (deprovisioning/helpers.go:125-165,339-366)
  bool has_deletion_cost = false;           // controller.kubernetes.io/pod-deletion-cost annotation parsed as a float
  double deletion_cost = 0;
  bool has_priority = false;                // Spec.Priority != nil
  int32_t priority = 0;
  bool do_not_evict = false;                // karpenter.sh/do-not-evict: "true"
  bool owned_by_node = false;               // static / mirror pod (ownerReference v1 Node)
};

struct Offering {
  std::string capacity_type, zone;
  double price = 0;
  bool available = true;
};

struct InstanceType {
  std::string name;
  std::vector<NodeSelectorRequirement> requirements;
  std::vector<Offering> offerings;
  ResourceList capacity;
  ResourceList kube_reserved, system_reserved, eviction_threshold;
};

struct Provisioner {
  std::string name;
  int32_t weight = 0;
  std::vector<NodeSelectorRequirement> requirements;
  Labels labels;
  std::vector<Taint> taints, startup_taints;
  bool has_limits = false;  // Spec.Limits != nil
  ResourceList limits;
  bool consolidation_enabled = false;       // Spec.Consolidation.Enabled (consolidation.go:104-118)
  bool has_ttl_until_expired = false;       // Spec.TTLSecondsUntilExpired != nil (helpers.go:275-287)
  int64_t ttl_seconds_until_expired = 0;
  std::vector<int32_t> instance_types;  // indices into Problem.instance_types (GetInstanceTypes result)
};

// state.Node as NewScheduler sees it (deep copy of the cluster cache).
struct StateNode {
  std::string name;
  Labels labels;
  std::vector<Taint> taints;          // Node.Spec.Taints
  std::vector<Taint> startup_taints;  // from the owning provisioner
  ResourceList allocatable, capacity;
  std::vector<Pod> pods;              // pods bound to the node (incl. daemonset pods)
  bool marked_for_deletion = false;
  // consolidation candidate data (deprovisioning/helpers.go:171-249)
  bool candidate = false;
  double disruption_cost = 0;
  // raw inputs of candidateNodes / sortAndFilterCandidates (used when Problem.derive_candidates is set)
  bool deleting = false;                    // DeletionTimestamp != nil (helpers.go:340)
  bool nominated = false;                   // state.Node.Nominated()
  int8_t do_not_consolidate = 0;            // karpenter.sh/do-not-consolidate annotation: 0 absent, 1 "true", 2 any other value
  double creation_ts = 0;                   // seconds (node.CreationTimestamp)
  std::map<std::string, int32_t> volume_limits;  // CSINode driver -> Allocatable.Count (state/cluster.go:292-303)
};

// policy/v1 PodDisruptionBudget as PDBLimits reads it (deprovisioning/pdblimits.go:34-80)
struct PodDisruptionBudget {
  std::string ns;
  LabelSelector selector;
  int32_t disruptions_allowed = 0;
};

// Derived, dictionary-independent facts about the cluster state that every encoding of the same Problem needs again
// (consolidation encodes one Problem once per probe): filled lazily by the encoder, owned by the Problem.
struct ProblemDerived {
  virtual ~ProblemDerived() = default;
};

// A process-unique id per Problem: a cache keyed on a Problem must not take a new Problem at a freed one's address for it.
inline uint64_t next_problem_id() {
  static std::atomic<uint64_t> last{0};
  return ++last;
}

struct Problem {
  const uint64_t id = next_problem_id();
  mutable std::shared_ptr<ProblemDerived> derived;   // see khost::encode; a Problem is immutable once built
  mutable std::mutex derived_mu;
  std::vector<std::string> extra_well_known_labels;  // v1alpha5.WellKnownLabels additions
  std::vector<InstanceType> instance_types;
  std::vector<Provisioner> provisioners;  // caller order; OrderByWeight applied by the solver
  std::vector<StateNode> nodes;
  std::vector<Pod> pods;            // pending pods handed to Solve
  std::vector<Pod> daemonset_pods;  // daemonset template pods (getDaemonSetPods)
  std::vector<PodDisruptionBudget> pdbs;
  double now_ts = 0;                 // the clock candidateNodes reads (seconds)
  bool derive_candidates = false;    // candidate / disruption_cost of every node come from rank_candidates, not from the fields
  bool simulation_mode = false;
  bool empty_topology = false;  // benchmark passes &scheduling.Topology{} (scheduling_benchmark_test.go:123)
};

// One new node in the result, in s.newNodes append order.
struct NewNodeResult {
  int32_t provisioner = -1;                   // index into the weight-ordered provisioner list
  std::vector<int32_t> pods;                  // indices into Problem.pods, in Add order
  std::vector<int32_t> instance_type_options; // indices into Problem.instance_types, input order preserved
  int32_t option_set = -1;                    // >= 0: the options are Result::option_sets[option_set] (nodes of one deployment share their set)
  ResourceList requests;
  // final requirement per key (hostname removed), rendered "key Op [v1 v2]" style for comparison
  std::map<std::string, std::string> requirements;
  // what the cloud provider would launch (fake/cloudprovider.go:74-84, cloudprovider/types.go:128-145); -1 = not computed
  int32_t launch_type = -1;                   // index into Problem.instance_types
  std::string launch_capacity_type, launch_zone;
  double launch_price = 0;
};

struct Result {
  std::vector<int32_t> assign;        // per pod: -1 unscheduled; [0,E) existing node idx; E+i new node i
  std::vector<int32_t> relax_level;   // per pod: number of successful Relax calls
  std::vector<NewNodeResult> new_nodes;
  std::vector<std::vector<int32_t>> option_sets;  // distinct InstanceTypeOptions lists, shared by the nodes that name them
  std::vector<int32_t> existing_node_index;  // s.existingNodes[i] -> index into Problem.nodes
  std::vector<std::vector<int32_t>> existing_pods;  // per existing node: pods in Add order
  int64_t nodes_visited = 0;  // sum over Add attempts of candidate nodes examined (SURVEY 8d K2 bytes)
  int64_t add_calls = 0;      // number of Scheduler.add calls (queue pops)
  std::string error;
};

// InstanceTypeOptions of a new node: its own list, or the shared one it names
inline const std::vector<int32_t>& node_options(const Result& r, const NewNodeResult& n) {
  return n.option_set >= 0 ? r.option_sets[(size_t)n.option_set] : n.instance_type_options;
}

}  // namespace kmodel
