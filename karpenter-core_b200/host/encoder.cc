// Problem -> flat C-ABI encoder (see encoder.h). Product code: it must not use anything under oracle/.
//
// Reference steps restated here because they happen before Solve, on the host, in the reference too:
//   provisioner.go:237-296   template order, instance types per provisioner, domain universe
//   scheduler.go:221-267     daemonset overhead, existing nodes, remaining provisioner limits
//   topology.go:56-117,183-322  topology groups, owners, inverse anti-affinity groups, countDomains
//   preferences.go:36-145    the relaxation chain of every pod (pre-computed as classes)
#include "encoder.h"

#include <algorithm>
#include <cmath>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <set>
#include <stdexcept>
#include <thread>

#include "reqmask.cuh"

namespace khost {
using namespace kmodel;
using ksched::KeyMeta;
using ksched::Req;

namespace {

[[noreturn]] void unsupported(const std::string& what) { throw std::runtime_error("unsupported: " + what); }

const char* kHostname = "kubernetes.io/hostname";
const char* kZone = "topology.kubernetes.io/zone";
const char* kCapacityType = "karpenter.sh/capacity-type";
const char* kProvisionerName = "karpenter.sh/provisioner-name";
const char* kInitialized = "karpenter.sh/initialized";
const char* kInstanceType = "node.kubernetes.io/instance-type";

std::string normalize_key(const std::string& k) {  // v1alpha5.NormalizedLabels, labels.go:103-109
  if (k == "failure-domain.beta.kubernetes.io/zone") return kZone;
  if (k == "beta.kubernetes.io/arch") return "kubernetes.io/arch";
  if (k == "beta.kubernetes.io/os") return "kubernetes.io/os";
  if (k == "beta.kubernetes.io/instance-type") return kInstanceType;
  if (k == "failure-domain.beta.kubernetes.io/region") return "topology.kubernetes.io/region";
  return k;
}

bool parse_int(const std::string& s, int64_t* out) {  // strconv.Atoi: optional sign, decimal digits, must fit in int64
  if (s.empty()) return false;
  size_t i = 0;
  bool neg = false;
  if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
  if (i >= s.size()) return false;
  unsigned __int128 v = 0;
  const unsigned __int128 lim = neg ? ((unsigned __int128)1 << 63) : (((unsigned __int128)1 << 63) - 1);
  for (; i < s.size(); ++i) {
    if (s[i] < '0' || s[i] > '9') return false;
    v = v * 10 + (unsigned)(s[i] - '0');
    if (v > lim) return false;
  }
  *out = neg ? (int64_t)(0 - (uint64_t)v) : (int64_t)v;
  return true;
}

// ---- resources (utils/resources/resources.go)
ResourceList merge(const ResourceList& a, const ResourceList& b) {
  ResourceList r = a;
  for (auto& kv : b) r[kv.first] += kv.second;
  return r;
}
ResourceList pod_requests(const Pod& p) {  // RequestsForPods(pod): Ceiling + pods:1
  ResourceList r;
  auto eff = [](const Container& c) {
    ResourceList x = c.requests;
    for (auto& kv : c.limits) if (!x.count(kv.first)) x[kv.first] = kv.second;
    return x;
  };
  for (auto& c : p.containers) r = merge(r, eff(c));
  for (auto& c : p.init_containers) {
    ResourceList x = eff(c);
    for (auto& kv : x) {
      auto it = r.find(kv.first);
      if (it == r.end() || kv.second > it->second) r[kv.first] = kv.second;
    }
  }
  r["pods"] = 1000;
  return r;
}

// ---- tolerations (k8s.io/api core/v1 Toleration.ToleratesTaint)
bool tolerates_taint(const Toleration& t, const Taint& taint) {
  if (!t.effect.empty() && t.effect != taint.effect) return false;
  if (!t.key.empty() && t.key != taint.key) return false;
  if (t.op.empty() || t.op == "Equal") return t.value == taint.value;
  return t.op == "Exists";
}
bool tolerates_all(const std::vector<Taint>& taints, const std::vector<Toleration>& tols) {  // taints.go:28-40
  for (auto& taint : taints) {
    bool ok = false;
    for (auto& t : tols) ok = ok || tolerates_taint(t, taint);
    if (!ok) return false;
  }
  return true;
}
std::string taints_key(const std::vector<Taint>& ts) {
  std::string s;
  for (auto& t : ts) s += t.key + "=" + t.value + ":" + t.effect + ";";
  return s;
}

// ---- label selectors (apimachinery): nil -> nothing, invalid -> nothing
bool selector_valid(const LabelSelector& s) {
  for (auto& e : s.match_expressions) {
    if ((e.op == Op::In || e.op == Op::NotIn) && e.values.empty()) return false;
    if ((e.op == Op::Exists || e.op == Op::DoesNotExist) && !e.values.empty()) return false;
    if (e.op == Op::Gt || e.op == Op::Lt) return false;
  }
  return true;
}
bool selector_matches(const LabelSelector& s, const Labels& labels) {  // s non-nil
  if (!selector_valid(s)) return false;
  for (auto& kv : s.match_labels) {
    auto it = labels.find(kv.first);
    if (it == labels.end() || it->second != kv.second) return false;
  }
  for (auto& e : s.match_expressions) {
    auto it = labels.find(e.key);
    bool has = it != labels.end();
    bool in = has && std::find(e.values.begin(), e.values.end(), it->second) != e.values.end();
    if (e.op == Op::In && !in) return false;
    if (e.op == Op::NotIn && has && in) return false;
    if (e.op == Op::Exists && !has) return false;
    if (e.op == Op::DoesNotExist && has) return false;
  }
  return true;
}
std::string selector_key(const LabelSelector& s) {
  if (s.is_nil) return "<nil>";
  std::string out = "{";
  for (auto& kv : s.match_labels) out += kv.first + "=" + kv.second + ",";
  out += "|";
  std::vector<std::string> ex;
  for (auto& e : s.match_expressions) {
    std::string x = e.key + ":" + std::to_string((int)e.op) + ":";
    std::vector<std::string> v = e.values;
    std::sort(v.begin(), v.end());
    for (auto& y : v) x += y + ",";
    ex.push_back(x);
  }
  std::sort(ex.begin(), ex.end());
  for (auto& x : ex) out += x + ";";
  return out + "}";
}

std::string reqs_key(const std::vector<NodeSelectorRequirement>& rs) {
  std::string s;
  for (auto& r : rs) {
    s += normalize_key(r.key) + ":" + std::to_string((int)r.op) + ":";
    for (auto& v : r.values) s += v + ",";
    s += ";";
  }
  return s;
}
std::string labels_key(const Labels& l) {
  std::string s;
  for (auto& kv : l) s += kv.first + "=" + kv.second + ",";
  return s;
}
std::string term_key(const PodAffinityTerm& t) {
  std::string s = t.topology_key + "|" + selector_key(t.selector) + "|";
  for (auto& n : t.namespaces) s += n + ",";
  return s;
}

// Structural equality of everything class_key reads (a SUFFICIENT condition for "same class": two pods whose containers
// differ but sum to the same requests still share a class, they just take the keyed path below). Consecutive pods of a batch
// usually come from one deployment, so the per-pod cost of interning is one such comparison instead of a key string.
bool same_reqs(const std::vector<NodeSelectorRequirement>& a, const std::vector<NodeSelectorRequirement>& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i) if (a[i].key != b[i].key || a[i].op != b[i].op || a[i].values != b[i].values) return false;
  return true;
}
bool same_selector(const LabelSelector& a, const LabelSelector& b) {
  return a.is_nil == b.is_nil && a.match_labels == b.match_labels && same_reqs(a.match_expressions, b.match_expressions);
}
bool same_term(const PodAffinityTerm& a, const PodAffinityTerm& b) {
  return a.topology_key == b.topology_key && a.namespaces == b.namespaces && same_selector(a.selector, b.selector);
}
template <class T, class F>
bool same_vec(const std::vector<T>& a, const std::vector<T>& b, F eq) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i) if (!eq(a[i], b[i])) return false;
  return true;
}
bool same_container(const Container& a, const Container& b) {
  return a.requests == b.requests && a.limits == b.limits &&
         same_vec(a.ports, b.ports, [](const HostPort& x, const HostPort& y) { return x.ip == y.ip && x.port == y.port && x.protocol == y.protocol; });
}
bool same_spec(const Pod& a, const Pod& b) {
  auto wterm = [](const WeightedPodAffinityTerm& x, const WeightedPodAffinityTerm& y) { return x.weight == y.weight && same_term(x.term, y.term); };
  if (!a.volumes.empty() || !b.volumes.empty()) return false;  // claims are per pod: the keyed path decides (volume signature)
  return a.ns == b.ns && a.labels == b.labels && same_vec(a.containers, b.containers, same_container) &&
         same_vec(a.init_containers, b.init_containers, same_container) && a.node_selector == b.node_selector &&
         a.has_node_affinity == b.has_node_affinity && a.has_required_node_affinity == b.has_required_node_affinity &&
         same_vec(a.required_node_terms, b.required_node_terms, same_reqs) &&
         same_vec(a.preferred_node_terms, b.preferred_node_terms,
                  [](const PreferredSchedulingTerm& x, const PreferredSchedulingTerm& y) { return x.weight == y.weight && same_reqs(x.preference, y.preference); }) &&
         same_vec(a.pod_affinity_required, b.pod_affinity_required, same_term) && same_vec(a.pod_affinity_preferred, b.pod_affinity_preferred, wterm) &&
         same_vec(a.pod_anti_affinity_required, b.pod_anti_affinity_required, same_term) &&
         same_vec(a.pod_anti_affinity_preferred, b.pod_anti_affinity_preferred, wterm) &&
         same_vec(a.topology_spread, b.topology_spread,
                  [](const TopologySpreadConstraint& x, const TopologySpreadConstraint& y) {
                    return x.max_skew == y.max_skew && x.topology_key == y.topology_key && x.schedule_anyway == y.schedule_anyway && same_selector(x.selector, y.selector);
                  }) &&
         same_vec(a.tolerations, b.tolerations,
                  [](const Toleration& x, const Toleration& y) { return x.key == y.key && x.op == y.op && x.value == y.value && x.effect == y.effect; });
}

// A hash of (a subset of) what same_spec compares: equal specs hash equally, so a pod that starts a new run of its batch
// finds the class of an earlier run by hash + one same_spec against that class's first pod, without building the key string.
uint64_t spec_hash(const Pod& p) {
  uint64_t h = 0xcbf29ce484222325ull;
  auto mix = [&](uint64_t v) { h = (h ^ v) * 0x100000001b3ull; h ^= h >> 29; };
  auto str = [&](const std::string& x) { mix(x.size()); for (unsigned char ch : x) h = (h ^ ch) * 0x100000001b3ull; };
  auto labels = [&](const Labels& l) { mix(l.size()); for (auto& kv : l) { str(kv.first); str(kv.second); } };
  auto resources = [&](const ResourceList& r) { mix(r.size()); for (auto& kv : r) { str(kv.first); mix((uint64_t)kv.second); } };
  auto containers = [&](const std::vector<Container>& cs) {
    mix(cs.size());
    for (auto& c : cs) { resources(c.requests); resources(c.limits); mix(c.ports.size()); for (auto& hp : c.ports) mix((uint64_t)hp.port); }
  };
  str(p.ns);
  labels(p.labels);
  containers(p.containers);
  containers(p.init_containers);
  labels(p.node_selector);
  mix((uint64_t)p.has_node_affinity * 2 + (uint64_t)p.has_required_node_affinity);
  mix(p.required_node_terms.size());
  for (auto& t : p.required_node_terms) { mix(t.size()); for (auto& r : t) { str(r.key); mix((uint64_t)r.op); mix(r.values.size()); } }
  mix(p.preferred_node_terms.size());
  for (auto& t : p.preferred_node_terms) mix((uint64_t)t.weight);
  mix(p.pod_affinity_required.size());
  for (auto& t : p.pod_affinity_required) str(t.topology_key);
  mix(p.pod_affinity_preferred.size());
  mix(p.pod_anti_affinity_required.size());
  for (auto& t : p.pod_anti_affinity_required) str(t.topology_key);
  mix(p.pod_anti_affinity_preferred.size());
  mix(p.topology_spread.size());
  for (auto& t : p.topology_spread) { mix((uint64_t)t.max_skew); str(t.topology_key); mix((uint64_t)t.schedule_anyway); }
  mix(p.tolerations.size());
  for (auto& t : p.tolerations) { str(t.key); str(t.effect); }
  return h;
}

// Everything the scheduler can observe about a pod except its identity (uid / name / timestamp).
std::string class_key(const Pod& p, const ResourceList& req) {
  // built by appending in place (no temporaries): this runs once per pod of the batch
  std::string s;
  s.reserve(256);
  auto num = [&](long long v) { char b[24]; int n = std::snprintf(b, sizeof b, "%lld", v); s.append(b, (size_t)n); };
  s += "ns="; s += p.ns; s += "|L="; s += labels_key(p.labels); s += "|R=";
  for (auto& kv : req) { s += kv.first; s += ':'; num(kv.second); s += ','; }
  s += "|S="; s += labels_key(p.node_selector); s += "|NA="; num(p.has_node_affinity); num(p.has_required_node_affinity);
  for (auto& t : p.required_node_terms) { s += '['; s += reqs_key(t); s += ']'; }
  s += "|NP=";
  for (auto& t : p.preferred_node_terms) { num(t.weight); s += '['; s += reqs_key(t.preference); s += ']'; }
  s += "|PA=";
  for (auto& t : p.pod_affinity_required) { s += '('; s += term_key(t); s += ')'; }
  s += "|PAP=";
  for (auto& t : p.pod_affinity_preferred) { num(t.weight); s += '('; s += term_key(t.term); s += ')'; }
  s += "|PAA=";
  for (auto& t : p.pod_anti_affinity_required) { s += '('; s += term_key(t); s += ')'; }
  s += "|PAAP=";
  for (auto& t : p.pod_anti_affinity_preferred) { num(t.weight); s += '('; s += term_key(t.term); s += ')'; }
  s += "|TS=";
  for (auto& t : p.topology_spread) {
    num(t.max_skew); s += ':'; s += t.topology_key; s += ':'; num(t.schedule_anyway); s += ':'; s += selector_key(t.selector); s += ';';
  }
  s += "|T=";
  for (auto& t : p.tolerations) { s += t.key; s += ':'; s += t.op; s += ':'; s += t.value; s += ':'; s += t.effect; s += ';'; }
  s += "|HP=";
  for (auto& c : p.containers)
    for (auto& hp : c.ports) { s += hp.ip; s += ':'; num(hp.port); s += ':'; s += hp.protocol; s += ';'; }
  return s;
}

// ---- Preferences.Relax restated (preferences.go:36-145); sorts are stable (tie order is unpinned in Go)
template <class T>
bool remove_heaviest(std::vector<T>& terms) {
  if (terms.empty()) return false;
  std::stable_sort(terms.begin(), terms.end(), [](const T& a, const T& b) { return a.weight > b.weight; });
  terms.erase(terms.begin());
  return true;
}
bool relax(Pod& p, bool tolerate_prefer_no_schedule) {
  if (p.has_node_affinity && p.has_required_node_affinity && p.required_node_terms.size() > 1) {
    p.required_node_terms.erase(p.required_node_terms.begin());
    return true;
  }
  if (remove_heaviest(p.pod_affinity_preferred)) return true;
  if (remove_heaviest(p.pod_anti_affinity_preferred)) return true;
  if (p.has_node_affinity && remove_heaviest(p.preferred_node_terms)) return true;
  for (size_t i = 0; i < p.topology_spread.size(); ++i)
    if (p.topology_spread[i].schedule_anyway) {
      p.topology_spread[i] = p.topology_spread.back();
      p.topology_spread.pop_back();
      return true;
    }
  if (tolerate_prefer_no_schedule) {
    for (auto& x : p.tolerations)
      if (x.key.empty() && x.effect == "PreferNoSchedule" && x.op == "Exists" && x.value.empty()) return false;
    p.tolerations.push_back({"", "Exists", "", "PreferNoSchedule"});
    return true;
  }
  return false;
}

struct HostPortEntry {
  std::string ip;
  int32_t port;
  std::string protocol;
  bool operator<(const HostPortEntry& o) const { return std::tie(ip, port, protocol) < std::tie(o.ip, o.port, o.protocol); }
};
bool ip_unspecified(const std::string& ip) { return ip == "0.0.0.0" || ip == "::"; }
bool hp_matches(const HostPortEntry& a, const HostPortEntry& b) {  // hostportusage.go:45-57
  if (a.protocol != b.protocol || a.port != b.port) return false;
  return a.ip == b.ip || ip_unspecified(a.ip) || ip_unspecified(b.ip);
}
std::vector<HostPortEntry> host_ports(const Pod& p) {  // hostportusage.go:118-144
  std::vector<HostPortEntry> out;
  for (auto& c : p.containers)
    for (auto& hp : c.ports)
      if (hp.port != 0) out.push_back({hp.ip.empty() ? "0.0.0.0" : hp.ip, hp.port, hp.protocol});
  return out;
}

// Facts about the cluster state that do not depend on which nodes are consolidation candidates nor on the dictionary:
// computed once per Problem (a consolidation pass encodes the same Problem once per probe), by exactly the code the
// encoder used to run per node on every call, so the encoding stays byte-identical (tests/test_encoding_digests.py).
std::vector<Taint> state_node_taints(const StateNode& n);
struct NodeFacts {
  ResourceList pod_req, ds_req;          // sum of RequestsForPods over the bound pods / over the bound daemonset pods
  std::vector<HostPortEntry> hostports;  // host ports of the bound pods, pod order
  std::vector<NodeSelectorRequirement> label_reqs;  // NewLabelRequirements(node.Labels), requirements.go:54-59
  std::vector<Taint> taints;             // state.Node.Taints(): Spec.Taints without the ephemeral / not-yet-removed startup ones
};
struct ClusterFacts : kmodel::ProblemDerived {
  std::vector<NodeFacts> node;           // parallel to Problem.nodes
  std::set<std::string> res_names;       // resource names mentioned by node allocatable / capacity / bound pods
  std::set<std::string> req_names;       // resource names some bound pod requests
  std::set<std::string> anti_keys;       // topology keys of the bound pods' required anti-affinity terms
  std::set<std::pair<std::string, std::string>> label_pairs;  // every (key, value) some node carries as a label
  std::set<std::pair<std::string, std::string>> named_pairs;  // (normalized key, value) a bound pod's node selector / affinity names
};
const ClusterFacts& cluster_facts(const Problem& P) {
  std::lock_guard<std::mutex> lock(P.derived_mu);
  if (!P.derived) {
    auto f = std::make_shared<ClusterFacts>();
    f->node.resize(P.nodes.size());
    for (size_t i = 0; i < P.nodes.size(); ++i) {
      const StateNode& n = P.nodes[i];
      NodeFacts& nf = f->node[i];
      for (auto& kv : n.allocatable) f->res_names.insert(kv.first);
      for (auto& kv : n.capacity) f->res_names.insert(kv.first);
      for (auto& p : n.pods) {
        const ResourceList r = pod_requests(p);
        for (auto& kv : r) { f->res_names.insert(kv.first); f->req_names.insert(kv.first); }
        auto name = [&](const std::vector<NodeSelectorRequirement>& rs) {
          for (auto& q : rs)
            if (q.op == Op::In || q.op == Op::NotIn)
              for (auto& v : q.values) f->named_pairs.insert({normalize_key(q.key), v});
        };
        for (auto& kv : p.node_selector) f->named_pairs.insert({normalize_key(kv.first), kv.second});
        for (auto& t : p.required_node_terms) name(t);
        for (auto& t : p.preferred_node_terms) name(t.preference);
        nf.pod_req = merge(nf.pod_req, r);
        if (p.is_daemonset) nf.ds_req = merge(nf.ds_req, r);
        for (auto& hp : host_ports(p)) nf.hostports.push_back(hp);
      }
      for (auto& kv : n.labels) nf.label_reqs.push_back({kv.first, Op::In, {kv.second}});
      nf.taints = state_node_taints(n);
      for (auto& p : n.pods)
        for (auto& t : p.pod_anti_affinity_required) f->anti_keys.insert(t.topology_key);
      for (auto& kv : n.labels) f->label_pairs.insert({kv.first, kv.second});
    }
    P.derived = f;
  }
  return static_cast<const ClusterFacts&>(*P.derived);
}

struct Builder {
  const Problem& P;
  Encoded& E;
  std::set<std::string> well_known;
  std::map<std::string, int> key_id;                       // mask key -> id
  std::vector<std::map<std::string, int>> value_id;        // per key
  std::map<std::string, int> res_id;
  std::vector<KeyMeta> key_meta;
  std::map<std::string, int> taintset_id;
  std::vector<std::vector<Taint>> taintsets;
  std::vector<HostPortEntry> hp_entries;
  std::map<std::string, int> type_col;                     // instance type name -> column
  bool res_pruned = false;                                 // resource names no request reads were left out of res_id

  Builder(const Problem& p, Encoded& e) : P(p), E(e) {}

  // ------------------------------------------------------------ requirement encoding
  int key_of(const std::string& k) const {
    auto it = key_id.find(normalize_key(k));
    return it == key_id.end() ? -1 : it->second;
  }
  Req encode_req(int k, Op op, const std::vector<std::string>& values) const {  // NewRequirement requirement.go:44-68
    Req r{0, 0, 0, true, true, false, false};
    r.complement = !(op == Op::In || op == Op::DoesNotExist);
    if (op == Op::In || op == Op::NotIn)
      for (auto& v : values) r.values |= 1ull << value_id[k].at(v);
    if (op == Op::Gt) { r.has_gt = true; parse_int(values.at(0), &r.gt); }
    if (op == Op::Lt) { r.has_lt = true; parse_int(values.at(0), &r.lt); }
    return r;
  }
  void add_req(ksched_reqset& rs, ksched_bounds& b, int k, const Req& r) const {  // Requirements.Add
    Req cur = ksched::req_load(rs, &b, k);
    ksched::req_store(rs, &b, k, ksched::key_add(cur, r, key_meta[k]));
  }
  // requirements on mask keys only; hostname / instance-type requirements are returned separately
  struct Special {
    std::vector<NodeSelectorRequirement> hostname, itype;
  };
  void add_selector_reqs(ksched_reqset& rs, ksched_bounds& b, const std::vector<NodeSelectorRequirement>& list, Special* sp) const {
    for (auto& r : list) {
      std::string key = normalize_key(r.key);
      if (key == kHostname) { if (sp) sp->hostname.push_back(r); else unsupported("hostname requirement here"); continue; }
      if (key == kInstanceType) { if (sp) sp->itype.push_back(r); else unsupported("instance-type requirement here"); continue; }
      int k = key_of(key);
      if (k < 0) continue;  // key inactive: cannot influence any decision
      add_req(rs, b, k, encode_req(k, r.op, r.values));
    }
  }
  static std::vector<NodeSelectorRequirement> label_reqs(const Labels& l) {  // NewLabelRequirements requirements.go:54-59
    std::vector<NodeSelectorRequirement> out;
    for (auto& kv : l) out.push_back({kv.first, Op::In, {kv.second}});
    return out;
  }
  // NewPodRequirements requirements.go:61-78 (the preferred-term sort is stable here)
  void pod_requirements(const Pod& pod, ksched_reqset& rs, ksched_bounds& b, Special* sp) const {
    add_selector_reqs(rs, b, label_reqs(pod.node_selector), sp);
    if (!pod.has_node_affinity) return;
    if (!pod.preferred_node_terms.empty()) {
      auto terms = pod.preferred_node_terms;
      std::stable_sort(terms.begin(), terms.end(), [](auto& x, auto& y) { return x.weight > y.weight; });
      add_selector_reqs(rs, b, terms[0].preference, sp);
    }
    if (pod.has_required_node_affinity && !pod.required_node_terms.empty())
      add_selector_reqs(rs, b, pod.required_node_terms[0], sp);
  }
  // Hand a requirement set over to the C-ABI: bounds become excluded regions + excluded out-of-range values (ksched.h:
  // ksched_key_regions). Applied at the very end, after every host-side use of the exact {values, gt, lt} form.
  void to_region_form(ksched_reqset& rs, const ksched_bounds& b) const {
    if (!(rs.meta >> KSCHED_META_HASGT_SHIFT)) return;
    for (int k = 0; k < (int)E.key_names.size(); ++k) {
      Req r = ksched::req_load(rs, &b, k);
      if (!r.present || (!r.has_gt && !r.has_lt)) continue;
      if (E.key_regions.empty() || !E.key_regions[k].region_mask) throw std::runtime_error("internal: bounded requirement on a key without regions");
      Req out;
      if (!ksched::req_to_region_form(r, E.key_regions[k], E.keys[k].dict_mask, &out)) throw std::runtime_error("internal: bound that is not a threshold of its key");
      ksched_bounds scratch{};
      ksched::req_store(rs, &scratch, k, out);
    }
  }
  bool compatible(const ksched_reqset& node, const ksched_bounds& nb, const ksched_reqset& inc, const ksched_bounds& ib) const {
    for (int k = 0; k < (int)E.key_names.size(); ++k) {
      Req n = ksched::req_load(node, &nb, k), i = ksched::req_load(inc, &ib, k);
      if (!ksched::key_compatible(n, i, E.keys[k].well_known != 0, key_meta[k])) return false;
    }
    return true;
  }

  int taintset(const std::vector<Taint>& ts) {
    std::string k = taints_key(ts);
    auto it = taintset_id.find(k);
    if (it != taintset_id.end()) return it->second;
    int id = (int)taintsets.size();
    if (id >= 64) unsupported("more than 64 distinct taint sets");
    taintset_id[k] = id;
    taintsets.push_back(ts);
    return id;
  }
  int hp_entry(const HostPortEntry& e) {
    for (size_t i = 0; i < hp_entries.size(); ++i)
      if (hp_entries[i].ip == e.ip && hp_entries[i].port == e.port && hp_entries[i].protocol == e.protocol) return (int)i;
    if (hp_entries.size() >= 64) unsupported("more than 64 distinct host-port entries");
    hp_entries.push_back(e);
    return (int)hp_entries.size() - 1;
  }
  int resource(const std::string& name) const {
    auto it = res_id.find(name);
    if (it == res_id.end()) throw std::runtime_error("internal: unknown resource " + name);
    return it->second;
  }
  uint32_t fill_resources(const ResourceList& r, int64_t* out) const {
    uint32_t present = 0;
    for (int i = 0; i < KSCHED_MAX_RES; ++i) out[i] = 0;
    for (auto& kv : r) {
      if (res_pruned && !res_id.count(kv.first)) continue;  // no request or limit reads it: it cannot change an answer
      int id = resource(kv.first);
      out[id] = kv.second;
      present |= 1u << id;
    }
    return present;
  }
};

std::vector<Taint> state_node_taints(const StateNode& n) {  // state/node.go:61-78
  auto lab = [&](const char* k) { auto it = n.labels.find(k); return it == n.labels.end() ? std::string() : it->second; };
  bool initialized = lab(kInitialized) == "true", owned = !lab(kProvisionerName).empty();
  std::vector<Taint> eph = {{"node.kubernetes.io/not-ready", "", "NoSchedule"}, {"node.kubernetes.io/unreachable", "", "NoSchedule"}};
  if (!initialized && owned) eph.insert(eph.end(), n.startup_taints.begin(), n.startup_taints.end());
  std::vector<Taint> out;
  for (auto& t : n.taints) {
    bool rej = false;
    for (auto& e : eph) rej = rej || (e.key == t.key && e.value == t.value && e.effect == t.effect);
    if (!rej) out.push_back(t);
  }
  return out;
}

// topology group under construction (topologygroup.go:53-86)
struct Group {
  int type;  // 0 spread, 1 affinity, 2 anti-affinity
  std::string key;
  int32_t max_skew;
  std::set<std::string> namespaces;
  LabelSelector selector;
  bool filter_nil = true;
  std::vector<std::pair<ksched_reqset, ksched_bounds>> filter;  // TopologyNodeFilter terms
  std::string filter_key;
  bool inverse = false;
  bool dormant = false;
  std::map<std::string, int32_t> counts;  // domain string -> count (countDomains / inverse Record)
  std::set<size_t> owner_specs;           // indices into the spec table (classes)
  bool selects(const Pod& p) const {      // topologygroup.go:246-252
    if (selector.is_nil) return false;
    return namespaces.count(p.ns) && selector_matches(selector, p.labels);
  }
  std::string hash() const {
    std::string h = key + "|" + std::to_string(type) + "|" + std::to_string(max_skew) + "|";
    for (auto& n : namespaces) h += n + ",";
    return h + "|" + selector_key(selector) + "|" + filter_key;
  }
};

}  // namespace

std::map<std::string, std::string> value_classes(const std::set<std::string>& values, const std::set<std::string>& named,
                                                 const std::set<int64_t>& thresholds) {
  std::map<std::string, std::string> rep_of;
  std::map<int, std::string> rep;  // class -> representative; class = region index of an integer (ksched.h), -1 non-integers
  for (auto& v : values) {         // ascending string order: a class's first member is its smallest
    int64_t iv;
    const bool is_int = parse_int(v, &iv);
    if (named.count(v) || (is_int && thresholds.count(iv))) continue;
    const int cls = is_int ? (int)std::distance(thresholds.begin(), thresholds.lower_bound(iv)) : -1;
    rep_of[v] = rep.emplace(cls, v).first->second;
  }
  return rep_of;
}

std::unique_ptr<Encoded> encode(const Problem& P, const std::vector<int>& candidates, bool cluster_superset) {
  static const bool prof = std::getenv("KSCHED_ENCODE_PROFILE") != nullptr;
  auto t_last = std::chrono::steady_clock::now();
  auto phase = [&](const char* name) {
    if (!prof) return;
    auto now = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[encode] %-28s %8.2f ms\n", name, std::chrono::duration<double, std::milli>(now - t_last).count());
    t_last = now;
  };
  auto enc = std::make_unique<Encoded>();
  Encoded& E = *enc;
  E.problem_ref = &P;
  Builder B(P, E);
  const ClusterFacts& facts = cluster_facts(P);

  // ------------------------------------------------------------------ who takes part
  std::vector<int> state_nodes;
  {
    std::set<int> cand(candidates.begin(), candidates.end());
    auto reschedulable = [](const Pod& p) { return !p.is_daemonset && !p.terminal && !p.terminating; };  // utils/node/node.go:30-50
    for (size_t i = 0; i < P.nodes.size(); ++i)
      if ((cluster_superset || !cand.count((int)i)) && !P.nodes[i].marked_for_deletion) state_nodes.push_back((int)i);
    for (auto& p : P.pods) E.pods.push_back(&p);
    if (cluster_superset) {
      // pending pods first (the pods of deleting nodes are pending in every simulation), then the candidates' pods node by node
      for (size_t i = 0; i < P.nodes.size(); ++i)
        if (!cand.count((int)i) && P.nodes[i].marked_for_deletion)
          for (auto& p : P.nodes[i].pods) if (reschedulable(p)) E.pods.push_back(&p);
      E.pod_node.assign(E.pods.size(), -1);
      for (int c : candidates) {
        if (P.nodes.at(c).marked_for_deletion) throw std::runtime_error("a candidate node is marked for deletion");
        for (auto& p : P.nodes[c].pods) if (reschedulable(p)) { E.pods.push_back(&p); E.pod_node.push_back(-2 - c); }  // slot resolved below
      }
    } else {
      for (int c : candidates)
        for (auto& p : P.nodes.at(c).pods) if (reschedulable(p)) E.pods.push_back(&p);
      for (size_t i = 0; i < P.nodes.size(); ++i)
        if (!cand.count((int)i) && P.nodes[i].marked_for_deletion)
          for (auto& p : P.nodes[i].pods) if (reschedulable(p)) E.pods.push_back(&p);
    }
  }
  const size_t NP = E.pods.size();
  // strictly ascending UIDs (the usual case: one informer list) are unique and already ranked; found out in the pass below
  // that visits every pod anyway
  bool uids_ascending = true;
  if (P.provisioners.empty()) throw std::runtime_error("no provisioners found");
  if (P.provisioners.size() > KSCHED_MAX_TEMPLATES) unsupported("more than 16 provisioners");

  B.well_known = {kProvisionerName, kZone, "topology.kubernetes.io/region", kInstanceType, "kubernetes.io/arch", "kubernetes.io/os", kCapacityType};
  B.well_known.insert(P.extra_well_known_labels.begin(), P.extra_well_known_labels.end());

  // template order: OrderByWeight (v1alpha5/provisioner.go:132-136), stable
  for (size_t i = 0; i < P.provisioners.size(); ++i) E.template_provisioner.push_back((int)i);
  std::stable_sort(E.template_provisioner.begin(), E.template_provisioner.end(),
                   [&](int a, int b) { return P.provisioners[a].weight > P.provisioners[b].weight; });
  bool tolerate_pns = false;  // scheduler.go:49-56
  for (auto& pr : P.provisioners)
    for (auto& t : pr.taints) if (t.effect == "PreferNoSchedule") tolerate_pns = true;

  phase("who takes part");
  // ------------------------------------------------------------------ CSI volume limits (ksched.h: ksched_class_volumes)
  // Drivers some owned state node limits; claims by how many pods (batch + bound) mount them: one -> counted, several -> tracked id.
  std::vector<std::string> vol_drivers;
  std::map<std::pair<std::string, std::string>, int> vol_tracked;  // (driver, claim) -> bit
  auto pod_claims = [&](const Pod& p) {  // VolumeUsage.validate's result: driver -> claim set, limited drivers only
    std::map<std::string, std::set<std::string>> m;
    for (auto& v : p.volumes)
      if (!v.driver.empty() && std::find(vol_drivers.begin(), vol_drivers.end(), v.driver) != vol_drivers.end()) m[v.driver].insert(v.pvc_id);
    return m;
  };
  {
    std::set<std::string> drivers;
    for (int si : state_nodes) for (auto& kv : P.nodes[si].volume_limits) drivers.insert(kv.first);
    vol_drivers.assign(drivers.begin(), drivers.end());
    if (vol_drivers.size() > KSCHED_MAX_VOLUME_DRIVERS) unsupported("more than 4 CSI drivers with node volume limits");
    if (!vol_drivers.empty()) {
      std::map<std::pair<std::string, std::string>, int> refs;
      auto count = [&](const Pod& p) { for (auto& kv : pod_claims(p)) for (auto& c : kv.second) refs[{kv.first, c}]++; };
      for (auto* p : E.pods) count(*p);
      for (int si : state_nodes) for (auto& p : P.nodes[si].pods) count(p);
      for (auto& kv : refs)
        if (kv.second > 1) {
          if (vol_tracked.size() >= 64) unsupported("more than 64 volume claims shared between pods");
          const int bit = (int)vol_tracked.size();
          vol_tracked[kv.first] = bit;
        }
    }
  }
  auto volume_signature = [&](const Pod& p, ksched_class_volumes* out) {
    ksched_class_volumes cv{};
    if (!vol_drivers.empty())
      for (auto& kv : pod_claims(p)) {
        const size_t d = (size_t)(std::find(vol_drivers.begin(), vol_drivers.end(), kv.first) - vol_drivers.begin());
        for (auto& c : kv.second) {
          auto t = vol_tracked.find({kv.first, c});
          if (t != vol_tracked.end()) cv.shared |= 1ull << t->second;
          else if (cv.priv[d] == 0xFFFF) unsupported("more than 65535 volume claims on one pod");
          else cv.priv[d]++;
        }
      }
    if (out) *out = cv;
    char b[96];
    std::snprintf(b, sizeof b, "|V=%llx:%u:%u:%u:%u", (unsigned long long)cv.shared, cv.priv[0], cv.priv[1], cv.priv[2], cv.priv[3]);
    return (cv.shared | cv.priv[0] | cv.priv[1] | cv.priv[2] | cv.priv[3]) ? std::string(b) : std::string();
  };

  // ------------------------------------------------------------------ pod specs: classes and relaxation chains
  struct Spec { Pod pod; ResourceList req; uint32_t next = KSCHED_NONE; };
  std::vector<Spec> specs;
  std::map<std::string, uint32_t> spec_id;
  std::function<uint32_t(const Pod&)> intern = [&](const Pod& p) -> uint32_t {
    ResourceList req = pod_requests(p);
    std::string k = class_key(p, req);
    if (!p.volumes.empty()) k += volume_signature(p, nullptr);
    auto it = spec_id.find(k);
    if (it != spec_id.end()) return it->second;
    uint32_t id = (uint32_t)specs.size();
    spec_id[k] = id;
    specs.push_back({p, req, KSCHED_NONE});
    Pod relaxed = p;
    // NewPodRequirements sorts the preferred terms in place before Relax ever runs (requirements.go:69)
    std::stable_sort(relaxed.preferred_node_terms.begin(), relaxed.preferred_node_terms.end(),
                     [](auto& a, auto& b) { return a.weight > b.weight; });
    if (relax(relaxed, tolerate_pns)) {
      uint32_t nx = intern(relaxed);
      specs[id].next = nx;
    }
    return id;
  };
  E.pod_class.resize(NP);
  {
    // "same deployment as the previous pod" is a pure comparison of two pods: every pair at once, on all cores; only the
    // class boundaries (a few hundred in a 100 000-pod batch) take the keyed path, in order
    std::vector<uint8_t> same(NP, 0), uid_order_broken((NP >> 12) + 2, 0);
    std::vector<uint64_t> run_hash(NP, 0);  // spec_hash of the pods that start a run
    E.pod_timestamp.resize(NP);
    parallel_ranges(NP, 4096, [&](size_t b, size_t e) {
      bool asc = true;
      if (b == 0 && e > 0) { E.pod_timestamp[0] = E.pods[0]->creation_ts; run_hash[0] = spec_hash(*E.pods[0]); }
      for (size_t i = std::max<size_t>(b, 1); i < e; ++i) {
        const Pod& p = *E.pods[i];
        const Pod& q = *E.pods[i - 1];
        same[i] = same_spec(p, q) ? 1 : 0;
        if (!same[i]) run_hash[i] = spec_hash(p);
        asc = asc && q.uid < p.uid;
        E.pod_timestamp[i] = p.creation_ts;  // queue.go:74-110 sorts by it (per-pod queue keys below)
      }
      if (!asc) uid_order_broken[b >> 12] = 1;  // (ranges start at multiples of >= 4096 pods or at 0: one flag each)
    });
    for (uint8_t f : uid_order_broken) uids_ascending = uids_ascending && !f;
    if (!uids_ascending) {
      std::unordered_set<std::string> uids;
      uids.reserve(NP * 2);
      for (auto* p : E.pods)
        if (!uids.insert(p->uid).second) throw std::runtime_error("pods must have unique UIDs: " + p->uid);
    }
    phase("  same_spec pairs");
    // a run's class: the class of an earlier run with the same spec (hash, then one same_spec against that class's first pod),
    // else the keyed path (new classes, pods with volumes, pods whose containers differ but sum to the same requests)
    std::unordered_map<uint64_t, std::vector<uint32_t>> by_hash;
    for (size_t i = 0; i < NP; ++i) {
      if (same[i]) { E.pod_class[i] = E.pod_class[i - 1]; continue; }
      const Pod& p = *E.pods[i];
      uint32_t id = KSCHED_NONE;
      if (p.volumes.empty()) {
        auto it = by_hash.find(run_hash[i]);
        if (it != by_hash.end())
          for (uint32_t cid : it->second)
            if (same_spec(p, specs[cid].pod)) { id = cid; break; }
      }
      if (id == KSCHED_NONE) {
        id = intern(p);
        if (p.volumes.empty()) {
          auto& v = by_hash[run_hash[i]];
          if (std::find(v.begin(), v.end(), id) == v.end()) v.push_back(id);
        }
      }
      E.pod_class[i] = id;
    }
    phase("  intern boundaries");
  }
  std::vector<Pod> daemons = P.daemonset_pods;

  phase("pod classes");
  // ------------------------------------------------------------------ active keys + dictionary
  // pod-side keys: anything a pod / daemonset / topology group / node filter can put into a node's requirements
  std::set<std::string> pod_side;
  auto note_reqs = [&](const std::vector<NodeSelectorRequirement>& rs) { for (auto& r : rs) pod_side.insert(normalize_key(r.key)); };
  auto note_pod = [&](const Pod& p) {
    for (auto& kv : p.node_selector) pod_side.insert(normalize_key(kv.first));
    for (auto& t : p.required_node_terms) note_reqs(t);
    for (auto& t : p.preferred_node_terms) note_reqs(t.preference);
    for (auto& t : p.pod_affinity_required) pod_side.insert(t.topology_key);
    for (auto& t : p.pod_affinity_preferred) pod_side.insert(t.term.topology_key);
    for (auto& t : p.pod_anti_affinity_required) pod_side.insert(t.topology_key);
    for (auto& t : p.pod_anti_affinity_preferred) pod_side.insert(t.term.topology_key);
    for (auto& t : p.topology_spread) pod_side.insert(t.topology_key);
  };
  for (auto& s : specs) note_pod(s.pod);
  for (auto& d : daemons) note_pod(d);
  if (!P.empty_topology)
    for (auto& k : facts.anti_keys) pod_side.insert(k);  // bound pods with required anti-affinity (ClusterFacts)
  std::set<std::string> type_keys, template_keys;
  for (auto& it : P.instance_types) for (auto& r : it.requirements) type_keys.insert(normalize_key(r.key));
  for (auto& pr : P.provisioners) {
    for (auto& r : pr.requirements) template_keys.insert(normalize_key(r.key));
    for (auto& kv : pr.labels) template_keys.insert(normalize_key(kv.first));
    template_keys.insert(kProvisionerName);
  }
  // Active keys: everything that can appear in a node's requirements (template or pod side). Keys that only
  // instance types define can never meet a node requirement (Intersects walks keys present on BOTH sides,
  // requirements.go:189-190) and are dropped.
  std::set<std::string> active = pod_side;
  active.insert(template_keys.begin(), template_keys.end());
  (void)type_keys;
  active.erase(kHostname);
  active.erase(kInstanceType);
  if (active.size() > KSCHED_MAX_KEYS) unsupported("more than 16 active label keys");
  for (auto& k : active) {
    B.key_id[k] = (int)E.key_names.size();
    E.key_names.push_back(k);
  }
  const int NK = (int)E.key_names.size();
  std::vector<std::set<std::string>> vals(NK);
  auto note_vals = [&](const std::vector<NodeSelectorRequirement>& rs) {
    for (auto& r : rs) {
      int k = B.key_of(r.key);
      if (k < 0) continue;
      if (r.op == Op::In || r.op == Op::NotIn) vals[k].insert(r.values.begin(), r.values.end());
    }
  };
  auto note_label_vals = [&](const Labels& l) {
    for (auto& kv : l) { int k = B.key_of(kv.first); if (k >= 0) vals[k].insert(kv.second); }
  };
  auto note_pod_vals = [&](const Pod& p) {
    note_label_vals(p.node_selector);
    for (auto& t : p.required_node_terms) note_vals(t);
    for (auto& t : p.preferred_node_terms) note_vals(t.preference);
  };
  for (auto& s : specs) note_pod_vals(s.pod);
  for (auto& d : daemons) note_pod_vals(d);
  for (auto& it : P.instance_types) note_vals(it.requirements);
  // offerings name zones / capacity types too (a node without a requirement on the key admits all of them)
  for (auto& it : P.instance_types)
    for (auto& o : it.offerings) {
      int kz = B.key_of(kZone), kc = B.key_of(kCapacityType);
      if (kz >= 0) vals[kz].insert(o.zone);
      if (kc >= 0) vals[kc].insert(o.capacity_type);
    }
  for (auto& pr : P.provisioners) {
    note_vals(pr.requirements);
    Labels l = pr.labels;
    l[kProvisionerName] = pr.name;
    note_label_vals(l);
  }
  for (auto& kv : facts.label_pairs) { int k = B.key_of(kv.first); if (k >= 0) vals[k].insert(kv.second); }  // every node's labels (ClusterFacts)
  const int zone_key = B.key_of(kZone), ct_key = B.key_of(kCapacityType);
  // Every threshold any requirement of this problem names, per key; a key also gets one region when an instance type has a
  // complement requirement on it (region form below).
  std::vector<std::set<int64_t>> thr(NK);
  std::vector<bool> type_complement(NK, false);
  {
    auto note_thr = [&](const std::vector<NodeSelectorRequirement>& rs, bool is_type) {
      for (auto& r : rs) {
        int k = B.key_of(r.key);
        if (k < 0) continue;
        if (r.op == Op::Gt || r.op == Op::Lt) { int64_t v = 0; if (!r.values.empty()) parse_int(r.values[0], &v); thr[k].insert(v); }
        if (is_type && r.op != Op::In && r.op != Op::DoesNotExist) type_complement[k] = true;
      }
    };
    auto note_pod_thr = [&](const Pod& p) {
      for (auto& t : p.required_node_terms) note_thr(t, false);
      for (auto& t : p.preferred_node_terms) note_thr(t.preference, false);
    };
    for (auto& sp : specs) note_pod_thr(sp.pod);
    for (auto& d : daemons) note_pod_thr(d);
    for (auto& it : P.instance_types) note_thr(it.requirements, true);
    for (auto& pr : P.provisioners) note_thr(pr.requirements, false);
  }
  // Value classes (DESIGN.md §3). A key whose values do not fit the word keeps the values some requirement of the problem
  // names, and one representative per class of the others: instance types' In values and node labels that no requirement
  // tells apart. Keys that fit are encoded as they always were.
  phase("  keys + thresholds");
  E.key_representatives.assign(NK, 0);
  std::vector<std::map<std::string, std::string>> rep_of(NK);  // unnamed value -> its class's representative
  {
    std::vector<int> wide;
    for (int k = 0; k < NK; ++k) {
      const size_t nd = vals[k].size(), m = thr[k].size();
      if (nd > 63 || ((m > 0 || type_complement[k]) && nd + m + 1 > 63)) wide.push_back(k);
    }
    if (!wide.empty()) {
      std::vector<std::set<std::string>> named(NK);
      std::vector<bool> all_named(NK, false);
      auto name_vals = [&](const std::vector<NodeSelectorRequirement>& rs, bool complement_only) {
        for (auto& r : rs) {
          int k = B.key_of(r.key);
          if (k < 0 || (complement_only && r.op == Op::In)) continue;
          if (r.op == Op::In || r.op == Op::NotIn) named[k].insert(r.values.begin(), r.values.end());
        }
      };
      auto name_labels = [&](const Labels& l) { for (auto& kv : l) { int k = B.key_of(kv.first); if (k >= 0) named[k].insert(kv.second); } };
      auto name_pod = [&](const Pod& p) {  // topology node filters are built from the same node selector and required terms
        name_labels(p.node_selector);
        for (auto& t : p.required_node_terms) name_vals(t, false);
        for (auto& t : p.preferred_node_terms) name_vals(t.preference, false);
        auto topo = [&](const std::string& key) { int k = B.key_of(key); if (k >= 0) all_named[k] = true; };
        for (auto& t : p.topology_spread) topo(t.topology_key);
        for (auto& t : p.pod_affinity_required) topo(t.topology_key);
        for (auto& t : p.pod_affinity_preferred) topo(t.term.topology_key);
        for (auto& t : p.pod_anti_affinity_required) topo(t.topology_key);
        for (auto& t : p.pod_anti_affinity_preferred) topo(t.term.topology_key);
      };
      for (auto& s : specs) name_pod(s.pod);
      for (auto& d : daemons) name_pod(d);
      for (auto& kv : facts.named_pairs) { int k = B.key_of(kv.first); if (k >= 0) named[k].insert(kv.second); }  // bound pods
      for (auto& key : facts.anti_keys) { int k = B.key_of(key); if (k >= 0) all_named[k] = true; }  // inverse anti-affinity groups
      for (auto& pr : P.provisioners) {
        name_vals(pr.requirements, false);
        Labels l = pr.labels;
        l[kProvisionerName] = pr.name;
        name_labels(l);
      }
      for (auto& it : P.instance_types) name_vals(it.requirements, true);
      if (zone_key >= 0) all_named[zone_key] = true;  // offering slots: they feed the launch choice
      if (ct_key >= 0) all_named[ct_key] = true;
      for (int k : wide) {
        if (all_named[k]) continue;  // refused below when it does not fit
        rep_of[k] = value_classes(vals[k], named[k], thr[k]);
        for (auto& kv : rep_of[k]) {
          if (kv.first != kv.second) vals[k].erase(kv.first);
          else E.key_representatives[k]++;
        }
      }
    }
  }
  phase("  value classes");
  B.value_id.resize(NK);
  E.key_values.resize(NK);
  E.keys.resize(NK);
  E.key_int_values.assign((size_t)NK * 64, 0);
  B.key_meta.resize(NK);
  for (int k = 0; k < NK; ++k) {
    if (vals[k].size() > 63) unsupported("label key " + E.key_names[k] + " has more than 63 distinct values");
    ksched_keyinfo& ki = E.keys[k];
    std::memset(&ki, 0, sizeof ki);
    int b = 0;
    for (auto& v : vals[k]) {
      B.value_id[k][v] = b;
      E.key_values[k].push_back(v);
      ki.dict_mask |= 1ull << b;
      int64_t iv;
      if (parse_int(v, &iv)) { ki.int_mask |= 1ull << b; E.key_int_values[(size_t)k * 64 + b] = iv; }
      ++b;
    }
    // every requirement, label and domain table looks an unnamed value up under its representative's id
    for (auto& kv : rep_of[k]) B.value_id[k][kv.first] = B.value_id[k].at(kv.second);
    ki.well_known = B.well_known.count(E.key_names[k]) ? 1 : 0;
    ki.is_zone = E.key_names[k] == kZone;
    ki.is_capacity_type = E.key_names[k] == kCapacityType;
  }
  for (int k = 0; k < NK; ++k) B.key_meta[k] = KeyMeta{E.keys[k].int_mask, &E.key_int_values[(size_t)k * 64], nullptr};
  // Region form of Gt/Lt (ksched.h: ksched_key_regions).
  {
    bool any = false;
    for (int k = 0; k < NK; ++k) any = any || !thr[k].empty() || type_complement[k];
    if (any) {
      E.key_regions.assign(NK, ksched_key_regions{});
      for (int k = 0; k < NK; ++k) {
        if (thr[k].empty() && !type_complement[k]) continue;
        const int m = (int)thr[k].size(), nd = (int)E.key_values[k].size();
        if (m > KSCHED_MAX_THRESHOLDS) unsupported("label key " + E.key_names[k] + " has more than 7 distinct Gt/Lt thresholds");
        if (nd + m + 1 > 63) unsupported("label key " + E.key_names[k] + " has too many values for its Gt/Lt regions");
        std::vector<int64_t> ts(thr[k].begin(), thr[k].end());
        ksched::regions_build(&E.key_regions[k], ts.data(), m, nd, E.keys[k].dict_mask, B.key_meta[k]);
      }
    }
  }

  phase("keys + dictionary");
  // ------------------------------------------------------------------ resources
  {
    std::set<std::string> names;
    auto note = [&](const ResourceList& r) { for (auto& kv : r) names.insert(kv.first); };
    for (auto& s : specs) note(s.req);
    for (auto& d : daemons) note(pod_requests(d));
    for (auto& it : P.instance_types) { note(it.capacity); }
    for (auto& pr : P.provisioners) note(pr.limits);
    for (auto& n : facts.res_names) names.insert(n);  // node allocatable / capacity / bound pods (ClusterFacts)
    E.res_names = {"cpu", "memory", "pods"};
    for (auto& n : names) if (n != "cpu" && n != "memory" && n != "pods") E.res_names.push_back(n);
    if (E.res_names.size() > KSCHED_MAX_RES) {
      // Fits reads the request's keys only (resources.go:138-145), the limits bookkeeping the limit's keys only
      // (scheduler.go:284-303): a name that no pod requests and no limit names cannot change an answer. Left out.
      std::set<std::string> read = facts.req_names;
      auto note_read = [&](const ResourceList& r) { for (auto& kv : r) read.insert(kv.first); };
      for (auto& s : specs) note_read(s.req);
      for (auto& d : daemons) note_read(pod_requests(d));
      for (auto& pr : P.provisioners) note_read(pr.limits);
      E.res_names = {"cpu", "memory", "pods"};
      for (auto& n : read) if (n != "cpu" && n != "memory" && n != "pods") E.res_names.push_back(n);
      B.res_pruned = true;
    }
    if (E.res_names.size() > KSCHED_MAX_RES) unsupported("more than 8 distinct resources");
    for (size_t i = 0; i < E.res_names.size(); ++i) B.res_id[E.res_names[i]] = (int)i;
  }

  phase("resources");
  // ------------------------------------------------------------------ instance types (columns, price order)
  const int NT = (int)P.instance_types.size();
  E.type_words = (NT + 63) / 64;
  if (E.type_words == 0) E.type_words = 1;
  {
    std::vector<double> min_price(NT, std::numeric_limits<double>::infinity());
    for (int i = 0; i < NT; ++i)
      for (auto& o : P.instance_types[i].offerings)
        if (o.available && o.price < min_price[i]) min_price[i] = o.price;
    E.type_input_index.resize(NT);
    for (int i = 0; i < NT; ++i) E.type_input_index[i] = i;
    std::stable_sort(E.type_input_index.begin(), E.type_input_index.end(), [&](int a, int b) { return min_price[a] < min_price[b]; });
    E.types.resize(NT);
    E.type_capacity.assign((size_t)NT * KSCHED_MAX_RES, 0);
    // launch-choice table: exact price order through ranks of the distinct (double) prices
    {
      std::set<double> prices;
      for (auto& it : P.instance_types)
        for (auto& o : it.offerings) if (o.available) prices.insert(o.price);
      E.price_by_rank.assign(prices.begin(), prices.end());
      E.offering_keys.assign((size_t)NT * 64, ~0ull);
    }
    for (int c = 0; c < NT; ++c) {
      const InstanceType& it = P.instance_types[E.type_input_index[c]];
      if (B.type_col.count(it.name)) unsupported("duplicate instance type name " + it.name);
      B.type_col[it.name] = c;
      ksched_type_row& row = E.types[c];
      std::memset(&row, 0, sizeof row);
      ksched_reqset rs{};
      ksched_bounds bd{};
      for (auto& r : it.requirements) {
        std::string key = normalize_key(r.key);
        if (key == kHostname) unsupported("instance type with a hostname requirement");
        if (key == kInstanceType) {
          if (!(r.op == Op::In && r.values.size() == 1 && r.values[0] == it.name)) unsupported("instance-type requirement of a type must be In [its own name]");
          continue;
        }
        int k = B.key_of(key);
        if (k < 0) continue;
        B.add_req(rs, bd, k, B.encode_req(k, r.op, r.values));
      }
      B.to_region_form(rs, bd);
      std::memcpy(row.values, rs.values, sizeof row.values);
      row.meta = rs.meta;
      ResourceList overhead = merge(merge(it.kube_reserved, it.system_reserved), it.eviction_threshold);
      ResourceList alloc = it.capacity;  // resources.Subtract only over keys of capacity
      for (auto& kv : alloc) { auto o = overhead.find(kv.first); if (o != overhead.end()) kv.second -= o->second; }
      row.res_present = B.fill_resources(alloc, row.allocatable);
      B.fill_resources(it.capacity, &E.type_capacity[(size_t)c * KSCHED_MAX_RES]);
      for (size_t oi = 0; oi < it.offerings.size(); ++oi) {
        const Offering& o = it.offerings[oi];
        if (!o.available) continue;
        int z = 0, ct = 0;
        if (zone_key >= 0) { auto f = B.value_id[zone_key].find(o.zone); if (f == B.value_id[zone_key].end()) continue; z = f->second; }
        if (ct_key >= 0) { auto f = B.value_id[ct_key].find(o.capacity_type); if (f == B.value_id[ct_key].end()) continue; ct = f->second; }
        if (z >= 16 || ct >= 4) unsupported("more than 16 zones or 4 capacity types");
        row.offerings |= 1ull << (ct * 16 + z);
        // (price rank, Offerings list position, slot): the smallest key of a slot wins when several offerings share it
        if (oi > 255) unsupported("instance type " + it.name + " has more than 256 offerings");
        const uint64_t rank = (uint64_t)(std::lower_bound(E.price_by_rank.begin(), E.price_by_rank.end(), o.price) - E.price_by_rank.begin());
        const uint64_t key = (rank << 16) | ((uint64_t)oi << 8) | (uint64_t)(ct * 16 + z);
        uint64_t& cell = E.offering_keys[(size_t)c * 64 + ct * 16 + z];
        if (key < cell) cell = key;
      }
      row.min_price = min_price[E.type_input_index[c]];
      row.input_index = (uint32_t)E.type_input_index[c];
    }
  }
  // offerings whose zone / capacity-type is not a dictionary value can never satisfy a *present* requirement,
  // but they do satisfy an absent one: keep them visible through a catch-all bit when the key is inactive.
  // (When zone/ct keys are inactive every offering maps to z=0/ct=0 above, which is exactly "key not constrained".)

  phase("instance types");
  // ------------------------------------------------------------------ templates
  const int NV = (int)E.template_provisioner.size();
  E.templates.resize(NV);
  E.template_bounds.resize(NV);
  std::vector<ksched_bounds> tb(NV);
  for (int v = 0; v < NV; ++v) {
    const Provisioner& pr = P.provisioners[E.template_provisioner[v]];
    ksched_template& t = E.templates[v];
    std::memset(&t, 0, sizeof t);
    std::memset(&tb[v], 0, sizeof(ksched_bounds));
    Builder::Special sp;
    B.add_selector_reqs(t.reqs, tb[v], pr.requirements, &sp);  // NewMachineTemplate machinetemplate.go:46-62
    Labels l = pr.labels;
    l[kProvisionerName] = pr.name;
    B.add_selector_reqs(t.reqs, tb[v], Builder::label_reqs(l), &sp);
    if (!sp.hostname.empty()) unsupported("provisioner with a hostname requirement");
    // instance-type requirement of the provisioner: fold into membership (types are singletons on that key)
    std::vector<bool> allowed(NT, true);
    for (auto& r : sp.itype) {
      std::set<std::string> names(r.values.begin(), r.values.end());
      for (int c = 0; c < NT; ++c) {
        const std::string& name = P.instance_types[E.type_input_index[c]].name;
        bool ok = true;
        if (r.op == Op::In) ok = names.count(name) > 0;
        else if (r.op == Op::NotIn) ok = !names.count(name);
        else if (r.op == Op::DoesNotExist) ok = false;
        else if (r.op == Op::Gt || r.op == Op::Lt) unsupported("Gt/Lt on instance-type");
        allowed[c] = allowed[c] && ok;
      }
    }
    for (int idx : pr.instance_types) {
      int c = B.type_col.at(P.instance_types.at(idx).name);
      if (allowed[c]) E.types[c].template_members |= 1ull << v;
    }
    t.taintset = (uint32_t)B.taintset(pr.taints);
    t.has_limits = pr.has_limits ? 1 : 0;
    t.limit_present = B.fill_resources(pr.limits, t.remaining);
    if (t.reqs.meta >> KSCHED_META_HASGT_SHIFT) E.any_template_bounds = true;
  }
  E.template_bounds = tb;

  phase("templates");
  // ------------------------------------------------------------------ daemonset overhead (scheduler.go:250-267)
  auto daemon_reqs = [&](const Pod& d, ksched_reqset& rs, ksched_bounds& bd) {
    Builder::Special sp;
    B.pod_requirements(d, rs, bd, &sp);
    return sp;
  };
  for (int v = 0; v < NV; ++v) {
    const Provisioner& pr = P.provisioners[E.template_provisioner[v]];
    ResourceList total;
    int count = 0;
    for (auto& d : daemons) {
      if (!tolerates_all(pr.taints, d.tolerations)) continue;
      ksched_reqset rs{}; ksched_bounds bd{};
      auto sp = daemon_reqs(d, rs, bd);
      if (!sp.hostname.empty() || !sp.itype.empty()) unsupported("daemonset pod with hostname / instance-type requirement");
      if (!B.compatible(E.templates[v].reqs, tb[v], rs, bd)) continue;
      total = merge(total, pod_requests(d));
      ++count;
    }
    total["pods"] = (int64_t)count * 1000;
    E.templates[v].daemon_res_present = B.fill_resources(total, E.templates[v].daemon_requests);
  }

  phase("daemonset overhead");
  // ------------------------------------------------------------------ existing nodes (scheduler.go:221-248, existingnode.go:41-75)
  std::map<std::string, int> hostname_slot;  // hostname -> existing slot
  for (int si : state_nodes) {
    const StateNode& n = P.nodes[si];
    auto own = n.labels.find(kProvisionerName);
    if (own == n.labels.end() || own->second.empty()) continue;  // !node.Owned()
    ksched_existing_node e;
    std::memset(&e, 0, sizeof e);
    ksched_bounds nb{};
    Builder::Special sp;
    const NodeFacts& nf = facts.node[(size_t)si];
    B.add_selector_reqs(e.reqs, nb, nf.label_reqs, &sp);
    ResourceList daemon_total;
    int dcount = 0;
    for (auto& d : daemons) {
      if (!tolerates_all(n.taints, d.tolerations)) continue;  // raw Spec.Taints (scheduler.go:231)
      ksched_reqset rs{}; ksched_bounds bd{};
      daemon_reqs(d, rs, bd);
      if (!B.compatible(e.reqs, nb, rs, bd)) continue;
      daemon_total = merge(daemon_total, pod_requests(d));
      ++dcount;
    }
    daemon_total["pods"] = (int64_t)dcount * 1000;
    const ResourceList& pod_req = nf.pod_req;
    const ResourceList& ds_req = nf.ds_req;
    ResourceList rem = daemon_total;  // resources.Subtract over keys of lhs, clamped at 0
    for (auto& kv : rem) { auto f = ds_req.find(kv.first); if (f != ds_req.end()) kv.second -= f->second; if (kv.second < 0) kv.second = 0; }
    ResourceList avail = n.allocatable;
    for (auto& kv : avail) { auto f = pod_req.find(kv.first); if (f != pod_req.end()) kv.second -= f->second; }
    e.available_present = B.fill_resources(avail, e.available);
    e.requests_present = B.fill_resources(rem, e.requests);
    e.taintset = (uint32_t)B.taintset(nf.taints);
    e.itype = KSCHED_NONE;
    auto itl = n.labels.find(kInstanceType);
    if (itl != n.labels.end()) { auto c = B.type_col.find(itl->second); if (c != B.type_col.end()) e.itype = (uint32_t)c->second; }
    for (auto& hp : nf.hostports) e.hostport_entries |= 1ull << B.hp_entry(hp);
    std::string hostname;
    auto h = n.labels.find(kHostname);
    if (h != n.labels.end()) hostname = h->second;
    if (hostname.empty()) hostname = n.name;
    hostname_slot[hostname] = (int)E.existing.size();
    E.existing_state_index.push_back(si);
    auto ini = n.labels.find(kInitialized);
    E.existing_initialized.push_back(ini != n.labels.end() && ini->second == "true");
    if (!vol_drivers.empty()) {  // state.Node.VolumeUsage() / VolumeLimits() (state/cluster.go:292-303,340-347)
      ksched_node_volumes nv{};
      std::map<std::string, std::set<std::string>> mounted;
      for (auto& p : n.pods) for (auto& kv : pod_claims(p)) mounted[kv.first].insert(kv.second.begin(), kv.second.end());
      bool over = false;
      for (size_t d = 0; d < KSCHED_MAX_VOLUME_DRIVERS; ++d) {
        nv.limit[d] = -1;
        if (d >= vol_drivers.size()) continue;
        auto l = n.volume_limits.find(vol_drivers[d]);
        if (l != n.volume_limits.end()) nv.limit[d] = l->second;
        int total = 0;
        for (auto& c : mounted[vol_drivers[d]]) {
          ++total;
          auto t = vol_tracked.find({vol_drivers[d], c});
          if (t != vol_tracked.end()) nv.mounted |= 1ull << t->second; else nv.used[d]++;
        }
        if (nv.limit[d] >= 0 && total > nv.limit[d]) over = true;
      }
      // a node already over a limit refuses every pod (VolumeCount.Exceeds walks the node's own drivers, volumeusage.go:101-112)
      if (over) { e.available[2] = std::numeric_limits<int64_t>::min() / 4; e.available_present |= 1u << 2; }
      E.existing_volumes.push_back(nv);
    }
    E.existing.push_back(e);
    int charged = -1;
    int64_t charged_cap[KSCHED_MAX_RES] = {};
    for (int v = 0; v < NV; ++v)  // scheduler.go:244-246
      if (P.provisioners[E.template_provisioner[v]].name == own->second && E.templates[v].has_limits) {
        int64_t cap[KSCHED_MAX_RES];
        uint32_t present = B.fill_resources(n.capacity, cap);
        for (int r = 0; r < KSCHED_MAX_RES; ++r)
          if ((E.templates[v].limit_present >> r) & 1 && (present >> r) & 1) { E.templates[v].remaining[r] -= cap[r]; charged_cap[r] = cap[r]; }
        charged = v;
      }
    if (cluster_superset) {
      E.existing_template.push_back(charged);
      E.existing_capacity.insert(E.existing_capacity.end(), charged_cap, charged_cap + KSCHED_MAX_RES);
    }
  }
  if (cluster_superset) {
    std::map<int, int> slot_of_state;
    for (size_t e = 0; e < E.existing_state_index.size(); ++e) slot_of_state[E.existing_state_index[e]] = (int)e;
    for (auto& pn : E.pod_node)
      if (pn <= -2) {
        auto f = slot_of_state.find(-2 - pn);
        if (f == slot_of_state.end()) throw std::runtime_error("a candidate node is not owned by a provisioner");
        pn = f->second;
      }
  }
  const int NE = (int)E.existing.size();

  phase("existing nodes");
  // ------------------------------------------------------------------ topology groups (topology.go)
  std::vector<Group> groups;
  std::map<std::string, size_t> group_of;          // hash -> index, non-inverse
  std::map<std::string, size_t> inverse_group_of;  // hash -> index, inverse
  // domain universe: provisioner.go:266-276 (requirement.Values() of every type + provisioner In requirements). Only topology
  // keys read it, and their values are never collapsed into classes, so the strings here are the dictionary's own.
  std::map<std::string, std::set<std::string>> universe;
  for (int v = 0; v < NV; ++v) {
    const Provisioner& pr = P.provisioners[E.template_provisioner[v]];
    for (int idx : pr.instance_types)
      for (auto& r : P.instance_types[idx].requirements)
        if (r.op == Op::In || r.op == Op::NotIn) universe[normalize_key(r.key)].insert(r.values.begin(), r.values.end());
    // NewNodeSelectorRequirements(provisioner.Spec.Requirements...) then Operator()==In
    std::map<std::string, std::vector<NodeSelectorRequirement>> by_key;
    for (auto& r : pr.requirements) by_key[normalize_key(r.key)].push_back(r);
    for (auto& kv : by_key) {
      int k = B.key_of(kv.first);
      if (k < 0) {  // inactive key: only needed when a single In requirement exists
        if (kv.second.size() == 1 && kv.second[0].op == Op::In) universe[kv.first].insert(kv.second[0].values.begin(), kv.second[0].values.end());
        continue;
      }
      ksched_reqset rs{}; ksched_bounds bd{};
      B.add_selector_reqs(rs, bd, kv.second, nullptr);
      Req r = ksched::req_load(rs, &bd, k);
      if (!r.complement && r.values)
        for (int b = 0; b < 64; ++b) if ((r.values >> b) & 1) universe[kv.first].insert(E.key_values[k][b]);
    }
  }
  auto namespace_list = [](const std::string& ns, const std::vector<std::string>& nss) {
    if (nss.empty()) return std::set<std::string>{ns};
    return std::set<std::string>(nss.begin(), nss.end());
  };
  auto make_filter = [&](Group& g, const Pod& p) {  // MakeTopologyNodeFilter topologynodefilter.go:30-47
    g.filter_nil = false;
    auto canon = [&](const ksched_reqset& rs, const ksched_bounds& bd) {
      std::string s;
      for (int k = 0; k < NK; ++k) {
        Req r = ksched::req_load(rs, &bd, k);
        if (!r.present) continue;
        s += std::to_string(k) + ":" + std::to_string(r.complement) + ":" + std::to_string(r.values) + ":" +
             (r.has_gt ? std::to_string(r.gt) : "") + ":" + (r.has_lt ? std::to_string(r.lt) : "") + ";";
      }
      return s;
    };
    std::vector<std::string> parts;
    auto add_term = [&](const std::vector<NodeSelectorRequirement>* term) {
      ksched_reqset rs{}; ksched_bounds bd{};
      Builder::Special sp;
      B.add_selector_reqs(rs, bd, Builder::label_reqs(p.node_selector), &sp);
      if (term) B.add_selector_reqs(rs, bd, *term, &sp);
      if (!sp.hostname.empty() || !sp.itype.empty()) unsupported("topology spread node filter on hostname / instance-type");
      g.filter.push_back({rs, bd});
      parts.push_back(canon(rs, bd));
    };
    if (!p.has_node_affinity || !p.has_required_node_affinity) add_term(nullptr);
    else for (auto& t : p.required_node_terms) add_term(&t);
    std::sort(parts.begin(), parts.end());
    for (auto& s : parts) g.filter_key += "(" + s + ")";
  };
  auto filter_matches_labels = [&](const Group& g, const Labels& labels) {  // TopologyNodeFilter.Matches
    if (g.filter_nil || g.filter.empty()) return true;
    ksched_reqset rs{}; ksched_bounds bd{};
    Builder::Special sp;
    B.add_selector_reqs(rs, bd, Builder::label_reqs(labels), &sp);
    for (auto& f : g.filter)
      if (B.compatible(rs, bd, f.first, f.second)) return true;
    return false;
  };
  // pods of the batch are not counted as cluster pods (topology.go:66-70); only consulted for pods bound to nodes
  std::unordered_set<std::string> excluded;
  {
    bool any_bound = false;
    for (auto& n : P.nodes) any_bound = any_bound || !n.pods.empty();
    if (any_bound) {
      excluded.reserve(NP * 2);
      for (auto* p : E.pods) excluded.insert(p->uid);
    }
  }
  auto new_group = [&](int type, const std::string& key, const Pod& p, std::set<std::string> nss, const LabelSelector& sel, int32_t skew) {
    Group g;
    g.type = type; g.key = key; g.max_skew = skew; g.namespaces = std::move(nss); g.selector = sel;
    if (type == 0) make_filter(g, p);
    else g.filter_key = "<nil>";
    auto u = universe.find(key);
    if (u != universe.end()) for (auto& d : u->second) g.counts[d] = 0;
    return g;
  };
  auto count_domains = [&](Group& g) {  // topology.go:231-276
    for (auto& n : P.nodes)
      for (auto& p : n.pods) {
        if (!g.namespaces.count(p.ns)) continue;
        if (!g.selector.is_nil && !selector_matches(g.selector, p.labels)) continue;  // TopologyListOptions: nil lists everything
        if (p.terminal || p.terminating) continue;
        if (excluded.count(p.uid)) continue;
        std::string domain;
        auto it = n.labels.find(g.key);
        bool ok = it != n.labels.end();
        if (ok) domain = it->second;
        if (!ok && g.key == kHostname) { domain = n.name; ok = true; }
        if (!ok) continue;
        if (!filter_matches_labels(g, n.labels)) continue;
        g.counts[domain]++;
      }
  };
  auto spec_groups = [&](const Pod& p) {  // newForTopologies + newForAffinities topology.go:278-322
    std::vector<Group> out;
    for (auto& cs : p.topology_spread) out.push_back(new_group(0, cs.topology_key, p, {p.ns}, cs.selector, cs.max_skew));
    for (auto& t : p.pod_affinity_required) out.push_back(new_group(1, t.topology_key, p, namespace_list(p.ns, t.namespaces), t.selector, INT32_MAX));
    for (auto& t : p.pod_affinity_preferred) out.push_back(new_group(1, t.term.topology_key, p, namespace_list(p.ns, t.term.namespaces), t.term.selector, INT32_MAX));
    for (auto& t : p.pod_anti_affinity_required) out.push_back(new_group(2, t.topology_key, p, namespace_list(p.ns, t.namespaces), t.selector, INT32_MAX));
    for (auto& t : p.pod_anti_affinity_preferred) out.push_back(new_group(2, t.term.topology_key, p, namespace_list(p.ns, t.term.namespaces), t.term.selector, INT32_MAX));
    return out;
  };
  auto inverse_groups = [&](const Pod& p, const Labels* node_labels, int owner_spec) {  // updateInverseAntiAffinity topology.go:202-227
    for (auto& term : p.pod_anti_affinity_required) {
      Group g = new_group(2, term.topology_key, p, namespace_list(p.ns, term.namespaces), term.selector, INT32_MAX);
      g.inverse = true;
      std::string h = g.hash();
      auto it = inverse_group_of.find(h);
      size_t gi;
      if (it == inverse_group_of.end()) { gi = groups.size(); inverse_group_of[h] = gi; groups.push_back(std::move(g)); }
      else gi = it->second;
      if (node_labels) {
        auto d = node_labels->find(groups[gi].key);
        if (d != node_labels->end()) groups[gi].counts[d->second]++;
      }
      if (owner_spec >= 0) groups[gi].owner_specs.insert((size_t)owner_spec);
    }
  };
  if (!P.empty_topology) {
    for (auto& n : P.nodes)  // updateInverseAffinities topology.go:185-198
      for (auto& p : n.pods) {
        if (p.pod_anti_affinity_required.empty() || excluded.count(p.uid)) continue;
        inverse_groups(p, &n.labels, -1);
      }
    // Topology.Update for every pod of the batch, in Solve's pod order (topology.go:73-75); group creation order
    // only matters for countDomains, which is order-independent.
    std::vector<bool> seen(specs.size(), false);
    for (size_t i = 0; i < NP; ++i) {
      uint32_t s = E.pod_class[i];
      if (seen[s]) continue;
      seen[s] = true;
      const Pod& p = specs[s].pod;
      if (!p.pod_anti_affinity_required.empty() || !p.pod_anti_affinity_preferred.empty()) inverse_groups(p, nullptr, (int)s);
      for (auto& g : spec_groups(p)) {
        std::string h = g.hash();
        auto it = group_of.find(h);
        size_t gi;
        if (it == group_of.end()) { gi = groups.size(); group_of[h] = gi; count_domains(g); groups.push_back(std::move(g)); }
        else gi = it->second;
        groups[gi].owner_specs.insert(s);
      }
    }
    // relaxed variants: Topology.Update after Relax (scheduler.go:119-123). Their groups must already exist.
    for (size_t s = 0; s < specs.size(); ++s) {
      if (seen[s]) continue;
      const Pod& p = specs[s].pod;
      if (!p.pod_anti_affinity_required.empty() || !p.pod_anti_affinity_preferred.empty()) {
        for (auto& term : p.pod_anti_affinity_required) {
          Group g = new_group(2, term.topology_key, p, namespace_list(p.ns, term.namespaces), term.selector, INT32_MAX);
          g.inverse = true;
          auto it = inverse_group_of.find(g.hash());
          if (it == inverse_group_of.end()) unsupported("relaxation creates a new inverse topology group");
          groups[it->second].owner_specs.insert(s);
        }
      }
      for (auto& g : spec_groups(p)) {
        std::string h = g.hash();
        auto it = group_of.find(h);
        size_t gi;
        if (it == group_of.end()) {
          // Topology.Update creates this group when the pod is relaxed (e.g. the node filter of a spread constraint
          // changes with the required node-affinity terms): counts come from the cluster at that moment, which is the
          // same static state countDomains sees at the start of the solve.
          gi = groups.size();
          group_of[h] = gi;
          g.dormant = true;
          count_domains(g);
          groups.push_back(std::move(g));
        } else {
          gi = it->second;
        }
        groups[gi].owner_specs.insert(s);
      }
    }
  }
  const int NG = (int)groups.size();
  E.groups.resize(NG);
  E.group_domain_counts.assign((size_t)NG * 64, 0);
  E.group_existing_counts.assign((size_t)NG * std::max(NE, 1), 0);
  for (int g = 0; g < NG; ++g) {
    Group& G = groups[g];
    ksched_topo_group& o = E.groups[g];
    std::memset(&o, 0, sizeof o);
    o.type = (uint8_t)G.type;
    o.inverse = G.inverse;
    o.dormant = G.dormant;
    o.max_skew = G.max_skew;
    o.filter_begin = (uint32_t)E.filter_terms.size();
    for (auto& f : G.filter) {
      ksched_reqset term = f.first;
      B.to_region_form(term, f.second);
      E.filter_terms.push_back(term);
    }
    o.filter_end = (uint32_t)E.filter_terms.size();
    if (G.key == kHostname) {
      o.key = KSCHED_KEY_HOSTNAME;
      for (auto& kv : G.counts) {
        auto s = hostname_slot.find(kv.first);
        if (s != hostname_slot.end()) E.group_existing_counts[(size_t)g * std::max(NE, 1) + s->second] = kv.second;
        else if (kv.second > 0) o.extra_nonzero_domains++;
      }
    } else {
      int k = B.key_of(G.key);
      if (k < 0) throw std::runtime_error("internal: topology key not active: " + G.key);
      o.key = (uint8_t)k;
      for (auto& kv : G.counts) {
        auto v = B.value_id[k].find(kv.first);
        if (v == B.value_id[k].end()) {
          if (kv.second > 0) unsupported("topology domain outside the dictionary: " + kv.first);
          // zero-count universe domain that no requirement mentions (e.g. a type-only value): it is still a
          // domain of the group; the dictionary holds every type / template / node value, so this is unreachable.
          throw std::runtime_error("internal: universe domain missing from dictionary: " + kv.first);
        }
        o.registered |= 1ull << v->second;
        E.group_domain_counts[(size_t)g * 64 + v->second] = kv.second;
      }
    }
  }

  if (cluster_superset && NG > 0) {
    // What countDomains (topology.go:231-276) and updateInverseAffinities (:183-227) would add for a bound pod of each class,
    // split into its class part (namespace, selector, owned inverse groups) and its node part (label value, node filter).
    const int NCs = (int)specs.size();
    E.class_count_begin.assign((size_t)NCs + 1, 0);
    for (int c = 0; c < NCs; ++c) {
      const Pod& p = specs[(size_t)c].pod;
      E.class_count_begin[(size_t)c] = (uint32_t)E.class_count.size();
      std::map<size_t, int> inverse_times;
      for (auto& term : p.pod_anti_affinity_required) {
        Group g = new_group(2, term.topology_key, p, namespace_list(p.ns, term.namespaces), term.selector, INT32_MAX);
        g.inverse = true;
        auto it = inverse_group_of.find(g.hash());
        if (it != inverse_group_of.end()) inverse_times[it->second]++;
      }
      for (int g = 0; g < NG; ++g) {
        const Group& G = groups[(size_t)g];
        if (G.inverse) {
          auto it = inverse_times.find((size_t)g);
          if (it != inverse_times.end()) E.class_count.push_back({(uint32_t)g, KSCHED_COUNT_INVERSE, (uint8_t)std::min(it->second, 255), 0});
        } else if (G.namespaces.count(p.ns) && (G.selector.is_nil || selector_matches(G.selector, p.labels))) {
          E.class_count.push_back({(uint32_t)g, KSCHED_COUNT_DOMAINS, 1, 0});
        }
      }
    }
    E.class_count_begin[(size_t)NCs] = (uint32_t)E.class_count.size();
    E.node_domain.assign((size_t)std::max(NK, 1) * std::max(NE, 1), -1);
    E.node_has_hostname_label.assign((size_t)std::max(NE, 1), 0);
    const int FW = (NE + 31) / 32;
    E.group_filter_match.assign((size_t)NG * std::max(FW, 1), 0);
    std::map<std::string, std::vector<char>> filter_memo;  // node labels without the hostname -> verdict per group
    for (int e = 0; e < NE; ++e) {
      const StateNode& n = P.nodes[(size_t)E.existing_state_index[(size_t)e]];
      for (int k = 0; k < NK; ++k) {
        auto l = n.labels.find(E.key_names[(size_t)k]);
        if (l == n.labels.end()) continue;
        auto v = B.value_id[(size_t)k].find(l->second);
        if (v != B.value_id[(size_t)k].end()) E.node_domain[(size_t)k * NE + e] = (int8_t)v->second;
      }
      E.node_has_hostname_label[(size_t)e] = n.labels.count(kHostname) ? 1 : 0;
      Labels sig = n.labels;
      sig.erase(kHostname);
      const std::string key = labels_key(sig);
      auto memo = filter_memo.find(key);
      if (memo == filter_memo.end()) {
        std::vector<char> v((size_t)NG, 1);
        for (int g = 0; g < NG; ++g) v[(size_t)g] = filter_matches_labels(groups[(size_t)g], n.labels) ? 1 : 0;
        memo = filter_memo.emplace(key, std::move(v)).first;
      }
      for (int g = 0; g < NG; ++g)
        if (memo->second[(size_t)g]) E.group_filter_match[(size_t)g * FW + (e >> 5)] |= 1u << (e & 31);
    }
  }

  phase("topology groups");
  // ------------------------------------------------------------------ class rows
  const int NC = (int)specs.size();
  E.classes.resize(NC);
  E.class_bounds.resize(NC);
  std::map<std::string, uint32_t> itype_req_id;
  // (class, group) relations: selector matches of every class against every group, on all cores (pure reads)
  std::vector<uint8_t> rel((size_t)NC * std::max(NG, 1), 0);
  parallel_ranges((size_t)NC, 16, [&](size_t cb, size_t ce) {
    for (size_t c = cb; c < ce; ++c)
      for (int g = 0; g < NG; ++g) {
        const Group& G = groups[g];
        const bool owns = G.owner_specs.count(c) > 0;
        const bool sel = G.selects(specs[c].pod);
        uint32_t flags = 0;
        if (sel) flags |= KSCHED_TOPO_SELECTS;
        if (!G.inverse && owns) flags |= KSCHED_TOPO_CONSTRAINS;
        if (G.inverse && sel) flags |= KSCHED_TOPO_CONSTRAINS;  // Counts(): nil node filter always matches
        if (!G.inverse && sel) flags |= KSCHED_TOPO_RECORDS;
        if (G.inverse && owns) flags |= KSCHED_TOPO_RECORDS_INVERSE;
        rel[c * NG + g] = (uint8_t)flags;
      }
  });
  phase("  class relations");
  for (int c = 0; c < NC; ++c) {
    const Pod& p = specs[c].pod;
    ksched_pod_row& row = E.classes[c];
    std::memset(&row, 0, sizeof row);
    std::memset(&E.class_bounds[c], 0, sizeof(ksched_bounds));
    row.res_present = B.fill_resources(specs[c].req, row.requests);
    ksched_reqset rs{};
    Builder::Special sp;
    B.pod_requirements(p, rs, E.class_bounds[c], &sp);
    std::memcpy(row.values, rs.values, sizeof row.values);
    row.meta = rs.meta;
    if (rs.meta >> KSCHED_META_HASGT_SHIFT) E.any_class_bounds = true;
    row.relax_next = specs[c].next;
    row.reserved = (uint64_t)c;  // class index, so a row copied into the FFD-ordered pod matrix knows its class
    row.itype_req = KSCHED_NONE;
    row.hostname_req = KSCHED_NONE;
    if (!sp.itype.empty()) {
      // intersection of all instance-type requirements of the pod as (complement, name set)
      bool comp = true;
      std::set<std::string> names;
      bool first = true;
      for (auto& r : sp.itype) {
        if (r.op == Op::Gt || r.op == Op::Lt) unsupported("Gt/Lt on instance-type");
        bool rc = !(r.op == Op::In || r.op == Op::DoesNotExist);
        std::set<std::string> rv;
        if (r.op == Op::In || r.op == Op::NotIn) rv.insert(r.values.begin(), r.values.end());
        if (first) { comp = rc; names = rv; first = false; continue; }
        std::set<std::string> nv;
        if (comp && rc) { nv = names; nv.insert(rv.begin(), rv.end()); }
        else if (comp && !rc) { for (auto& x : rv) if (!names.count(x)) nv.insert(x); }
        else if (!comp && rc) { for (auto& x : names) if (!rv.count(x)) nv.insert(x); }
        else { for (auto& x : names) if (rv.count(x)) nv.insert(x); }
        comp = comp && rc;
        names = nv;
      }
      std::string key = std::to_string(comp) + ":";
      for (auto& n : names) key += n + ",";
      auto it = itype_req_id.find(key);
      if (it == itype_req_id.end()) {
        uint32_t id = (uint32_t)E.itype_req_complement.size();
        itype_req_id[key] = id;
        E.itype_req_complement.push_back(comp ? 1 : 0);
        size_t base = E.itype_req_sets.size();
        E.itype_req_sets.resize(base + E.type_words, 0);
        for (int col = 0; col < NT; ++col) {
          bool in = names.count(P.instance_types[E.type_input_index[col]].name) > 0;
          if (comp ? !in : in) E.itype_req_sets[base + col / 64] |= 1ull << (col % 64);
        }
        row.itype_req = id;
      } else {
        row.itype_req = it->second;
      }
    }
    if (!sp.hostname.empty()) {
      if (sp.hostname.size() != 1) unsupported("more than one hostname requirement on a pod");
      auto& r = sp.hostname[0];
      int32_t comp, slot = -1;
      if (r.op == Op::In && r.values.size() == 1) comp = 0;
      else if (r.op == Op::NotIn && r.values.size() == 1) comp = 1;
      else if (r.op == Op::Exists) comp = 1;
      else unsupported("hostname requirement form");
      if (!r.values.empty()) { auto s = hostname_slot.find(r.values[0]); if (s != hostname_slot.end()) slot = s->second; }
      row.hostname_req = (uint32_t)(E.hostname_reqs.size() / 2);
      E.hostname_reqs.push_back(comp);
      E.hostname_reqs.push_back(slot);
    }
    auto hps = host_ports(p);
    for (auto& hp : hps) row.hostport_entries |= 1ull << B.hp_entry(hp);
    // topology relations
    row.topo_begin = (uint32_t)E.class_topo.size();
    for (int g = 0; g < NG; ++g) {
      const uint32_t flags = rel[(size_t)c * NG + g];
      if (flags & ~KSCHED_TOPO_SELECTS) E.class_topo.push_back({(uint32_t)g, flags});
    }
    row.topo_end = (uint32_t)E.class_topo.size();
  }
  if (!vol_drivers.empty()) {
    E.class_volumes.resize(NC);
    bool any = false;
    for (int c = 0; c < NC; ++c) any = !volume_signature(specs[c].pod, &E.class_volumes[c]).empty() || any;
    if (!any) E.class_volumes.clear();  // no pod of the batch mounts a limited claim: the kernels never look
    for (auto& kv : vol_tracked) {
      const size_t d = (size_t)(std::find(vol_drivers.begin(), vol_drivers.end(), kv.first.first) - vol_drivers.begin());
      E.volume_driver_mask[d] |= 1ull << kv.second;
    }
  }
  // host-port conflict masks and tolerated taint sets need the complete entry / taint-set tables
  for (int c = 0; c < NC; ++c) {
    const Pod& p = specs[c].pod;
    for (auto& hp : host_ports(p))
      for (size_t e = 0; e < B.hp_entries.size(); ++e)
        if (hp_matches(hp, B.hp_entries[e])) E.classes[c].hostport_conflicts |= 1ull << e;
    for (size_t s = 0; s < B.taintsets.size(); ++s)
      if (tolerates_all(B.taintsets[s], p.tolerations)) E.classes[c].tolerated_taintsets |= 1ull << s;
  }

  phase("class rows");
  // ------------------------------------------------------------------ per-pod queue keys (queue.go:74-110)
  E.pod_uid_rank.resize(NP);
  {
    if (uids_ascending) {
      for (size_t i = 0; i < NP; ++i) E.pod_uid_rank[i] = (uint32_t)i;
    } else {
      std::vector<uint32_t> order(NP);
      for (size_t i = 0; i < NP; ++i) order[i] = (uint32_t)i;
      std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return E.pods[a]->uid < E.pods[b]->uid; });
      for (size_t r = 0; r < NP; ++r) E.pod_uid_rank[order[r]] = (uint32_t)r;
    }
  }

  phase("queue keys");
  // ------------------------------------------------------------------ wire up the flat structs
  ksched_catalog& cat = E.catalog;
  cat.n_keys = NK; cat.n_res = (int)E.res_names.size(); cat.n_types = NT; cat.n_templates = NV;
  cat.keys = E.keys.data();
  cat.key_int_values = E.key_int_values.data();
  cat.types = E.types.data();
  cat.type_bounds = nullptr;
  cat.type_capacity = E.type_capacity.data();
  cat.templates = E.templates.data();
  cat.template_bounds = nullptr;
  cat.offering_keys = E.offering_keys.data();
  ksched_problem& pr = E.problem;
  pr.n_pods = (int)NP; pr.n_classes = NC; pr.n_existing = NE; pr.n_groups = NG;
  pr.classes = E.classes.data();
  pr.class_bounds = nullptr;
  pr.pod_class = E.pod_class.data();
  pr.pod_timestamp = E.pod_timestamp.data();
  pr.pod_uid_rank = E.pod_uid_rank.data();
  pr.existing = E.existing.data();
  pr.existing_bounds = nullptr;
  pr.groups = E.groups.data();
  pr.group_domain_counts = E.group_domain_counts.data();
  pr.group_existing_counts = E.group_existing_counts.data();
  pr.class_topo = E.class_topo.data();
  pr.n_class_topo = (int)E.class_topo.size();
  pr.filter_terms = E.filter_terms.data();
  pr.n_filter_terms = (int)E.filter_terms.size();
  pr.itype_req_sets = E.itype_req_sets.data();
  pr.itype_req_complement = E.itype_req_complement.data();
  pr.n_itype_reqs = (int)E.itype_req_complement.size();
  pr.hostname_reqs = E.hostname_reqs.data();
  pr.n_hostname_reqs = (int)E.hostname_reqs.size() / 2;
  pr.max_new_nodes = (int)NP;
  pr.write_feasibility = 0;
  if (!E.class_volumes.empty() && NE > 0) {
    pr.class_volumes = E.class_volumes.data();
    pr.existing_volumes = E.existing_volumes.data();
    for (int d = 0; d < KSCHED_MAX_VOLUME_DRIVERS; ++d) pr.volume_driver_mask[d] = E.volume_driver_mask[d];
  }
  pr.count_nodes_visited = 0;  // the exact nodes_visited statistic is opt-in (kh_set_count_visited / tests): it turns the pack kernel's steady-state paths off
  // Gt/Lt leave the host algebra here: templates and pod classes in region form (types and filter terms already are)
  for (int v = 0; v < NV; ++v) B.to_region_form(E.templates[v].reqs, tb[v]);
  for (int c = 0; c < NC; ++c) {
    ksched_reqset rs{};
    std::memcpy(rs.values, E.classes[c].values, sizeof rs.values);
    rs.meta = E.classes[c].meta;
    B.to_region_form(rs, E.class_bounds[c]);
    std::memcpy(E.classes[c].values, rs.values, sizeof rs.values);
    E.classes[c].meta = rs.meta;
  }
  cat.key_regions = E.key_regions.empty() ? nullptr : E.key_regions.data();
  return enc;
}

bool label_selector_matches(const kmodel::LabelSelector& sel, const kmodel::Labels& labels) { return !sel.is_nil && selector_matches(sel, labels); }

std::string render_requirement(const Encoded& E, const ksched_reqset& rs, int k) {
  static const ksched_bounds zero{};
  Req r = ksched::req_load(rs, &zero, k);
  // results come back in region form (ksched.h: ksched_key_regions): recover the excluded set proper and the bounds
  std::string bounds;
  if (r.complement && !E.key_regions.empty() && E.key_regions[k].region_mask) {
    const ksched_key_regions& g = E.key_regions[k];
    const int low = ksched::region_low(r.values, g), high = ksched::region_high(r.values, g);
    r.values = ksched::req_excluded(r, KeyMeta{0, nullptr, &g});
    if (low > 0) bounds += " >" + std::to_string(g.thresholds[low - 1]);
    if (high > 0) bounds += " <" + std::to_string(g.thresholds[g.n_thresholds - high]);
  }
  const char* op;
  if (r.complement) op = r.values ? "NotIn" : "Exists";
  else op = r.values ? "In" : "DoesNotExist";
  std::string s = std::string(op) + " [";
  bool first = true;
  for (size_t b = 0; b < E.key_values[k].size(); ++b)
    if ((r.values >> b) & 1) { if (!first) s += " "; s += E.key_values[k][b]; first = false; }
  return s + "]" + bounds;
}

}  // namespace khost
