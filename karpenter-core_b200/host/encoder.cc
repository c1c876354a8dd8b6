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
#include <limits>
#include <optional>
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

// NewRequirement (requirement.go:44-68) on a dictionary: id maps a value to its bit
Req new_requirement(Op op, const std::vector<std::string>& values, const std::map<std::string, int>& id) {
  Req r{0, 0, 0, true, !(op == Op::In || op == Op::DoesNotExist), false, false};
  if (op == Op::In || op == Op::NotIn)
    for (auto& v : values) r.values |= 1ull << id.at(v);
  if (op == Op::Gt) { r.has_gt = true; parse_int(values.at(0), &r.gt); }
  if (op == Op::Lt) { r.has_lt = true; parse_int(values.at(0), &r.lt); }
  return r;
}

// A requirement on kubernetes.io/hostname in the reference's string algebra: NewRequirement (requirement.go:44-68),
// Intersection (:117-150), Has (:171-176), Operator (:186-197). Hostnames are not dictionary values, so the encoder
// evaluates these on strings and hands the device the existing slots they admit (DESIGN.md §3, hostname requirements).
// The daemonset overhead uses the same algebra on node.kubernetes.io/instance-type (string_compatible).
constexpr const char* kPlaceholderPrefix = "hostname-placeholder-";  // a new node's hostname (node.go:46, a per-Solve counter)
struct HostnameReq {
  bool comp = true;  // (true, {}, no bounds): Exists
  std::set<std::string> values;
  bool has_gt = false, has_lt = false;
  int64_t gt = 0, lt = 0;
  static HostnameReq make(const NodeSelectorRequirement& r) {
    for (auto& v : r.values)
      if (v.rfind(kPlaceholderPrefix, 0) == 0) unsupported("hostname requirement naming a placeholder hostname: " + v);
    return of(r);
  }
  static HostnameReq of(const NodeSelectorRequirement& r) {  // NewRequirement on any key
    HostnameReq h;
    h.comp = !(r.op == Op::In || r.op == Op::DoesNotExist);
    if (r.op == Op::In || r.op == Op::NotIn) h.values.insert(r.values.begin(), r.values.end());
    if (r.op == Op::Gt) { h.has_gt = true; parse_int(r.values.at(0), &h.gt); }
    if (r.op == Op::Lt) { h.has_lt = true; parse_int(r.values.at(0), &h.lt); }
    return h;
  }
  bool within(const std::string& v) const {
    if (!has_gt && !has_lt) return true;
    int64_t x;
    if (!parse_int(v, &x)) return false;
    return !(has_gt && gt >= x) && !(has_lt && lt <= x);
  }
  bool has(const std::string& v) const { return (values.count(v) > 0) != comp && within(v); }
  HostnameReq intersect(const HostnameReq& o) const {
    HostnameReq r;
    r.has_gt = has_gt || o.has_gt;
    r.gt = has_gt && o.has_gt ? std::max(gt, o.gt) : (has_gt ? gt : o.gt);
    r.has_lt = has_lt || o.has_lt;
    r.lt = has_lt && o.has_lt ? std::min(lt, o.lt) : (has_lt ? lt : o.lt);
    if (r.has_gt && r.has_lt && r.gt >= r.lt) return HostnameReq{false, {}, false, false, 0, 0};  // DoesNotExist
    r.comp = comp && o.comp;
    if (comp && o.comp) { r.values = values; r.values.insert(o.values.begin(), o.values.end()); }
    else if (comp) { for (auto& v : o.values) if (!values.count(v)) r.values.insert(v); }
    else if (o.comp) { for (auto& v : values) if (!o.values.count(v)) r.values.insert(v); }
    else { for (auto& v : values) if (o.values.count(v)) r.values.insert(v); }
    for (auto it = r.values.begin(); it != r.values.end();) it = r.within(*it) ? std::next(it) : r.values.erase(it);
    if (!r.comp) r.has_gt = r.has_lt = false;
    return r;
  }
  // Operator() is NotIn or DoesNotExist: Compatible with a node that has no hostname label (requirements.go:123-133)
  bool admits_unlabelled() const { return comp ? !values.empty() : values.empty(); }
  // A new node's hostname is a placeholder: not an integer, and never one of `values` (make refuses such values)
  bool admits_new() const { return comp && !has_gt && !has_lt; }
  std::string key() const {
    std::string s = comp ? "!" : "=";
    for (auto& v : values) s += v + ",";
    return s + "|" + (has_gt ? std::to_string(gt) : "") + "|" + (has_lt ? std::to_string(lt) : "");
  }
};
// A requirement on node.kubernetes.io/instance-type as (complement, names): the names it admits, or for a complement the
// names it excludes (itype_intersection).
using ItypeSet = std::pair<bool, std::set<std::string>>;

// Requirements.Add of a pod's hostname requirements, in order (requirements.go:87-94)
HostnameReq hostname_intersection(const std::vector<NodeSelectorRequirement>& rs) {
  HostnameReq h = HostnameReq::make(rs.at(0));
  for (size_t i = 1; i < rs.size(); ++i) h = HostnameReq::make(rs[i]).intersect(h);
  return h;
}
// Requirements.Add of a list of requirements on one key, on strings; nullopt for an empty list (the key is not defined)
std::optional<HostnameReq> string_requirement(const std::vector<NodeSelectorRequirement>& rs) {
  if (rs.empty()) return std::nullopt;
  HostnameReq h = HostnameReq::of(rs[0]);
  for (size_t i = 1; i < rs.size(); ++i) h = HostnameReq::of(rs[i]).intersect(h);
  return h;
}
// One key of Requirements.Compatible (requirements.go:123-133) on strings, `node` the receiver and nullopt where a side does
// not define the key: an undefined node key admits anything on a well-known key and only NotIn / DoesNotExist on another;
// a defined one must Intersect (:189-206): a non-empty intersection, or NotIn / DoesNotExist on both sides.
bool string_compatible(const std::optional<HostnameReq>& node, const std::optional<HostnameReq>& inc, bool well_known) {
  if (!inc) return true;
  if (!node) return well_known || inc->admits_unlabelled();
  const HostnameReq i = node->intersect(*inc);
  if (i.comp || !i.values.empty()) return true;  // Len() of a complement is never 0
  return node->admits_unlabelled() && inc->admits_unlabelled();
}

// ---- resources (utils/resources/resources.go)
ResourceList merge(const ResourceList& a, const ResourceList& b) {  // checked: sums stay inside kQuantityBound
  ResourceList r = a;
  for (auto& kv : b) r[kv.first] = checked_quantity((__int128)r[kv.first] + kv.second, kv.first);
  return r;
}
// lhs[k] -= rhs[k] for the keys of lhs that rhs has (resources.Subtract), checked like merge
void subtract_in_place(ResourceList& lhs, const ResourceList& rhs) {
  for (auto& kv : lhs) {
    auto f = rhs.find(kv.first);
    if (f != rhs.end()) kv.second = checked_quantity((__int128)kv.second - f->second, kv.first);
  }
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
  return selector_valid(s) && selector_matches_labels(s, labels);
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
  if (!t.namespace_selector.is_nil) s += "|ns=" + selector_key(t.namespace_selector);
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
  return a.topology_key == b.topology_key && a.namespaces == b.namespaces && same_selector(a.selector, b.selector) &&
         same_selector(a.namespace_selector, b.namespace_selector);
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
  // a namespace selector is mixed in only where one is set: pods without one hash as they always did
  auto ns_selector = [&](const PodAffinityTerm& t) {
    if (!t.namespace_selector.is_nil) { labels(t.namespace_selector.match_labels); mix(t.namespace_selector.match_expressions.size() + 1); }
  };
  mix(p.pod_affinity_required.size());
  for (auto& t : p.pod_affinity_required) { str(t.topology_key); ns_selector(t); }
  mix(p.pod_affinity_preferred.size());
  for (auto& t : p.pod_affinity_preferred) ns_selector(t.term);
  mix(p.pod_anti_affinity_required.size());
  for (auto& t : p.pod_anti_affinity_required) { str(t.topology_key); ns_selector(t); }
  mix(p.pod_anti_affinity_preferred.size());
  for (auto& t : p.pod_anti_affinity_preferred) ns_selector(t.term);
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

std::vector<NodeSelectorRequirement> label_reqs(const Labels& l) {  // NewLabelRequirements requirements.go:54-59
  std::vector<NodeSelectorRequirement> out;
  for (auto& kv : l) out.push_back({kv.first, Op::In, {kv.second}});
  return out;
}
Labels template_labels(const Provisioner& pr) {  // NewMachineTemplate's labels (machinetemplate.go:46-62)
  Labels l = pr.labels;
  l[kProvisionerName] = pr.name;
  return l;
}
// The requirement lists a pod can put into a node's requirements (NewPodRequirements, requirements.go:61-78): its node
// selector as labels, every required term and every preferred term.
template <class F>
void pod_requirement_lists(const Pod& p, F f) {
  f(label_reqs(p.node_selector));
  for (auto& t : p.required_node_terms) f(t);
  for (auto& t : p.preferred_node_terms) f(t.preference);
}
// The topology terms of a pod, in the order newForTopologies + newForAffinities make groups of them (topology.go:278-322):
// f(type, topology key, namespaces, selector, max skew) with type 0 spread, 1 affinity, 2 anti-affinity. Empty namespaces
// stand for the pod's own.
template <class F>
void pod_topology_terms(const Pod& p, F f) {
  static const std::vector<std::string> own;
  for (auto& t : p.topology_spread) f(0, t.topology_key, own, t.selector, t.max_skew);
  for (auto& t : p.pod_affinity_required) f(1, t.topology_key, t.namespaces, t.selector, INT32_MAX);
  for (auto& t : p.pod_affinity_preferred) f(1, t.term.topology_key, t.term.namespaces, t.term.selector, INT32_MAX);
  for (auto& t : p.pod_anti_affinity_required) f(2, t.topology_key, t.namespaces, t.selector, INT32_MAX);
  for (auto& t : p.pod_anti_affinity_preferred) f(2, t.term.topology_key, t.term.namespaces, t.term.selector, INT32_MAX);
}
// Resource ids: cpu, memory and pods first, then the other names in order.
std::vector<std::string> resource_order(const std::set<std::string>& names) {
  std::vector<std::string> out = {"cpu", "memory", "pods"};
  for (auto& n : names) if (std::find(out.begin(), out.begin() + 3, n) == out.begin() + 3) out.push_back(n);
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
        pod_requirement_lists(p, [&](const std::vector<NodeSelectorRequirement>& rs) {
          for (auto& q : rs)
            if (q.op == Op::In || q.op == Op::NotIn)
              for (auto& v : q.values) f->named_pairs.insert({normalize_key(q.key), v});
        });
        nf.pod_req = merge(nf.pod_req, r);
        if (p.is_daemonset) nf.ds_req = merge(nf.ds_req, r);
        for (auto& hp : host_ports(p)) nf.hostports.push_back(hp);
        for (auto& t : p.pod_anti_affinity_required) f->anti_keys.insert(t.topology_key);
      }
      nf.label_reqs = label_reqs(n.labels);
      nf.taints = state_node_taints(n);
      for (auto& kv : n.labels) f->label_pairs.insert({kv.first, kv.second});
    }
    P.derived = f;
  }
  return static_cast<const ClusterFacts&>(*P.derived);
}

struct Profile {  // KSCHED_ENCODE_PROFILE: one line per phase of encode() on stderr
  std::chrono::steady_clock::time_point last = std::chrono::steady_clock::now();
  void operator()(const char* name) {
    static const bool on = std::getenv("KSCHED_ENCODE_PROFILE") != nullptr;
    if (!on) return;
    auto now = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[encode] %-28s %8.2f ms\n", name, std::chrono::duration<double, std::milli>(now - last).count());
    last = now;
  }
};

struct Spec { Pod pod; ResourceList req; uint32_t next = KSCHED_NONE; };  // a pod class and the class its relaxation leads to
// a daemonset pod's requirements (on the mask keys, and on the hostname / instance-type keys when it names them) and requests
struct Daemon { const Pod* pod; ksched_reqset rs; ksched_bounds bd; std::optional<HostnameReq> hostname, itype; ResourceList req; };

// The encoder's state: what one phase of encode() hands to the next.
struct Builder {
  Profile phase;
  const Problem& P;
  Encoded& E;
  const ClusterFacts& facts;
  const bool superset;                                     // encode(..., cluster_superset)
  std::vector<int> state_nodes;                            // Problem.nodes that stay existing nodes
  bool tolerate_pns = false;                               // scheduler.go:49-56
  bool uids_ascending = true;                              // the batch's UIDs: unique and already in rank order
  std::vector<std::string> vol_drivers;                    // CSI drivers some owned state node limits
  std::map<std::pair<std::string, std::string>, int> vol_tracked;  // (driver, claim) -> bit
  std::vector<Spec> specs;                                 // pod classes, relaxed variants included (intern)
  std::map<std::string, uint32_t> spec_id;
  std::set<std::string> well_known;
  std::map<std::string, int> key_id;                       // mask key -> id
  std::vector<std::map<std::string, int>> value_id;        // per key
  std::map<std::string, int> res_id;
  std::vector<KeyMeta> key_meta;
  std::map<std::string, int> taintset_id;
  std::vector<std::vector<Taint>> taintsets;
  std::vector<HostPortEntry> hp_entries;                   // host-port entries in id order (host_port_table)
  std::map<HostPortEntry, int> hp_id;                      // every entry of the problem -> id, -1 = left out
  std::map<std::string, int> type_col;                    // instance type name -> column
  bool res_pruned = false;                                 // resource names no request reads were left out of res_id
  std::vector<Daemon> daemons;
  std::map<std::string, int> hostname_slot;                // hostname -> existing slot
  std::vector<std::string> slot_hostname;                  // existing slot -> hostname (label, or the node's name)
  // hostname_reqs entries: the string form of a table entry (admitted slots read from E.hostname_slots), none for the
  // {complement, slot} pair form
  std::vector<std::optional<HostnameReq>> hostname_forms;
  std::map<std::string, uint32_t> hostname_table_id;       // HostnameReq::key() -> entry
  bool filter_names_hostname = false;                      // some topology node filter term has a hostname part
  std::map<std::string, uint32_t> itype_req_id;            // (complement, names) -> itype_req entry (itype_entry)
  // instance-type parts of topology node filter terms, in filter_terms order, and the templates' requirements on the key
  std::vector<std::optional<ItypeSet>> filter_itype, template_itype;
  std::string itype_unlisted;                              // a type name outside the catalog that a requirement keeps, or ""

  Builder(const Problem& p, Encoded& e, bool cluster_superset) : P(p), E(e), facts(cluster_facts(p)), superset(cluster_superset) {}

  // ------------------------------------------------------------ requirement encoding
  int key_of(const std::string& k) const {
    auto it = key_id.find(normalize_key(k));
    return it == key_id.end() ? -1 : it->second;
  }
  Req encode_req(int k, Op op, const std::vector<std::string>& values) const { return new_requirement(op, values, value_id[k]); }
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
    int id = (int)taintsets.size();  // ids from 64 on only ever go to existing nodes' sets (class_tolerated_ext, ksched.h)
    taintset_id[k] = id;
    taintsets.push_back(ts);
    return id;
  }
  // hostname_reqs entries (ksched.h): the {complement, slot} pair of In / NotIn one value and Exists, as before tables
  // existed, or an entry whose admitted existing slots are a row of the table (one per distinct requirement)
  uint32_t hostname_pair(int32_t comp, int32_t slot) {
    E.hostname_reqs.push_back(comp);
    E.hostname_reqs.push_back(slot);
    hostname_forms.emplace_back();
    return (uint32_t)hostname_forms.size() - 1;
  }
  uint32_t hostname_table(const HostnameReq& h) {
    auto id = hostname_table_id.emplace(h.key(), (uint32_t)hostname_forms.size());
    if (!id.second) return id.first->second;
    E.hostname_reqs.push_back(h.admits_new() ? 1 : 0);
    E.hostname_reqs.push_back(KSCHED_HOSTNAME_TABLE);
    hostname_forms.push_back(h);
    return id.first->second;
  }
  int hp_entry(const HostPortEntry& e) const {  // id of an entry (host_port_table), -1 when it was left out
    auto it = hp_id.find(e);
    if (it == hp_id.end()) throw std::runtime_error("internal: host-port entry missing from the table");
    return it->second;
  }
  // host-port entry or tracked volume claim `id`'s bit: of `word` below 64, of ext[(id - 64) / 64] (a table row of
  // E.hostport_ext_words / E.volume_ext_words words) from 64 on
  static void id_bit(int id, uint64_t& word, uint64_t* ext) {
    if (id < 0) return;  // a host-port entry left out: it can turn no pod away
    if (id < 64) word |= 1ull << id;
    else ext[(id - 64) / 64] |= 1ull << ((id - 64) % 64);
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
      if (id >= KSCHED_MAX_RES) continue;  // an ext resource: fill_ext
      out[id] = kv.second;
      present |= 1u << id;
    }
    return present;
  }
  // ext resources (ids from KSCHED_MAX_RES on) of r into out[E.n_res_ext]; bit x of the result: ext resource x is a key of r
  uint32_t fill_ext(const ResourceList& r, int64_t* out) const {
    uint32_t present = 0;
    for (int i = 0; i < E.n_res_ext; ++i) out[i] = 0;
    for (auto& kv : r) {
      auto it = res_id.find(kv.first);
      if (it == res_id.end() || it->second < KSCHED_MAX_RES) continue;
      out[it->second - KSCHED_MAX_RES] = kv.second;
      present |= 1u << (it->second - KSCHED_MAX_RES);
    }
    return present;
  }

  // ------------------------------------------------------------ CSI volume limits (ksched.h: ksched_class_volumes)
  size_t driver_index(const std::string& driver) const {  // vol_drivers.size() when the driver has no limit
    return (size_t)(std::find(vol_drivers.begin(), vol_drivers.end(), driver) - vol_drivers.begin());
  }
  std::map<std::string, std::set<std::string>> pod_claims(const Pod& p) const {  // VolumeUsage.validate: driver -> claims, limited drivers only
    std::map<std::string, std::set<std::string>> m;
    for (auto& v : p.volumes)
      if (!v.driver.empty() && driver_index(v.driver) < vol_drivers.size()) m[v.driver].insert(v.pvc_id);
    return m;
  }
  // The class's claims (out, and its tracked claims from id 64 on into ext[E.volume_ext_words] when given) and their part of
  // the class key: "" without a claim. The key carries every word, so pods that differ in a claim beyond 64 stay apart.
  std::string volume_signature(const Pod& p, ksched_class_volumes* out, uint64_t* ext = nullptr) const {
    ksched_class_volumes cv{};
    std::vector<uint64_t> words((size_t)E.volume_ext_words, 0);
    if (!vol_drivers.empty())
      for (auto& kv : pod_claims(p)) {
        const size_t d = driver_index(kv.first);
        for (auto& c : kv.second) {
          auto t = vol_tracked.find({kv.first, c});
          if (t != vol_tracked.end()) id_bit(t->second, cv.shared, words.data());
          else if (cv.priv[d] == 0xFFFF) unsupported("more than 65535 volume claims on one pod");
          else cv.priv[d]++;
        }
      }
    if (out) *out = cv;
    if (ext) std::copy(words.begin(), words.end(), ext);
    char b[96];
    std::snprintf(b, sizeof b, "|V=%llx:%u:%u:%u:%u", (unsigned long long)cv.shared, cv.priv[0], cv.priv[1], cv.priv[2], cv.priv[3]);
    std::string key(b);
    bool any = (cv.shared | cv.priv[0] | cv.priv[1] | cv.priv[2] | cv.priv[3]) != 0;
    for (uint64_t w : words) {
      std::snprintf(b, sizeof b, ":%llx", (unsigned long long)w);
      key += b;
      any = any || w != 0;
    }
    return any ? key : std::string();
  }

  // ------------------------------------------------------------ pod classes and relaxation chains
  uint32_t intern(const Pod& p) {
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
  }
  // the pods whose requirements can reach a node: every pod class (relaxed variants included) and every daemonset pod
  template <class F>
  void for_class_and_daemon_pods(F f) const {
    for (auto& s : specs) f(s.pod);
    for (auto& d : P.daemonset_pods) f(d);
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
  std::vector<std::optional<HostnameReq>> filter_host;          // per term: its hostname part, if it names the hostname
  std::vector<std::optional<ItypeSet>> filter_itype;            // per term: its instance-type part, if it names the key
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

// Requirement::Canonical() of the oracle: "<Operator()> [values in string order]", then the bounds (" >gt", " <lt")
std::string render_canonical(bool complement, uint64_t values, const std::vector<std::string>& dict, const std::string& bounds) {
  const char* op;
  if (complement) op = values ? "NotIn" : "Exists";
  else op = values ? "In" : "DoesNotExist";
  std::string s = std::string(op) + " [";
  bool first = true;
  for (size_t b = 0; b < dict.size(); ++b)
    if ((values >> b) & 1) { if (!first) s += " "; s += dict[b]; first = false; }
  return s + "]" + bounds;
}

// One template-only key (DESIGN.md §3) in the host algebra of reqmask.cuh, on a dictionary of its own: the values that the
// given requirement lists name, in string order. Intersects only ever meets values both sides name, so this is exact.
struct FoldedKey {
  std::map<std::string, int> id;
  std::vector<std::string> values;
  uint64_t int_mask = 0;
  int64_t ints[64] = {};
  explicit FoldedKey(std::initializer_list<const std::vector<NodeSelectorRequirement>*> lists) {
    std::set<std::string> named;
    for (auto* l : lists)
      for (auto& r : *l)
        if (r.op == Op::In || r.op == Op::NotIn) named.insert(r.values.begin(), r.values.end());
    if (named.size() > 64) unsupported("a template-only label key whose requirements name more than 64 values");
    for (auto& v : named) {
      const int b = (int)values.size();
      id[v] = b;
      values.push_back(v);
      if (parse_int(v, &ints[b])) int_mask |= 1ull << b;
    }
  }
  KeyMeta meta() const { return KeyMeta{int_mask, ints, nullptr}; }
  // NewRequirement (requirement.go:44-68) of every requirement, combined by Requirements.Add (requirements.go:87-94)
  Req req(const std::vector<NodeSelectorRequirement>& rs) const {
    Req cur = ksched::req_absent();
    for (auto& r : rs) cur = ksched::key_add(cur, new_requirement(r.op, r.values, id), meta());
    return cur;
  }
  std::string render(const Req& r) const {
    std::string bounds;
    if (r.has_gt) bounds += " >" + std::to_string(r.gt);
    if (r.has_lt) bounds += " <" + std::to_string(r.lt);
    return render_canonical(r.complement, r.values, values, bounds);
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

namespace {

// ------------------------------------------------------------------ who takes part
// The nodes that stay existing nodes, Solve's pod list (provisioner.go:119-144, deprovisioning/helpers.go:42-93), the
// well-known keys and the template order.
void participants(Builder& B, const std::vector<int>& candidates) {
  const Problem& P = B.P;
  Encoded& E = B.E;
  std::set<int> cand(candidates.begin(), candidates.end());
  auto reschedulable = [](const Pod& p) { return !p.is_daemonset && !p.terminal && !p.terminating; };  // utils/node/node.go:30-50
  for (size_t i = 0; i < P.nodes.size(); ++i)
    if ((B.superset || !cand.count((int)i)) && !P.nodes[i].marked_for_deletion) B.state_nodes.push_back((int)i);
  for (auto& p : P.pods) E.pods.push_back(&p);
  auto deleting_nodes_pods = [&] {  // pending in every simulation
    for (size_t i = 0; i < P.nodes.size(); ++i)
      if (!cand.count((int)i) && P.nodes[i].marked_for_deletion)
        for (auto& p : P.nodes[i].pods) if (reschedulable(p)) E.pods.push_back(&p);
  };
  if (B.superset) {
    // pending pods first, then the candidates' pods node by node
    deleting_nodes_pods();
    E.pod_node.assign(E.pods.size(), -1);
    for (int c : candidates) {
      if (P.nodes.at(c).marked_for_deletion) throw std::runtime_error("a candidate node is marked for deletion");
      for (auto& p : P.nodes[c].pods) if (reschedulable(p)) { E.pods.push_back(&p); E.pod_node.push_back(-2 - c); }  // slot resolved in existing_nodes
    }
  } else {
    for (int c : candidates)
      for (auto& p : P.nodes.at(c).pods) if (reschedulable(p)) E.pods.push_back(&p);
    deleting_nodes_pods();
  }
  if (P.provisioners.empty()) throw std::runtime_error("no provisioners found");
  if (P.provisioners.size() > KSCHED_MAX_TEMPLATES) unsupported("more than 64 provisioners");

  B.well_known = {kProvisionerName, kZone, "topology.kubernetes.io/region", kInstanceType, "kubernetes.io/arch", "kubernetes.io/os", kCapacityType};
  B.well_known.insert(P.extra_well_known_labels.begin(), P.extra_well_known_labels.end());

  // template order: OrderByWeight (v1alpha5/provisioner.go:132-136), stable
  for (size_t i = 0; i < P.provisioners.size(); ++i) E.template_provisioner.push_back((int)i);
  std::stable_sort(E.template_provisioner.begin(), E.template_provisioner.end(),
                   [&](int a, int b) { return P.provisioners[a].weight > P.provisioners[b].weight; });
  for (auto& pr : P.provisioners)
    for (auto& t : pr.taints) if (t.effect == "PreferNoSchedule") B.tolerate_pns = true;
}

// ------------------------------------------------------------------ CSI volume limits (ksched.h: ksched_class_volumes)
// Drivers some owned state node limits; claims by how many pods (batch + bound) mount them: one -> counted, several -> tracked id.
// When that would track more than 64 claims, a claim is tracked only when two different pods mount it and one of them is a pod
// of the batch (DESIGN.md §3, volume claims beyond the word). A claim only bound pods mount stays in their nodes' used[], which
// count it once per node already; a claim exactly one pod mounts is private to it. Problems that fit keep their encoding.
void csi_volumes(Builder& B) {
  std::set<std::string> drivers;
  for (int si : B.state_nodes) for (auto& kv : B.P.nodes[si].volume_limits) drivers.insert(kv.first);
  B.vol_drivers.assign(drivers.begin(), drivers.end());
  if (B.vol_drivers.size() > KSCHED_MAX_VOLUME_DRIVERS) unsupported("more than 4 CSI drivers with node volume limits");
  if (B.vol_drivers.empty()) return;
  struct Mounts { int refs = 0; const Pod* first = nullptr; bool two_pods = false, batch = false; };
  std::map<std::pair<std::string, std::string>, Mounts> claims;
  // (a candidate's pod is reached through E.pods and through its node's pod list: one Pod object, one pod)
  auto count = [&](const Pod& p, bool batch) {
    for (auto& kv : B.pod_claims(p))
      for (auto& c : kv.second) {
        Mounts& m = claims[{kv.first, c}];
        m.refs++;
        if (!m.first) m.first = &p; else m.two_pods = m.two_pods || m.first != &p;
        m.batch = m.batch || batch;
      }
  };
  for (auto* p : B.E.pods) count(*p, true);
  for (int si : B.state_nodes) for (auto& p : B.P.nodes[si].pods) count(p, false);
  size_t shared = 0;
  for (auto& kv : claims) shared += kv.second.refs > 1;
  for (auto& kv : claims)
    if (shared <= 64 ? kv.second.refs > 1 : kv.second.two_pods && kv.second.batch) {
      B.vol_tracked[kv.first] = (int)B.E.volume_claims.size();
      B.E.volume_claims.push_back(kv.first);
    }
  const size_t n = B.E.volume_claims.size();
  B.E.volume_ext_words = n > 64 ? (int)((n - 64 + 63) / 64) : 0;
}

// ------------------------------------------------------------------ pod specs: classes and relaxation chains
void pod_classes(Builder& B) {
  Encoded& E = B.E;
  const size_t NP = E.pods.size();
  E.pod_class.resize(NP);
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
      E.pod_timestamp[i] = p.creation_ts;  // queue.go:74-110 sorts by it (per-pod queue keys)
    }
    if (!asc) uid_order_broken[b >> 12] = 1;  // (ranges start at multiples of >= 4096 pods or at 0: one flag each)
  });
  // strictly ascending UIDs (the usual case: one informer list) are unique and already ranked
  for (uint8_t f : uid_order_broken) B.uids_ascending = B.uids_ascending && !f;
  if (!B.uids_ascending) {
    std::unordered_set<std::string> uids;
    uids.reserve(NP * 2);
    for (auto* p : E.pods)
      if (!uids.insert(p->uid).second) throw std::runtime_error("pods must have unique UIDs: " + p->uid);
  }
  B.phase("  same_spec pairs");
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
          if (same_spec(p, B.specs[cid].pod)) { id = cid; break; }
    }
    if (id == KSCHED_NONE) {
      id = B.intern(p);
      if (p.volumes.empty()) {
        auto& v = by_hash[run_hash[i]];
        if (std::find(v.begin(), v.end(), id) == v.end()) v.push_back(id);
      }
    }
    E.pod_class[i] = id;
  }
  B.phase("  intern boundaries");
}

// ------------------------------------------------------------------ active keys + dictionary
// Active keys: everything that can appear in a node's requirements (template or pod side). Keys that only instance types
// define can never meet a node requirement (Intersects walks keys present on BOTH sides, requirements.go:189-190) and are
// dropped. Template-only keys (DESIGN.md §3) go to *foldable: no pod-side source names them, so a node's requirement on one is
// always its template's own and the key only decides which instance types the template admits. Zone and capacity-type stay
// mask keys: offerings, the launch choice and the price helpers read them.
std::set<std::string> active_keys(const Builder& B, std::set<std::string>* foldable) {
  // pod-side keys: anything a pod / daemonset / topology group / node filter can put into a node's requirements
  std::set<std::string> pod_side;
  B.for_class_and_daemon_pods([&](const Pod& p) {
    pod_requirement_lists(p, [&](const std::vector<NodeSelectorRequirement>& rs) { for (auto& r : rs) pod_side.insert(normalize_key(r.key)); });
    pod_topology_terms(p, [&](int, const std::string& key, auto&&...) { pod_side.insert(key); });
  });
  if (!B.P.empty_topology)
    for (auto& k : B.facts.anti_keys) pod_side.insert(k);  // bound pods with required anti-affinity (ClusterFacts)
  std::set<std::string> active = pod_side;
  for (auto& pr : B.P.provisioners) {
    for (auto& r : pr.requirements) active.insert(normalize_key(r.key));
    for (auto& kv : template_labels(pr)) active.insert(normalize_key(kv.first));
  }
  active.erase(kHostname);
  active.erase(kInstanceType);
  for (auto& k : active)
    if (!pod_side.count(k) && k != kZone && k != kCapacityType) foldable->insert(k);
  return active;
}

// The dictionary of a set of mask keys under construction: values, thresholds and value classes per key.
struct Dictionary {
  std::vector<std::set<std::string>> vals;
  std::vector<std::set<int64_t>> thr;
  std::vector<bool> type_complement;                       // an instance type has a complement requirement on the key
  std::vector<std::map<std::string, std::string>> rep_of;  // unnamed value -> its class's representative
  bool fits(int k) const {  // what the checks of install_dictionary accept: a key that fails them is refused
    const size_t nd = vals[k].size(), m = thr[k].size();
    return nd <= 63 && m <= KSCHED_MAX_THRESHOLDS && !((m > 0 || type_complement[k]) && nd + m + 1 > 63);
  }
};
// Adds to out[k] the values that In / NotIn requirements of rs on mask key k name (NotIn only when complement_only).
void note_values(const Builder& B, const std::vector<NodeSelectorRequirement>& rs, std::vector<std::set<std::string>>& out, bool complement_only = false) {
  for (auto& r : rs) {
    int k = B.key_of(r.key);
    if (k < 0 || (complement_only && r.op == Op::In)) continue;
    if (r.op == Op::In || r.op == Op::NotIn) out[k].insert(r.values.begin(), r.values.end());
  }
}

// Value classes (DESIGN.md §3). A key whose values do not fit the word keeps the values some requirement of the problem
// names, and one representative per class of the others: instance types' In values and node labels that no requirement
// tells apart. Keys that fit are encoded as they always were.
void collapse_value_classes(Builder& B, Dictionary& D) {
  const int NK = (int)B.E.key_names.size();
  std::vector<int> wide;
  for (int k = 0; k < NK; ++k) {
    const size_t nd = D.vals[k].size(), m = D.thr[k].size();
    if (nd > 63 || ((m > 0 || D.type_complement[k]) && nd + m + 1 > 63)) wide.push_back(k);
  }
  if (wide.empty()) return;
  std::vector<std::set<std::string>> named(NK);
  std::vector<bool> all_named(NK, false);
  auto name_key = [&](const std::string& key) { int k = B.key_of(key); if (k >= 0) all_named[k] = true; };
  B.for_class_and_daemon_pods([&](const Pod& p) {  // topology node filters are built from the same node selector and required terms
    pod_requirement_lists(p, [&](const std::vector<NodeSelectorRequirement>& rs) { note_values(B, rs, named); });
    pod_topology_terms(p, [&](int, const std::string& key, auto&&...) { name_key(key); });
  });
  for (auto& kv : B.facts.named_pairs) { int k = B.key_of(kv.first); if (k >= 0) named[k].insert(kv.second); }  // bound pods
  for (auto& key : B.facts.anti_keys) name_key(key);  // inverse anti-affinity groups
  for (auto& pr : B.P.provisioners) {
    note_values(B, pr.requirements, named);
    note_values(B, label_reqs(template_labels(pr)), named);
  }
  for (auto& it : B.P.instance_types) note_values(B, it.requirements, named, true);
  name_key(kZone);  // offering slots: they feed the launch choice
  name_key(kCapacityType);
  for (int k : wide) {
    if (all_named[k]) continue;  // refused in install_dictionary when it does not fit
    D.rep_of[k] = value_classes(D.vals[k], named[k], D.thr[k]);
    for (auto& kv : D.rep_of[k]) {
      if (kv.first != kv.second) D.vals[k].erase(kv.first);
      else B.E.key_representatives[k]++;
    }
  }
}
Dictionary dictionary(Builder& B, const std::set<std::string>& keys) {
  Encoded& E = B.E;
  B.key_id.clear();
  E.key_names.clear();
  for (auto& k : keys) {
    B.key_id[k] = (int)E.key_names.size();
    E.key_names.push_back(k);
  }
  const int NK = (int)E.key_names.size();
  Dictionary D;
  D.vals.assign(NK, {});
  auto note_vals = [&](const std::vector<NodeSelectorRequirement>& rs) { note_values(B, rs, D.vals); };
  B.for_class_and_daemon_pods([&](const Pod& p) { pod_requirement_lists(p, note_vals); });
  for (auto& it : B.P.instance_types) note_vals(it.requirements);
  // offerings name zones / capacity types too (a node without a requirement on the key admits all of them)
  for (auto& it : B.P.instance_types)
    for (auto& o : it.offerings) {
      int kz = B.key_of(kZone), kc = B.key_of(kCapacityType);
      if (kz >= 0) D.vals[kz].insert(o.zone);
      if (kc >= 0) D.vals[kc].insert(o.capacity_type);
    }
  for (auto& pr : B.P.provisioners) {
    note_vals(pr.requirements);
    note_vals(label_reqs(template_labels(pr)));
  }
  for (auto& kv : B.facts.label_pairs) { int k = B.key_of(kv.first); if (k >= 0) D.vals[k].insert(kv.second); }  // every node's labels (ClusterFacts)
  // Every threshold any requirement of this problem names, per key; a key also gets one region when an instance type has a
  // complement requirement on it (region form in install_dictionary).
  D.thr.assign(NK, {});
  D.type_complement.assign(NK, false);
  auto note_thr = [&](const std::vector<NodeSelectorRequirement>& rs, bool is_type) {
    for (auto& r : rs) {
      int k = B.key_of(r.key);
      if (k < 0) continue;
      if (r.op == Op::Gt || r.op == Op::Lt) { int64_t v = 0; if (!r.values.empty()) parse_int(r.values[0], &v); D.thr[k].insert(v); }
      if (is_type && r.op != Op::In && r.op != Op::DoesNotExist) D.type_complement[k] = true;
    }
  };
  B.for_class_and_daemon_pods([&](const Pod& p) { pod_requirement_lists(p, [&](const std::vector<NodeSelectorRequirement>& rs) { note_thr(rs, false); }); });
  for (auto& it : B.P.instance_types) note_thr(it.requirements, true);
  for (auto& pr : B.P.provisioners) note_thr(pr.requirements, false);
  B.phase("  keys + thresholds");
  E.key_representatives.assign(NK, 0);
  D.rep_of.assign(NK, {});
  collapse_value_classes(B, D);
  return D;
}
// Value ids, key infos and the region form of Gt/Lt (ksched.h: ksched_key_regions) of the dictionary.
void install_dictionary(Builder& B, const Dictionary& D) {
  Encoded& E = B.E;
  const int NK = (int)E.key_names.size();
  B.value_id.resize(NK);
  E.key_values.resize(NK);
  E.keys.resize(NK);
  E.key_int_values.assign((size_t)NK * 64, 0);
  B.key_meta.resize(NK);
  for (int k = 0; k < NK; ++k) {
    if (D.vals[k].size() > 63) unsupported("label key " + E.key_names[k] + " has more than 63 distinct values");
    ksched_keyinfo& ki = E.keys[k];
    std::memset(&ki, 0, sizeof ki);
    int b = 0;
    for (auto& v : D.vals[k]) {
      B.value_id[k][v] = b;
      E.key_values[k].push_back(v);
      ki.dict_mask |= 1ull << b;
      int64_t iv;
      if (parse_int(v, &iv)) { ki.int_mask |= 1ull << b; E.key_int_values[(size_t)k * 64 + b] = iv; }
      ++b;
    }
    // every requirement, label and domain table looks an unnamed value up under its representative's id
    for (auto& kv : D.rep_of[k]) B.value_id[k][kv.first] = B.value_id[k].at(kv.second);
    ki.well_known = B.well_known.count(E.key_names[k]) ? 1 : 0;
    ki.is_zone = E.key_names[k] == kZone;
    ki.is_capacity_type = E.key_names[k] == kCapacityType;
  }
  for (int k = 0; k < NK; ++k) B.key_meta[k] = KeyMeta{E.keys[k].int_mask, &E.key_int_values[(size_t)k * 64], nullptr};
  bool any = false;
  for (int k = 0; k < NK; ++k) any = any || !D.thr[k].empty() || D.type_complement[k];
  if (!any) return;
  E.key_regions.assign(NK, ksched_key_regions{});
  for (int k = 0; k < NK; ++k) {
    if (D.thr[k].empty() && !D.type_complement[k]) continue;
    const int m = (int)D.thr[k].size(), nd = (int)E.key_values[k].size();
    if (m > KSCHED_MAX_THRESHOLDS) unsupported("label key " + E.key_names[k] + " has more than 7 distinct Gt/Lt thresholds");
    if (nd + m + 1 > 63) unsupported("label key " + E.key_names[k] + " has too many values for its Gt/Lt regions");
    std::vector<int64_t> ts(D.thr[k].begin(), D.thr[k].end());
    ksched::regions_build(&E.key_regions[k], ts.data(), m, nd, E.keys[k].dict_mask, B.key_meta[k]);
  }
}
void keys_and_dictionary(Builder& B) {
  std::set<std::string> foldable;
  std::set<std::string> active = active_keys(B, &foldable);
  // Folding is conditional, so that every problem that fits the word keeps its encoding byte for byte: the template-only keys
  // are folded only when the problem would be refused otherwise, for more than 16 keys or for a template-only key whose values
  // do not fit (karpenter.sh/provisioner-name with 64 provisioners).
  bool fold = active.size() > KSCHED_MAX_KEYS;
  Dictionary D;
  if (!fold) {
    D = dictionary(B, active);
    for (auto& k : foldable) fold = fold || !D.fits(B.key_id.at(k));
  }
  if (fold) {
    for (auto& k : foldable) active.erase(k);
    if (active.size() > KSCHED_MAX_KEYS) unsupported("more than 16 active label keys");
    B.E.folded_keys.assign(foldable.begin(), foldable.end());
    D = dictionary(B, active);
  }
  B.phase("  value classes");
  install_dictionary(B, D);
}

// ------------------------------------------------------------------ resources
void resources(Builder& B) {
  const Problem& P = B.P;
  Encoded& E = B.E;
  // bound: what a daemonset requests or a provisioner limit names; read: that and what some pod requests; names: every
  // resource name of the problem
  std::set<std::string> bound, read = B.facts.req_names, names = B.facts.res_names;  // ClusterFacts: node allocatable / capacity / bound pods
  for (auto& d : P.daemonset_pods) for (auto& kv : pod_requests(d)) bound.insert(kv.first);
  for (auto& pr : P.provisioners) for (auto& kv : pr.limits) bound.insert(kv.first);
  for (auto& s : B.specs) for (auto& kv : s.req) read.insert(kv.first);
  read.insert(bound.begin(), bound.end());
  names.insert(read.begin(), read.end());
  for (auto& it : P.instance_types) for (auto& kv : it.capacity) names.insert(kv.first);
  E.res_names = resource_order(names);
  if (E.res_names.size() > KSCHED_MAX_RES) {
    // Fits reads the request's keys only (resources.go:138-145), the limits bookkeeping the limit's keys only
    // (scheduler.go:284-303): a name that no pod requests and no limit names cannot change an answer. Left out.
    E.res_names = resource_order(read);
    B.res_pruned = true;
  }
  if (E.res_names.size() > KSCHED_MAX_RES) {
    // Ext resources (DESIGN.md §3): the 8 row slots take cpu, memory, pods and every resource a daemonset requests or a
    // provisioner limit names, then the other read resources by descending number of requesting pods (ties by name).
    // The rest is requested by pod classes only, and only the classes requesting it ever read it.
    std::vector<std::string> order = resource_order(bound);
    if (order.size() > KSCHED_MAX_RES) unsupported("more than 8 resources that a daemonset requests or a provisioner limit names");
    if (E.res_names.size() > KSCHED_MAX_RES + KSCHED_MAX_RES_EXT) unsupported("more than 32 resources that a pod requests or a limit names");
    std::map<std::string, size_t> requesting;
    for (size_t i = 0; i < E.pods.size(); ++i) for (auto& kv : B.specs[E.pod_class[i]].req) ++requesting[kv.first];
    std::vector<std::string> rest;
    for (size_t i = 3; i < E.res_names.size(); ++i) if (!bound.count(E.res_names[i])) rest.push_back(E.res_names[i]);
    std::stable_sort(rest.begin(), rest.end(), [&](const std::string& a, const std::string& b) { return requesting[a] > requesting[b]; });
    order.insert(order.end(), rest.begin(), rest.end());
    E.res_names = order;
    E.n_res_ext = (int)E.res_names.size() - KSCHED_MAX_RES;
  }
  for (size_t i = 0; i < E.res_names.size(); ++i) B.res_id[E.res_names[i]] = (int)i;
}

// ------------------------------------------------------------------ instance types (columns, price order)
void instance_types(Builder& B) {
  const Problem& P = B.P;
  Encoded& E = B.E;
  const int NT = (int)P.instance_types.size();
  const int zone_key = B.key_of(kZone), ct_key = B.key_of(kCapacityType);
  E.type_words = (NT + 63) / 64;
  if (E.type_words == 0) E.type_words = 1;
  std::vector<double> min_price(NT, std::numeric_limits<double>::infinity());
  for (int i = 0; i < NT; ++i)
    for (auto& o : P.instance_types[i].offerings)
      if (o.available && o.price < min_price[i]) min_price[i] = o.price;
  E.type_input_index.resize(NT);
  for (int i = 0; i < NT; ++i) E.type_input_index[i] = i;
  std::stable_sort(E.type_input_index.begin(), E.type_input_index.end(), [&](int a, int b) { return min_price[a] < min_price[b]; });
  E.types.resize(NT);
  E.type_capacity.assign((size_t)NT * KSCHED_MAX_RES, 0);
  E.type_alloc_ext.assign((size_t)NT * E.n_res_ext, 0);
  // launch-choice table: exact price order through ranks of the distinct (double) prices
  std::set<double> prices;
  for (auto& it : P.instance_types)
    for (auto& o : it.offerings) if (o.available) prices.insert(o.price);
  E.price_by_rank.assign(prices.begin(), prices.end());
  E.offering_keys.assign((size_t)NT * 64, ~0ull);
  // Offering slots. An available offering whose zone / capacity type is not a dictionary value can never satisfy a *present*
  // requirement and gets no slot; when a key is inactive every offering counts as its value 0, which is exactly "key not
  // constrained". The pair (ct, z) is slot ct*16 + z while every pair fits that; otherwise the distinct pairs are numbered
  // densely in ascending (ct, z) order, and the slot tables of ksched_catalog say which pairs the slots are.
  auto offering_pair = [&](const Offering& o, int& z, int& ct) {
    z = 0; ct = 0;
    if (zone_key >= 0) { auto f = B.value_id[zone_key].find(o.zone); if (f == B.value_id[zone_key].end()) return false; z = f->second; }
    if (ct_key >= 0) { auto f = B.value_id[ct_key].find(o.capacity_type); if (f == B.value_id[ct_key].end()) return false; ct = f->second; }
    return true;
  };
  std::set<std::pair<int, int>> pairs;  // (ct, z)
  for (auto& it : P.instance_types)
    for (auto& o : it.offerings) {
      int z, ct;
      if (o.available && offering_pair(o, z, ct)) pairs.insert({ct, z});
    }
  const bool formula = std::all_of(pairs.begin(), pairs.end(), [](const std::pair<int, int>& p) { return p.first < 4 && p.second < 16; });
  std::map<std::pair<int, int>, int> slot_of;
  if (formula) {
    for (auto& p : pairs) slot_of[p] = p.first * 16 + p.second;
  } else {
    if (pairs.size() > 64)
      unsupported("more than 64 (capacity type, zone) pairs with an available offering (" + std::to_string(pairs.size()) + " pairs)");
    E.offering_slots = (int)pairs.size();
    E.offering_slot_tables.assign(128, 0);
    for (auto& p : pairs) {
      const int s = (int)slot_of.size();
      slot_of[p] = s;
      E.offering_slot_tables[(size_t)p.second] |= 1ull << s;
      E.offering_slot_tables[64 + (size_t)p.first] |= 1ull << s;
    }
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
    subtract_in_place(alloc, overhead);
    row.res_present = B.fill_resources(alloc, row.allocatable);
    B.fill_resources(it.capacity, &E.type_capacity[(size_t)c * KSCHED_MAX_RES]);
    if (E.n_res_ext) B.fill_ext(alloc, &E.type_alloc_ext[(size_t)c * E.n_res_ext]);
    for (size_t oi = 0; oi < it.offerings.size(); ++oi) {
      const Offering& o = it.offerings[oi];
      int z, ct;
      if (!o.available || !offering_pair(o, z, ct)) continue;
      const int slot = slot_of.at({ct, z});
      row.offerings |= 1ull << slot;
      // (price rank, Offerings list position, slot): the smallest key of a slot wins when several offerings share it
      if (oi > 255) unsupported("instance type " + it.name + " has more than 256 offerings");
      const uint64_t rank = (uint64_t)(std::lower_bound(E.price_by_rank.begin(), E.price_by_rank.end(), o.price) - E.price_by_rank.begin());
      const uint64_t key = (rank << 16) | ((uint64_t)oi << 8) | (uint64_t)slot;
      uint64_t& cell = E.offering_keys[(size_t)c * 64 + slot];
      if (key < cell) cell = key;
    }
    row.min_price = min_price[E.type_input_index[c]];
    row.input_index = (uint32_t)E.type_input_index[c];
  }
}

// The instance types that every one of a list of instance-type requirements admits, as (complement, names).
std::pair<bool, std::set<std::string>> itype_intersection(const std::vector<NodeSelectorRequirement>& rs) {
  bool comp = true;  // (true, {}): every type
  std::set<std::string> names;
  for (auto& r : rs) {
    if (r.op == Op::Gt || r.op == Op::Lt) unsupported("Gt/Lt on instance-type");
    bool rc = !(r.op == Op::In || r.op == Op::DoesNotExist);
    std::set<std::string> rv;
    if (r.op == Op::In || r.op == Op::NotIn) rv.insert(r.values.begin(), r.values.end());
    std::set<std::string> nv;
    if (comp && rc) { nv = names; nv.insert(rv.begin(), rv.end()); }
    else if (comp && !rc) { for (auto& x : rv) if (!names.count(x)) nv.insert(x); }
    else if (!comp && rc) { for (auto& x : names) if (!rv.count(x)) nv.insert(x); }
    else { for (auto& x : names) if (rv.count(x)) nv.insert(x); }
    comp = comp && rc;
    names = nv;
  }
  return {comp, names};
}
// Requirements.Intersects on the instance-type key of two requirements that both name it (requirements.go:189-206): the
// intersection is not empty, or both operators are NotIn / DoesNotExist.
bool itype_intersects(const ItypeSet& a, const ItypeSet& b) {
  bool any = a.first && b.first;
  for (auto& n : a.second) any = any || (a.first ? false : (b.first ? !b.second.count(n) : b.second.count(n) > 0));
  for (auto& n : b.second) any = any || (!b.first && a.first && !a.second.count(n));
  if (any) return true;
  auto negative = [](const ItypeSet& s) { return s.first ? !s.second.empty() : s.second.empty(); };  // NotIn / DoesNotExist
  return negative(a) && negative(b);
}
// Its instance-type columns: bit col % 64 of word col / 64 is set when the type of column col is admitted.
std::vector<uint64_t> itype_columns(const Builder& B, const std::pair<bool, std::set<std::string>>& set) {
  std::vector<uint64_t> words((size_t)B.E.type_words, 0);
  for (int col = 0; col < (int)B.E.types.size(); ++col) {
    bool in = set.second.count(B.P.instance_types[B.E.type_input_index[col]].name) > 0;
    if (set.first ? !in : in) words[col / 64] |= 1ull << (col % 64);
  }
  return words;
}
// The itype_req entry of a requirement, added when it is new. The columns keep only names of the catalog; the first other
// name a requirement keeps is remembered, since a node filter that names the key needs such names told apart
// (itype_filter_tables).
uint32_t itype_entry(Builder& B, const ItypeSet& set) {
  std::string key = std::to_string(set.first) + ":";
  for (auto& n : set.second) {
    key += n + ",";
    if (B.itype_unlisted.empty() && !B.type_col.count(n)) B.itype_unlisted = n;
  }
  auto id = B.itype_req_id.emplace(key, (uint32_t)B.E.itype_req_complement.size());
  if (id.second) {
    B.E.itype_req_complement.push_back(set.first ? 1 : 0);
    const std::vector<uint64_t> words = itype_columns(B, set);
    B.E.itype_req_sets.insert(B.E.itype_req_sets.end(), words.begin(), words.end());
  }
  return id.first->second;
}

// ------------------------------------------------------------------ templates
void templates(Builder& B) {
  const Problem& P = B.P;
  Encoded& E = B.E;
  const int NV = (int)E.template_provisioner.size(), NT = (int)P.instance_types.size();
  E.templates.resize(NV);
  E.template_bounds.resize(NV);
  for (int v = 0; v < NV; ++v) {
    const Provisioner& pr = P.provisioners[E.template_provisioner[v]];
    ksched_template& t = E.templates[v];
    std::memset(&t, 0, sizeof t);
    std::memset(&E.template_bounds[v], 0, sizeof(ksched_bounds));
    Builder::Special sp;
    B.add_selector_reqs(t.reqs, E.template_bounds[v], pr.requirements, &sp);  // NewMachineTemplate machinetemplate.go:46-62
    B.add_selector_reqs(t.reqs, E.template_bounds[v], label_reqs(template_labels(pr)), &sp);
    if (!sp.hostname.empty()) unsupported("provisioner with a hostname requirement");
    // instance-type requirement of the provisioner: fold into membership (types are singletons on that key); without instance
    // types nothing is folded (nor refused)
    const std::vector<uint64_t> allowed = NT ? itype_columns(B, itype_intersection(sp.itype)) : std::vector<uint64_t>((size_t)E.type_words, 0);
    B.template_itype.push_back(sp.itype.empty() ? std::nullopt : std::optional<ItypeSet>(itype_intersection(sp.itype)));
    for (int idx : pr.instance_types) {
      int c = B.type_col.at(P.instance_types.at(idx).name);
      if ((allowed[c / 64] >> (c % 64)) & 1) E.types[c].template_members |= 1ull << v;
    }
    t.taintset = (uint32_t)B.taintset(pr.taints);
    // at most KSCHED_MAX_TEMPLATES templates, encoded before any existing node: the template side reads only the 64-bit word
    if (t.taintset >= 64) throw std::runtime_error("internal: template taint set id beyond 63");
    t.has_limits = pr.has_limits ? 1 : 0;
    t.limit_present = B.fill_resources(pr.limits, t.remaining);
    if (t.reqs.meta >> KSCHED_META_HASGT_SHIFT) E.any_template_bounds = true;
  }
  // Template-only keys (DESIGN.md §3): filterInstanceTypesByRequirements (node.go:137-145) keeps a type only when its
  // requirements intersect the node's, and on such a key the node's requirement is always its template's
  // (NewMachineTemplate: provisioner requirements, then labels, machinetemplate.go:46-62). Types that fail it on some folded
  // key leave the template's list; the requirement itself is kept, rendered, for the new nodes' requirements.
  if (!E.folded_keys.empty()) E.template_folded.assign(NV, {});
  for (auto& key : E.folded_keys) {
    auto on_key = [&](const std::vector<NodeSelectorRequirement>& rs) {
      std::vector<NodeSelectorRequirement> out;
      for (auto& r : rs) if (normalize_key(r.key) == key) out.push_back(r);
      return out;
    };
    std::map<std::string, std::pair<std::vector<NodeSelectorRequirement>, std::vector<int>>> type_groups;  // by requirements on the key
    for (int c = 0; c < NT; ++c) {
      auto rs = on_key(P.instance_types[E.type_input_index[c]].requirements);
      if (rs.empty()) continue;  // Intersects skips a key the type does not define
      auto& g = type_groups[reqs_key(rs)];
      g.first = std::move(rs);
      g.second.push_back(c);
    }
    for (int v = 0; v < NV; ++v) {
      const Provisioner& pr = P.provisioners[E.template_provisioner[v]];
      std::vector<NodeSelectorRequirement> tmpl = on_key(pr.requirements);
      for (auto& r : on_key(label_reqs(template_labels(pr)))) tmpl.push_back(r);
      if (tmpl.empty()) continue;
      const FoldedKey own({&tmpl});
      E.template_folded[v][key] = own.render(own.req(tmpl));
      for (auto& g : type_groups) {
        const FoldedKey d({&tmpl, &g.second.first});
        if (ksched::key_intersects(d.req(g.second.first), d.req(tmpl), d.meta())) continue;
        for (int c : g.second.second) E.types[c].template_members &= ~(1ull << v);
      }
    }
  }
}

// ------------------------------------------------------------------ daemonset overhead (scheduler.go:250-267)
// The daemonset pods a node with these taints and requirements runs (Taints.Tolerates, then Requirements.Compatible with
// the daemon's NewPodRequirements): their requests, and one pod each. `itype` / `hostname` are the node's requirements on
// those keys, nullopt where it defines none. Instance-type is well-known, so a node that does not define it is compatible
// with any instance-type requirement. A template refuses a daemon that tolerates its taints and names a hostname.
ResourceList daemon_overhead(const Builder& B, const std::vector<Taint>& taints, const ksched_reqset& rs, const ksched_bounds& bd,
                             const std::optional<HostnameReq>& itype, const std::optional<HostnameReq>& hostname, bool is_template) {
  ResourceList total;
  int count = 0;
  for (auto& d : B.daemons) {
    if (!tolerates_all(taints, d.pod->tolerations)) continue;
    if (is_template && d.hostname) unsupported("daemonset pod with a hostname requirement");
    if (!B.compatible(rs, bd, d.rs, d.bd)) continue;
    if (!string_compatible(itype, d.itype, true) || !string_compatible(hostname, d.hostname, false)) continue;
    total = merge(total, d.req);
    ++count;
  }
  total["pods"] = (int64_t)count * 1000;
  return total;
}
void daemonset_overhead(Builder& B) {
  for (auto& d : B.P.daemonset_pods) {
    Daemon x{&d, {}, {}, std::nullopt, std::nullopt, pod_requests(d)};
    Builder::Special sp;
    B.pod_requirements(d, x.rs, x.bd, &sp);
    x.hostname = string_requirement(sp.hostname);
    x.itype = string_requirement(sp.itype);
    B.daemons.push_back(x);
  }
  // per template, as getDaemonOverhead does: a template that does not define the instance-type key charges a daemon with an
  // instance-type requirement on every type it offers (DESIGN.md §3, daemonset overhead)
  for (size_t v = 0; v < B.E.templates.size(); ++v) {
    ksched_template& t = B.E.templates[v];
    std::optional<HostnameReq> itype;  // the template's own requirement on the key: provisioner requirements and labels
    if (const auto& own = B.template_itype[v]) itype = HostnameReq{own->first, own->second};
    const ResourceList total = daemon_overhead(B, B.P.provisioners[B.E.template_provisioner[v]].taints, t.reqs, B.E.template_bounds[v],
                                               itype, std::nullopt, true);
    t.daemon_res_present = B.fill_resources(total, t.daemon_requests);
  }
}

// ------------------------------------------------------------------ existing nodes (scheduler.go:221-248, existingnode.go:41-75)
// ------------------------------------------------------------------ host-port entries (hostportusage.go)
// Ids in order of first appearance: the bound pods of the owned state nodes that stay, then the pod classes. With more than
// 64 entries, the ones that can never turn a pod away are left out (no id, no bit). HostPortUsage.validate
// (hostportusage.go:80-93) refuses pod p on a node only for an entry e that a DIFFERENT pod q on that node holds and a port
// of p matches. So e is kept iff some pod of the problem holds it (bound to a node that stays, or a pod of the batch, which
// can be committed) and another pod of the batch has a port matching it. Two pods of one class are different pods; a pod
// whose containers repeat a port is one. Matching is not transitive, so each entry is tested against ports.
// Problems with at most 64 entries keep their ids and encode as before.
void host_port_table(Builder& B) {
  const Problem& P = B.P;
  Encoded& E = B.E;
  std::vector<HostPortEntry> seen;  // every entry, first appearance order
  std::map<HostPortEntry, int> index;
  auto note = [&](const HostPortEntry& e) { if (index.emplace(e, (int)seen.size()).second) seen.push_back(e); };
  std::vector<int> owned;  // state nodes that become existing nodes (existing_nodes)
  for (int si : B.state_nodes) {
    auto own = P.nodes[si].labels.find(kProvisionerName);
    if (own == P.nodes[si].labels.end() || own->second.empty()) continue;
    owned.push_back(si);
    for (auto& hp : B.facts.node[(size_t)si].hostports) note(hp);
  }
  const size_t NC = B.specs.size();
  std::vector<std::vector<HostPortEntry>> ports(NC);
  for (size_t c = 0; c < NC; ++c) {
    ports[c] = host_ports(B.specs[c].pod);
    for (auto& hp : ports[c]) note(hp);
  }
  std::vector<uint8_t> keep(seen.size(), 1);
  if (seen.size() > 64) {
    struct Pods {  // distinct pods seen, counted up to two, and the first one
      int n = 0;
      const Pod* first = nullptr;
      void add(const Pod* p) { if (n == 0) { n = 1; first = p; } else if (n == 1 && p != first) n = 2; }
    };
    std::vector<Pods> holders(seen.size()), matchers(seen.size());
    for (int si : owned)
      for (auto& p : P.nodes[si].pods)
        for (auto& hp : host_ports(p)) holders[(size_t)index.at(hp)].add(&p);
    std::vector<std::vector<int>> matched(NC);  // entries some port of the class matches
    for (size_t c = 0; c < NC; ++c)
      for (size_t u = 0; u < seen.size() && !ports[c].empty(); ++u)
        for (auto& hp : ports[c])
          if (hp_matches(hp, seen[u])) { matched[c].push_back((int)u); break; }
    for (size_t i = 0; i < E.pods.size(); ++i) {
      const uint32_t c = E.pod_class[i];
      for (auto& hp : ports[c]) holders[(size_t)index.at(hp)].add(E.pods[i]);
      for (int u : matched[c]) matchers[(size_t)u].add(E.pods[i]);
    }
    for (size_t u = 0; u < seen.size(); ++u) {
      const Pods &h = holders[u], &m = matchers[u];
      keep[u] = h.n > 0 && m.n > 0 && !(h.n == 1 && m.n == 1 && h.first == m.first);
    }
  }
  for (size_t u = 0; u < seen.size(); ++u) {
    B.hp_id[seen[u]] = keep[u] ? (int)B.hp_entries.size() : -1;
    if (!keep[u]) continue;
    B.hp_entries.push_back(seen[u]);
    E.hostports.push_back(seen[u].ip + " " + std::to_string(seen[u].port) + " " + seen[u].protocol);
  }
  const size_t n = B.hp_entries.size();
  E.hostport_ext_words = n > 64 ? (int)((n - 64 + 63) / 64) : 0;
}

void existing_nodes(Builder& B) {
  const Problem& P = B.P;
  Encoded& E = B.E;
  const int NV = (int)E.templates.size();
  E.remaining_exact.resize((size_t)NV * KSCHED_MAX_RES);
  for (int v = 0; v < NV; ++v)
    for (int r = 0; r < KSCHED_MAX_RES; ++r) E.remaining_exact[(size_t)v * KSCHED_MAX_RES + r] = E.templates[v].remaining[r];
  bool daemon_itype = false, daemon_hostname = false;
  for (auto& d : B.daemons) { daemon_itype = daemon_itype || d.itype; daemon_hostname = daemon_hostname || d.hostname; }
  for (int si : B.state_nodes) {
    const StateNode& n = P.nodes[si];
    auto own = n.labels.find(kProvisionerName);
    if (own == n.labels.end() || own->second.empty()) continue;  // !node.Owned()
    ksched_existing_node e;
    std::memset(&e, 0, sizeof e);
    ksched_bounds nb{};
    Builder::Special sp;
    const NodeFacts& nf = B.facts.node[(size_t)si];
    B.add_selector_reqs(e.reqs, nb, nf.label_reqs, &sp);
    // the daemonsets' requests not yet bound: resources.Subtract over keys of lhs, clamped at 0. The node's labels define its
    // instance type and hostname (In [label], both instance-type label keys when a node carries both); a key no daemon names
    // cannot turn one away, so it is only read when some daemon does.
    ResourceList rem = daemon_overhead(B, n.taints, e.reqs, nb, daemon_itype ? string_requirement(sp.itype) : std::nullopt,
                                       daemon_hostname ? string_requirement(sp.hostname) : std::nullopt, false);  // raw Spec.Taints (scheduler.go:231)
    subtract_in_place(rem, nf.ds_req);
    for (auto& kv : rem) if (kv.second < 0) kv.second = 0;
    ResourceList avail = n.allocatable;
    subtract_in_place(avail, nf.pod_req);
    e.available_present = B.fill_resources(avail, e.available);
    e.requests_present = B.fill_resources(rem, e.requests);
    if (E.n_res_ext) {
      E.existing_available_ext.resize(E.existing_available_ext.size() + E.n_res_ext);
      B.fill_ext(avail, &E.existing_available_ext[E.existing_available_ext.size() - E.n_res_ext]);
    }
    e.taintset = (uint32_t)B.taintset(nf.taints);
    e.itype = KSCHED_NONE;
    auto itl = n.labels.find(kInstanceType);
    if (itl != n.labels.end()) { auto c = B.type_col.find(itl->second); if (c != B.type_col.end()) e.itype = (uint32_t)c->second; }
    if (const int W = E.hostport_ext_words) {
      E.existing_hostport_ext.resize(E.existing_hostport_ext.size() + W, 0);
      for (auto& hp : nf.hostports) B.id_bit(B.hp_entry(hp), e.hostport_entries, &E.existing_hostport_ext[E.existing_hostport_ext.size() - W]);
    } else {
      for (auto& hp : nf.hostports) B.id_bit(B.hp_entry(hp), e.hostport_entries, nullptr);
    }
    std::string hostname;
    auto h = n.labels.find(kHostname);
    if (h != n.labels.end()) hostname = h->second;
    if (hostname.empty()) hostname = n.name;
    B.hostname_slot[hostname] = (int)E.existing.size();
    B.slot_hostname.push_back(hostname);
    E.existing_state_index.push_back(si);
    auto ini = n.labels.find(kInitialized);
    E.existing_initialized.push_back(ini != n.labels.end() && ini->second == "true");
    if (!B.vol_drivers.empty()) {  // state.Node.VolumeUsage() / VolumeLimits() (state/cluster.go:292-303,340-347)
      ksched_node_volumes nv{};
      const int VW = E.volume_ext_words;
      E.existing_volumes_mounted_ext.resize(E.existing_volumes_mounted_ext.size() + VW, 0);
      uint64_t* ext = VW ? &E.existing_volumes_mounted_ext[E.existing_volumes_mounted_ext.size() - VW] : nullptr;
      std::map<std::string, std::set<std::string>> mounted;
      for (auto& p : n.pods) for (auto& kv : B.pod_claims(p)) mounted[kv.first].insert(kv.second.begin(), kv.second.end());
      bool over = false;
      for (size_t d = 0; d < KSCHED_MAX_VOLUME_DRIVERS; ++d) {
        nv.limit[d] = -1;
        if (d >= B.vol_drivers.size()) continue;
        auto l = n.volume_limits.find(B.vol_drivers[d]);
        if (l != n.volume_limits.end()) nv.limit[d] = l->second;
        int total = 0;
        for (auto& c : mounted[B.vol_drivers[d]]) {
          ++total;
          auto t = B.vol_tracked.find({B.vol_drivers[d], c});
          if (t != B.vol_tracked.end()) B.id_bit(t->second, nv.mounted, ext); else nv.used[d]++;
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
          if ((E.templates[v].limit_present >> r) & 1 && (present >> r) & 1) {
            E.templates[v].remaining[r] = remaining_minus(E.templates[v].remaining[r], cap[r]);
            E.remaining_exact[(size_t)v * KSCHED_MAX_RES + r] -= cap[r];
            charged_cap[r] = cap[r];
          }
        charged = v;
      }
    if (B.superset) {
      E.existing_template.push_back(charged);
      E.existing_capacity.insert(E.existing_capacity.end(), charged_cap, charged_cap + KSCHED_MAX_RES);
    }
  }
  if (!B.superset) return;
  std::map<int, int> slot_of_state;
  for (size_t e = 0; e < E.existing_state_index.size(); ++e) slot_of_state[E.existing_state_index[e]] = (int)e;
  for (auto& pn : E.pod_node)
    if (pn <= -2) {
      auto f = slot_of_state.find(-2 - pn);
      if (f == slot_of_state.end()) throw std::runtime_error("a candidate node is not owned by a provisioner");
      pn = f->second;
    }
}

// ------------------------------------------------------------------ topology groups (topology.go)
struct Topology {
  const Builder& B;
  std::vector<Group> groups;
  std::map<std::string, size_t> group_of;          // hash -> index, non-inverse
  std::map<std::string, size_t> inverse_group_of;  // hash -> index, inverse
  // domain universe: provisioner.go:266-276 (requirement.Values() of every type + provisioner In requirements). Only topology
  // keys read it, and their values are never collapsed into classes, so the strings here are the dictionary's own.
  std::map<std::string, std::set<std::string>> universe;
  std::unordered_set<std::string> excluded;  // pods of the batch are not counted as cluster pods (topology.go:66-70)
  explicit Topology(const Builder& b) : B(b) {
    const Problem& P = B.P;
    for (int pi : B.E.template_provisioner) {
      const Provisioner& pr = P.provisioners[pi];
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
          for (int b = 0; b < 64; ++b) if ((r.values >> b) & 1) universe[kv.first].insert(B.E.key_values[k][b]);
      }
    }
    bool any_bound = false;  // only consulted for pods bound to nodes
    for (auto& n : P.nodes) any_bound = any_bound || !n.pods.empty();
    if (any_bound) {
      excluded.reserve(B.E.pods.size() * 2);
      for (auto* p : B.E.pods) excluded.insert(p->uid);
    }
  }
  void make_filter(Group& g, const Pod& p) const {  // MakeTopologyNodeFilter topologynodefilter.go:30-47
    g.filter_nil = false;
    auto canon = [&](const ksched_reqset& rs, const ksched_bounds& bd) {
      std::string s;
      for (int k = 0; k < (int)B.E.key_names.size(); ++k) {
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
      B.add_selector_reqs(rs, bd, label_reqs(p.node_selector), &sp);
      if (term) B.add_selector_reqs(rs, bd, *term, &sp);
      std::optional<HostnameReq> host;
      if (!sp.hostname.empty()) host = hostname_intersection(sp.hostname);
      std::optional<ItypeSet> itype;  // Gt/Lt refused by itype_intersection
      std::string itype_key;
      if (!sp.itype.empty()) {
        itype = itype_intersection(sp.itype);
        itype_key = "itype:" + std::to_string(itype->first) + ":";
        for (auto& n : itype->second) itype_key += n + ",";
      }
      g.filter.push_back({rs, bd});
      g.filter_host.push_back(host);
      g.filter_itype.push_back(itype);
      parts.push_back(canon(rs, bd) + (host ? "hostname:" + host->key() : "") + itype_key);
    };
    if (!p.has_node_affinity || !p.has_required_node_affinity) add_term(nullptr);
    else for (auto& t : p.required_node_terms) add_term(&t);
    std::sort(parts.begin(), parts.end());
    for (auto& s : parts) g.filter_key += "(" + s + ")";
  }
  bool filter_matches_labels(const Group& g, const Labels& labels) const {  // TopologyNodeFilter.Matches
    if (g.filter_nil || g.filter.empty()) return true;
    ksched_reqset rs{}; ksched_bounds bd{};
    Builder::Special sp;
    B.add_selector_reqs(rs, bd, label_reqs(labels), &sp);
    for (size_t t = 0; t < g.filter.size(); ++t) {
      if (!B.compatible(rs, bd, g.filter[t].first, g.filter[t].second)) continue;
      if (const auto& h = g.filter_host[t]) {  // the labels' hostname In [label], or no hostname key at all
        auto l = labels.find(kHostname);
        if (l == labels.end() ? !h->admits_unlabelled() : !h->has(l->second)) continue;
      }
      // the labels' instance type In [label], on strings; a node without the label does not have the key
      if (g.filter_itype[t] && !sp.itype.empty() && !itype_intersects(itype_intersection(sp.itype), *g.filter_itype[t])) continue;
      return true;
    }
    return false;
  }
  Group new_group(int type, const std::string& key, const Pod& p, const std::vector<std::string>& nss, const LabelSelector& sel, int32_t skew) const {
    Group g;
    g.type = type; g.key = key; g.max_skew = skew; g.selector = sel;
    if (nss.empty()) g.namespaces = {p.ns};
    else g.namespaces.insert(nss.begin(), nss.end());
    if (type == 0) make_filter(g, p);
    else g.filter_key = "<nil>";
    auto u = universe.find(key);
    if (u != universe.end()) for (auto& d : u->second) g.counts[d] = 0;
    return g;
  }
  void count_domains(Group& g) const {  // topology.go:231-276
    for (auto& n : B.P.nodes)
      for (auto& p : n.pods) {
        if (!g.namespaces.count(p.ns)) continue;
        if (!g.selector.is_nil && !selector_matches(g.selector, p.labels)) continue;  // TopologyListOptions: nil lists everything
        if (p.terminal || p.terminating) continue;
        if (excluded.count(p.uid)) continue;
        auto it = n.labels.find(g.key);
        if (it == n.labels.end() && g.key != kHostname) continue;  // a node without a hostname label is its own domain
        if (!filter_matches_labels(g, n.labels)) continue;
        g.counts[it != n.labels.end() ? it->second : n.name]++;
      }
  }
  // The group of a topology term, made and counted (countDomains) when it is new; a relaxed variant's new group is dormant.
  size_t add_group(Group g, bool dormant) {
    const std::string h = g.hash();
    auto it = group_of.find(h);
    if (it != group_of.end()) return it->second;
    group_of[h] = groups.size();
    g.dormant = dormant;
    count_domains(g);
    groups.push_back(std::move(g));
    return groups.size() - 1;
  }
  // The inverse anti-affinity group of a required anti-affinity term (updateInverseAntiAffinity topology.go:202-227), made
  // when it is new and `create`; -1 when it does not exist.
  int inverse_group(const Pod& p, const PodAffinityTerm& term, bool create) {
    Group g = new_group(2, term.topology_key, p, term.namespaces, term.selector, INT32_MAX);
    g.inverse = true;
    const std::string h = g.hash();
    auto it = inverse_group_of.find(h);
    if (it != inverse_group_of.end()) return (int)it->second;
    if (!create) return -1;
    inverse_group_of[h] = groups.size();
    groups.push_back(std::move(g));
    return (int)groups.size() - 1;
  }
  void build() {
    for (auto& n : B.P.nodes)  // updateInverseAffinities topology.go:185-198
      for (auto& p : n.pods) {
        if (p.pod_anti_affinity_required.empty() || excluded.count(p.uid)) continue;
        for (auto& term : p.pod_anti_affinity_required) {
          Group& g = groups[(size_t)inverse_group(p, term, true)];
          auto d = n.labels.find(g.key);
          if (d != n.labels.end()) g.counts[d->second]++;
        }
      }
    // Topology.Update of every class of the batch, in Solve's pod order (topology.go:73-75); group creation order only matters
    // for countDomains, which is order-independent. Then of the relaxed variants (Topology.Update after Relax,
    // scheduler.go:119-123): their inverse groups must already exist, and a new group (e.g. the node filter of a spread
    // constraint changes with the required node-affinity terms) is dormant and counts the cluster at that moment, which is the
    // same static state countDomains sees at the start of the solve.
    std::vector<bool> seen(B.specs.size(), false);
    std::vector<uint32_t> order;
    for (uint32_t s : B.E.pod_class) if (!seen[s]) { seen[s] = true; order.push_back(s); }
    const size_t n_batch = order.size();
    for (uint32_t s = 0; s < (uint32_t)B.specs.size(); ++s) if (!seen[s]) order.push_back(s);
    for (size_t i = 0; i < order.size(); ++i) {
      const uint32_t s = order[i];
      const bool relaxed = i >= n_batch;
      const Pod& p = B.specs[s].pod;
      for (auto& term : p.pod_anti_affinity_required) {
        const int gi = inverse_group(p, term, !relaxed);
        if (gi < 0) unsupported("relaxation creates a new inverse topology group");
        groups[(size_t)gi].owner_specs.insert(s);
      }
      pod_topology_terms(p, [&](int type, const std::string& key, const std::vector<std::string>& nss, const LabelSelector& sel, int32_t skew) {
        groups[add_group(new_group(type, key, p, nss, sel, skew), relaxed)].owner_specs.insert(s);
      });
    }
  }
};

// The groups' flat rows, their node filters and their counts per domain / per existing node.
void group_tables(Builder& B, const std::vector<Group>& groups) {
  Encoded& E = B.E;
  const int NG = (int)groups.size(), NE = (int)E.existing.size();
  E.groups.resize(NG);
  E.group_domain_counts.assign((size_t)NG * 64, 0);
  E.group_existing_counts.assign((size_t)NG * std::max(NE, 1), 0);
  for (int g = 0; g < NG; ++g) {
    const Group& G = groups[g];
    ksched_topo_group& o = E.groups[g];
    std::memset(&o, 0, sizeof o);
    o.type = (uint8_t)G.type;
    o.inverse = G.inverse;
    o.dormant = G.dormant;
    o.max_skew = G.max_skew;
    o.filter_begin = (uint32_t)E.filter_terms.size();
    for (size_t t = 0; t < G.filter.size(); ++t) {
      ksched_reqset term = G.filter[t].first;
      B.to_region_form(term, G.filter[t].second);
      E.filter_terms.push_back(term);
      const auto& h = G.filter_host[t];
      E.filter_term_hostname.push_back(h ? B.hostname_table(*h) : KSCHED_NONE);
      if (h) B.filter_names_hostname = true;
      B.filter_itype.push_back(G.filter_itype[t]);  // entries after the classes' (itype_filter_tables)
    }
    o.filter_end = (uint32_t)E.filter_terms.size();
    if (G.key == kHostname) {
      o.key = KSCHED_KEY_HOSTNAME;
      for (auto& kv : G.counts) {
        auto s = B.hostname_slot.find(kv.first);
        if (s != B.hostname_slot.end()) E.group_existing_counts[(size_t)g * std::max(NE, 1) + s->second] = kv.second;
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
}

// What countDomains (topology.go:231-276) and updateInverseAffinities (:183-227) would add for a bound pod of each class,
// split into its class part (namespace, selector, owned inverse groups) and its node part (label value, node filter).
void superset_counts(Builder& B, Topology& T) {
  Encoded& E = B.E;
  const int NG = (int)T.groups.size(), NE = (int)E.existing.size(), NK = (int)E.key_names.size();
  const int NCs = (int)B.specs.size();
  E.class_count_begin.assign((size_t)NCs + 1, 0);
  for (int c = 0; c < NCs; ++c) {
    const Pod& p = B.specs[(size_t)c].pod;
    E.class_count_begin[(size_t)c] = (uint32_t)E.class_count.size();
    std::map<size_t, int> inverse_times;
    for (auto& term : p.pod_anti_affinity_required) {
      const int gi = T.inverse_group(p, term, false);
      if (gi >= 0) inverse_times[(size_t)gi]++;
    }
    for (int g = 0; g < NG; ++g) {
      const Group& G = T.groups[(size_t)g];
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
  // node labels -> verdict per group; without the hostname unless some filter term names it
  std::map<std::string, std::vector<char>> filter_memo;
  for (int e = 0; e < NE; ++e) {
    const StateNode& n = B.P.nodes[(size_t)E.existing_state_index[(size_t)e]];
    for (int k = 0; k < NK; ++k) {
      auto l = n.labels.find(E.key_names[(size_t)k]);
      if (l == n.labels.end()) continue;
      auto v = B.value_id[(size_t)k].find(l->second);
      if (v != B.value_id[(size_t)k].end()) E.node_domain[(size_t)k * NE + e] = (int8_t)v->second;
    }
    E.node_has_hostname_label[(size_t)e] = n.labels.count(kHostname) ? 1 : 0;
    Labels sig = n.labels;
    if (!B.filter_names_hostname) sig.erase(kHostname);
    const std::string key = labels_key(sig);
    auto memo = filter_memo.find(key);
    if (memo == filter_memo.end()) {
      std::vector<char> v((size_t)NG, 1);
      for (int g = 0; g < NG; ++g) v[(size_t)g] = T.filter_matches_labels(T.groups[(size_t)g], n.labels) ? 1 : 0;
      memo = filter_memo.emplace(key, std::move(v)).first;
    }
    for (int g = 0; g < NG; ++g)
      if (memo->second[(size_t)g]) E.group_filter_match[(size_t)g * FW + (e >> 5)] |= 1u << (e & 31);
  }
}
std::vector<Group> topology_groups(Builder& B) {
  Topology T(B);
  if (!B.P.empty_topology) T.build();
  group_tables(B, T.groups);
  if (B.superset && !T.groups.empty()) superset_counts(B, T);
  return std::move(T.groups);
}

// ------------------------------------------------------------------ hostname requirement table
// Row i holds the existing slots hostname_reqs entry i admits: ExistingNode's requirement hostname In [label or name]
// (existingnode.go) is Compatible with the requirement exactly when the requirement Has that hostname. Pair-form entries get
// the row their {complement, slot} means. Without a table entry there is no table, so older problems encode as before.
void hostname_slot_table(Builder& B) {
  Encoded& E = B.E;
  if (!B.filter_names_hostname) E.filter_term_hostname.clear();
  if (B.hostname_table_id.empty()) return;
  const int NE = (int)E.existing.size(), W = std::max(1, (NE + 63) / 64);
  if (B.slot_hostname.size() != (size_t)NE) throw std::runtime_error("internal: hostname of an existing slot missing");
  E.hostname_words = W;
  E.hostname_slots.assign(B.hostname_forms.size() * (size_t)W, 0);
  for (size_t i = 0; i < B.hostname_forms.size(); ++i) {
    uint64_t* row = &E.hostname_slots[i * (size_t)W];
    const auto& f = B.hostname_forms[i];
    const int32_t comp = E.hostname_reqs[2 * i], slot = E.hostname_reqs[2 * i + 1];
    for (int e = 0; e < NE; ++e)
      if (f ? f->has(B.slot_hostname[(size_t)e]) : ((e == slot) != (comp != 0))) row[e / 64] |= 1ull << (e % 64);
  }
}

// ------------------------------------------------------------------ class rows
void class_rows(Builder& B, const std::vector<Group>& groups) {
  Encoded& E = B.E;
  const int NC = (int)B.specs.size(), NG = (int)groups.size();
  E.classes.resize(NC);
  E.class_bounds.resize(NC);
  // (class, group) relations: selector matches of every class against every group, on all cores (pure reads)
  std::vector<uint8_t> rel((size_t)NC * std::max(NG, 1), 0);
  parallel_ranges((size_t)NC, 16, [&](size_t cb, size_t ce) {
    for (size_t c = cb; c < ce; ++c)
      for (int g = 0; g < NG; ++g) {
        const Group& G = groups[g];
        const bool owns = G.owner_specs.count(c) > 0;
        const bool sel = G.selects(B.specs[c].pod);
        uint32_t flags = 0;
        if (sel) flags |= KSCHED_TOPO_SELECTS;
        if (!G.inverse && owns) flags |= KSCHED_TOPO_CONSTRAINS;
        if (G.inverse && sel) flags |= KSCHED_TOPO_CONSTRAINS;  // Counts(): nil node filter always matches
        if (!G.inverse && sel) flags |= KSCHED_TOPO_RECORDS;
        if (G.inverse && owns) flags |= KSCHED_TOPO_RECORDS_INVERSE;
        rel[c * NG + g] = (uint8_t)flags;
      }
  });
  B.phase("  class relations");
  // Sets from id 64 on are existing nodes' only; their bits go to a table of their own, so problems with at most 64 sets encode
  // as before.
  const size_t NS = B.taintsets.size();
  E.n_taintsets = (int)NS;
  E.tolerated_ext_words = NS > 64 ? (int)((NS - 64 + 63) / 64) : 0;
  E.class_tolerated_ext.assign((size_t)NC * E.tolerated_ext_words, 0);
  E.class_requests_ext.assign((size_t)NC * E.n_res_ext, 0);
  E.class_res_ext_present.assign(E.n_res_ext ? NC : 0, 0);
  const int HW = E.hostport_ext_words;
  E.class_hostport_conflicts_ext.assign((size_t)NC * HW, 0);
  E.class_hostport_entries_ext.assign((size_t)NC * HW, 0);
  for (int c = 0; c < NC; ++c) {
    const Spec& s = B.specs[c];
    ksched_pod_row& row = E.classes[c];
    std::memset(&row, 0, sizeof row);
    std::memset(&E.class_bounds[c], 0, sizeof(ksched_bounds));
    row.res_present = B.fill_resources(s.req, row.requests);
    if (E.n_res_ext) E.class_res_ext_present[c] = B.fill_ext(s.req, &E.class_requests_ext[(size_t)c * E.n_res_ext]);
    ksched_reqset rs{};
    Builder::Special sp;
    B.pod_requirements(s.pod, rs, E.class_bounds[c], &sp);
    std::memcpy(row.values, rs.values, sizeof row.values);
    row.meta = rs.meta;
    if (rs.meta >> KSCHED_META_HASGT_SHIFT) E.any_class_bounds = true;
    row.relax_next = s.next;
    row.reserved = (uint64_t)c;  // class index, so a row copied into the FFD-ordered pod matrix knows its class
    row.itype_req = KSCHED_NONE;
    row.hostname_req = KSCHED_NONE;
    if (!sp.itype.empty()) row.itype_req = itype_entry(B, itype_intersection(sp.itype));
    std::optional<HostnameReq> host;
    if (!sp.hostname.empty()) {
      // every hostname requirement of the class at its relaxation level (node selector, required term, heaviest preferred
      // term), intersected as Requirements.Add does; placeholder-named values are refused by HostnameReq::make
      const HostnameReq h = hostname_intersection(sp.hostname);
      host = h;
      auto& r = sp.hostname[0];
      const bool pair = sp.hostname.size() == 1 && (((r.op == Op::In || r.op == Op::NotIn) && r.values.size() == 1) || r.op == Op::Exists);
      if (pair) {  // the {complement, slot} form
        int32_t slot = -1;
        if (!r.values.empty()) { auto f = B.hostname_slot.find(r.values[0]); if (f != B.hostname_slot.end()) slot = f->second; }
        row.hostname_req = B.hostname_pair(r.op == Op::In ? 0 : 1, slot);
      } else {
        row.hostname_req = B.hostname_table(h);
      }
    }
    for (auto& hp : host_ports(s.pod)) {  // the entry table is complete: host_port_table ran before the existing nodes
      B.id_bit(B.hp_entry(hp), row.hostport_entries, HW ? &E.class_hostport_entries_ext[(size_t)c * HW] : nullptr);
      for (size_t e = 0; e < B.hp_entries.size(); ++e)
        if (hp_matches(hp, B.hp_entries[e])) B.id_bit((int)e, row.hostport_conflicts, HW ? &E.class_hostport_conflicts_ext[(size_t)c * HW] : nullptr);
    }
    for (size_t t = 0; t < NS; ++t) {  // the taint-set table is complete: templates and existing nodes are encoded
      if (!tolerates_all(B.taintsets[t], s.pod.tolerations)) continue;
      if (t < 64) row.tolerated_taintsets |= 1ull << t;
      else E.class_tolerated_ext[(size_t)c * E.tolerated_ext_words + (t - 64) / 64] |= 1ull << ((t - 64) % 64);
    }
    // topology relations
    row.topo_begin = (uint32_t)E.class_topo.size();
    for (int g = 0; g < NG; ++g) {
      uint32_t flags = rel[(size_t)c * NG + g];
      const Group& G = groups[g];
      if (host && G.key == kHostname && G.type == 1 && (flags & KSCHED_TOPO_CONSTRAINS))  // nextDomainAffinity's options
        for (auto& kv : G.counts)  // a domain with a count that is no existing slot is never counted on the device
          if (kv.second > 0 && !B.hostname_slot.count(kv.first) && host->has(kv.first)) { flags |= KSCHED_TOPO_HOST_EXTRA; break; }
      if (flags & ~KSCHED_TOPO_SELECTS) E.class_topo.push_back({(uint32_t)g, flags});
    }
    row.topo_end = (uint32_t)E.class_topo.size();
  }
  hostname_slot_table(B);
  if (!B.vol_drivers.empty()) {
    const int VW = E.volume_ext_words;
    E.class_volumes.resize(NC);
    E.class_volumes_shared_ext.assign((size_t)NC * VW, 0);
    E.volume_driver_mask_ext.assign((size_t)KSCHED_MAX_VOLUME_DRIVERS * VW, 0);
    bool any = false;
    for (int c = 0; c < NC; ++c)
      any = !B.volume_signature(B.specs[c].pod, &E.class_volumes[c], VW ? &E.class_volumes_shared_ext[(size_t)c * VW] : nullptr).empty() || any;
    if (!any) E.class_volumes.clear();  // no pod of the batch mounts a limited claim: the kernels never look
    for (auto& kv : B.vol_tracked)
      B.id_bit(kv.second, E.volume_driver_mask[B.driver_index(kv.first.first)],
               VW ? &E.volume_driver_mask_ext[B.driver_index(kv.first.first) * VW] : nullptr);
  }
}

// ------------------------------------------------------------------ instance-type filter tables
// When some topology node filter term names the instance type, Topology.Record and countDomains ask whether the node's
// requirement on the key Intersects the term's. A new node's requirement is its template's (NewMachineTemplate) ∩ its pods',
// an existing node's In [its label] ∩ its pods' (ExistingNode.Add). The device carries them as itype_req entries, which
// keep only names of the catalog: every name outside it is then one that no requirement names, and the entry's complement
// bit stands for all of them at once. An existing node's label outside the catalog is such a name of its own
// (KSCHED_ITYPE_UNLISTED). A requirement that keeps a name outside the catalog would need that name told apart: refused.
// Entries are added after the classes', so problems without such terms encode as before.
void itype_filter_tables(Builder& B) {
  Encoded& E = B.E;
  bool any = false;
  for (auto& f : B.filter_itype) any = any || f.has_value();
  if (!any) return;
  for (auto& f : B.filter_itype) E.filter_term_itype.push_back(f ? itype_entry(B, *f) : KSCHED_NONE);
  for (auto& t : B.template_itype) E.template_itype.push_back(t ? itype_entry(B, *t) : KSCHED_NONE);
  for (size_t e = 0; e < E.existing.size(); ++e) {
    const StateNode& n = B.P.nodes[(size_t)E.existing_state_index[e]];
    Builder::Special sp;
    ksched_reqset rs{}; ksched_bounds bd{};
    B.add_selector_reqs(rs, bd, label_reqs(n.labels), &sp);
    uint32_t v = KSCHED_NONE;
    if (!sp.itype.empty()) {
      const ItypeSet own = itype_intersection(sp.itype);  // In [label] (both label keys when a node carries both)
      bool listed = true;  // at most one name: In [a] ∩ In [b] is DoesNotExist
      for (auto& name : own.second) listed = listed && B.type_col.count(name) > 0;
      v = listed ? itype_entry(B, own) : KSCHED_ITYPE_UNLISTED;
    }
    E.existing_itype.push_back(v);
  }
  if (!B.itype_unlisted.empty())
    unsupported("instance-type requirement naming " + B.itype_unlisted + ", a type outside the catalog, with an instance-type node filter");
}

// ------------------------------------------------------------------ per-pod queue keys (queue.go:74-110)
void queue_keys(Builder& B) {
  Encoded& E = B.E;
  const size_t NP = E.pods.size();
  E.pod_uid_rank.resize(NP);
  if (B.uids_ascending) {
    for (size_t i = 0; i < NP; ++i) E.pod_uid_rank[i] = (uint32_t)i;
    return;
  }
  std::vector<uint32_t> order(NP);
  for (size_t i = 0; i < NP; ++i) order[i] = (uint32_t)i;
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return E.pods[a]->uid < E.pods[b]->uid; });
  for (size_t r = 0; r < NP; ++r) E.pod_uid_rank[order[r]] = (uint32_t)r;
}

// ------------------------------------------------------------------ wire up the flat structs
void wire(Builder& B) {
  Encoded& E = B.E;
  const int NE = (int)E.existing.size(), NC = (int)E.classes.size(), NV = (int)E.templates.size();
  ksched_catalog& cat = E.catalog;
  cat.n_keys = (int)E.key_names.size(); cat.n_res = (int)E.res_names.size() - E.n_res_ext; cat.n_types = (int)E.types.size(); cat.n_templates = NV;
  cat.n_res_ext = E.n_res_ext;
  cat.type_alloc_ext = E.n_res_ext ? E.type_alloc_ext.data() : nullptr;
  cat.keys = E.keys.data();
  cat.key_int_values = E.key_int_values.data();
  cat.types = E.types.data();
  cat.type_capacity = E.type_capacity.data();
  cat.templates = E.templates.data();
  cat.offering_keys = E.offering_keys.data();
  cat.zone_slots = E.offering_slots ? E.offering_slot_tables.data() : nullptr;
  cat.ct_slots = E.offering_slots ? E.offering_slot_tables.data() + 64 : nullptr;
  ksched_problem& pr = E.problem;
  pr.n_pods = (int)E.pods.size(); pr.n_classes = NC; pr.n_existing = NE; pr.n_groups = (int)E.groups.size();
  pr.classes = E.classes.data();
  pr.pod_class = E.pod_class.data();
  pr.pod_timestamp = E.pod_timestamp.data();
  pr.pod_uid_rank = E.pod_uid_rank.data();
  pr.existing = E.existing.data();
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
  if (E.hostname_words) {
    pr.hostname_slots = E.hostname_slots.data();
    pr.n_hostname_words = E.hostname_words;
    pr.filter_term_hostname = E.filter_term_hostname.empty() ? nullptr : E.filter_term_hostname.data();
  }
  if (!E.filter_term_itype.empty()) {
    pr.filter_term_itype = E.filter_term_itype.data();
    pr.template_itype = E.template_itype.data();
    pr.existing_itype = NE > 0 ? E.existing_itype.data() : nullptr;
  }
  pr.max_new_nodes = (int)E.pods.size();
  if (!E.class_volumes.empty() && NE > 0) {
    pr.class_volumes = E.class_volumes.data();
    pr.existing_volumes = E.existing_volumes.data();
    for (int d = 0; d < KSCHED_MAX_VOLUME_DRIVERS; ++d) pr.volume_driver_mask[d] = E.volume_driver_mask[d];
    if (E.volume_ext_words) {
      pr.class_volumes_shared_ext = E.class_volumes_shared_ext.data();
      pr.existing_volumes_mounted_ext = E.existing_volumes_mounted_ext.data();
      pr.volume_driver_mask_ext = E.volume_driver_mask_ext.data();
      pr.n_volume_ext_words = E.volume_ext_words;
    }
  }
  pr.class_tolerated_ext = E.class_tolerated_ext.empty() ? nullptr : E.class_tolerated_ext.data();
  pr.n_tolerated_ext_words = E.tolerated_ext_words;
  if (E.hostport_ext_words) {
    pr.class_hostport_conflicts_ext = E.class_hostport_conflicts_ext.data();
    pr.class_hostport_entries_ext = E.class_hostport_entries_ext.data();
    pr.existing_hostport_ext = NE > 0 ? E.existing_hostport_ext.data() : nullptr;
    pr.n_hostport_ext_words = E.hostport_ext_words;
  }
  if (E.n_res_ext) {
    pr.class_requests_ext = E.class_requests_ext.data();
    pr.class_res_ext_present = E.class_res_ext_present.data();
    pr.existing_available_ext = E.existing_available_ext.data();
  }
  pr.count_nodes_visited = 0;  // the exact nodes_visited statistic is opt-in (kh_set_count_visited / tests): it turns the pack kernel's steady-state paths off
  // Gt/Lt leave the host algebra here: templates and pod classes in region form (types and filter terms already are)
  for (int v = 0; v < NV; ++v) B.to_region_form(E.templates[v].reqs, E.template_bounds[v]);
  for (int c = 0; c < NC; ++c) {
    ksched_reqset rs{};
    std::memcpy(rs.values, E.classes[c].values, sizeof rs.values);
    rs.meta = E.classes[c].meta;
    B.to_region_form(rs, E.class_bounds[c]);
    std::memcpy(E.classes[c].values, rs.values, sizeof rs.values);
    E.classes[c].meta = rs.meta;
  }
  cat.key_regions = E.key_regions.empty() ? nullptr : E.key_regions.data();
}

}  // namespace

std::unique_ptr<Encoded> encode(const Problem& P, const std::vector<int>& candidates, bool cluster_superset) {
  auto enc = std::make_unique<Encoded>();
  enc->problem_ref = &P;
  Builder B(P, *enc, cluster_superset);
  participants(B, candidates);
  B.phase("who takes part");
  csi_volumes(B);
  pod_classes(B);
  B.phase("pod classes");
  keys_and_dictionary(B);
  B.phase("keys + dictionary");
  resources(B);
  B.phase("resources");
  instance_types(B);
  B.phase("instance types");
  templates(B);
  B.phase("templates");
  daemonset_overhead(B);
  B.phase("daemonset overhead");
  host_port_table(B);
  B.phase("host-port entries");
  existing_nodes(B);
  B.phase("existing nodes");
  const std::vector<Group> groups = topology_groups(B);
  B.phase("topology groups");
  class_rows(B, groups);
  B.phase("class rows");
  itype_filter_tables(B);
  queue_keys(B);
  B.phase("queue keys");
  wire(B);
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
  return render_canonical(r.complement, r.values, E.key_values[k], bounds);
}

}  // namespace khost
