// ORACLE — TEST INFRASTRUCTURE ONLY (see requirements.h header).
//
// Single-threaded CPU restatement of the reference's provisioning scheduler:
//   pkg/controllers/provisioning/scheduling/{scheduler,queue,node,existingnode,machinetemplate,
//       preferences,topology,topologygroup,topologynodefilter}.go
//   pkg/scheduling/{taints,hostportusage}.go, pkg/utils/resources/resources.go,
//   pkg/cloudprovider/types.go:87-145, pkg/controllers/state/node.go:61-143,
//   pkg/controllers/provisioning/provisioner.go:237-296 (NewScheduler input marshalling),
//   pkg/controllers/deprovisioning/{helpers.go:42-157,292-315, consolidation.go:190-287,
//       multinodeconsolidation.go:74-165}.
// Third-party semantics restated from k8s.io/api v0.25.4 (Toleration.ToleratesTaint,
// Toleration.MatchToleration) and k8s.io/apimachinery v0.25.4 (label selector matching,
// resource.Quantity as exact int64 milli-units).
//
// PARITY PINNING: the Go reference cannot be built here (no Go toolchain), so this oracle is
// pinned by the reference's own golden vectors (tests/golden/*.json, extracted from
// pkg/scheduling/requirement_test.go and requirements_test.go by tests/golden/extract_golden.py)
// and by the known-answer scheduling tests restated in tests/test_oracle_known_answers.py.
// Pod->node INDEX parity is "unpinned" by the reference (its tests shuffle inputs and assert
// order-free invariants only); the canonical rules below define it:
//   R1 sort.Slice(newNodes, len(Pods)<) (scheduler.go:183, pdqsort, unstable) -> STABLE sort of the
//      persistent slice (identical to Go for <=12 nodes, where pdqsort is insertion sort).
//   R2 existing nodes are visited in caller-given order (Go: map order).
//   R3 every `for x := range map` over domains/groups -> ascending string order.
//   R4 OrderByWeight / preferred-term sorts (sort.Slice) -> stable sorts.
//   R5 NewQueue sort is total because pods must carry unique UIDs.
//   R6 hostname placeholders use a per-Solve counter (Go: process-global), same %04d format.
#include "oracle.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <functional>
#include <memory>
#include <stdexcept>

namespace oracle {
using namespace kmodel;

// FAST MODE (oracle_set_fast / ORACLE_FAST=1) — still test infrastructure. The literal restatement below is O(nodes x
// instance types x string-set work) per Add and needs ~20 h for BASELINE C4 at full size. Fast mode adds RESULT-NEUTRAL
// shortcuts only (each one derives the same verdict / the same committed state as the literal code next to it; they are
// marked "fast:" and tests/test_oracle_fast_mode.py asserts digest equality with the literal path on every known answer,
// the fuzz corpus and C3/C4/C5 samples):
//   F1 a node whose merged requests exceed the per-resource maximum allocatable of its remaining options is rejected
//      before the requirement / topology stages (node_add has no side effects before its commit, so only `false` matters);
//   F2 filter_types evaluates Fits first and memoises the requirement part (Intersects && hasOffering) per distinct
//      requirement set (restricted to the keys instance types define);
//   F3 hostname-keyed spread / anti-affinity groups look up the node's concrete hostname set instead of walking every
//      registered hostname (same visiting order, same result); the "any empty domain" emptiness test uses a maintained
//      zero-count counter;
//   F4 getMatchingTopologies / Record memoise, per pod, which groups own / select it (pure in the pod and the group set;
//      flushed by every Topology.Update);
//   F5 per-pod requests_for_pod / new_pod_requirements are cached until the pod is relaxed.
// cpu_baseline and every small-size parity test use the LITERAL path; fast mode exists for the full-size golden digests.
bool g_fast = false;
void set_fast(bool on) { g_fast = on; }

// ---------------------------------------------------------------- resources (utils/resources/resources.go)
// Sums and differences are checked against kQuantityBound (model.h): out of range is refused, like the product does.
static ResourceList merge(const ResourceList& a, const ResourceList& b) {  // :47-60
  ResourceList r = a;
  for (auto& kv : b) r[kv.first] = checked_quantity((__int128)r[kv.first] + kv.second, kv.first);
  return r;
}
static ResourceList subtract(const ResourceList& lhs, const ResourceList& rhs) {  // :62-75
  ResourceList r = lhs;
  for (auto& kv : lhs) {
    auto it = rhs.find(kv.first);
    if (it != rhs.end()) r[kv.first] = checked_quantity((__int128)kv.second - it->second, kv.first);
  }
  return r;
}
// A node's requests plus one pod's, unchecked: requests are >= 0 (the loader refuses others) and a node's requests never
// pass an allocatable inside kQuantityBound, so the sum is below 2^63 and exact; Fits then answers as the reference does.
static ResourceList add_requests(const ResourceList& a, const ResourceList& b) {
  ResourceList r = a;
  for (auto& kv : b) r[kv.first] += kv.second;
  return r;
}
static ResourceList max_resources(const ResourceList& a, const ResourceList& b) {  // :92-102
  ResourceList r = a;
  for (auto& kv : b) {
    auto it = r.find(kv.first);
    if (it == r.end() || kv.second > it->second) r[kv.first] = kv.second;
  }
  return r;
}
static ResourceList limits_into_requests(const Container& c) {  // :105-118
  ResourceList r = c.requests;
  for (auto& kv : c.limits)
    if (!r.count(kv.first)) r[kv.first] = kv.second;
  return r;
}
static ResourceList ceiling_requests(const Pod& p) {  // :78-89
  ResourceList r;
  for (auto& c : p.containers) r = merge(r, limits_into_requests(c));
  for (auto& c : p.init_containers) r = max_resources(r, limits_into_requests(c));
  return r;
}
ResourceList requests_for_pods(const std::vector<const Pod*>& pods) {  // :25-33
  ResourceList r;
  for (auto* p : pods) r = merge(r, ceiling_requests(*p));
  r["pods"] = (int64_t)pods.size() * 1000;
  return r;
}
static ResourceList requests_for_pod(const Pod& p) { return requests_for_pods({&p}); }
static bool fits(const ResourceList& candidate, const ResourceList& total) {  // :138-145
  for (auto& kv : candidate) {
    auto it = total.find(kv.first);
    int64_t t = it == total.end() ? 0 : it->second;
    if (kv.second > t) return false;
  }
  return true;
}
static int64_t getq(const ResourceList& r, const std::string& k) {
  auto it = r.find(k);
  return it == r.end() ? 0 : it->second;
}

// ---------------------------------------------------------------- taints (pkg/scheduling/taints.go:28-40)
static bool tolerates_taint(const Toleration& t, const Taint& taint) {  // k8s.io/api core/v1 Toleration.ToleratesTaint
  if (!t.effect.empty() && t.effect != taint.effect) return false;
  if (!t.key.empty() && t.key != taint.key) return false;
  if (t.op.empty() || t.op == "Equal") return t.value == taint.value;
  if (t.op == "Exists") return true;
  return false;
}
static bool tolerates(const std::vector<Taint>& taints, const Pod& pod) {
  for (auto& taint : taints) {
    bool ok = false;
    for (auto& t : pod.tolerations) ok = ok || tolerates_taint(t, taint);
    if (!ok) return false;
  }
  return true;
}

// ---------------------------------------------------------------- host ports (pkg/scheduling/hostportusage.go)
struct HostPortEntry {
  std::string ip;  // canonical text; "0.0.0.0"/"::" are unspecified
  int32_t port;
  std::string protocol;
};
static bool ip_unspecified(const std::string& ip) { return ip == "0.0.0.0" || ip == "::"; }
static bool hp_matches(const HostPortEntry& a, const HostPortEntry& b) {  // :45-57
  if (a.protocol != b.protocol) return false;
  if (a.port != b.port) return false;
  if (a.ip != b.ip && !ip_unspecified(a.ip) && !ip_unspecified(b.ip)) return false;
  return true;
}
static std::vector<HostPortEntry> get_host_ports(const Pod& p) {  // :118-144
  std::vector<HostPortEntry> out;
  for (auto& c : p.containers)
    for (auto& hp : c.ports) {
      if (hp.port == 0) continue;
      out.push_back({hp.ip.empty() ? "0.0.0.0" : hp.ip, hp.port, hp.protocol});
    }
  return out;
}
struct HostPortUsage {
  std::map<std::string, std::vector<HostPortEntry>> reserved;  // ns/name -> entries
  static std::string key(const Pod& p) { return p.ns + "/" + p.name; }
  bool validate(const Pod& p) const {  // :81-94
    auto nu = get_host_ports(p);
    for (auto& ne : nu)
      for (auto& kv : reserved)
        for (auto& ex : kv.second)
          if (hp_matches(ne, ex) && kv.first != key(p)) return false;
    return true;
  }
  void add(const Pod& p) { reserved[key(p)] = get_host_ports(p); }  // :65-71
};

// ---------------------------------------------------------------- label selectors (apimachinery labels)
// metav1.LabelSelectorAsSelector + Selector.Matches. nil selector -> Nothing for `selects`
// (topologygroup.go:246-252); invalid selector -> Nothing as well.
static bool selector_valid(const LabelSelector& s) {
  for (auto& e : s.match_expressions) {
    if ((e.op == Op::In || e.op == Op::NotIn) && e.values.empty()) return false;
    if ((e.op == Op::Exists || e.op == Op::DoesNotExist) && !e.values.empty()) return false;
    if (e.op == Op::Gt || e.op == Op::Lt) return false;
  }
  return true;
}
static bool selector_matches_nonnil(const LabelSelector& s, const Labels& labels) {
  if (!selector_valid(s)) return false;
  for (auto& kv : s.match_labels) {
    auto it = labels.find(kv.first);
    if (it == labels.end() || it->second != kv.second) return false;
  }
  for (auto& e : s.match_expressions) {
    auto it = labels.find(e.key);
    bool has = it != labels.end();
    bool in = has && std::find(e.values.begin(), e.values.end(), it->second) != e.values.end();
    switch (e.op) {
      case Op::In: if (!in) return false; break;
      case Op::NotIn: if (has && in) return false; break;
      case Op::Exists: if (!has) return false; break;
      case Op::DoesNotExist: if (has) return false; break;
      default: return false;
    }
  }
  return true;
}
static std::string selector_canonical(const LabelSelector& s) {
  if (s.is_nil) return "<nil>";
  std::string out = "{";
  for (auto& kv : s.match_labels) out += kv.first + "=" + kv.second + ",";
  out += "|";
  // SlicesAsSets in the reference's hash: order-insensitive
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

// ---------------------------------------------------------------- pod requirements (requirements.go:61-78)
static Requirements new_pod_requirements(Pod& pod) {
  Requirements r = Requirements::FromLabels(pod.node_selector);
  if (!pod.has_node_affinity) return r;
  if (!pod.preferred_node_terms.empty()) {
    // sort.Slice by weight desc, in place on the pod (R4: stable)
    std::stable_sort(pod.preferred_node_terms.begin(), pod.preferred_node_terms.end(),
                     [](const PreferredSchedulingTerm& a, const PreferredSchedulingTerm& b) { return a.weight > b.weight; });
    r.AddAll(Requirements::FromNodeSelector(pod.preferred_node_terms[0].preference));
  }
  if (pod.has_required_node_affinity && !pod.required_node_terms.empty())
    r.AddAll(Requirements::FromNodeSelector(pod.required_node_terms[0]));
  return r;
}

// ---------------------------------------------------------------- topology node filter (topologynodefilter.go)
struct TopologyNodeFilter {
  std::vector<Requirements> terms;
  bool is_nil = true;  // nil filter (affinity / anti-affinity groups) always matches
  static TopologyNodeFilter Make(const Pod& p) {  // :30-47
    TopologyNodeFilter f;
    f.is_nil = false;
    Requirements sel = Requirements::FromLabels(p.node_selector);
    if (!p.has_node_affinity || !p.has_required_node_affinity) {
      f.terms.push_back(sel);
      return f;
    }
    for (auto& term : p.required_node_terms) {
      Requirements r;
      r.AddAll(sel);
      r.AddAll(Requirements::FromNodeSelector(term));
      f.terms.push_back(r);
    }
    return f;
  }
  bool MatchesRequirements(const Requirements& req, const std::set<std::string>& wk) const {  // :57-70
    if (terms.empty()) return true;
    for (auto& t : terms)
      if (req.Compatible(t, wk)) return true;
    return false;
  }
  std::string canonical() const {
    if (is_nil) return "<nil>";
    std::vector<std::string> parts;
    for (auto& t : terms) {
      std::string s;
      for (auto& kv : t.m) s += kv.first + " " + kv.second.Canonical() + ";";
      parts.push_back(s);
    }
    std::sort(parts.begin(), parts.end());
    std::string out;
    for (auto& p : parts) out += "(" + p + ")";
    return out;
  }
};

// ---------------------------------------------------------------- topology group (topologygroup.go)
enum class TopologyType { Spread = 0, PodAffinity = 1, PodAntiAffinity = 2 };

struct TopologyGroup {
  std::string key;
  TopologyType type;
  int32_t max_skew;
  std::set<std::string> namespaces;
  LabelSelector selector;
  TopologyNodeFilter node_filter;
  std::set<std::string> owners;
  std::map<std::string, int32_t> domains;

  std::string hash() const {  // :137-153 (any injective key works)
    std::string h = key + "|" + std::to_string((int)type) + "|" + std::to_string(max_skew) + "|";
    for (auto& n : namespaces) h += n + ",";
    h += "|" + selector_canonical(selector) + "|" + node_filter.canonical();
    return h;
  }
  bool selects(const Pod& p) const {  // :246-252
    if (selector.is_nil) return false;
    return namespaces.count(p.ns) && selector_matches_nonnil(selector, p.labels);
  }
  bool Counts(const Pod& p, const Requirements& req, const std::set<std::string>& wk) const {  // :109-111
    return selects(p) && node_filter.MatchesRequirements(req, wk);
  }
  int64_t zero_domains = 0;  // fast: number of registered domains whose count is 0 (maintained by Record / Register)
  void Record(const std::string& d) {                                                   // :101-105
    auto it = domains.find(d);
    if (it == domains.end()) { domains[d] = 1; return; }
    if (it->second == 0) --zero_domains;
    it->second++;
  }
  void Register(const std::string& d) { if (!domains.count(d)) { domains[d] = 0; ++zero_domains; } }  // :114-120

  int32_t domainMinCount(const Requirement& pod_domains) const {  // :184-200
    if (key == kHostname) return 0;
    int32_t mn = INT32_MAX;
    for (auto& kv : domains)
      if (pod_domains.Has(kv.first) && kv.second < mn) mn = kv.second;
    return mn;
  }
  Requirement nextDomainTopologySpread(const Pod& pod, const Requirement& pod_domains, const Requirement& node_domains) const {  // :155-182
    int32_t mn = domainMinCount(pod_domains);
    bool self = selects(pod);
    std::string min_domain;
    bool found = false;
    int32_t min_count = INT32_MAX;
    for (auto& kv : domains) {  // R3: ascending domain order
      if (!node_domains.Has(kv.first)) continue;
      int64_t count = kv.second;
      if (self) count++;
      if (count - (int64_t)mn <= max_skew && count < min_count) {
        min_domain = kv.first;
        min_count = (int32_t)count;
        found = true;
      }
    }
    if (!found || min_domain.empty()) return Requirement::New(pod_domains.key, Op::DoesNotExist);
    return Requirement::New(pod_domains.key, Op::In, {min_domain});
  }
  Requirement nextDomainAffinity(const Pod& pod, const Requirement& pod_domains, const Requirement& node_domains) const {  // :202-233
    Requirement options = Requirement::New(pod_domains.key, Op::DoesNotExist);
    for (auto& kv : domains)
      if (pod_domains.Has(kv.first) && kv.second > 0) options.values.insert(kv.first);
    if (options.Len() == 0 && selects(pod)) {
      Requirement inter = pod_domains.Intersection(node_domains);
      for (auto& kv : domains)
        if (inter.Has(kv.first)) { options.values.insert(kv.first); break; }
      for (auto& kv : domains)
        if (pod_domains.Has(kv.first)) { options.values.insert(kv.first); break; }
    }
    return options;
  }
  Requirement nextDomainAntiAffinity(const Requirement& pod_domains) const {  // :235-243
    Requirement options = Requirement::New(pod_domains.key, Op::DoesNotExist);
    for (auto& kv : domains)
      if (pod_domains.Has(kv.first) && kv.second == 0) options.values.insert(kv.first);
    return options;
  }
  // fast (F3): hostname groups hold one domain per node ever attempted. When the node's own requirement for the key is a
  // concrete set (always: hostname In [own name]) the literal loops below only ever admit members of that set, so they are
  // walked in the same ascending order instead of all domains. Anti-affinity: the literal result is {d : count==0 and the pod
  // allows d}; its emptiness (the `Len()==0` reject in AddRequirements) is decided by zero_domains when the pod allows
  // everything, and the caller only intersects the result with the node's set, so returning the members of the node's set
  // that qualify leaves the merged requirement identical.
  bool fast_applicable(const Requirement& pd, const Requirement& nd) const {
    return key == kHostname && !nd.complement && pd.complement && pd.values.empty() && !pd.greater_than && !pd.less_than &&
           (type == TopologyType::Spread || type == TopologyType::PodAntiAffinity);
  }
  Requirement GetFast(const Pod& pod, const Requirement& pd, const Requirement& nd) const {
    if (type == TopologyType::Spread) {
      bool self = selects(pod);
      std::string min_domain;
      bool found = false;
      int32_t min_count = INT32_MAX;
      for (auto& v : nd.values) {  // ascending, like the literal walk restricted to node_domains.Has
        auto it = domains.find(v);
        if (it == domains.end() || !nd.Has(v)) continue;
        int64_t count = it->second;
        if (self) count++;
        if (count - 0 <= max_skew && count < min_count) { min_domain = v; min_count = (int32_t)count; found = true; }
      }
      if (!found || min_domain.empty()) return Requirement::New(pd.key, Op::DoesNotExist);
      return Requirement::New(pd.key, Op::In, {min_domain});
    }
    Requirement options = Requirement::New(pd.key, Op::DoesNotExist);
    if (zero_domains == 0) return options;  // literal: no domain with count 0 -> Len()==0
    bool any_in_node = false;
    for (auto& v : nd.values) {
      auto it = domains.find(v);
      if (it != domains.end() && it->second == 0) { options.values.insert(v); any_in_node = true; }
    }
    if (!any_in_node) {
      // literal result is non-empty but disjoint from the node's set: keep ONE witness domain outside the node's set so
      // that Len()!=0 here and the later intersection / Compatible behave exactly as with the full set
      for (auto& kv : domains)
        if (kv.second == 0 && !nd.values.count(kv.first)) { options.values.insert(kv.first); break; }
    }
    return options;
  }
  Requirement Get(const Pod& pod, const Requirement& pd, const Requirement& nd) const {  // :88-99
    if (g_fast && fast_applicable(pd, nd)) return GetFast(pod, pd, nd);
    switch (type) {
      case TopologyType::Spread: return nextDomainTopologySpread(pod, pd, nd);
      case TopologyType::PodAffinity: return nextDomainAffinity(pod, pd, nd);
      default: return nextDomainAntiAffinity(pd);
    }
  }
};

// ---------------------------------------------------------------- topology (topology.go)
struct ClusterView {
  // every bound pod with the labels of the node it is bound to (kubeClient List/Get in the reference)
  struct Bound { const Pod* pod; const StateNode* node; };
  std::vector<Bound> bound;
};

struct Topology {
  bool inert = false;  // &scheduling.Topology{} as used by the reference benchmark
  std::map<std::string, TopologyGroup> topologies, inverse;
  std::map<std::string, std::set<std::string>> domains;
  std::set<std::string> excluded;
  const ClusterView* cluster = nullptr;
  const std::set<std::string>* wk = nullptr;

  static std::set<std::string> namespace_list(const std::string& ns, const std::vector<std::string>& nss) {  // :326-347 (no namespaceSelector)
    if (nss.empty()) return {ns};
    return std::set<std::string>(nss.begin(), nss.end());
  }
  TopologyGroup make_group(TopologyType t, const std::string& key, const Pod& pod, std::set<std::string> nss,
                           const LabelSelector& sel, int32_t max_skew) {  // topologygroup.go:66-86
    TopologyGroup g;
    g.type = t; g.key = key; g.namespaces = std::move(nss); g.selector = sel; g.max_skew = max_skew;
    auto it = domains.find(key);
    if (it != domains.end()) for (auto& d : it->second) g.Register(d);
    if (t == TopologyType::Spread) g.node_filter = TopologyNodeFilter::Make(pod);
    return g;
  }
  void countDomains(TopologyGroup& tg) {  // :231-276
    for (auto& b : cluster->bound) {
      const Pod& p = *b.pod;
      if (!tg.namespaces.count(p.ns)) continue;
      // TopologyListOptions: nil selector lists everything (:366-370); invalid -> nothing
      if (!tg.selector.is_nil && !selector_matches_nonnil(tg.selector, p.labels)) continue;
      if (p.node_name.empty() || p.terminal || p.terminating) continue;  // IgnoredForTopology :404-406
      if (excluded.count(p.uid)) continue;
      std::string domain;
      auto it = b.node->labels.find(tg.key);
      bool ok = it != b.node->labels.end();
      if (ok) domain = it->second;
      if (!ok && tg.key == kHostname) { domain = b.node->name; ok = true; }
      if (!ok) continue;
      if (!tg.node_filter.MatchesRequirements(Requirements::FromLabels(b.node->labels), *wk)) continue;
      tg.Record(domain);
    }
  }
  void updateInverseAntiAffinity(const Pod& pod, const Labels* node_labels) {  // :202-227
    for (auto& term : pod.pod_anti_affinity_required) {
      TopologyGroup tg = make_group(TopologyType::PodAntiAffinity, term.topology_key, pod,
                                    namespace_list(pod.ns, term.namespaces), term.selector, INT32_MAX);
      std::string h = tg.hash();
      auto it = inverse.find(h);
      if (it == inverse.end()) it = inverse.emplace(h, std::move(tg)).first;
      if (node_labels) {
        auto d = node_labels->find(it->second.key);
        if (d != node_labels->end()) it->second.Record(d->second);
      }
      it->second.owners.insert(pod.uid);
    }
  }
  // fast (F4): per pod uid, the groups that own it / the inverse groups and groups whose selector matches it. Pure in
  // (pod, set of groups); every Update (the only place groups or owners change after NewTopology) flushes the memo.
  struct PodMemo { std::vector<TopologyGroup*> owned, inverse_selecting, selecting, inverse_owned; };
  std::map<std::string, PodMemo> memo;
  const PodMemo& memo_for(const Pod& p) {
    auto it = memo.find(p.uid);
    if (it != memo.end()) return it->second;
    PodMemo m;
    for (auto& kv : topologies) {
      if (kv.second.owners.count(p.uid)) m.owned.push_back(&kv.second);
      if (kv.second.selects(p)) m.selecting.push_back(&kv.second);
    }
    for (auto& kv : inverse) {
      if (kv.second.selects(p)) m.inverse_selecting.push_back(&kv.second);
      if (kv.second.owners.count(p.uid)) m.inverse_owned.push_back(&kv.second);
    }
    return memo.emplace(p.uid, std::move(m)).first->second;
  }
  void Update(const Pod& p) {  // :86-117
    memo.clear();
    for (auto& kv : topologies) kv.second.owners.erase(p.uid);
    bool has_anti = !p.pod_anti_affinity_required.empty() || !p.pod_anti_affinity_preferred.empty();
    if (has_anti) updateInverseAntiAffinity(p, nullptr);
    std::vector<TopologyGroup> groups;
    for (auto& cs : p.topology_spread)  // newForTopologies :278-284
      groups.push_back(make_group(TopologyType::Spread, cs.topology_key, p, {p.ns}, cs.selector, cs.max_skew));
    // newForAffinities :287-322 (required then preferred; affinity then anti-affinity — Go ranges a map, order-free)
    for (auto& t : p.pod_affinity_required)
      groups.push_back(make_group(TopologyType::PodAffinity, t.topology_key, p, namespace_list(p.ns, t.namespaces), t.selector, INT32_MAX));
    for (auto& t : p.pod_affinity_preferred)
      groups.push_back(make_group(TopologyType::PodAffinity, t.term.topology_key, p, namespace_list(p.ns, t.term.namespaces), t.term.selector, INT32_MAX));
    for (auto& t : p.pod_anti_affinity_required)
      groups.push_back(make_group(TopologyType::PodAntiAffinity, t.topology_key, p, namespace_list(p.ns, t.namespaces), t.selector, INT32_MAX));
    for (auto& t : p.pod_anti_affinity_preferred)
      groups.push_back(make_group(TopologyType::PodAntiAffinity, t.term.topology_key, p, namespace_list(p.ns, t.term.namespaces), t.term.selector, INT32_MAX));
    for (auto& tg : groups) {
      std::string h = tg.hash();
      auto it = topologies.find(h);
      if (it == topologies.end()) {
        countDomains(tg);
        it = topologies.emplace(h, std::move(tg)).first;
      }
      it->second.owners.insert(p.uid);
    }
  }
  void Register(const std::string& key, const std::string& domain) {  // :170-181
    if (inert) return;
    for (auto& kv : topologies) if (kv.second.key == key) kv.second.Register(domain);
    for (auto& kv : inverse) if (kv.second.key == key) kv.second.Register(domain);
  }
  void Record(const Pod& p, const Requirements& req) {  // :120-143
    if (inert) return;
    if (g_fast) {  // same two loops over the memoised subsets, in the same (ascending hash) order
      const PodMemo& m = memo_for(p);
      for (auto* tc : m.selecting) {
        if (!tc->node_filter.MatchesRequirements(req, *wk)) continue;
        Requirement d = req.Get(tc->key);
        if (tc->type == TopologyType::PodAntiAffinity) {
          for (auto& v : d.values) tc->Record(v);
        } else if (d.Len() == 1) {
          tc->Record(*d.values.begin());
        }
      }
      for (auto* tc : m.inverse_owned) {
        Requirement d = req.Get(tc->key);
        for (auto& v : d.values) tc->Record(v);
      }
      return;
    }
    for (auto& kv : topologies) {
      TopologyGroup& tc = kv.second;
      if (!tc.Counts(p, req, *wk)) continue;
      Requirement d = req.Get(tc.key);
      if (tc.type == TopologyType::PodAntiAffinity) {
        for (auto& v : d.values) tc.Record(v);
      } else if (d.Len() == 1) {
        tc.Record(*d.values.begin());
      }
    }
    for (auto& kv : inverse) {
      TopologyGroup& tc = kv.second;
      if (tc.owners.count(p.uid)) {
        Requirement d = req.Get(tc.key);
        for (auto& v : d.values) tc.Record(v);
      }
    }
  }
  // :149-167; returns false on "unsatisfiable topology constraint"
  bool AddRequirements(const Requirements& pod_req, const Requirements& node_req, const Pod& p, Requirements* out) {
    Requirements req;
    req.AddAll(node_req);
    if (!inert) {
      std::vector<const TopologyGroup*> matching;  // getMatchingTopologies :351-364
      if (g_fast) {
        const PodMemo& m = memo_for(p);
        for (auto* tg : m.owned) matching.push_back(tg);
        for (auto* tg : m.inverse_selecting) if (tg->node_filter.MatchesRequirements(node_req, *wk)) matching.push_back(tg);
      } else {
        for (auto& kv : topologies) if (kv.second.owners.count(p.uid)) matching.push_back(&kv.second);
        for (auto& kv : inverse) if (kv.second.Counts(p, node_req, *wk)) matching.push_back(&kv.second);
      }
      for (auto* tg : matching) {
        Requirement pd = pod_req.Has(tg->key) ? pod_req.Get(tg->key) : Requirement::New(tg->key, Op::Exists);
        Requirement nd = node_req.Has(tg->key) ? node_req.Get(tg->key) : Requirement::New(tg->key, Op::Exists);
        Requirement d = tg->Get(p, pd, nd);
        if (d.Len() == 0) return false;
        req.Add(d);
      }
    }
    *out = std::move(req);
    return true;
  }
};

// ---------------------------------------------------------------- preferences (preferences.go)
struct Preferences {
  bool tolerate_prefer_no_schedule = false;
  static bool removeRequiredNodeAffinityTerm(Pod& p) {  // :73-87
    if (!p.has_node_affinity || !p.has_required_node_affinity || p.required_node_terms.empty()) return false;
    if (p.required_node_terms.size() > 1) {
      p.required_node_terms.erase(p.required_node_terms.begin());
      return true;
    }
    return false;
  }
  template <class T>
  static bool remove_heaviest(std::vector<T>& terms) {
    if (terms.empty()) return false;
    std::stable_sort(terms.begin(), terms.end(), [](const T& a, const T& b) { return a.weight > b.weight; });
    terms.erase(terms.begin());
    return true;
  }
  static bool removePreferredPodAffinityTerm(Pod& p) { return remove_heaviest(p.pod_affinity_preferred); }          // :101-114
  static bool removePreferredPodAntiAffinityTerm(Pod& p) { return remove_heaviest(p.pod_anti_affinity_preferred); }  // :116-129
  static bool removePreferredNodeAffinityTerm(Pod& p) {  // :58-71
    if (!p.has_node_affinity) return false;
    return remove_heaviest(p.preferred_node_terms);
  }
  static bool removeTopologySpreadScheduleAnyway(Pod& p) {  // :89-99
    for (size_t i = 0; i < p.topology_spread.size(); ++i)
      if (p.topology_spread[i].schedule_anyway) {
        p.topology_spread[i] = p.topology_spread.back();
        p.topology_spread.pop_back();
        return true;
      }
    return false;
  }
  static bool toleratePreferNoScheduleTaints(Pod& p) {  // :131-145
    Toleration t{"", "Exists", "", "PreferNoSchedule"};
    for (auto& x : p.tolerations)
      if (x.key == t.key && x.effect == t.effect && x.op == t.op && x.value == t.value) return false;  // MatchToleration
    p.tolerations.push_back(t);
    return true;
  }
  bool Relax(Pod& p) const {  // :36-56
    if (removeRequiredNodeAffinityTerm(p)) return true;
    if (removePreferredPodAffinityTerm(p)) return true;
    if (removePreferredPodAntiAffinityTerm(p)) return true;
    if (removePreferredNodeAffinityTerm(p)) return true;
    if (removeTopologySpreadScheduleAnyway(p)) return true;
    if (tolerate_prefer_no_schedule && toleratePreferNoScheduleTaints(p)) return true;
    return false;
  }
};

// ---------------------------------------------------------------- instance types (cloudprovider/types.go)
struct IType {
  int index;  // into Problem.instance_types
  const InstanceType* it;
  Requirements req;
  ResourceList allocatable;  // :87-89, precomputed (pure function of the type)
};

// What the cloud provider launches for a finished node (the step after Solve). Instance type: the options sorted by the
// price of Offerings.Available().Requirements(reqs).Cheapest(), element 0 (cloudprovider/fake/cloudprovider.go:74-84;
// sort.Slice taken as a stable sort over the provider's input order, canonical rule R4). Offering: that type's cheapest
// compatible available offering, lo.MinBy = first minimum in list order (cloudprovider/types.go:120-145).
static void launch_choice(const Requirements& reqs, const std::vector<const IType*>& options, NewNodeResult& out) {
  auto compatible = [&](const Offering& o) {  // Offerings.Requirements, types.go:120-126
    return (!reqs.Has("topology.kubernetes.io/zone") || reqs.Get("topology.kubernetes.io/zone").Has(o.zone)) &&
           (!reqs.Has("karpenter.sh/capacity-type") || reqs.Get("karpenter.sh/capacity-type").Has(o.capacity_type));
  };
  auto cheapest = [&](const InstanceType& it) -> const Offering* {
    const Offering* best = nullptr;
    for (auto& o : it.offerings) {
      if (!o.available || !compatible(o)) continue;
      if (!best || o.price < best->price) best = &o;
    }
    return best;
  };
  std::vector<const IType*> ordered(options.begin(), options.end());
  std::stable_sort(ordered.begin(), ordered.end(), [](const IType* a, const IType* b) { return a->index < b->index; });  // provider order
  const IType* chosen = nullptr;
  const Offering* chosen_of = nullptr;
  for (auto* t : ordered) {
    const Offering* of = cheapest(*t->it);
    if (!of) continue;
    if (!chosen || of->price < chosen_of->price) { chosen = t; chosen_of = of; }
  }
  if (!chosen) return;
  out.launch_type = chosen->index;
  out.launch_capacity_type = chosen_of->capacity_type;
  out.launch_zone = chosen_of->zone;
  out.launch_price = chosen_of->price;
}

// ---------------------------------------------------------------- machine template / nodes
struct MachineTemplate {  // machinetemplate.go:32-62
  int provisioner;        // index in weight order
  std::string name;
  std::vector<Taint> taints;
  Requirements req;
};

struct SchedNode {  // node.go:34-40
  int tmpl;
  Requirements req;
  ResourceList requests;
  std::vector<const IType*> options;
  std::vector<int> pods;
  HostPortUsage ports;
  ResourceList max_alloc;  // fast (F1): per-resource maximum of allocatable over `options` (valid when max_alloc_valid)
  bool max_alloc_valid = false;
};

// volumeusage.go:33-131. The API Gets of validate() (:133-190) happen on the host: a pod arrives with (driver, pvc id) pairs.
struct VolumeUsage {
  std::map<std::string, std::set<std::string>> volumes;  // driver -> mounted pvc ids
  static std::map<std::string, std::set<std::string>> of(const Pod& pod) {
    std::map<std::string, std::set<std::string>> v;
    for (auto& pv : pod.volumes) if (!pv.driver.empty()) v[pv.driver].insert(pv.pvc_id);  // :180-183 non-CSI volumes are not tracked
    return v;
  }
  // Validate :121-131 -> VolumeCount; Exceeds :101-112
  bool exceeds(const Pod& pod, const std::map<std::string, int32_t>& limits) const {
    auto u = volumes;
    for (auto& kv : of(pod)) u[kv.first].insert(kv.second.begin(), kv.second.end());
    for (auto& kv : u) {
      auto l = limits.find(kv.first);
      if (l == limits.end()) continue;
      if ((int64_t)kv.second.size() > (int64_t)l->second) return true;
    }
    return false;
  }
  void add(const Pod& pod) {  // Add :91-98
    for (auto& kv : of(pod)) volumes[kv.first].insert(kv.second.begin(), kv.second.end());
  }
};

struct ExistingNode {  // existingnode.go:28-39
  int state_index;
  std::vector<int> pods;
  ResourceList requests, available;
  Requirements req;
  std::vector<Taint> taints;
  HostPortUsage ports;
  VolumeUsage volumes;
  std::map<std::string, int32_t> volume_limits;
  bool initialized;
};

// state/node.go:61-78
static std::vector<Taint> state_node_taints(const StateNode& n) {
  bool initialized = false, owned = false;
  {
    auto it = n.labels.find(kInitialized);
    initialized = it != n.labels.end() && it->second == "true";
    auto o = n.labels.find(kProvisionerName);
    owned = o != n.labels.end() && !o->second.empty();
  }
  std::vector<Taint> eph = {{"node.kubernetes.io/not-ready", "", "NoSchedule"}, {"node.kubernetes.io/unreachable", "", "NoSchedule"}};
  if (!initialized && owned) eph.insert(eph.end(), n.startup_taints.begin(), n.startup_taints.end());
  std::vector<Taint> out;
  for (auto& t : n.taints) {
    bool rej = false;
    for (auto& e : eph) if (e.key == t.key && e.value == t.value && e.effect == t.effect) rej = true;
    if (!rej) out.push_back(t);
  }
  return out;
}

struct Scheduler {
  const Problem& P;
  std::set<std::string> wk;
  std::vector<Pod> pods;  // working copies (relaxation mutates them)
  std::vector<IType> itypes;
  std::vector<int> prov_order;  // weight order -> Problem.provisioners index
  std::vector<MachineTemplate> templates;
  std::vector<std::vector<const IType*>> template_types;
  std::vector<ResourceList> daemon_overhead;
  std::vector<bool> has_remaining;
  std::vector<ResourceList> remaining;
  std::vector<SchedNode> new_nodes_storage;  // creation order (result order)
  std::vector<int> new_nodes;                // s.newNodes: permutation of storage indices (sorted in place)
  std::vector<ExistingNode> existing;
  Topology topology;
  ClusterView cluster;
  Preferences prefs;
  int64_t node_id = 0;
  int64_t nodes_visited = 0, add_calls = 0;

  explicit Scheduler(const Problem& p) : P(p) {}

  // compatible/fits/hasOffering node.go:143-159
  bool has_offering(const IType& t, const Requirements& req) const {
    for (auto& o : t.it->offerings) {
      if (!o.available) continue;
      if ((!req.Has(kZone) || req.Get(kZone).Has(o.zone)) && (!req.Has(kCapacityType) || req.Get(kCapacityType).Has(o.capacity_type)))
        return true;
    }
    return false;
  }
  // fast (F2): requirement part of the filter per distinct requirement set, over ALL instance types
  std::map<std::string, std::vector<char>> req_part_memo;
  std::set<std::string> type_keys;  // keys any instance type defines (+ zone / capacity-type, read by hasOffering)
  const std::vector<char>& req_part(const Requirements& req) {
    std::string key;
    for (auto& kv : req.m)
      if (type_keys.count(kv.first)) key += kv.first + "\x01" + kv.second.Canonical() + "\x02";
    auto it = req_part_memo.find(key);
    if (it != req_part_memo.end()) return it->second;
    std::vector<char> v(itypes.size());
    for (auto& t : itypes) v[t.index] = t.req.Intersects(req) && has_offering(t, req);
    return req_part_memo.emplace(key, std::move(v)).first->second;
  }
  // fast (F5)
  std::vector<ResourceList> pod_requests_memo;
  std::vector<char> pod_requests_valid;
  ResourceList pod_requests(int pi) {
    if (!g_fast) return requests_for_pod(pods[pi]);
    if (pod_requests_valid.size() != pods.size()) { pod_requests_valid.assign(pods.size(), 0); pod_requests_memo.resize(pods.size()); }
    if (!pod_requests_valid[pi]) { pod_requests_memo[pi] = requests_for_pod(pods[pi]); pod_requests_valid[pi] = 1; }
    return pod_requests_memo[pi];
  }
  std::vector<const IType*> filter_types(const std::vector<const IType*>& in, const Requirements& req, const ResourceList& requests) {  // node.go:137-141
    std::vector<const IType*> out;
    if (g_fast) {
      const std::vector<char>& ok = req_part(req);
      for (auto* t : in)
        if (fits(requests, t->allocatable) && ok[t->index]) out.push_back(t);
      return out;
    }
    for (auto* t : in)
      if (t->req.Intersects(req) && fits(requests, t->allocatable) && has_offering(*t, req)) out.push_back(t);
    return out;
  }

  bool node_add(SchedNode& n, int pi) {  // node.go:62-107
    Pod& pod = pods[pi];
    if (g_fast) {  // F1: no remaining option can hold the merged requests -> filter_types below would come back empty
      if (!n.max_alloc_valid) {
        n.max_alloc.clear();  // max over options of allocatable[r], a missing entry counting as 0 exactly like fits() does
        for (auto* t : n.options) for (auto& kv : t->allocatable) n.max_alloc.emplace(kv.first, INT64_MIN);
        for (auto* t : n.options)
          for (auto& kv : n.max_alloc) kv.second = std::max(kv.second, getq(t->allocatable, kv.first));
        n.max_alloc_valid = true;
      }
      if (!fits(add_requests(n.requests, pod_requests(pi)), n.max_alloc)) return false;
    }
    if (!tolerates(templates[n.tmpl].taints, pod)) return false;
    if (!n.ports.validate(pod)) return false;
    Requirements node_req;
    node_req.AddAll(n.req);
    Requirements pod_req = new_pod_requirements(pod);
    if (!node_req.Compatible(pod_req, wk)) return false;
    node_req.AddAll(pod_req);
    Requirements topo_req;
    if (!topology.AddRequirements(pod_req, node_req, pod, &topo_req)) return false;
    if (!node_req.Compatible(topo_req, wk)) return false;
    node_req.AddAll(topo_req);
    ResourceList requests = add_requests(n.requests, pod_requests(pi));
    auto types = filter_types(n.options, node_req, requests);
    if (types.empty()) return false;
    n.pods.push_back(pi);
    n.max_alloc_valid = false;
    n.options = std::move(types);
    n.requests = std::move(requests);
    n.req = std::move(node_req);
    topology.Record(pod, n.req);
    n.ports.add(pod);
    return true;
  }
  bool existing_add(ExistingNode& n, int pi) {  // existingnode.go:77-130
    Pod& pod = pods[pi];
    if (!tolerates(n.taints, pod)) return false;
    if (!n.ports.validate(pod)) return false;
    if (n.volumes.exceeds(pod, n.volume_limits)) return false;  // :88-96
    ResourceList requests = add_requests(n.requests, requests_for_pod(pod));
    if (!fits(requests, n.available)) return false;
    Requirements node_req;
    node_req.AddAll(n.req);
    Requirements pod_req = new_pod_requirements(pod);
    if (!node_req.Compatible(pod_req, wk)) return false;
    node_req.AddAll(pod_req);
    Requirements topo_req;
    if (!topology.AddRequirements(pod_req, node_req, pod, &topo_req)) return false;
    if (!node_req.Compatible(topo_req, wk)) return false;
    node_req.AddAll(topo_req);
    n.pods.push_back(pi);
    n.requests = std::move(requests);
    n.req = std::move(node_req);
    topology.Record(pod, n.req);
    n.ports.add(pod);
    n.volumes.add(pod);
    return true;
  }

  // scheduler.go:174-219
  bool add(int pi) {
    ++add_calls;
    for (auto& n : existing) {
      ++nodes_visited;
      if (existing_add(n, pi)) return true;
    }
    // R1: stable sort of the persistent slice by len(Pods)
    std::stable_sort(new_nodes.begin(), new_nodes.end(), [&](int a, int b) {
      return new_nodes_storage[a].pods.size() < new_nodes_storage[b].pods.size();
    });
    for (int idx : new_nodes) {
      ++nodes_visited;
      if (node_add(new_nodes_storage[idx], pi)) return true;
    }
    for (size_t v = 0; v < templates.size(); ++v) {
      ++nodes_visited;  // one per template considered (statistic defined by this repo, see Result::nodes_visited)
      std::vector<const IType*> types = template_types[v];
      if (has_remaining[v]) {
        types = filter_by_remaining(template_types[v], remaining[v]);
        if (types.empty()) continue;
      }
      // NewNode node.go:44-60
      SchedNode n;
      n.tmpl = (int)v;
      char host[64];
      std::snprintf(host, sizeof host, "hostname-placeholder-%04lld", (long long)++node_id);
      topology.Register(kHostname, host);
      n.req.AddAll(templates[v].req);
      n.req.Add(Requirement::New(kHostname, Op::In, {host}));
      n.options = types;
      n.requests = daemon_overhead[v];
      if (!node_add(n, pi)) continue;
      new_nodes_storage.push_back(std::move(n));
      new_nodes.push_back((int)new_nodes_storage.size() - 1);
      if (has_remaining[v]) remaining[v] = subtract_max(remaining[v], new_nodes_storage.back().options);
      return true;
    }
    return false;
  }
  static ResourceList subtract_max(const ResourceList& rem, const std::vector<const IType*>& types) {  // scheduler.go:273-290
    if (types.empty()) return rem;
    ResourceList mx;
    for (auto* t : types) mx = max_resources(mx, t->it->capacity);
    ResourceList out;
    for (auto& kv : rem) out[kv.first] = kv.second - getq(mx, kv.first);
    return out;
  }
  static std::vector<const IType*> filter_by_remaining(const std::vector<const IType*>& types, const ResourceList& rem) {  // scheduler.go:293-309
    std::vector<const IType*> out;
    for (auto* t : types) {
      bool viable = true;
      for (auto& kv : rem)
        if (getq(t->it->capacity, kv.first) > kv.second) viable = false;
      if (viable) out.push_back(t);
    }
    return out;
  }

  // provisioner.go:237-296 + scheduler.go:42-78,221-267
  void init(const std::vector<int>& state_nodes, const std::vector<const Pod*>& solve_pods) {
    wk = well_known_labels(P.extra_well_known_labels);
    for (auto* p : solve_pods) pods.push_back(*p);
    {
      std::set<std::string> uids;
      for (auto& p : pods)
        if (!uids.insert(p.uid).second) throw std::runtime_error("pods must have unique UIDs (R5): " + p.uid);
    }
    itypes.reserve(P.instance_types.size());
    for (size_t i = 0; i < P.instance_types.size(); ++i) {
      IType t;
      t.index = (int)i;
      t.it = &P.instance_types[i];
      t.req = Requirements::FromNodeSelector(t.it->requirements);
      ResourceList overhead = merge(merge(t.it->kube_reserved, t.it->system_reserved), t.it->eviction_threshold);
      t.allocatable = subtract(t.it->capacity, overhead);
      itypes.push_back(std::move(t));
    }
    for (auto& t : itypes) for (auto& kv : t.req.m) type_keys.insert(kv.first);
    type_keys.insert(kZone);
    type_keys.insert(kCapacityType);
    // OrderByWeight (R4 stable)
    for (size_t i = 0; i < P.provisioners.size(); ++i) prov_order.push_back((int)i);
    std::stable_sort(prov_order.begin(), prov_order.end(), [&](int a, int b) { return P.provisioners[a].weight > P.provisioners[b].weight; });
    for (size_t v = 0; v < prov_order.size(); ++v) {
      const Provisioner& pr = P.provisioners[prov_order[v]];
      MachineTemplate mt;  // NewMachineTemplate machinetemplate.go:46-62
      mt.provisioner = (int)v;
      mt.name = pr.name;
      mt.taints = pr.taints;
      mt.req.AddAll(Requirements::FromNodeSelector(pr.requirements));
      Labels l = pr.labels;
      l[kProvisionerName] = pr.name;
      mt.req.AddAll(Requirements::FromLabels(l));
      templates.push_back(std::move(mt));
      std::vector<const IType*> ts;
      for (int idx : pr.instance_types) ts.push_back(&itypes.at(idx));
      // topology domain universe provisioner.go:266-276
      for (auto* t : ts)
        for (auto& kv : t->req.m) topology.domains[kv.first].insert(kv.second.values.begin(), kv.second.values.end());
      Requirements preq = Requirements::FromNodeSelector(pr.requirements);
      for (auto& kv : preq.m)
        if (kv.second.Operator() == Op::In) topology.domains[kv.first].insert(kv.second.values.begin(), kv.second.values.end());
      template_types.push_back(std::move(ts));
      for (auto& t : pr.taints)
        if (t.effect == "PreferNoSchedule") prefs.tolerate_prefer_no_schedule = true;  // scheduler.go:49-56
      has_remaining.push_back(pr.has_limits);
      remaining.push_back(pr.limits);
    }
    if (templates.empty()) throw std::runtime_error("no provisioners found");
    // cluster view for countDomains / inverse anti-affinity
    for (auto& n : P.nodes)
      for (auto& p : n.pods) cluster.bound.push_back({&p, &n});
    // NewTopology topology.go:56-80
    topology.inert = P.empty_topology;
    topology.cluster = &cluster;
    topology.wk = &wk;
    if (!topology.inert) {
      for (auto& p : pods) topology.excluded.insert(p.uid);
      for (auto& b : cluster.bound) {  // updateInverseAffinities :185-198
        if (b.pod->pod_anti_affinity_required.empty()) continue;
        if (topology.excluded.count(b.pod->uid)) continue;
        topology.updateInverseAntiAffinity(*b.pod, &b.node->labels);
      }
      for (auto& p : pods) topology.Update(p);
    }
    // getDaemonOverhead scheduler.go:250-267
    std::vector<Pod> daemons = P.daemonset_pods;
    for (auto& mt : templates) {
      std::vector<const Pod*> ds;
      for (auto& p : daemons) {
        if (!tolerates(mt.taints, p)) continue;
        if (!mt.req.Compatible(new_pod_requirements(p), wk)) continue;
        ds.push_back(&p);
      }
      daemon_overhead.push_back(requests_for_pods(ds));
    }
    // calculateExistingMachines scheduler.go:221-248
    for (int si : state_nodes) {
      const StateNode& n = P.nodes[si];
      auto own = n.labels.find(kProvisionerName);
      bool owned = own != n.labels.end() && !own->second.empty();
      if (!owned) continue;
      std::vector<const Pod*> ds;
      for (auto& p : daemons) {
        if (!tolerates(n.taints, p)) continue;  // raw Node.Spec.Taints here (scheduler.go:231)
        if (!Requirements::FromLabels(n.labels).Compatible(new_pod_requirements(p), wk)) continue;
        ds.push_back(&p);
      }
      ResourceList daemon_res = requests_for_pods(ds);
      // NewExistingNode existingnode.go:41-75
      std::vector<const Pod*> bound_all, bound_ds;
      for (auto& p : n.pods) {
        bound_all.push_back(&p);
        if (p.is_daemonset) bound_ds.push_back(&p);
      }
      ResourceList pod_requests, ds_requests;  // state.Node.PodRequests / DaemonSetRequests: Merge of per-pod RequestsForPods
      for (auto* p : bound_all) pod_requests = merge(pod_requests, requests_for_pod(*p));
      for (auto* p : bound_ds) ds_requests = merge(ds_requests, requests_for_pod(*p));
      ResourceList rem_daemon = subtract(daemon_res, ds_requests);
      for (auto& kv : rem_daemon) if (kv.second < 0) kv.second = 0;
      ExistingNode e;
      e.state_index = si;
      e.available = subtract(n.allocatable, pod_requests);  // state/node.go:113
      e.taints = state_node_taints(n);
      e.requests = rem_daemon;
      e.req = Requirements::FromLabels(n.labels);
      for (auto& p : n.pods) e.ports.add(p);
      for (auto& p : n.pods) e.volumes.add(p);  // state.Node.VolumeUsage(): every pod bound to the node (state/cluster.go:340-347)
      e.volume_limits = n.volume_limits;
      auto init_it = n.labels.find(kInitialized);
      e.initialized = init_it != n.labels.end() && init_it->second == "true";
      std::string hostname;
      auto h = n.labels.find(kHostname);
      if (h != n.labels.end()) hostname = h->second;
      if (hostname.empty()) hostname = n.name;
      e.req.Add(Requirement::New(kHostname, Op::In, {hostname}));
      topology.Register(kHostname, hostname);
      existing.push_back(std::move(e));
      auto pit = std::find_if(templates.begin(), templates.end(), [&](const MachineTemplate& m) { return m.name == own->second; });
      if (pit != templates.end() && has_remaining[pit - templates.begin()]) {
        size_t v = pit - templates.begin();
        for (auto& kv : remaining[v]) {  // resources.Subtract over the limits' keys, held at remaining_minus's floor
          auto c = n.capacity.find(kv.first);
          if (c != n.capacity.end()) kv.second = remaining_minus(kv.second, c->second);
        }
      }
    }
  }

  // scheduler.go:96-133 with queue.go
  void solve(Result& out) {
    size_t n = pods.size();
    std::vector<int> order(n);
    for (size_t i = 0; i < n; ++i) order[i] = (int)i;
    std::vector<int64_t> cpu(n), mem(n);
    for (size_t i = 0; i < n; ++i) {
      ResourceList r = requests_for_pod(pods[i]);
      cpu[i] = getq(r, "cpu");
      mem[i] = getq(r, "memory");
    }
    std::sort(order.begin(), order.end(), [&](int a, int b) {  // queue.go:74-110 (total order by R5)
      if (cpu[a] != cpu[b]) return cpu[a] > cpu[b];
      if (mem[a] != mem[b]) return mem[a] > mem[b];
      if (pods[a].creation_ts != pods[b].creation_ts) return pods[a].creation_ts < pods[b].creation_ts;
      return pods[a].uid < pods[b].uid;
    });
    std::vector<int> q(order.begin(), order.end());
    size_t head = 0;
    std::map<int, size_t> last_len;
    out.assign.assign(n, -1);
    out.relax_level.assign(n, 0);
    for (;;) {
      size_t len = q.size() - head;
      if (len == 0) break;
      int p = q[head];
      auto ll = last_len.find(p);
      if (ll != last_len.end() && ll->second == len) break;  // queue.go:52
      ++head;
      if (add(p)) continue;
      bool relaxed = prefs.Relax(pods[p]);
      if (relaxed && !pod_requests_valid.empty()) pod_requests_valid[p] = 0;
      q.push_back(p);
      if (relaxed) {
        last_len.clear();
        out.relax_level[p]++;
        if (!topology.inert) topology.Update(pods[p]);
      } else {
        last_len[p] = q.size() - head;
      }
    }
    // results
    size_t E = existing.size();
    out.existing_node_index.clear();
    out.existing_pods.clear();
    for (size_t e = 0; e < E; ++e) {
      out.existing_node_index.push_back(existing[e].state_index);
      out.existing_pods.push_back(existing[e].pods);
      for (int pi : existing[e].pods) out.assign[pi] = (int32_t)e;
    }
    out.new_nodes.clear();
    for (size_t i = 0; i < new_nodes_storage.size(); ++i) {
      SchedNode& nn = new_nodes_storage[i];
      nn.req.m.erase(kHostname);  // FinalizeScheduling node.go:111-115
      NewNodeResult r;
      r.provisioner = nn.tmpl;
      r.pods = nn.pods;
      for (auto* t : nn.options) r.instance_type_options.push_back(t->index);
      r.requests = nn.requests;
      for (auto& kv : nn.req.m) r.requirements[kv.first] = kv.second.Canonical();
      launch_choice(nn.req, nn.options, r);
      for (int pi : nn.pods) out.assign[pi] = (int32_t)(E + i);
      out.new_nodes.push_back(std::move(r));
    }
    out.nodes_visited = nodes_visited;
    out.add_calls = add_calls;
  }
};

// which nodes / pods a Solve sees: provisioner.go:119-144 (plain) and deprovisioning/helpers.go:42-93 (simulation)
static void gather(const Problem& P, const std::vector<int>& candidates, std::vector<int>* state_nodes, std::vector<const Pod*>* pods) {
  std::set<int> cand(candidates.begin(), candidates.end());
  for (size_t i = 0; i < P.nodes.size(); ++i)
    if (!cand.count((int)i) && !P.nodes[i].marked_for_deletion) state_nodes->push_back((int)i);
  for (auto& p : P.pods) pods->push_back(&p);
  auto reschedulable = [](const Pod& p) { return !p.is_daemonset && !p.terminal && !p.terminating; };  // utils/node/node.go:30-50
  for (int c : candidates)
    for (auto& p : P.nodes[c].pods) if (reschedulable(p)) pods->push_back(&p);
  for (size_t i = 0; i < P.nodes.size(); ++i)
    if (!cand.count((int)i) && P.nodes[i].marked_for_deletion)
      for (auto& p : P.nodes[i].pods) if (reschedulable(p)) pods->push_back(&p);
}

void solve(const Problem& P, const std::vector<int>& candidates, Result& out) {
  out = Result();
  try {
    std::vector<int> state_nodes;
    std::vector<const Pod*> pods;
    gather(P, candidates, &state_nodes, &pods);
    Scheduler s(P);
    s.init(state_nodes, pods);
    s.solve(out);
  } catch (const std::exception& e) {
    out.error = e.what();
  }
}

// ---------------------------------------------------------------- consolidation simulator
namespace {
struct Candidate {
  int node;
  const InstanceType* it;
  std::string capacity_type, zone;
  double cost;
};

double worst_launch_price(const InstanceType& it, const std::map<std::string, std::string>& req_canon, const Requirements& reqs) {  // helpers.go:292-315
  (void)req_canon;
  auto worst = [&](const char* ct, double* out) {
    bool any = false;
    double mx = 0;
    for (auto& o : it.offerings) {
      if (!o.available) continue;
      if (o.capacity_type == ct && reqs.Get(kZone).Has(o.zone)) {
        if (!any || o.price > mx) mx = o.price;
        any = true;
      }
    }
    *out = mx;
    return any;
  };
  double p;
  if (reqs.Get(kCapacityType).Has("spot") && worst("spot", &p)) return p;
  if (reqs.Get(kCapacityType).Has("on-demand") && worst("on-demand", &p)) return p;
  return std::numeric_limits<double>::max();
}
}  // namespace

// GetPodEvictionCost helpers.go:125-146
static double clampd(double lo, double v, double hi) { return v < lo ? lo : (v > hi ? hi : v); }
double pod_eviction_cost(const Pod& p) {
  double cost = 1.0;
  if (p.has_deletion_cost) cost += p.deletion_cost / 134217728.0;   // math.Pow(2, 27)
  if (p.has_priority) cost += (double)p.priority / 33554432.0;      // math.Pow(2, 25)
  return clampd(-10.0, cost, 10.0);
}

// candidateNodes (helpers.go:171-249) with consolidation.ShouldDeprovision (consolidation.go:104-118) as the filter, then
// sortAndFilterCandidates (consolidation.go:85-103): canBeTerminated (helpers.go:339-366, PDBLimits pdblimits.go:55-68) and the
// sort by disruption cost (R4: stable). Without Problem.derive_candidates the `candidate` / `disruption_cost` fields are inputs.
void rank_candidates(const Problem& P, std::vector<int>* order, std::vector<double>* cost_out) {
  struct C { int node; double cost; };
  std::vector<C> cands;
  for (size_t i = 0; i < P.nodes.size(); ++i) {
    const StateNode& n = P.nodes[i];
    if (!P.derive_candidates) {
      if (n.candidate) cands.push_back({(int)i, n.disruption_cost});
      continue;
    }
    const Provisioner* prov = nullptr;
    auto pl = n.labels.find(kProvisionerName);
    if (pl != n.labels.end())
      for (auto& pr : P.provisioners) if (pr.name == pl->second) prov = &pr;
    if (n.marked_for_deletion) continue;                    // :186-188
    if (!prov) continue;                                    // :190-192
    auto itn = n.labels.find(kInstanceType);                // :194-198 instance type must be one the provisioner offers
    bool it_ok = false;
    if (itn != n.labels.end())
      for (int idx : prov->instance_types) if (P.instance_types[(size_t)idx].name == itn->second) it_ok = true;
    if (!it_ok) continue;
    if (!n.labels.count(kCapacityType) || !n.labels.count(kZone)) continue;  // :201-208
    auto ini = n.labels.find(kInitialized);
    if (ini == n.labels.end() || ini->second != "true") continue;            // :211-213
    if (n.nominated) continue;                                               // :215-217
    // ShouldDeprovision consolidation.go:104-118
    if (n.do_not_consolidate != 0) { if (n.do_not_consolidate == 1) continue; }
    else if (!prov->consolidation_enabled) continue;
    double cost = 0.0;                                      // disruptionCost helpers.go:159-165
    for (auto& p : n.pods) cost += pod_eviction_cost(p);
    double remaining = 1.0;                                 // calculateLifetimeRemaining helpers.go:275-287
    if (prov->has_ttl_until_expired) {
      const double age = P.now_ts - n.creation_ts, total = (double)prov->ttl_seconds_until_expired;
      remaining = clampd(0.0, (total - age) / total, 1.0);
    }
    cost *= remaining;
    // canBeTerminated helpers.go:339-351
    if (n.deleting) continue;
    bool blocked = false;
    for (auto& p : n.pods) {                                // CanEvictPods pdblimits.go:55-68
      for (auto& b : P.pdbs)
        if (b.ns == p.ns && !b.selector.is_nil && selector_matches_nonnil(b.selector, p.labels) && b.disruptions_allowed == 0) blocked = true;
    }
    for (auto& p : n.pods) {                                // PodsPreventEviction helpers.go:354-366
      if (p.terminating || p.terminal || p.owned_by_node) continue;
      if (p.do_not_evict) blocked = true;
    }
    if (blocked) continue;
    cands.push_back({(int)i, cost});
  }
  // R8: a NaN cost (a "NaN" deletion-cost annotation, a TTL of 0 at age 0) sorts after every number, stable among NaNs
  std::stable_sort(cands.begin(), cands.end(), [](const C& a, const C& b) { return !std::isnan(a.cost) && (std::isnan(b.cost) || a.cost < b.cost); });
  order->clear();
  if (cost_out) cost_out->clear();
  for (auto& c : cands) { order->push_back(c.node); if (cost_out) cost_out->push_back(c.cost); }
}

// The scheduler result keeps requirements only as canonical strings; for the price guard we need the
// Requirements object of the single new node, so the simulation is re-run here with access to internals.
// mode 0: firstNNodeConsolidationOption (multinodeconsolidation.go:74-114); only_count > 0: ONE computeConsolidation (+ the
// multi-node caller's filterOutSameType) over that many cheapest candidates; mode 1: SingleNodeConsolidation.ComputeCommand
// (singlenodeconsolidation.go:43-84, Validation taken as valid: it re-runs the same simulation after a TTL).
static void consolidate_impl(const Problem& P, ConsolidationResult& out, int only_count, int mode, int single_only) {
  out = ConsolidationResult();
  try {
    std::vector<Candidate> cands;
    {
      std::vector<int> order;
      std::vector<double> costs;
      rank_candidates(P, &order, &costs);
      for (size_t q = 0; q < order.size(); ++q) {
        const StateNode& n = P.nodes[(size_t)order[q]];
        Candidate c;
        c.node = order[q];
        c.cost = costs[q];
        auto itn = n.labels.find(kInstanceType);
        c.it = nullptr;
        if (itn != n.labels.end())
          for (auto& t : P.instance_types) if (t.name == itn->second) c.it = &t;
        auto ct = n.labels.find(kCapacityType);
        c.capacity_type = ct == n.labels.end() ? "" : ct->second;
        auto z = n.labels.find(kZone);
        c.zone = z == n.labels.end() ? "" : z->second;
        cands.push_back(c);
      }
    }
    for (auto& c : cands) out.candidate_order.push_back(c.node);

    struct Cmd { int action = 0; std::vector<int> options; };
    auto compute_set = [&](const std::vector<int>& which, bool multi) -> Cmd {  // consolidation.go:190-274 on the given candidates
      Cmd cmd;
      const int count = (int)which.size();
      std::vector<Candidate> sel;
      for (int i : which) sel.push_back(cands[(size_t)i]);
      const std::vector<Candidate>& cands = sel;  // the code below indexes the selected candidates 0..count-1
      std::vector<int> nodes;
      for (int i = 0; i < count; ++i) nodes.push_back(cands[i].node);
      std::vector<int> state_nodes;
      std::vector<const Pod*> pods;
      gather(P, nodes, &state_nodes, &pods);
      Problem sim_flags = Problem();  // unused, kept for clarity
      (void)sim_flags;
      Scheduler s(P);
      s.init(state_nodes, pods);
      Result r;
      s.solve(r);
      ++out.simulations;
      size_t scheduled = 0;
      for (auto a : r.assign) if (a >= 0) ++scheduled;
      for (auto& e : s.existing)  // helpers.go:109-113: EVERY existing node Solve returns, whether or not a pod landed on it
        if (!e.initialized) return cmd;
      if (scheduled != pods.size()) return cmd;
      if (s.new_nodes_storage.empty()) { cmd.action = 1; return cmd; }
      if (s.new_nodes_storage.size() != 1) return cmd;
      double price = 0;  // getNodePrices :277-287
      for (int i = 0; i < count; ++i) {
        const Candidate& c = cands[i];
        if (!c.it) throw std::runtime_error("candidate without instance type");
        bool ok = false;
        for (auto& o : c.it->offerings)
          if (o.capacity_type == c.capacity_type && o.zone == c.zone) { price += o.price; ok = true; break; }
        if (!ok) throw std::runtime_error("unable to determine offering");
      }
      SchedNode& nn = s.new_nodes_storage[0];
      std::vector<const IType*> opts;  // filterByPrice helpers.go:148-157
      for (auto* t : nn.options)
        if (worst_launch_price(*t->it, {}, nn.req) < price) opts.push_back(t);
      if (opts.empty()) return cmd;
      bool all_spot = true;
      for (int i = 0; i < count; ++i) if (cands[i].capacity_type != "spot") all_spot = false;
      if (all_spot && nn.req.Get(kCapacityType).Has("spot")) return cmd;
      Requirement ct = nn.req.Get(kCapacityType);
      if (ct.Has("spot") && ct.Has("on-demand")) nn.req.Add(Requirement::New(kCapacityType, Op::In, {"spot"}));
      if (!multi) {  // single-node consolidation returns computeConsolidation's command as it is
        cmd.action = 2;
        for (auto* t : opts) cmd.options.push_back(t->index);
        return cmd;
      }
      // filterOutSameType multinodeconsolidation.go:132-165 (applied by the multi-node caller)
      std::set<std::string> existing_types;
      std::map<std::string, double> by_type;
      for (int i = 0; i < count; ++i) {
        const Candidate& c = cands[i];
        existing_types.insert(c.it->name);
        for (auto& o : c.it->offerings)
          if (o.capacity_type == c.capacity_type && o.zone == c.zone) {
            double ex = by_type.count(c.it->name) ? by_type[c.it->name] : std::numeric_limits<double>::max();
            if (o.price < ex) by_type[c.it->name] = o.price;
            break;
          }
      }
      double max_price = std::numeric_limits<double>::max();
      for (auto* t : opts)
        if (existing_types.count(t->it->name) && by_type[t->it->name] < max_price) max_price = by_type[t->it->name];
      std::vector<const IType*> opts2;
      for (auto* t : opts)
        if (worst_launch_price(*t->it, {}, nn.req) < max_price) opts2.push_back(t);
      if (opts2.empty()) return cmd;
      cmd.action = 2;
      for (auto* t : opts2) cmd.options.push_back(t->index);
      return cmd;
    };
    auto compute = [&](int count) -> Cmd {
      std::vector<int> which;
      for (int i = 0; i < count; ++i) which.push_back(i);
      return compute_set(which, true);
    };
    if (mode == 1) {
      if (single_only >= 0) {  // one candidate's computeConsolidation (position in the cost order)
        if (single_only >= (int)cands.size()) throw std::runtime_error("candidate out of range");
        Cmd c = compute_set({single_only}, false);
        out.action = c.action;
        out.nodes_removed = (c.action == 1 || c.action == 2) ? 1 : 0;
        out.replacement_options = c.options;
        out.single_node = (c.action == 1 || c.action == 2) ? cands[(size_t)single_only].node : -1;
        return;
      }
      for (size_t i = 0; i < cands.size(); ++i) {  // singlenodeconsolidation.go:54-77
        Cmd c = compute_set({(int)i}, false);
        out.probes.push_back((int)i);
        out.probe_actions.push_back(c.action);
        if (c.action == 1 || c.action == 2) {
          out.action = c.action;
          out.nodes_removed = 1;
          out.replacement_options = c.options;
          out.single_node = cands[i].node;
          return;
        }
      }
      return;
    }

    if (only_count > 0) {  // one computeConsolidation over the `only_count` cheapest candidates (tests of the price guards)
      if (only_count > (int)cands.size()) throw std::runtime_error("probe size out of range");
      Cmd c = compute(only_count);
      out.action = c.action;
      out.nodes_removed = (c.action == 1 || c.action == 2) ? only_count : 0;
      out.replacement_options = c.options;
      return;
    }
    // firstNNodeConsolidationOption multinodeconsolidation.go:74-114
    if (cands.size() < 2) return;
    int mn = 1, mx = (int)cands.size() - 1;
    Cmd last;
    int last_count = 0;
    while (mn <= mx) {
      int mid = (mn + mx) / 2;
      Cmd c = compute(mid + 1);
      out.probes.push_back(mid + 1);
      out.probe_actions.push_back(c.action);
      if (c.action == 1 || c.action == 2) {
        last = c;
        last_count = mid + 1;
        mn = mid + 1;
      } else {
        mx = mid - 1;
      }
    }
    out.action = last.action;
    out.nodes_removed = last_count;
    out.replacement_options = last.options;
  } catch (const std::exception& e) {
    out.error = e.what();
  }
}

void consolidate(const Problem& P, ConsolidationResult& out, int only_count) { consolidate_impl(P, out, only_count, 0, -1); }
void consolidate_single(const Problem& P, ConsolidationResult& out, int only_candidate) { consolidate_impl(P, out, 0, 1, only_candidate); }

}  // namespace oracle
