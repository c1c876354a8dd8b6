// JSON -> kmodel::Problem loader and k8s resource.Quantity string parser.
// Field names follow the Go structs the reference's tests build
// (pkg/test/pods.go:62-111, pkg/test/provisioner.go, pkg/cloudprovider/fake/instancetype.go).
#include "loader.h"

#include <cctype>
#include <set>
#include <stdexcept>

#include "json.h"

namespace kmodel {

// resource.MustParse restated for the suffixes the reference uses. Exact: the result
// must be a whole number of milli-units, otherwise the quantity is rejected
// (SURVEY.md 7-H6). |milli| must stay below kQuantityBound = 2^62 (DESIGN §2): sums of two
// admitted values then never wrap int64, and the device's sort key adds 2^62.
int64_t parse_quantity_milli(const std::string& s) {
  if (s.empty()) throw std::runtime_error("empty quantity");
  size_t i = 0;
  bool neg = false;
  if (s[i] == '+' || s[i] == '-') neg = s[i++] == '-';
  __int128 mant = 0;
  int frac_digits = 0;
  bool seen_dot = false, any = false;
  for (; i < s.size(); ++i) {
    char c = s[i];
    if (c >= '0' && c <= '9') {
      mant = mant * 10 + (c - '0');
      if (seen_dot) ++frac_digits;
      // mant * (suffix multiplier < 2^61) and 10^frac_digits must stay exact in __int128, so mantissas of 21 or more
      // digits (leading zeros aside) and more than 30 fractional digits are refused; an admitted value has at most 19
      // digits of milli-units
      if (mant >= (__int128)100000000000LL * 1000000000LL || frac_digits > 30)
        throw std::runtime_error("quantity has too many digits: " + s);
      any = true;
    } else if (c == '.' && !seen_dot) {
      seen_dot = true;
    } else {
      break;
    }
  }
  if (!any) throw std::runtime_error("bad quantity: " + s);
  std::string suf = s.substr(i);
  __int128 mul = 1000;  // to milli
  __int128 div = 1;
  if (suf == "") {
  } else if (suf == "m") mul = 1;
  else if (suf == "k") mul = (__int128)1000 * 1000;
  else if (suf == "M") mul = (__int128)1000 * 1000000;
  else if (suf == "G") mul = (__int128)1000 * 1000000000LL;
  else if (suf == "T") mul = (__int128)1000 * 1000000000000LL;
  else if (suf == "P") mul = (__int128)1000 * 1000000000000000LL;
  else if (suf == "Ki") mul = (__int128)1000 << 10;
  else if (suf == "Mi") mul = (__int128)1000 << 20;
  else if (suf == "Gi") mul = (__int128)1000 << 30;
  else if (suf == "Ti") mul = (__int128)1000 << 40;
  else if (suf == "Pi") mul = (__int128)1000 << 50;
  else throw std::runtime_error("unsupported quantity suffix: " + s);
  for (int k = 0; k < frac_digits; ++k) div *= 10;
  __int128 num = mant * mul;
  if (num % div != 0) throw std::runtime_error("sub-milli quantity rejected: " + s);
  __int128 v = num / div;
  if (v >= (__int128)kQuantityBound) throw std::runtime_error("quantity out of range (|milli| >= 2^62): " + s);
  int64_t r = (int64_t)v;
  return neg ? -r : r;
}

namespace {
using kjson::Value;

ResourceList resources(const Value* v) {
  ResourceList r;
  if (!v || v->is_null()) return r;
  for (auto& kv : v->obj) {
    try {
      r[kv.first] = parse_quantity_milli(kv.second.str);  // a string, or the raw text of a number
    } catch (const std::runtime_error& e) {
      throw std::runtime_error("resource " + kv.first + ": " + e.what());
    }
  }
  return r;
}
// Capacities charged against provisioner limits must not be negative: remaining_minus (model.h) relies on it
ResourceList capacity(const Value* v, const std::string& owner) {
  ResourceList r = resources(v);
  for (auto& kv : r)
    if (kv.second < 0) throw std::runtime_error(owner + ": negative capacity of resource " + kv.first);
  return r;
}
Labels labels(const Value* v) {
  Labels r;
  if (!v || v->is_null()) return r;
  for (auto& kv : v->obj) r[kv.first] = kv.second.str;
  return r;
}
Op parse_op(const std::string& s) {
  if (s == "In") return Op::In;
  if (s == "NotIn") return Op::NotIn;
  if (s == "Exists") return Op::Exists;
  if (s == "DoesNotExist") return Op::DoesNotExist;
  if (s == "Gt") return Op::Gt;
  if (s == "Lt") return Op::Lt;
  throw std::runtime_error("bad operator: " + s);
}
std::vector<NodeSelectorRequirement> reqs(const Value* v) {
  std::vector<NodeSelectorRequirement> out;
  if (!v || v->is_null()) return out;
  for (auto& e : v->arr) {
    NodeSelectorRequirement r;
    r.key = e.s("key");
    r.op = parse_op(e.s("operator", "In"));
    if (const Value* vals = e.get("values"))
      for (auto& x : vals->arr) r.values.push_back(x.str);
    out.push_back(std::move(r));
  }
  return out;
}
LabelSelector selector(const Value* v) {
  LabelSelector s;
  if (!v || v->is_null()) return s;
  s.is_nil = false;
  s.match_labels = labels(v->get("matchLabels"));
  s.match_expressions = reqs(v->get("matchExpressions"));
  return s;
}
// k8s.io/apimachinery validation: a label name part / value ([A-Za-z0-9]([-A-Za-z0-9_.]*[A-Za-z0-9])?, at most 63) and a
// qualified name (an optional DNS-1123 subdomain prefix and '/' before the name part).
bool label_name_part(const std::string& s) {
  if (s.empty() || s.size() > 63 || !std::isalnum((unsigned char)s.front()) || !std::isalnum((unsigned char)s.back())) return false;
  for (unsigned char c : s)
    if (!std::isalnum(c) && c != '-' && c != '_' && c != '.') return false;
  return true;
}
bool qualified_name(const std::string& s) {
  const size_t slash = s.find('/');
  if (slash == std::string::npos) return label_name_part(s);
  const std::string prefix = s.substr(0, slash), name = s.substr(slash + 1);
  if (prefix.empty() || prefix.size() > 253 || name.find('/') != std::string::npos) return false;
  for (size_t i = 0; i < prefix.size(); ++i) {
    const char c = prefix[i];
    const bool alnum = (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9');
    const bool edge = i == 0 || i + 1 == prefix.size() || prefix[i - 1] == '.' || prefix[i + 1] == '.';
    if (!alnum && (edge || (c != '-' && c != '.'))) return false;
  }
  return label_name_part(name);
}
// metav1.LabelSelectorAsSelector's checks (labels.NewRequirement): buildNamespaceList returns its error, so NewScheduler
// fails on a namespaceSelector it rejects.
void check_namespace_selector(const LabelSelector& s) {
  auto fail = [](const std::string& why) { throw std::runtime_error("invalid namespaceSelector: " + why); };
  for (auto& kv : s.match_labels) {
    if (!qualified_name(kv.first)) fail("label key \"" + kv.first + "\"");
    if (!kv.second.empty() && !label_name_part(kv.second)) fail("label value \"" + kv.second + "\"");
  }
  for (auto& r : s.match_expressions) {
    if (r.op != Op::In && r.op != Op::NotIn && r.op != Op::Exists && r.op != Op::DoesNotExist)
      fail("\"" + r.key + "\": operator is not one of In, NotIn, Exists, DoesNotExist");
    if (!qualified_name(r.key)) fail("label key \"" + r.key + "\"");
    const bool set_op = r.op == Op::In || r.op == Op::NotIn;
    if (set_op && r.values.empty()) fail("\"" + r.key + "\": In and NotIn need values");
    if (!set_op && !r.values.empty()) fail("\"" + r.key + "\": Exists and DoesNotExist take no values");
    for (auto& v : r.values)
      if (!v.empty() && !label_name_part(v)) fail("label value \"" + v + "\"");
  }
}
PodAffinityTerm affinity_term(const Value& e) {
  PodAffinityTerm t;
  t.selector = selector(e.get("labelSelector"));
  if (const Value* ns = e.get("namespaces"))
    for (auto& x : ns->arr) t.namespaces.push_back(x.str);
  t.namespace_selector = selector(e.get("namespaceSelector"));
  if (!t.namespace_selector.is_nil) check_namespace_selector(t.namespace_selector);
  t.topology_key = e.s("topologyKey");
  return t;
}
// buildNamespaceList (topology.go:326-347) of every term with a namespaceSelector, done once here because the document
// holds all it reads: the term's `namespaces` become the Namespace objects the selector matches plus the ones the term
// named (the pod's own namespace is not added), {kNoNamespace} when that is empty (model.h). A batch repeats one term
// thousands of times, so each distinct selector is matched against the Namespaces once.
void resolve_namespace_selectors(Problem& P, bool listed) {
  std::map<std::string, std::vector<std::string>> matched;  // selector -> the Namespaces it matches
  auto resolve = [&](PodAffinityTerm& t) {
    if (t.namespace_selector.is_nil) return;
    if (!listed) throw std::runtime_error("a pod affinity term has a namespaceSelector but the document lists no namespaces");
    std::string key;
    for (auto& kv : t.namespace_selector.match_labels) key += kv.first + "=" + kv.second + ",";
    for (auto& r : t.namespace_selector.match_expressions) {
      key += "|" + r.key + ":" + std::to_string((int)r.op) + ":";
      for (auto& v : r.values) key += v + ",";
    }
    auto it = matched.find(key);
    if (it == matched.end()) {
      std::vector<std::string> names;
      for (auto& n : P.namespaces)
        if (selector_matches_labels(t.namespace_selector, n.labels)) names.push_back(n.name);
      it = matched.emplace(key, std::move(names)).first;
    }
    std::set<std::string> out(it->second.begin(), it->second.end());
    out.insert(t.namespaces.begin(), t.namespaces.end());
    if (out.empty()) out.insert(kNoNamespace);
    t.namespaces.assign(out.begin(), out.end());
  };
  auto pod_terms = [&](Pod& p) {
    if (p.ns == kNoNamespace) throw std::runtime_error("a pod may not be in namespace " + p.ns);
    for (auto* terms : {&p.pod_affinity_required, &p.pod_anti_affinity_required})
      for (auto& t : *terms) resolve(t);
    for (auto* terms : {&p.pod_affinity_preferred, &p.pod_anti_affinity_preferred})
      for (auto& t : *terms) resolve(t.term);
  };
  for (auto* ps : {&P.pods, &P.daemonset_pods})
    for (auto& p : *ps) pod_terms(p);
  for (auto& n : P.nodes)
    for (auto& p : n.pods) pod_terms(p);
}
std::vector<Taint> taints(const Value* v) {
  std::vector<Taint> out;
  if (!v || v->is_null()) return out;
  for (auto& e : v->arr) out.push_back({e.s("key"), e.s("value"), e.s("effect")});
  return out;
}
Container container(const Value& e) {
  Container c;
  c.requests = resources(e.get("requests"));
  c.limits = resources(e.get("limits"));
  // the API server refuses negative requests and limits (ValidateResourceRequirements); node sums rely on it (oracle.cc)
  for (auto* l : {&c.requests, &c.limits})
    for (auto& kv : *l)
      if (kv.second < 0) throw std::runtime_error("resource " + kv.first + ": negative request or limit");
  if (const Value* ports = e.get("ports"))
    for (auto& p : ports->arr) {
      HostPort hp;
      hp.ip = p.s("hostIP");
      hp.port = (int32_t)p.i("hostPort");
      hp.protocol = p.s("protocol", "TCP");
      c.ports.push_back(hp);
    }
  return c;
}
Pod pod(const Value& e, size_t index) {
  Pod p;
  p.name = e.s("name", "pod-" + std::to_string(index));
  p.ns = e.s("namespace", "default");
  p.uid = e.s("uid", p.name);
  p.creation_ts = e.i("creationTimestamp");
  p.labels = labels(e.get("labels"));
  if (const Value* cs = e.get("containers"))
    for (auto& c : cs->arr) p.containers.push_back(container(c));
  if (e.has("requests") || e.has("limits") || e.has("ports")) p.containers.push_back(container(e));
  if (const Value* cs = e.get("initContainers"))
    for (auto& c : cs->arr) p.init_containers.push_back(container(c));
  p.node_selector = labels(e.get("nodeSelector"));
  if (const Value* na = e.get("nodeAffinity"); na && !na->is_null()) {
    p.has_node_affinity = true;
    if (const Value* r = na->get("required"); r && !r->is_null()) {
      p.has_required_node_affinity = true;
      for (auto& term : r->arr) {
        Value tmp = term;
        p.required_node_terms.push_back(reqs(&tmp));
      }
    }
    if (const Value* pr = na->get("preferred"))
      for (auto& t : pr->arr) {
        PreferredSchedulingTerm pt;
        pt.weight = (int32_t)t.i("weight");
        pt.preference = reqs(t.get("terms"));
        p.preferred_node_terms.push_back(std::move(pt));
      }
  }
  auto load_aff = [&](const char* key, std::vector<PodAffinityTerm>& req, std::vector<WeightedPodAffinityTerm>& pref) {
    const Value* a = e.get(key);
    if (!a || a->is_null()) return;
    if (const Value* r = a->get("required"))
      for (auto& t : r->arr) req.push_back(affinity_term(t));
    if (const Value* pr = a->get("preferred"))
      for (auto& t : pr->arr) {
        WeightedPodAffinityTerm w;
        w.weight = (int32_t)t.i("weight");
        w.term = affinity_term(*t.get("term"));
        pref.push_back(std::move(w));
      }
  };
  load_aff("podAffinity", p.pod_affinity_required, p.pod_affinity_preferred);
  load_aff("podAntiAffinity", p.pod_anti_affinity_required, p.pod_anti_affinity_preferred);
  if (const Value* ts = e.get("topologySpreadConstraints"))
    for (auto& t : ts->arr) {
      TopologySpreadConstraint c;
      c.max_skew = (int32_t)t.i("maxSkew", 1);
      c.topology_key = t.s("topologyKey");
      c.schedule_anyway = t.s("whenUnsatisfiable", "DoNotSchedule") == "ScheduleAnyway";
      c.selector = selector(t.get("labelSelector"));
      p.topology_spread.push_back(std::move(c));
    }
  if (const Value* ts = e.get("tolerations"))
    for (auto& t : ts->arr) p.tolerations.push_back({t.s("key"), t.s("operator"), t.s("value"), t.s("effect")});
  p.node_name = e.s("nodeName");
  p.is_daemonset = e.boolean("isDaemonSet");
  p.terminal = e.boolean("terminal");
  p.terminating = e.boolean("terminating");
  if (const Value* vs = e.get("volumes"))
    for (auto& v : vs->arr) p.volumes.push_back({v.s("driver"), v.s("pvc")});
  if (e.has("deletionCost")) { p.has_deletion_cost = true; p.deletion_cost = e.d("deletionCost"); }
  if (e.has("priority")) { p.has_priority = true; p.priority = (int32_t)e.i("priority"); }
  p.do_not_evict = e.boolean("doNotEvict");
  p.owned_by_node = e.boolean("ownedByNode");
  return p;
}
}  // namespace

Problem* problem_from_json(const char* text) {
  Value root = kjson::Parser(text).parse();
  auto prob = std::make_unique<Problem>();
  Problem& P = *prob;
  if (const Value* w = root.get("wellKnownLabels"))
    for (auto& x : w->arr) P.extra_well_known_labels.push_back(x.str);
  if (const Value* its = root.get("instanceTypes"))
    for (auto& e : its->arr) {
      InstanceType it;
      it.name = e.s("name");
      it.requirements = reqs(e.get("requirements"));
      if (const Value* ofs = e.get("offerings"))
        for (auto& o : ofs->arr)
          it.offerings.push_back({o.s("capacityType"), o.s("zone"), o.d("price"), o.boolean("available", true)});
      it.capacity = capacity(e.get("capacity"), "instance type " + it.name);
      if (const Value* ov = e.get("overhead"); ov && !ov->is_null()) {
        it.kube_reserved = resources(ov->get("kubeReserved"));
        it.system_reserved = resources(ov->get("systemReserved"));
        it.eviction_threshold = resources(ov->get("evictionThreshold"));
      }
      P.instance_types.push_back(std::move(it));
    }
  if (const Value* ps = root.get("provisioners"))
    for (auto& e : ps->arr) {
      Provisioner pr;
      pr.name = e.s("name", "default");
      pr.weight = (int32_t)e.i("weight");
      pr.requirements = reqs(e.get("requirements"));
      pr.labels = labels(e.get("labels"));
      pr.taints = taints(e.get("taints"));
      pr.startup_taints = taints(e.get("startupTaints"));
      if (const Value* l = e.get("limits"); l && !l->is_null()) {
        pr.has_limits = true;
        pr.limits = resources(l);
      }
      pr.consolidation_enabled = e.boolean("consolidationEnabled");
      if (e.has("ttlSecondsUntilExpired")) { pr.has_ttl_until_expired = true; pr.ttl_seconds_until_expired = e.i("ttlSecondsUntilExpired"); }
      if (const Value* its = e.get("instanceTypes"); its && its->kind == Value::Arr) {
        for (auto& x : its->arr) pr.instance_types.push_back((int32_t)x.num);
      } else {
        for (size_t k = 0; k < P.instance_types.size(); ++k) pr.instance_types.push_back((int32_t)k);
      }
      P.provisioners.push_back(std::move(pr));
    }
  if (const Value* ns = root.get("nodes"))
    for (auto& e : ns->arr) {
      StateNode n;
      n.name = e.s("name");
      n.labels = labels(e.get("labels"));
      n.taints = taints(e.get("taints"));
      n.startup_taints = taints(e.get("startupTaints"));
      n.allocatable = resources(e.get("allocatable"));
      n.capacity = capacity(e.get("capacity"), "node " + n.name);
      if (n.capacity.empty()) n.capacity = capacity(e.get("allocatable"), "node " + n.name);
      if (const Value* ps = e.get("pods")) {
        size_t k = 0;
        for (auto& p : ps->arr) {
          n.pods.push_back(pod(p, k++));
          n.pods.back().node_name = n.name;
        }
      }
      n.marked_for_deletion = e.boolean("markedForDeletion");
      n.candidate = e.boolean("candidate");
      n.disruption_cost = e.d("disruptionCost");
      n.deleting = e.boolean("deleting");
      n.nominated = e.boolean("nominated");
      if (e.has("doNotConsolidate")) n.do_not_consolidate = e.s("doNotConsolidate") == "true" ? 1 : 2;
      n.creation_ts = e.d("creationTimestamp");
      if (const Value* vl = e.get("volumeLimits"); vl && !vl->is_null())
        for (auto& kv : vl->obj) n.volume_limits[kv.first] = (int32_t)kv.second.num;
      P.nodes.push_back(std::move(n));
    }
  if (const Value* ps = root.get("pods")) {
    size_t k = 0;
    for (auto& e : ps->arr) P.pods.push_back(pod(e, k++));
  }
  if (const Value* ps = root.get("daemonSetPods")) {
    size_t k = 0;
    for (auto& e : ps->arr) {
      P.daemonset_pods.push_back(pod(e, k++));
      P.daemonset_pods.back().is_daemonset = true;
    }
  }
  if (const Value* ps = root.get("pdbs"))
    for (auto& e : ps->arr) {
      PodDisruptionBudget b;
      b.ns = e.s("namespace", "default");
      b.selector = selector(e.get("selector"));
      b.disruptions_allowed = (int32_t)e.i("disruptionsAllowed");
      P.pdbs.push_back(std::move(b));
    }
  const Value* nss = root.get("namespaces");
  const bool listed = nss && !nss->is_null();
  if (listed) {
    std::set<std::string> names;
    for (auto& e : nss->arr) {
      Namespace n{e.s("name"), labels(e.get("labels"))};
      if (n.name == kNoNamespace) throw std::runtime_error("a Namespace may not be named " + n.name);
      if (!names.insert(n.name).second) throw std::runtime_error("duplicate namespace " + n.name);
      P.namespaces.push_back(std::move(n));
    }
  }
  resolve_namespace_selectors(P, listed);
  P.now_ts = root.d("now");
  P.derive_candidates = root.boolean("deriveCandidates");
  P.simulation_mode = root.boolean("simulationMode");
  P.empty_topology = root.boolean("emptyTopology");
  return prob.release();
}

}  // namespace kmodel
