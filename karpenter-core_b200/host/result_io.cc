// Result accessors shared by every producer of a kmodel::Result (the GPU scheduler facade and,
// in tests, the oracle): flat copies for numpy, a canonical JSON dump, and a 64-bit digest.
#include <cstdio>
#include <cstring>
#include <sstream>

#include "loader.h"
#include "model.h"
#include "synth.h"

using namespace kmodel;

static uint64_t fnv(uint64_t h, const void* data, size_t n) {
  const unsigned char* p = (const unsigned char*)data;
  for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ULL; }
  return h;
}
static uint64_t fnv_str(uint64_t h, const std::string& s) { h = fnv(h, s.data(), s.size()); return fnv(h, "\0", 1); }
static void json_str(std::ostringstream& o, const std::string& s) {
  o << '"';
  for (char c : s) { if (c == '"' || c == '\\') o << '\\'; o << c; }
  o << '"';
}
static thread_local std::string g_err;

extern "C" {
const char* kh_last_error() { return g_err.c_str(); }

Problem* kh_problem_from_json(const char* text) {
  try { return problem_from_json(text); } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
Problem* kh_problem_synth(int config, long long n_pods, long long n_types, unsigned long long seed, long long n_nodes) {
  try { return synth_problem(config, n_pods, n_types, seed, n_nodes); } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void kh_problem_free(Problem* p) { delete p; }
// counts: [pods, instance types, provisioners, nodes, daemonset pods, bound pods]
void kh_problem_counts(const Problem* p, long long* out) {
  out[0] = (long long)p->pods.size();
  out[1] = (long long)p->instance_types.size();
  out[2] = (long long)p->provisioners.size();
  out[3] = (long long)p->nodes.size();
  out[4] = (long long)p->daemonset_pods.size();
  long long b = 0;
  for (auto& n : p->nodes) b += (long long)n.pods.size();
  out[5] = b;
}
long long kh_parse_quantity(const char* s) {
  try { return parse_quantity_milli(s); } catch (const std::exception& e) { g_err = e.what(); return INT64_MIN; }
}

Result* kh_result_new() { return new Result(); }
void kh_result_free(Result* r) { delete r; }
const char* kh_result_error(const Result* r) { return r->error.c_str(); }
long long kh_result_num_pods(const Result* r) { return (long long)r->assign.size(); }
long long kh_result_num_new_nodes(const Result* r) { return (long long)r->new_nodes.size(); }
long long kh_result_num_existing(const Result* r) { return (long long)r->existing_node_index.size(); }
long long kh_result_nodes_visited(const Result* r) { return r->nodes_visited; }
long long kh_result_add_calls(const Result* r) { return r->add_calls; }
int kh_result_all_pods_scheduled(const Result* r) { return r->all_pods_scheduled ? 1 : 0; }
int kh_result_uninitialized_existing(const Result* r) { return r->uninitialized_existing ? 1 : 0; }
void kh_result_assign(const Result* r, int* out) { std::memcpy(out, r->assign.data(), r->assign.size() * sizeof(int32_t)); }
void kh_result_relax(const Result* r, int* out) { std::memcpy(out, r->relax_level.data(), r->relax_level.size() * sizeof(int32_t)); }
// per new node: [provisioner, n_pods, n_options]
void kh_result_new_node_info(const Result* r, int* out) {
  for (size_t i = 0; i < r->new_nodes.size(); ++i) {
    out[3 * i] = r->new_nodes[i].provisioner;
    out[3 * i + 1] = (int)r->new_nodes[i].pods.size();
    out[3 * i + 2] = (int)kmodel::node_options(*r, r->new_nodes[i]).size();
  }
}
long long kh_result_new_node_options(const Result* r, long long i, int* out, long long cap) {
  auto& v = kmodel::node_options(*r, r->new_nodes.at(i));
  for (size_t k = 0; k < v.size() && (long long)k < cap; ++k) out[k] = v[k];
  return (long long)v.size();
}
// Order-sensitive digest of everything parity is judged on: assignment, relax levels, and for every new node
// its provisioner, pods, surviving instance-type options, requests and final requirements.
unsigned long long kh_result_digest(const Result* r) {
  uint64_t h = 1469598103934665603ULL;
  h = fnv(h, r->assign.data(), r->assign.size() * 4);
  h = fnv(h, r->relax_level.data(), r->relax_level.size() * 4);
  for (auto& n : r->new_nodes) {
    h = fnv(h, &n.provisioner, 4);
    h = fnv(h, n.pods.data(), n.pods.size() * 4);
    h = fnv(h, kmodel::node_options(*r, n).data(), kmodel::node_options(*r, n).size() * 4);
    for (auto& kv : n.requests) { h = fnv_str(h, kv.first); h = fnv(h, &kv.second, 8); }
    for (auto& kv : n.requirements) { h = fnv_str(h, kv.first); h = fnv_str(h, kv.second); }
  }
  for (auto& e : r->existing_pods) h = fnv(h, e.data(), e.size() * 4);
  return h;
}
// Per pod, the facts an independent checker of placements needs (tests): [cpu milli, memory milli, id of the "app"
// label (-1 without), required hostname anti-affinity on its own app (0/1), max skew of a DoNotSchedule zone spread (0 =
// none), max skew of a DoNotSchedule hostname spread (0 = none)].
void kh_problem_pod_summary(const Problem* p, long long* out) {
  std::map<std::string, long long> app_id;
  for (size_t i = 0; i < p->pods.size(); ++i) {
    const Pod& pd = p->pods[i];
    long long* o = out + i * 6;
    long long cpu = 0, mem = 0;
    for (auto& c : pd.containers) {
      auto a = c.requests.find("cpu"); if (a != c.requests.end()) cpu += a->second;
      auto b = c.requests.find("memory"); if (b != c.requests.end()) mem += b->second;
    }
    o[0] = cpu; o[1] = mem;
    auto app = pd.labels.find("app");
    o[2] = -1;
    if (app != pd.labels.end()) {
      auto it = app_id.find(app->second);
      if (it == app_id.end()) it = app_id.emplace(app->second, (long long)app_id.size()).first;
      o[2] = it->second;
    }
    o[3] = 0; o[4] = 0; o[5] = 0;
    for (auto& t : pd.pod_anti_affinity_required)
      if (t.topology_key == "kubernetes.io/hostname" && app != pd.labels.end() && !t.selector.is_nil && t.selector.match_labels.count("app") &&
          t.selector.match_labels.at("app") == app->second) o[3] = 1;
    for (auto& t : pd.topology_spread) {
      if (t.schedule_anyway) continue;
      if (t.topology_key == "topology.kubernetes.io/zone") o[4] = t.max_skew;
      if (t.topology_key == "kubernetes.io/hostname") o[5] = t.max_skew;
    }
  }
}

// Canonical JSON dump (small problems). Returns the required size; writes only if it fits.
static long long result_json(const Result* r, char* buf, long long cap, bool brief);
long long kh_result_to_json(const Result* r, char* buf, long long cap) { return result_json(r, buf, cap, false); }
// the same without the per-node instance-type lists ("nOptions" instead): full-size problems
long long kh_result_to_json_brief(const Result* r, char* buf, long long cap) { return result_json(r, buf, cap, true); }
}
static long long result_json(const Result* r, char* buf, long long cap, bool brief) {
  std::ostringstream o;
  o << "{\"error\":";
  json_str(o, r->error);
  o << ",\"assign\":[";
  for (size_t i = 0; i < r->assign.size(); ++i) o << (i ? "," : "") << r->assign[i];
  o << "],\"relax\":[";
  for (size_t i = 0; i < r->relax_level.size(); ++i) o << (i ? "," : "") << r->relax_level[i];
  o << "],\"existing\":[";
  for (size_t e = 0; e < r->existing_pods.size(); ++e) {
    o << (e ? "," : "") << "{\"node\":" << r->existing_node_index[e] << ",\"pods\":[";
    for (size_t i = 0; i < r->existing_pods[e].size(); ++i) o << (i ? "," : "") << r->existing_pods[e][i];
    o << "]}";
  }
  o << "],\"newNodes\":[";
  for (size_t n = 0; n < r->new_nodes.size(); ++n) {
    auto& nn = r->new_nodes[n];
    o << (n ? "," : "") << "{\"provisioner\":" << nn.provisioner << ",\"pods\":[";
    for (size_t i = 0; i < nn.pods.size(); ++i) o << (i ? "," : "") << nn.pods[i];
    const std::vector<int32_t>& nn_options = kmodel::node_options(*r, nn);
    if (brief) {
      o << "],\"nOptions\":" << nn_options.size() << ",\"requests\":{";
    } else {
      o << "],\"options\":[";
      for (size_t i = 0; i < nn_options.size(); ++i) o << (i ? "," : "") << nn_options[i];
      o << "],\"requests\":{";
    }
    bool first = true;
    for (auto& kv : nn.requests) { o << (first ? "" : ","); json_str(o, kv.first); o << ":" << kv.second; first = false; }
    o << "},\"requirements\":{";
    first = true;
    for (auto& kv : nn.requirements) { o << (first ? "" : ","); json_str(o, kv.first); o << ":"; json_str(o, kv.second); first = false; }
    o << "}";
    if (nn.launch_type >= 0) {
      o << ",\"launch\":{\"type\":" << nn.launch_type << ",\"capacityType\":";
      json_str(o, nn.launch_capacity_type);
      o << ",\"zone\":";
      json_str(o, nn.launch_zone);
      char pb[64];
      std::snprintf(pb, sizeof pb, "%.17g", nn.launch_price);
      o << ",\"price\":" << pb << "}";
    }
    o << "}";
  }
  o << "],\"nodesVisited\":" << r->nodes_visited << ",\"addCalls\":" << r->add_calls << "}";
  std::string s = o.str();
  if ((long long)s.size() + 1 <= cap) std::memcpy(buf, s.c_str(), s.size() + 1);
  return (long long)s.size() + 1;
}

