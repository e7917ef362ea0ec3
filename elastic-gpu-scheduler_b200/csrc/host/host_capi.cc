// host_capi.cc -- flat C entry points over egs::CudaUnitScheduler so that tests (ctypes) can drive
// the C++ mirror of the reference's plugin interface.  A fake apiserver = a table of registered nodes.
#include <cstring>
#include <map>
#include <string>

#include "resource_scheduler.h"

using namespace egs;

struct HostCtx {
  std::map<std::string, NodeInfo> cluster;     // the "apiserver"
  CudaUnitScheduler *sch = nullptr;
  std::string buf;
};

static const char *ret(HostCtx *c, const std::string &s) { c->buf = s; return c->buf.c_str(); }

extern "C" {

// g_max: the widest node (EGS_MAX_GPUS, or up to EGS_MAX_GPUS_WIDE)
void *egsh_create(int policy, int max_nodes, int device, int g_max) {
  HostCtx *c = new HostCtx();
  c->sch = new CudaUnitScheduler(policy, max_nodes, device, [c](const std::string &name, NodeInfo *out) -> std::string {
    auto it = c->cluster.find(name);
    if (it == c->cluster.end()) return "nodes \"" + name + "\" not found";
    *out = it->second;
    return "";
  }, g_max);
  if (!c->sch->ok()) { delete c->sch; delete c; return nullptr; }
  return c;
}
void egsh_destroy(void *h) { if (!h) return; HostCtx *c = (HostCtx *)h; delete c->sch; delete c; }
void egsh_register_node(void *h, const char *name, int64_t core_alloc, int64_t mem_alloc) {
  NodeInfo &n = ((HostCtx *)h)->cluster[name];
  n.core_allocatable = core_alloc; n.mem_allocatable = mem_alloc;
}
void egsh_register_assumed_pod(void *h, const char *node, void *pod) {
  ((HostCtx *)h)->cluster[node].assumed_pods.push_back(*(Pod *)pod);
}

void *egsh_pod_new(const char *ns, const char *name, const char *uid, const char *node_name) {
  Pod *p = new Pod(); p->ns = ns; p->name = name; p->uid = uid; p->node_name = node_name; return p;
}
void egsh_pod_free(void *p) { delete (Pod *)p; }
// has_* == 0 leaves the key out of Requests (absent keys read as 0, pod.go:94-108)
void egsh_pod_add_container(void *p, const char *cname, int has_core, int64_t core, int has_mem, int64_t mem) {
  Container c; c.name = cname;
  if (has_core) c.requests[kResourceGPUCore] = core;
  if (has_mem) c.requests[kResourceGPUMemory] = mem;
  ((Pod *)p)->containers.push_back(c);
}
void egsh_pod_set_annotation(void *p, const char *k, const char *v) { ((Pod *)p)->annotations[k] = v; }
// annotations and labels as "A\tkey\tvalue\n" / "L\tkey\tvalue\n"
const char *egsh_pod_meta(void *h, void *p) {
  std::string s;
  for (auto &kv : ((Pod *)p)->annotations) s += "A\t" + kv.first + "\t" + kv.second + "\n";
  for (auto &kv : ((Pod *)p)->labels) s += "L\t" + kv.first + "\t" + kv.second + "\n";
  return ret((HostCtx *)h, s);
}
int egsh_handles(void *p) { return CudaUnitScheduler::Handles(*(Pod *)p) ? 1 : 0; }

// "E\t<error>\n" or per node "F\t<name>\n" (filtered, input order) / "X\t<name>\t<message>\n" (failedNodes)
const char *egsh_assume(void *h, void *pod, const char **nodes, int n) {
  HostCtx *c = (HostCtx *)h;
  std::vector<std::string> names(nodes, nodes + n), filtered;
  std::map<std::string, std::string> failed;
  std::string e = c->sch->Assume(names, *(Pod *)pod, &filtered, &failed);
  if (!e.empty()) return ret(c, "E\t" + e + "\n");
  std::string s;
  for (auto &f : filtered) s += "F\t" + f + "\n";
  for (auto &kv : failed) s += "X\t" + kv.first + "\t" + kv.second + "\n";
  return ret(c, s);
}
void egsh_score(void *h, void *pod, const char **nodes, int n, int64_t *out) {
  std::vector<std::string> names(nodes, nodes + n);
  auto sc = ((HostCtx *)h)->sch->Score(names, *(Pod *)pod);
  for (int i = 0; i < n; i++) out[i] = sc[i];
}
const char *egsh_bind(void *h, const char *node, void *pod) { return ret((HostCtx *)h, ((HostCtx *)h)->sch->Bind(node, (Pod *)pod)); }
const char *egsh_add_pod(void *h, void *pod) { return ret((HostCtx *)h, ((HostCtx *)h)->sch->AddPod(*(Pod *)pod)); }
const char *egsh_forget_pod(void *h, void *pod) { return ret((HostCtx *)h, ((HostCtx *)h)->sch->ForgetPod(*(Pod *)pod)); }
int egsh_known_pod(void *h, void *pod) { return ((HostCtx *)h)->sch->KnownPod(*(Pod *)pod); }
int egsh_released_pod(void *h, void *pod) { return ((HostCtx *)h)->sch->ReleasedPod(*(Pod *)pod); }
const char *egsh_status(void *h) { return ret((HostCtx *)h, ((HostCtx *)h)->sch->Status()); }

}  // extern "C"

// ---- extender JSON codec (no GPU needed) ----------------------------------------------------------
#include "extender_json.h"

struct JsonCtx { NodeInterner nodes; ExtenderArgs args; BindingArgs bind; std::string buf; };

// ---- the three extender routes end to end: HTTP body -> JSON decode -> plugin verb (libegs on the GPU) -> JSON body.
// pkg/routes/routes.go:39-163 over pkg/server/{predicate,priority,bind}.go.  *http_status receives 200 / 500;
// a request the reference answers by panicking (routes.go:98-109) yields status -1 and the panic text.
struct RouteCtx {
  HostCtx *host;
  NodeInterner nodes;                                  // per-process interning of the request's node names
  std::map<std::string, Pod> pods;                     // the "apiserver": ns/name -> pod (GetPod of bind.go:36)
  std::string buf;
};
static const char kNotCacheCapable[] = "elastic-gpu-scheduler extender must be configured with nodeCacheCapable=true";

extern "C" {
void *egsr_new(void *host) { RouteCtx *r = new RouteCtx(); r->host = (HostCtx *)host; return r; }
void egsr_free(void *r) { delete (RouteCtx *)r; }
void egsr_register_pod(void *r, void *pod) { Pod *p = (Pod *)pod; ((RouteCtx *)r)->pods[p->ns + "/" + p->name] = *p; }

// POST /scheduler/filter
const char *egsr_filter(void *rc, const char *json, int64_t len, int *http_status) {
  RouteCtx *r = (RouteCtx *)rc;
  *http_status = 200;
  ExtenderArgs a;
  std::string err = ParseExtenderArgs(std::string_view(json, (size_t)len), &r->nodes, &a);
  if (!err.empty()) { r->buf = EncodeFilterResult({}, {}, err, false); return r->buf.c_str(); }                 // routes.go:51-58
  if (!a.has_nodenames) { r->buf = EncodeFilterResult({}, {}, kNotCacheCapable, false); return r->buf.c_str(); } // routes.go:59-64
  if (!CudaUnitScheduler::Handles(a.pod)) {                                                                     // predicate.go:19-24
    r->buf = EncodeFilterResult({}, {}, "cannot find scheduler for pod " + a.pod.ns + "/" + a.pod.name, false);
    return r->buf.c_str();
  }
  std::vector<std::string> names; names.reserve(a.node_ids.size());
  for (int32_t id : a.node_ids) names.push_back(r->nodes.Name(id));
  std::vector<std::string> filtered; std::map<std::string, std::string> failed;
  err = r->host->sch->Assume(names, a.pod, &filtered, &failed);
  if (!err.empty()) { r->buf = EncodeFilterResult({}, {}, err, false); return r->buf.c_str(); }                 // predicate.go:27-31
  r->buf = EncodeFilterResult(filtered, failed, "", true);
  return r->buf.c_str();
}

// POST /scheduler/priorities
const char *egsr_priorities(void *rc, const char *json, int64_t len, int *http_status) {
  RouteCtx *r = (RouteCtx *)rc;
  *http_status = 200;
  ExtenderArgs a;
  std::string err = ParseExtenderArgs(std::string_view(json, (size_t)len), &r->nodes, &a);
  if (!err.empty()) { *http_status = -1; r->buf = "panic: " + err; return r->buf.c_str(); }                     // routes.go:98-100
  if (!a.has_nodenames) { *http_status = -1; r->buf = "panic: runtime error: invalid memory address or nil pointer dereference"; return r->buf.c_str(); }   // priority.go:19
  if (!CudaUnitScheduler::Handles(a.pod)) { *http_status = -1; r->buf = "panic: cannot find scheduler for pod " + a.pod.ns + "/" + a.pod.name; return r->buf.c_str(); }
  std::vector<std::string> names; names.reserve(a.node_ids.size());
  for (int32_t id : a.node_ids) names.push_back(r->nodes.Name(id));
  std::vector<int64_t> scores = r->host->sch->Score(names, a.pod);
  std::vector<std::pair<std::string, int64_t>> list; list.reserve(names.size());
  for (size_t i = 0; i < names.size(); i++) list.emplace_back(names[i], scores[i]);
  r->buf = EncodeHostPriorityList(list);
  return r->buf.c_str();
}

// POST /scheduler/bind
const char *egsr_bind(void *rc, const char *json, int64_t len, int *http_status) {
  RouteCtx *r = (RouteCtx *)rc;
  BindingArgs b;
  std::string err = ParseBindingArgs(std::string_view(json, (size_t)len), &b);
  if (err.empty()) {
    auto it = r->pods.find(b.pod_namespace + "/" + b.pod_name);
    if (it == r->pods.end()) err = "pods \"" + b.pod_name + "\" not found";                                    // GetPod, pod.go:110-126
    else if (!CudaUnitScheduler::Handles(it->second)) err = "cannot find scheduler for pod " + b.pod_namespace + "/" + b.pod_name;
    else err = r->host->sch->Bind(b.node, &it->second);
  }
  *http_status = err.empty() ? 200 : 500;                                                                       // routes.go:146-158
  r->buf = EncodeBindingResult(err);
  return r->buf.c_str();
}
}

extern "C" {
void *egsj_new() { return new JsonCtx(); }
void egsj_free(void *c) { delete (JsonCtx *)c; }
// returns "" or the error; afterwards egsj_* accessors read the parsed request
const char *egsj_parse_args(void *c, const char *json, int64_t len) {
  JsonCtx *j = (JsonCtx *)c;
  j->buf = ParseExtenderArgs(std::string_view(json, (size_t)len), &j->nodes, &j->args);
  return j->buf.c_str();
}
int egsj_has_nodenames(void *c) { return ((JsonCtx *)c)->args.has_nodenames; }
int egsj_n_nodes(void *c) { return (int)((JsonCtx *)c)->args.node_ids.size(); }
const int32_t *egsj_node_ids(void *c) { return ((JsonCtx *)c)->args.node_ids.data(); }
int egsj_interned(void *c) { return ((JsonCtx *)c)->nodes.size(); }
const char *egsj_node_name(void *c, int id) { return ((JsonCtx *)c)->nodes.Name(id).c_str(); }
// "ns\tname\tuid\tnodeName\n" then per container "C\tname\thasCore\tcore\thasMem\tmem\n", annotations "A\tk\tv\n"
const char *egsj_pod_dump(void *c) {
  JsonCtx *j = (JsonCtx *)c;
  const Pod &p = j->args.pod;
  std::string s = p.ns + "\t" + p.name + "\t" + p.uid + "\t" + p.node_name + "\n";
  for (const auto &ct : p.containers) {
    auto ci = ct.requests.find(kResourceGPUCore), mi = ct.requests.find(kResourceGPUMemory);
    s += "C\t" + ct.name + "\t" + (ci != ct.requests.end() ? "1\t" + std::to_string(ci->second) : std::string("0\t0")) + "\t" +
         (mi != ct.requests.end() ? "1\t" + std::to_string(mi->second) : std::string("0\t0")) + "\n";
  }
  for (const auto &kv : p.annotations) s += "A\t" + kv.first + "\t" + kv.second + "\n";
  j->buf = s;
  return j->buf.c_str();
}
const char *egsj_parse_binding(void *c, const char *json, int64_t len) {
  JsonCtx *j = (JsonCtx *)c;
  std::string e = ParseBindingArgs(std::string_view(json, (size_t)len), &j->bind);
  j->buf = e.empty() ? ("\t" + j->bind.pod_name + "\t" + j->bind.pod_namespace + "\t" + j->bind.pod_uid + "\t" + j->bind.node) : e;
  return j->buf.c_str();
}
int egsj_quantity(const char *q, int64_t *out) { return ParseQuantityValue(q, out) ? 1 : 0; }
// names / failed as "\n"-separated lists ("name\tmsg" for failed)
const char *egsj_encode_filter(void *c, const char *names, const char *failed, const char *error) {
  JsonCtx *j = (JsonCtx *)c;
  std::vector<std::string> nn; std::map<std::string, std::string> ff;
  auto split = [](const std::string &s, auto f) { size_t b = 0; while (b < s.size()) { size_t e = s.find('\n', b); if (e == std::string::npos) e = s.size(); if (e > b) f(s.substr(b, e - b)); b = e + 1; } };
  split(names, [&](const std::string &l) { nn.push_back(l); });
  split(failed, [&](const std::string &l) { size_t t = l.find('\t'); ff[l.substr(0, t)] = t == std::string::npos ? "" : l.substr(t + 1); });
  j->buf = EncodeFilterResult(nn, ff, error);
  return j->buf.c_str();
}
// an error path of the filter verb: NodeNames stays nil (predicate.go:21-31, routes.go:51-64)
const char *egsj_encode_filter_error(void *c, const char *error) {
  JsonCtx *j = (JsonCtx *)c;
  j->buf = EncodeFilterResult({}, {}, error, false);
  return j->buf.c_str();
}
const char *egsj_encode_priorities(void *c, const char *names, const int64_t *scores, int n) {
  JsonCtx *j = (JsonCtx *)c;
  std::vector<std::pair<std::string, int64_t>> v;
  std::string s(names); size_t b = 0;
  for (int i = 0; i < n; i++) { size_t e = s.find('\n', b); if (e == std::string::npos) e = s.size(); v.emplace_back(s.substr(b, e - b), scores[i]); b = e + 1; }
  j->buf = EncodeHostPriorityList(v);
  return j->buf.c_str();
}
const char *egsj_encode_binding(void *c, const char *error) { JsonCtx *j = (JsonCtx *)c; j->buf = EncodeBindingResult(error); return j->buf.c_str(); }
}
