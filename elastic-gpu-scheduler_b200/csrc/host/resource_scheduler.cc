// resource_scheduler.cc -- see resource_scheduler.h.  Only include/egs.h is used: this file is the
// C++ twin of the cgo shim shown in INTEGRATION.md.
#include "resource_scheduler.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sstream>

namespace egs {

static int64_t requestOf(const Container &c, const char *key) {   // GetGPUCoreFromContainer pod.go:94-108
  auto it = c.requests.find(key);
  return it == c.requests.end() ? 0 : it->second;
}

CudaUnitScheduler::CudaUnitScheduler(int policy, int max_nodes, int device, NodeProvider provider, int g_max, int c_max)
    : max_nodes_(max_nodes), g_max_(g_max), c_max_(c_max < EGS_MAX_CONTAINERS ? EGS_MAX_CONTAINERS : c_max),
      provider_(std::move(provider)) {
  if (egs_create_ex(policy, max_nodes, g_max, c_max, device, &h_) != EGS_OK) h_ = nullptr;
}

std::string CudaUnitScheduler::tooWide() const {
  return "libegs: pods with more than " + std::to_string(c_max_) + " containers are not supported by the device path";
}

// The GPU ids of container c's mask (EGS_MASK_BYTES(g_max) little-endian bytes at masks[c * EGS_MASK_BYTES]), joined.
std::string CudaUnitScheduler::gpuList(const uint8_t *masks, size_t c, const char *sep) const {
  const int nb = EGS_MASK_BYTES(g_max_);
  uint32_t m = 0;
  for (int b = 0; b < nb; b++) m |= (uint32_t)masks[c * nb + b] << (8 * b);
  std::string v;
  for (int g = 0; g < 8 * nb; g++) if (m >> g & 1) v += (v.empty() ? "" : sep) + std::to_string(g);
  return v;
}
CudaUnitScheduler::~CudaUnitScheduler() {
  if (h_) egs_destroy(h_);
}

bool CudaUnitScheduler::Handles(const Pod &pod) {
  for (const auto &c : pod.containers)
    if (c.requests.count(kResourceGPUCore) || c.requests.count(kResourceGPUMemory)) return true;
  return false;
}

// max_containers: c_max for the verbs that Trade (Assume / Score / Bind), EGS_MAX_CONTAINERS_APPLY for the
// ones that only account a pod somebody placed (AddPod / ForgetPod / replay)
bool CudaUnitScheduler::RequestOf(const Pod &pod, std::vector<egs_unit> *out, size_t max_containers) {
  out->clear();
  for (const auto &c : pod.containers) {
    egs_unit u;
    if (egs_unit_from_requests(requestOf(c, kResourceGPUCore), requestOf(c, kResourceGPUMemory), &u) != EGS_OK) return false;
    out->push_back(u);
  }
  return !out->empty() && out->size() <= max_containers;
}

std::string CudaUnitScheduler::RequestString(const std::vector<egs_unit> &req) {
  std::ostringstream os;
  for (const auto &u : req) os << "(core: " << u.core << ", memory: " << u.mem << ", gpu count: " << u.count << ")";
  return os.str();
}

// The pod UID crosses the C ABI as its 64-bit FNV-1a hash (as in integration/cuda_scheduler.go): no table that
// grows with every pod ever seen and needs cleaning on ForgetPod.
uint64_t CudaUnitScheduler::uidOf(const std::string &uid) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (unsigned char c : uid) { h ^= c; h *= 0x100000001b3ull; }
  return h;
}

void CudaUnitScheduler::optionFromPod(const Pod &pod, std::vector<int32_t> *off, std::vector<int32_t> *idx) {
  off->assign(1, 0);
  idx->clear();
  for (const auto &c : pod.containers) {
    auto it = pod.annotations.find(std::string(kAnnotationContainerPrefix) + c.name);
    if (it != pod.annotations.end()) {            // strings.Split(v, ",") + strconv.Atoi (errors -> 0)
      std::stringstream ss(it->second);
      std::string tok;
      if (it->second.empty()) idx->push_back(0);  // Split("") == [""] -> Atoi error -> 0
      while (std::getline(ss, tok, ',')) {
        char *end = nullptr;
        long v = std::strtol(tok.c_str(), &end, 10);
        idx->push_back((end && *end == '\0' && !tok.empty()) ? (int32_t)v : 0);
      }
    }
    off->push_back((int32_t)idx->size());
  }
  idx->push_back(0);
}

int CudaUnitScheduler::getNodeInfo(const std::string &name, std::string *err) {
  auto it = node_ids_.find(name);
  if (it != node_ids_.end()) return it->second;
  NodeInfo info;
  std::string e = provider_ ? provider_(name, &info) : std::string("no node provider");
  if (!e.empty()) { *err = e; return -1; }
  if ((int)node_names_.size() >= max_nodes_) { *err = "node cache full"; return -1; }
  const int id = (int)node_names_.size();
  int st = egs_node_set_allocatable(h_, id, info.core_allocatable, info.mem_allocatable);   // NewNodeAllocator node.go:23-59
  if (st == EGS_ERR_NO_GPU) { *err = "no gpu available on node " + name; return -1; }         // node.go:29
  if (st != EGS_OK) { *err = std::string("libegs: ") + egs_status_string(st); return -1; }
  node_names_.push_back(name);
  node_ids_.emplace(name, id);
  for (const auto &p : info.assumed_pods) {                                                    // node.go:52-54: na.Add(&pods[i], nil)
    std::vector<egs_unit> req;
    if (!RequestOf(p, &req, EGS_MAX_CONTAINERS_APPLY)) {   // not representable on the device path: say so, loudly -- the node's rows
      fprintf(stderr, "libegs: assumed pod %s/%s on node %s has more than %d containers (or an out-of-range request): "   // would
              "its GPU share is NOT subtracted from the node cache\n", p.ns.c_str(), p.name.c_str(), name.c_str(), EGS_MAX_CONTAINERS_APPLY);  // otherwise be silently wrong
      unsupported_.push_back(p.ns + "/" + p.name);
      continue;
    }
    std::vector<int32_t> off, idx;
    optionFromPod(p, &off, &idx);
    egs_node_replay_pod(h_, id, (int)req.size(), req.data(), off.data(), idx.data(), uidOf(p.uid));
  }
  return id;
}

std::string CudaUnitScheduler::Assume(const std::vector<std::string> &nodes, const Pod &pod,
                                      std::vector<std::string> *filtered, std::map<std::string, std::string> *failed) {
  filtered->clear();
  failed->clear();
  std::vector<egs_unit> req;
  if (!RequestOf(pod, &req, c_max_)) return tooWide();
  std::vector<int32_t> ids(nodes.size(), -1);
  std::vector<std::string> load_err(nodes.size());
  for (size_t i = 0; i < nodes.size(); i++) ids[i] = getNodeInfo(nodes[i], &load_err[i]);   // scheduler.go:119-127
  std::vector<uint8_t> fit(nodes.size() + 1, 0);
  int st = egs_filter(h_, (int)nodes.size(), ids.data(), (int)req.size(), req.data(), fit.data());
  if (st != EGS_OK) return std::string("libegs: ") + egs_status_string(st) + " " + egs_last_error(h_);
  for (size_t i = 0; i < nodes.size(); i++) {                                                 // scheduler.go:158-167
    if (fit[i]) filtered->push_back(nodes[i]);
    else if (ids[i] < 0) (*failed)[nodes[i]] = "elastic gpu scheduler get node failed: " + load_err[i];
    else (*failed)[nodes[i]] = egs_status_string(EGS_ERR_NOFIT);
  }
  return "";
}

std::vector<int64_t> CudaUnitScheduler::Score(const std::vector<std::string> &nodes, const Pod &pod) {
  std::vector<int64_t> out(nodes.size(), 0);
  std::vector<egs_unit> req;
  if (!RequestOf(pod, &req, c_max_)) return out;
  std::vector<int32_t> ids(nodes.size(), -1), sc(nodes.size() + 1, 0);
  std::string err;
  for (size_t i = 0; i < nodes.size(); i++) ids[i] = getNodeInfo(nodes[i], &err);            // error -> ScoreMin (scheduler.go:176-179)
  egs_score(h_, (int)nodes.size(), ids.data(), (int)req.size(), req.data(), sc.data());
  for (size_t i = 0; i < nodes.size(); i++) out[i] = sc[i];
  return out;
}

std::string CudaUnitScheduler::gpusJson(int node_id) {
  int32_t core[EGS_MAX_GPUS_WIDE], mem[EGS_MAX_GPUS_WIDE], gc = 0, mt = 0;   // EGS_ROW_WIDTH(g_max) cells used
  if (egs_state_dump(h_, node_id, 1, core, mem, &gc, &mt) != EGS_OK) return "[]";
  std::ostringstream os;
  os << "[";
  for (int g = 0; g < gc; g++)
    os << (g ? "," : "") << "{\"CoreAvailable\":" << core[g] << ",\"MemoryAvailable\":" << mem[g]
       << ",\"CoreTotal\":" << EGS_CORE_PER_GPU << ",\"MemoryTotal\":" << mt << "}";
  os << "]";
  return os.str();
}

std::string CudaUnitScheduler::Bind(const std::string &node, Pod *pod) {
  std::string err;
  int id = getNodeInfo(node, &err);
  if (id < 0) return err;                                                                     // scheduler.go:190-193
  std::vector<egs_unit> req;
  if (!RequestOf(*pod, &req, c_max_)) return tooWide();
  uint8_t masks[2 * EGS_MAX_CONTAINERS_APPLY] = {};            // room for EGS_MASKS_PER_POD <= 8 masks of EGS_MASK_BYTES <= 2
  // option text for the Transact error has to be read before the entry is consumed
  int32_t valid = 0, score = 0; uint8_t pm[2 * EGS_MAX_CONTAINERS_APPLY] = {};
  egs_option_peek(h_, id, (int)req.size(), req.data(), &valid, &score, pm);
  const std::string gpus_before = gpusJson(id);
  int st = egs_bind(h_, id, (int)req.size(), req.data(), uidOf(pod->uid), masks);
  if (st == EGS_ERR_NO_OPTION)                                                                // node.go:95
    return "cannot find option of GPU request " + RequestString(req) + " on " + gpus_before;
  if (st == EGS_ERR_TRANSACT) {                                                               // gpu.go:160,168
    std::ostringstream os;
    os << "can't trade option &{Request:" << RequestString(req) << " Allocated:[";
    for (size_t c = 0; c < req.size(); c++) {
      os << (c ? " " : "") << "[" << gpuList(pm, c, " ") << "]";
    }
    os << "] Score:" << score << "} on " << gpusJson(id) << " because the GPU's residual memory or core can't satisfy the container";
    return os.str();
  }
  if (st != EGS_OK) return std::string("libegs: ") + egs_status_string(st);
  // GetUpdatedPodAnnotationSpec pod.go:57-78
  for (size_t c = 0; c < pod->containers.size(); c++) {
    pod->annotations[std::string(kAnnotationContainerPrefix) + pod->containers[c].name] = gpuList(masks, c, ",");
  }
  pod->annotations[kEGPUAssumed] = "true";
  pod->labels[kEGPUAssumed] = "true";
  return "";                                   // Pods.Update / Pods.Bind stay in the Go host (scheduler.go:200-222)
}

std::string CudaUnitScheduler::AddPod(const Pod &pod) {
  if (pod.node_name.empty()) return "pod " + pod.ns + "/" + pod.name + " nodename is empty";  // scheduler.go:232-234
  std::string err;
  int id = getNodeInfo(pod.node_name, &err);
  if (id < 0) return err;
  std::vector<egs_unit> req;
  if (!RequestOf(pod, &req, EGS_MAX_CONTAINERS_APPLY)) {   // never drop silently: the caller (controller.go:330) logs the error
    unsupported_.push_back(pod.ns + "/" + pod.name);
    return "libegs: pod " + pod.ns + "/" + pod.name + " has more than 8 containers (or an out-of-range request): not accounted on the device path";
  }
  std::vector<int32_t> off, idx;
  optionFromPod(pod, &off, &idx);
  egs_pod_apply(h_, id, (int)req.size(), req.data(), off.data(), idx.data(), uidOf(pod.uid));  // error discarded, scheduler.go:242
  return "";
}

std::string CudaUnitScheduler::ForgetPod(const Pod &pod) {
  int id = -1;
  std::string err;
  if (!pod.node_name.empty()) {                                                                // scheduler.go:252-260
    id = getNodeInfo(pod.node_name, &err);
    if (id < 0) return err;
  }
  std::vector<egs_unit> req;
  std::vector<int32_t> off, idx;
  if (!RequestOf(pod, &req, EGS_MAX_CONTAINERS_APPLY)) { req.assign(1, egs_unit{-1, -1, 0}); off = {0, 0}; idx = {0}; }
  else optionFromPod(pod, &off, &idx);
  egs_pod_cancel(h_, id, (int)req.size(), req.data(), off.data(), idx.data(), uidOf(pod.uid));
  return "";
}

bool CudaUnitScheduler::KnownPod(const Pod &pod) { return egs_pod_known(h_, uidOf(pod.uid)) != 0; }
bool CudaUnitScheduler::ReleasedPod(const Pod &pod) { return egs_pod_released(h_, uidOf(pod.uid)) != 0; }

std::string CudaUnitScheduler::Status() {      // json.Marshal(map[string]GPUs): keys sorted (scheduler.go:283-290)
  std::map<std::string, int> sorted(node_ids_.begin(), node_ids_.end());
  std::ostringstream os;
  os << "{";
  bool first = true;
  for (const auto &kv : sorted) { os << (first ? "" : ",") << "\"" << kv.first << "\":" << gpusJson(kv.second); first = false; }
  os << "}";
  return os.str();
}

}  // namespace egs
