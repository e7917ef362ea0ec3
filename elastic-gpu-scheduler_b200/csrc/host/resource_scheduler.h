// resource_scheduler.h -- C++ mirror of the reference's plugin interface for the hot path.
//
//   type ResourceScheduler interface { Assume; Score; Bind; AddPod; ForgetPod; KnownPod;
//                                      ReleasedPod; Status }          pkg/scheduler/scheduler.go:30-39
//
// CudaUnitScheduler is what a cgo `CudaUnitScheduler` registered in BuildResourceSchedulers
// (scheduler.go:292-321) would be: same method names, argument meaning and error texts as
// GPUUnitScheduler (scheduler.go:108-290), with the Filter/Score/Allocate arithmetic done by
// libegs (include/egs.h) on the GPU.  Kubernetes objects are reduced to the fields the path reads.
#pragma once
#include <cstdint>
#include <functional>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/egs.h"

namespace egs {

constexpr const char *kResourceGPUCore = "elasticgpu.io/gpu-core";       // elastic-gpu v1alpha1 (README.md:58-61)
constexpr const char *kResourceGPUMemory = "elasticgpu.io/gpu-memory";
constexpr const char *kEGPUAssumed = "elasticgpu.io/assumed";           // pkg/utils/types.go:8
constexpr const char *kAnnotationContainerPrefix = "elasticgpu.io/container-";  // pkg/utils/types.go:9

struct Container {                       // v1.Container: Name + Resources.Requests
  std::string name;
  std::map<std::string, int64_t> requests;   // already through resource.Quantity.Value() (pod.go:94-108)
};
struct Pod {                             // v1.Pod fields the path touches
  std::string ns, name, uid, node_name;
  std::vector<Container> containers;
  std::map<std::string, std::string> annotations, labels;
};
struct NodeInfo {                        // what getNodeInfo fetches on a cache miss (scheduler.go:62-84)
  int64_t core_allocatable = 0, mem_allocatable = 0;   // node.Status.Allocatable (node.go:24-27)
  std::vector<Pod> assumed_pods;                       // pods labelled elasticgpu.io/assumed=true on the node
};
// returns "" and fills `out`, or the apiserver error text
using NodeProvider = std::function<std::string(const std::string &name, NodeInfo *out)>;

class ResourceScheduler {                // scheduler.go:30-39 (errors are "" for nil)
 public:
  virtual ~ResourceScheduler() = default;
  virtual std::string Assume(const std::vector<std::string> &nodes, const Pod &pod,
                             std::vector<std::string> *filtered, std::map<std::string, std::string> *failed) = 0;
  virtual std::vector<int64_t> Score(const std::vector<std::string> &nodes, const Pod &pod) = 0;
  virtual std::string Bind(const std::string &node, Pod *pod) = 0;   // pod receives the annotations/label
  virtual std::string AddPod(const Pod &pod) = 0;
  virtual std::string ForgetPod(const Pod &pod) = 0;
  virtual bool KnownPod(const Pod &pod) = 0;
  virtual bool ReleasedPod(const Pod &pod) = 0;
  virtual std::string Status() = 0;
};

class CudaUnitScheduler : public ResourceScheduler {
 public:
  // policy: EGS_BINPACK / EGS_SPREAD (cmd/main.go:45-54); max_nodes bounds the dense node-id space; g_max is the widest
  // node (egs_create): EGS_MAX_GPUS, or up to EGS_MAX_GPUS_WIDE for servers with more GPUs
  CudaUnitScheduler(int policy, int max_nodes, int device, NodeProvider provider, int g_max = EGS_MAX_GPUS);
  ~CudaUnitScheduler() override;
  bool ok() const { return h_ != nullptr; }

  std::string Assume(const std::vector<std::string> &nodes, const Pod &pod, std::vector<std::string> *filtered,
                     std::map<std::string, std::string> *failed) override;
  std::vector<int64_t> Score(const std::vector<std::string> &nodes, const Pod &pod) override;
  std::string Bind(const std::string &node, Pod *pod) override;
  std::string AddPod(const Pod &pod) override;
  std::string ForgetPod(const Pod &pod) override;
  bool KnownPod(const Pod &pod) override;
  bool ReleasedPod(const Pod &pod) override;
  std::string Status() override;

  // GetResourceScheduler (scheduler.go:323-334): does any container request a managed resource?
  static bool Handles(const Pod &pod);
  // NewGPURequest (allocate.go:35-58)
  static bool RequestOf(const Pod &pod, std::vector<egs_unit> *out, size_t max_containers = EGS_MAX_CONTAINERS);
  // GPURequest.String (allocate.go:22-28)
  static std::string RequestString(const std::vector<egs_unit> &req);

 private:
  int getNodeInfo(const std::string &name, std::string *err);   // scheduler.go:62-84 -> dense id or -1
  static uint64_t uidOf(const std::string &uid);
  std::string gpusJson(int node_id);                            // GPUs.String (gpu.go:60-63)
  std::string gpuList(const uint8_t *masks, size_t c, const char *sep) const;   // GPU ids of container c's mask
  static void optionFromPod(const Pod &pod, std::vector<int32_t> *off, std::vector<int32_t> *idx);  // allocate.go:75-93

  egs_handle *h_ = nullptr;
  int max_nodes_;
  int g_max_;
  NodeProvider provider_;
  std::unordered_map<std::string, int> node_ids_;
  std::vector<std::string> node_names_;
  std::vector<std::string> unsupported_;          // pods the device path could not account (reported, never dropped silently)
};

}  // namespace egs
