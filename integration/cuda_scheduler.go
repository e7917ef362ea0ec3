// cuda_scheduler.go -- CudaUnitScheduler: the reference's ResourceScheduler plugin (pkg/scheduler/scheduler.go:30-39)
// backed by libegs, the H100 scheduler core (include/egs.h), through cgo.
//
// Drop this file into pkg/scheduler/ of elastic-ai/elastic-gpu-scheduler and add the case shown in
// BuildResourceSchedulersCuda (bottom of the file) to BuildResourceSchedulers (scheduler.go:292-321).
// The Docker build of the reference already sets CGO_ENABLED=1 and CGO_LDFLAGS_ALLOW (Dockerfile:4,12).
//
// What lives where:
//   - node rows (free core / memory per GPU), the per-node option cache `allocated` (node.go:19) and the per-node
//     podsMap (node.go:16) live in libegs, on the GPU;
//   - node-name -> dense id interning, BaseScheduler.podMaps / releasedPodMap (scheduler.go:47-49), the apiserver
//     calls of Bind and the pod annotations stay here, in Go, byte for byte the reference's own code;
//   - a pod UID crosses the C ABI as its 64-bit FNV-1a hash: no UID table to grow or to clean on ForgetPod.
//
// This toolchain-less repository cannot compile Go; the call sequence below is replayed against libegs.so by the C
// test double integration/shim_double.c (tests/test_shim_double.py) with the same C calls in the same order.
package scheduler

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -legs
#include <stdlib.h>
#include "egs.h"
// the layout macros of egs.h (cgo cannot expand function-like macros)
static int row_width(int g_max) { return EGS_ROW_WIDTH(g_max); }
static int mask_bytes(int g_max) { return EGS_MASK_BYTES(g_max); }
*/
import "C"

import (
	"context"
	"encoding/json"
	"fmt"
	"hash/fnv"
	"strconv"
	"strings"
	"unsafe"

	v1 "k8s.io/api/core/v1"
	metav1 "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/fields"
	"k8s.io/apimachinery/pkg/types"
	log "k8s.io/klog/v2"

	"elasticgpu.io/elastic-gpu/apis/elasticgpu/v1alpha1"

	schetypes "elasticgpu.io/elastic-gpu-scheduler/pkg/utils"
)

// CudaUnitScheduler implements ResourceScheduler.  BaseScheduler supplies the config, the single lock every verb
// takes (scheduler.go:113,171,187,230,248,270,277) and podMaps / releasedPodMap; nodeMaps is not used.
type CudaUnitScheduler struct {
	BaseScheduler
	h        *C.egs_handle
	nodeIDs  map[string]int32 // node name -> dense id (interning stays in Go, SURVEY 8b "Ownership")
	nodeName []string
	nodeErr  map[string]error // nodes whose NodeAllocator could not be built (node.go:28-30)
	maxNodes int
	gMax     int // widest node the handle takes (egs_create's g_max): rows and masks are laid out for it
}

// NewCudaUnitScheduler mirrors NewGPUUnitScheduler (scheduler.go:86-106): nodes that already carry assumed pods are
// loaded up front, every other node on first use.  gMax is the widest node of the cluster, C.EGS_MAX_GPUS for 8-GPU
// servers, up to C.EGS_MAX_GPUS_WIDE (a wide handle: 16-wide rows, two mask bytes per container, per-pod engine).
func NewCudaUnitScheduler(config ElasticSchedulerConfig, coreName v1.ResourceName, memName v1.ResourceName,
	maxNodes int, device int, gMax int) (ResourceScheduler, error) {
	policy := C.int(C.EGS_BINPACK)
	if _, ok := config.Rater.(*Spread); ok {
		policy = C.int(C.EGS_SPREAD)
	}
	d := &CudaUnitScheduler{
		BaseScheduler: newBaseScheduler(config, coreName, memName),
		nodeIDs:       map[string]int32{},
		nodeErr:       map[string]error{},
		maxNodes:      maxNodes,
		gMax:          gMax,
	}
	if st := C.egs_create(policy, C.int(maxNodes), C.int(gMax), C.int(device), &d.h); st != C.EGS_OK {
		return nil, fmt.Errorf("egs_create failed: status %d (no CUDA device?)", int(st))
	}
	pods, err := d.Clientset.CoreV1().Pods(metav1.NamespaceAll).List(context.Background(), metav1.ListOptions{
		LabelSelector: fmt.Sprintf("%s=%s", schetypes.EGPUAssumed, "true"),
	})
	if err != nil {
		return nil, err
	}
	for _, pod := range pods.Items {
		if pod.Spec.NodeName == "" {
			continue
		}
		if _, err := d.getNodeID(pod.Spec.NodeName); err != nil {
			log.Errorf("Failed to get node %s: %s", pod.Spec.NodeName, err.Error())
			continue
		}
	}
	return d, nil
}

// uidKey: the pod UID as it crosses the C ABI.
func uidKey(uid types.UID) C.uint64_t {
	f := fnv.New64a()
	_, _ = f.Write([]byte(uid))
	return C.uint64_t(f.Sum64())
}

// requestOf == NewGPURequest (allocate.go:35-58) through egs_unit_from_requests.
// maxContainers: EGS_MAX_CONTAINERS for the verbs that Trade (Assume / Score / Bind), EGS_MAX_CONTAINERS_APPLY for the
// ones that only account a pod somebody placed (AddPod / ForgetPod / replay at node load).
func (d *CudaUnitScheduler) requestOf(pod *v1.Pod, maxContainers int) ([]C.egs_unit, error) {
	if len(pod.Spec.Containers) > maxContainers {
		return nil, fmt.Errorf("pod %s/%s: more than %d containers are not handled by the device path", pod.Namespace, pod.Name, maxContainers)
	}
	units := make([]C.egs_unit, len(pod.Spec.Containers))
	for i := range pod.Spec.Containers {
		c := &pod.Spec.Containers[i]
		core := GetGPUCoreFromContainer(c, d.coreName)
		mem := GetGPUMemoryFromContainer(c, d.memName)
		if st := C.egs_unit_from_requests(C.int64_t(core), C.int64_t(mem), &units[i]); st != C.EGS_OK {
			return nil, fmt.Errorf("pod %s/%s container %s: %s", pod.Namespace, pod.Name, c.Name, C.GoString(C.egs_status_string(st)))
		}
	}
	return units, nil
}

// allocFromAnnotations == NewGPUOptionFromPod (allocate.go:75-93): Atoi errors read as 0.
func allocFromAnnotations(pod *v1.Pod) (off []C.int32_t, idx []C.int32_t) {
	off = make([]C.int32_t, len(pod.Spec.Containers)+1)
	for i, c := range pod.Spec.Containers {
		if v, ok := pod.Annotations[fmt.Sprintf(schetypes.AnnotationEGPUContainer, c.Name)]; ok {
			for _, s := range strings.Split(v, ",") {
				id, _ := strconv.Atoi(s)
				idx = append(idx, C.int32_t(id))
			}
		}
		off[i+1] = C.int32_t(len(idx))
	}
	if len(idx) == 0 {
		idx = []C.int32_t{0}
	}
	return off, idx
}

// getNodeID == getNodeInfo (scheduler.go:62-84): first use loads the node (NewNodeAllocator, node.go:23-59) and
// replays the pods already assumed on it (node.go:52-54).
func (d *CudaUnitScheduler) getNodeID(name string) (int32, error) {
	if id, ok := d.nodeIDs[name]; ok {
		return id, nil
	}
	node, err := d.Clientset.CoreV1().Nodes().Get(context.TODO(), name, metav1.GetOptions{})
	if err != nil {
		return -1, err
	}
	pods, err := d.Clientset.CoreV1().Pods(metav1.NamespaceAll).List(context.Background(), metav1.ListOptions{
		LabelSelector: fmt.Sprintf("%s=%s", schetypes.EGPUAssumed, "true"),
		FieldSelector: fields.OneTermEqualSelector(schetypes.NodeNameField, name).String(),
	})
	if err != nil {
		return -1, err
	}
	if len(d.nodeName) >= d.maxNodes {
		return -1, fmt.Errorf("node table full (%d nodes)", d.maxNodes)
	}
	id := int32(len(d.nodeName))
	coreAvail := node.Status.Allocatable[d.coreName]
	memAvail := node.Status.Allocatable[d.memName]
	st := C.egs_node_set_allocatable(d.h, C.int(id), C.int64_t(coreAvail.Value()), C.int64_t(memAvail.Value()))
	if st == C.EGS_ERR_NO_GPU {
		return -1, fmt.Errorf("no gpu available on node %s", name) // node.go:29
	}
	if st != C.EGS_OK {
		return -1, fmt.Errorf("node %s: %s", name, C.GoString(C.egs_status_string(st)))
	}
	d.nodeIDs[name] = id
	d.nodeName = append(d.nodeName, name)
	for i := range pods.Items {
		pod := &pods.Items[i]
		units, err := d.requestOf(pod, C.EGS_MAX_CONTAINERS_APPLY)
		if err != nil {
			log.Errorf("replay of pod %s/%s on node %s skipped: %v", pod.Namespace, pod.Name, name, err)
			continue
		}
		off, idx := allocFromAnnotations(pod)
		C.egs_node_replay_pod(d.h, C.int(id), C.int(len(units)), &units[0], &off[0], &idx[0], uidKey(pod.UID))
	}
	return id, nil
}

// Assume (scheduler.go:112-168): filteredNodes in input order, failedNodes[name] = per-node message.
func (d *CudaUnitScheduler) Assume(nodes []string, pod *v1.Pod) ([]string, map[string]string, error) {
	d.lock.Lock()
	defer d.lock.Unlock()
	filteredNodes := []string{}
	failedNodes := map[string]string{}
	units, err := d.requestOf(pod, C.EGS_MAX_CONTAINERS)
	if err != nil {
		return nil, nil, err
	}
	ids := make([]C.int32_t, 0, len(nodes))
	pos := make([]int, 0, len(nodes))
	res := make([]string, len(nodes))
	fit := make([]bool, len(nodes))
	for i, name := range nodes {
		id, err := d.getNodeID(name)
		if err != nil {
			res[i] = fmt.Sprintf("elastic gpu scheduler get node failed: %v", err) // scheduler.go:124
			continue
		}
		ids = append(ids, C.int32_t(id))
		pos = append(pos, i)
	}
	if len(ids) > 0 {
		out := make([]C.uint8_t, len(ids))
		if st := C.egs_filter(d.h, C.int(len(ids)), &ids[0], C.int(len(units)), &units[0], &out[0]); st != C.EGS_OK {
			return nil, nil, fmt.Errorf("egs_filter: %s", C.GoString(C.egs_last_error(d.h)))
		}
		for k, i := range pos {
			fit[i] = out[k] != 0
			if !fit[i] {
				res[i] = C.GoString(C.egs_status_string(C.EGS_ERR_NOFIT)) // "no enough resource to allocate", gpu.go:126
			}
		}
	}
	for i, name := range nodes {
		if fit[i] {
			filteredNodes = append(filteredNodes, name)
		} else {
			failedNodes[name] = res[i]
		}
	}
	return filteredNodes, failedNodes, nil
}

// Score (scheduler.go:170-184): cached option.Score per node; a node that cannot be loaded scores ScoreMin.
func (d *CudaUnitScheduler) Score(nodes []string, pod *v1.Pod) []int {
	d.lock.Lock()
	defer d.lock.Unlock()
	scores := make([]int, len(nodes))
	units, err := d.requestOf(pod, C.EGS_MAX_CONTAINERS)
	if err != nil {
		return scores
	}
	ids := make([]C.int32_t, 0, len(nodes))
	pos := make([]int, 0, len(nodes))
	for i, name := range nodes {
		id, err := d.getNodeID(name)
		if err != nil {
			log.Errorf("Fail to score pod %s/%s because not found target node %s: %s", pod.Namespace, pod.Name, name, err.Error())
			scores[i] = ScoreMin
			continue
		}
		ids = append(ids, C.int32_t(id))
		pos = append(pos, i)
	}
	if len(ids) == 0 {
		return scores
	}
	out := make([]C.int32_t, len(ids))
	st := C.egs_score(d.h, C.int(len(ids)), &ids[0], C.int(len(units)), &units[0], &out[0])
	if st == C.EGS_ERR_PANIC {
		// node.go:84 dereferences a nil option when Score runs on a node Assume never saw and the request fits
		panic("runtime error: invalid memory address or nil pointer dereference (NodeAllocator.Score, node.go:84)")
	}
	for k, i := range pos {
		scores[i] = int(out[k])
	}
	return scores
}

// maskToIDs decodes container c's GPU mask: EGS_MASK_BYTES(gMax) little-endian bytes at masks[c*EGS_MASK_BYTES].
func (d *CudaUnitScheduler) maskToIDs(masks []C.uint8_t, c int) []int {
	nb := int(C.mask_bytes(C.int(d.gMax)))
	mask := 0
	for b := 0; b < nb; b++ {
		mask |= int(masks[c*nb+b]) << uint(8*b)
	}
	ids := []int{}
	for g := 0; g < 8*nb; g++ {
		if (mask>>uint(g))&1 != 0 {
			ids = append(ids, g)
		}
	}
	return ids
}

// Bind (scheduler.go:186-227): Allocate on the node, annotate, Update (+ one retry on the optimistic-lock error),
// Bind, then podMaps.
func (d *CudaUnitScheduler) Bind(node string, pod *v1.Pod) (err error) {
	d.lock.Lock()
	defer d.lock.Unlock()
	id, err := d.getNodeID(node)
	if err != nil {
		return err
	}
	units, err := d.requestOf(pod, C.EGS_MAX_CONTAINERS)
	if err != nil {
		return err
	}
	var masks [2 * C.EGS_MAX_CONTAINERS]C.uint8_t // room for EGS_MASK_BYTES <= 2
	switch st := C.egs_bind(d.h, C.int(id), C.int(len(units)), &units[0], uidKey(pod.UID), &masks[0]); st {
	case C.EGS_OK:
	case C.EGS_ERR_NO_OPTION:
		return fmt.Errorf("cannot find option of GPU request %+v on node %s", NewGPURequest(pod, d.coreName, d.memName), node) // node.go:95
	case C.EGS_ERR_TRANSACT:
		return fmt.Errorf("can't trade option of pod %s/%s on node %s because the GPU's residual memory or core can't satisfy the container", pod.Namespace, pod.Name, node) // gpu.go:160,168
	default:
		return fmt.Errorf("egs_bind: %s", C.GoString(C.egs_last_error(d.h)))
	}
	ids := make([][]int, len(units))
	for i := range units {
		ids[i] = d.maskToIDs(masks[:], i)
	}
	newPod := GetUpdatedPodAnnotationSpec(pod, ids) // pod.go:57-78
	if _, err := d.Clientset.CoreV1().Pods(newPod.Namespace).Update(context.Background(), newPod, metav1.UpdateOptions{}); err != nil {
		if err.Error() == schetypes.OptimisticLockErrorMsg {
			pod, err = d.Clientset.CoreV1().Pods(pod.Namespace).Get(context.Background(), pod.Name, metav1.GetOptions{})
			if err != nil {
				return err
			}
			newPod = GetUpdatedPodAnnotationSpec(pod, ids)
			if _, err = d.Clientset.CoreV1().Pods(pod.Namespace).Update(context.Background(), newPod, metav1.UpdateOptions{}); err != nil {
				return err
			}
		} else {
			return nil
		}
	}
	if err := d.Clientset.CoreV1().Pods(newPod.Namespace).Bind(context.Background(), &v1.Binding{
		ObjectMeta: metav1.ObjectMeta{Namespace: newPod.Namespace, Name: newPod.Name, UID: newPod.UID},
		Target:     v1.ObjectReference{Kind: "Node", Name: node},
	}, metav1.CreateOptions{}); err != nil {
		return err
	}
	d.podMaps[pod.UID] = newPod
	return nil
}

// AddPod (scheduler.go:229-245).
func (d *CudaUnitScheduler) AddPod(pod *v1.Pod) error {
	d.lock.Lock()
	defer d.lock.Unlock()
	if pod.Spec.NodeName == "" {
		return fmt.Errorf("pod %s/%s nodename is empty", pod.Namespace, pod.Name)
	}
	id, err := d.getNodeID(pod.Spec.NodeName)
	if err != nil {
		return err
	}
	if _, ok := d.podMaps[pod.UID]; ok {
		return nil
	}
	units, err := d.requestOf(pod, C.EGS_MAX_CONTAINERS_APPLY)
	if err != nil {
		return err
	}
	off, idx := allocFromAnnotations(pod)
	// ni.Add(pod, nil): node-level podsMap + Transact of the option rebuilt from the annotations (node.go:148-160)
	C.egs_node_replay_pod(d.h, C.int(id), C.int(len(units)), &units[0], &off[0], &idx[0], uidKey(pod.UID))
	d.podMaps[pod.UID] = pod
	return nil
}

// ForgetPod (scheduler.go:247-267).
func (d *CudaUnitScheduler) ForgetPod(pod *v1.Pod) error {
	d.lock.Lock()
	defer d.lock.Unlock()
	if pod.Spec.NodeName != "" {
		id, err := d.getNodeID(pod.Spec.NodeName)
		if err != nil {
			return err
		}
		units, err := d.requestOf(pod, C.EGS_MAX_CONTAINERS_APPLY)
		if err != nil {
			return err
		}
		off, idx := allocFromAnnotations(pod)
		// ni.Forget(pod): only if the UID is in that node's podsMap -- libegs checks it (node.go:131)
		C.egs_pod_cancel(d.h, C.int(id), C.int(len(units)), &units[0], &off[0], &idx[0], uidKey(pod.UID))
	}
	if _, ok := d.podMaps[pod.UID]; ok {
		delete(d.podMaps, pod.UID)
		d.releasedPodMap[pod.UID] = struct{}{}
	}
	return nil
}

// KnownPod (scheduler.go:269-274).
func (d *CudaUnitScheduler) KnownPod(pod *v1.Pod) bool {
	d.lock.Lock()
	defer d.lock.Unlock()
	_, ok := d.podMaps[pod.UID]
	return ok
}

// ReleasedPod (scheduler.go:276-281).
func (d *CudaUnitScheduler) ReleasedPod(pod *v1.Pod) bool {
	d.lock.Lock()
	defer d.lock.Unlock()
	_, ok := d.releasedPodMap[pod.UID]
	return ok
}

// Status (scheduler.go:283-290): {"<node>": [{"CoreAvailable":..,"MemoryAvailable":..,"CoreTotal":..,"MemoryTotal":..}, ..]}.
func (d *CudaUnitScheduler) Status() string {
	n := len(d.nodeName)
	gpus := make(map[string]GPUs, n)
	if n == 0 {
		result, _ := json.Marshal(gpus)
		return string(result)
	}
	g := int(C.row_width(C.int(d.gMax)))
	core := make([]C.int32_t, n*g)
	mem := make([]C.int32_t, n*g)
	cnt := make([]C.int32_t, n)
	tot := make([]C.int32_t, n)
	if st := C.egs_state_dump(d.h, 0, C.int(n), &core[0], &mem[0], &cnt[0], &tot[0]); st != C.EGS_OK {
		return "{}"
	}
	for i, name := range d.nodeName {
		row := make(GPUs, int(cnt[i]))
		for k := range row {
			row[k] = &GPU{CoreAvailable: int(core[i*g+k]), MemoryAvailable: int(mem[i*g+k]),
				CoreTotal: schetypes.GPUCoreEachCard, MemoryTotal: int(tot[i])}
		}
		gpus[name] = row
	}
	result, _ := json.Marshal(gpus)
	return string(result)
}

// Close releases the device state (the reference has no shutdown hook; call it from main's signal handler).
func (d *CudaUnitScheduler) Close() {
	d.lock.Lock()
	defer d.lock.Unlock()
	if d.h != nil {
		C.egs_destroy(d.h)
		d.h = nil
	}
}

var _ = unsafe.Pointer(nil)

// BuildResourceSchedulersCuda is BuildResourceSchedulers (scheduler.go:292-321) with one more mode: "gpushare-cuda"
// registers the same CudaUnitScheduler instance under both resource names, exactly as "gpushare" does with the
// GPUUnitScheduler.  In the reference tree add this case to the existing switch instead of calling this function.
func BuildResourceSchedulersCuda(modes []string, config ElasticSchedulerConfig) (map[v1.ResourceName]ResourceScheduler, error) {
	sches, err := BuildResourceSchedulers(modes, config)
	if err != nil {
		return nil, err
	}
	for _, m := range modes {
		switch m {
		case "gpushare-cuda":
			d, err := NewCudaUnitScheduler(config, v1alpha1.ResourceGPUCore, v1alpha1.ResourceGPUMemory, 1<<20, 0, int(C.EGS_MAX_GPUS))
			if err != nil {
				return nil, err
			}
			sches[v1alpha1.ResourceGPUCore] = d
			sches[v1alpha1.ResourceGPUMemory] = d
		}
	}
	return sches, nil
}
