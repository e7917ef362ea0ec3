// pod_book.h -- the reference's UID bookkeeping, which never reaches the device: NodeAllocator.podsMap (node.go:16)
// and BaseScheduler.podMaps / releasedPodMap (scheduler.go:47-49).  Host-only C++17; the CPU test suite runs it
// through csrc/host_test/pod_book_on_host.cc (tests/test_pod_book_host.py).
//
// Every key has exactly one home, so an insert, an erase and a query all go to the same place:
//  * A batch with library-assigned uids [uid0, uid0+n) becomes a Run: each pod's winning node and a flags byte.  A
//    uid inside a run has its podMaps home in the run's IN_MAPS bit; the key (node, uid) has its podsMap home in the
//    run's IN_PODS bit when node is the pod's winning node there.  A million-pod batch costs 5 B per pod and no hash
//    insert.
//  * Every other key lives in the hash sets.
// A run whose bits are all clear holds no key and is dropped.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <unordered_set>
#include <vector>

#include "../../include/egs.h"

class PodBook {
 public:
  // One finished batch of library-assigned uids [uid0, uid0+n): a pod with node >= 0 entered the node's podsMap
  // before its Transact (node.go:150), and also podMaps when it bound (scheduler.go:224).  uid0 is past every
  // earlier run.
  void add_run(uint64_t uid0, int n, const int32_t *node, const int32_t *status) {
    Run R;
    R.uid0 = uid0; R.node.assign(node, node + n); R.flags.resize((size_t)n);
    const bool absorb = hash_uid_max_ >= uid0;          // a caller already used one of these uids: move its keys here
    for (int p = 0; p < n; p++) {
      uint8_t f = node[p] >= 0 ? (uint8_t)(IN_PODS | (status[p] == EGS_OK ? IN_MAPS : 0)) : 0;
      if (absorb) {
        if (pods_.erase(NodeUid{node[p], uid0 + p})) f |= IN_PODS;
        if (maps_.erase(uid0 + p)) f |= IN_MAPS;
      }
      R.flags[p] = f; R.n_pods += (f & IN_PODS) != 0; R.n_maps += (f & IN_MAPS) != 0;
    }
    if (R.n_pods || R.n_maps) runs_.push_back(std::move(R));
  }
  // the same for a batch with caller-given uids
  void add_batch(const uint64_t *uids, int n, const int32_t *node, const int32_t *status) {
    for (int p = 0; p < n; p++)
      if (node[p] >= 0) {
        insert_pods(node[p], uids[p]);                                      // node.go:150
        if (status[p] == EGS_OK) insert_pod_maps(uids[p]);                  // scheduler.go:224
      }
  }

  bool in_pods_map(int node, uint64_t uid) const {
    const Home h = pods_home(node, uid);
    return h.r >= 0 ? (runs_[(size_t)h.r].flags[h.i] & IN_PODS) != 0 : pods_.count(NodeUid{node, uid}) != 0;
  }
  bool in_pod_maps(uint64_t uid) const {
    const Home h = maps_home(uid);
    return h.r >= 0 ? (runs_[(size_t)h.r].flags[h.i] & IN_MAPS) != 0 : maps_.count(uid) != 0;
  }
  bool released(uint64_t uid) const { return released_.count(uid) != 0; }

  // The end of Bind: Allocate put the pod in the node's podsMap when it found an option, before Transact
  // (node.go:150), unless the pod was `known` there already; a bind that succeeded puts it in podMaps
  // (scheduler.go:224).
  void record_bind(int node, uint64_t uid, bool had_entry, bool known, int status) {
    if (had_entry && !known) insert_pods(node, uid);
    if (status == EGS_OK) insert_pod_maps(uid);
  }

  // The podsMap / podMaps decision of one EGS_MUT_* record on `node`, in the reference's order.  apply(cancel) makes
  // the row update the reference would make, before the bookkeeping that follows it; a failing apply ends the record.
  // The single verbs validate a pod's index lists inside apply, i.e. only when the record reaches a row update, which
  // is when the reference parses the annotations: a known uid with a malformed list is EGS_OK there.  The mutation
  // stream validates every record's lists before it applies any, so the same record fails the whole stream.
  template <class F>
  int account(int kind, int node, uint64_t uid, F &&apply) {
    if (kind == EGS_MUT_FORGET) {                                           // ForgetPod scheduler.go:247-267
      if (node >= 0 && in_pods_map(node, uid)) {                            // node.go:131
        const int rc = apply(1);
        if (rc != EGS_OK) return rc;
        erase_pods(node, uid);
      }
      if (erase_pod_maps(uid)) released_.insert(uid);                       // scheduler.go:261-264
      return EGS_OK;
    }
    if (kind == EGS_MUT_ADD && in_pod_maps(uid)) return EGS_OK;            // scheduler.go:239-241
    if (!in_pods_map(node, uid)) {                                          // node.go:149
      const int rc = apply(0);
      if (rc != EGS_OK) return rc;
      insert_pods(node, uid);
    }
    if (kind == EGS_MUT_ADD) insert_pod_maps(uid);                          // scheduler.go:243
    return EGS_OK;
  }

  // podsMap entries of nodes [node0, node0+n) vanish with their NodeAllocator (node.go:42-50); podMaps, held by
  // the scheduler, survives
  void drop_nodes(int node0, int n) {
    for (size_t r = runs_.size(); r-- > 0;) {
      Run &R = runs_[r];
      if (R.n_pods == 0) continue;
      for (size_t i = 0; i < R.node.size(); i++)
        if ((R.flags[i] & IN_PODS) && R.node[i] >= node0 && R.node[i] < node0 + n) { R.flags[i] &= (uint8_t)~IN_PODS; R.n_pods--; }
      if (R.n_pods == 0 && R.n_maps == 0) runs_.erase(runs_.begin() + (std::ptrdiff_t)r);
    }
    for (auto it = pods_.begin(); it != pods_.end();)
      if (it->node >= node0 && it->node < node0 + n) it = pods_.erase(it); else ++it;
  }

  void clear() {
    runs_.clear(); pods_.clear(); maps_.clear(); released_.clear();
    hash_uid_max_ = 0;
  }

 private:
  enum : uint8_t { IN_PODS = 1, IN_MAPS = 2 };
  struct Run {
    uint64_t uid0 = 0;
    std::vector<int32_t> node;          // winning node of pod uid0 + i, -1 when none
    std::vector<uint8_t> flags;         // IN_PODS: (node[i], uid) is in podsMap; IN_MAPS: uid is in podMaps
    size_t n_pods = 0, n_maps = 0;      // set bits of each kind
  };
  struct NodeUid {
    int node; uint64_t uid;
    bool operator==(const NodeUid &o) const { return node == o.node && uid == o.uid; }
  };
  struct NodeUidHash {
    size_t operator()(const NodeUid &k) const { return std::hash<uint64_t>()(k.uid ^ ((uint64_t)(uint32_t)k.node << 40)); }
  };
  struct Home { int r; size_t i; };     // pod i of runs_[r]; r < 0: the hash set

  Home maps_home(uint64_t uid) const {
    auto it = std::upper_bound(runs_.begin(), runs_.end(), uid, [](uint64_t u, const Run &R) { return u < R.uid0; });
    if (it == runs_.begin()) return Home{-1, 0};
    --it;
    if (uid - it->uid0 >= it->node.size()) return Home{-1, 0};
    return Home{(int)(it - runs_.begin()), (size_t)(uid - it->uid0)};
  }
  Home pods_home(int node, uint64_t uid) const {
    const Home h = maps_home(uid);
    return h.r >= 0 && runs_[(size_t)h.r].node[h.i] == node ? h : Home{-1, 0};
  }
  // sets or clears `bit` of a pod in a run; false when it already had that value
  bool set_bit(Home h, uint8_t bit, bool on) {
    Run &R = runs_[(size_t)h.r];
    if (((R.flags[h.i] & bit) != 0) == on) return false;
    R.flags[h.i] ^= bit;
    size_t &count = bit == IN_PODS ? R.n_pods : R.n_maps;
    if (on) count++; else count--;
    if (R.n_pods == 0 && R.n_maps == 0) runs_.erase(runs_.begin() + h.r);
    return true;
  }

  void insert_pods(int node, uint64_t uid) {
    const Home h = pods_home(node, uid);
    if (h.r >= 0) { set_bit(h, IN_PODS, true); return; }
    pods_.insert(NodeUid{node, uid}); hash_uid_max_ = std::max(hash_uid_max_, uid);
  }
  bool erase_pods(int node, uint64_t uid) {
    const Home h = pods_home(node, uid);
    return h.r >= 0 ? set_bit(h, IN_PODS, false) : pods_.erase(NodeUid{node, uid}) != 0;
  }
  void insert_pod_maps(uint64_t uid) {
    const Home h = maps_home(uid);
    if (h.r >= 0) { set_bit(h, IN_MAPS, true); return; }
    maps_.insert(uid); hash_uid_max_ = std::max(hash_uid_max_, uid);
  }
  bool erase_pod_maps(uint64_t uid) {
    const Home h = maps_home(uid);
    return h.r >= 0 ? set_bit(h, IN_MAPS, false) : maps_.erase(uid) != 0;
  }

  std::vector<Run> runs_;                               // sorted by uid0, disjoint
  std::unordered_set<NodeUid, NodeUidHash> pods_;       // podsMap keys with no home in a run
  std::unordered_set<uint64_t> maps_, released_;        // podMaps uids with no home in a run; releasedPodMap
  uint64_t hash_uid_max_ = 0;                           // no uid above it was ever put in pods_ or maps_
};
