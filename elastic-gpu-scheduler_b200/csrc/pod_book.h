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
//
// Checkpoint: while one is open, every primitive change also pushes its inverse onto an undo journal, so that a
// rollback costs the changes made since the save, not the size of the book.  With none open the book does exactly
// what it did before, behind one branch per change.
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
        if (set_erase(pods_, NodeUid{node[p], uid0 + p})) f |= IN_PODS;
        if (set_erase(maps_, uid0 + p)) f |= IN_MAPS;
      }
      R.flags[p] = f; R.n_pods += (f & IN_PODS) != 0; R.n_maps += (f & IN_MAPS) != 0;
    }
    if (R.n_pods || R.n_maps) {
      runs_.push_back(std::move(R));
      if (journal_on_) log(Undo{U_RUN_ADD});
    }
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
      if (erase_pod_maps(uid)) set_insert(released_, uid);                  // scheduler.go:261-264
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
        if ((R.flags[i] & IN_PODS) && R.node[i] >= node0 && R.node[i] < node0 + n) {
          log_flags(r, i);
          R.flags[i] &= (uint8_t)~IN_PODS; R.n_pods--;
        }
      if (R.n_pods == 0 && R.n_maps == 0) erase_run(r);
    }
    for (auto it = pods_.begin(); it != pods_.end();)
      if (it->node >= node0 && it->node < node0 + n) {
        if (journal_on_) log(Undo{U_POD_ERA, 0, it->node, it->uid});
        it = pods_.erase(it);
      } else {
        ++it;
      }
  }

  void clear() {
    if (journal_on_) {                                  // the whole book moves into the journal: O(1)
      cleared_.push_back(Cleared{std::move(runs_), std::move(pods_), std::move(maps_), std::move(released_), hash_uid_max_});
      log(Undo{U_CLEAR});
    }
    runs_.clear(); pods_.clear(); maps_.clear(); released_.clear();
    hash_uid_max_ = 0;
  }

  // Checkpoint of the whole book.  checkpoint() opens one (replacing an open one); rollback() returns the book to it
  // by replaying the journal backwards and keeps it open; drop_checkpoint() closes it and keeps the current book.
  void checkpoint() { clear_journal(); journal_on_ = true; }
  void drop_checkpoint() { clear_journal(); journal_on_ = false; }
  void rollback() {
    for (size_t k = undo_.size(); k-- > 0;) {
      const Undo &u = undo_[k];
      switch (u.kind) {
        case U_POD_INS: pods_.erase(NodeUid{u.node, u.uid}); break;
        case U_POD_ERA: pods_.insert(NodeUid{u.node, u.uid}); break;
        case U_MAP_INS: maps_.erase(u.uid); break;
        case U_MAP_ERA: maps_.insert(u.uid); break;
        case U_REL_INS: released_.erase(u.uid); break;
        case U_REL_ERA: released_.insert(u.uid); break;
        case U_FLAGS: {
          Run &R = runs_[u.r];
          R.flags[u.i] = u.flags; R.n_pods = u.n_pods; R.n_maps = u.n_maps;
          break;
        }
        case U_RUN_ADD: runs_.pop_back(); break;
        case U_RUN_ERA:
          runs_.insert(runs_.begin() + (std::ptrdiff_t)u.r, std::move(dead_runs_.back()));
          dead_runs_.pop_back();
          break;
        case U_UID_MAX: hash_uid_max_ = u.uid; break;
        case U_CLEAR: {
          Cleared &c = cleared_.back();
          runs_ = std::move(c.runs); pods_ = std::move(c.pods); maps_ = std::move(c.maps);
          released_ = std::move(c.released); hash_uid_max_ = c.hash_uid_max;
          cleared_.pop_back();
          break;
        }
      }
    }
    clear_journal();
  }
  uint64_t hash_uid_max() const { return hash_uid_max_; }

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
    log_flags((size_t)h.r, h.i);
    R.flags[h.i] ^= bit;
    size_t &count = bit == IN_PODS ? R.n_pods : R.n_maps;
    if (on) count++; else count--;
    if (R.n_pods == 0 && R.n_maps == 0) erase_run((size_t)h.r);
    return true;
  }

  void insert_pods(int node, uint64_t uid) {
    const Home h = pods_home(node, uid);
    if (h.r >= 0) { set_bit(h, IN_PODS, true); return; }
    set_insert(pods_, NodeUid{node, uid}); raise_uid_max(uid);
  }
  bool erase_pods(int node, uint64_t uid) {
    const Home h = pods_home(node, uid);
    return h.r >= 0 ? set_bit(h, IN_PODS, false) : set_erase(pods_, NodeUid{node, uid});
  }
  void insert_pod_maps(uint64_t uid) {
    const Home h = maps_home(uid);
    if (h.r >= 0) { set_bit(h, IN_MAPS, true); return; }
    set_insert(maps_, uid); raise_uid_max(uid);
  }
  bool erase_pod_maps(uint64_t uid) {
    const Home h = maps_home(uid);
    return h.r >= 0 ? set_bit(h, IN_MAPS, false) : set_erase(maps_, uid);
  }

  // ---- the undo journal: each primitive change below pushes its inverse while a checkpoint is open
  enum UndoKind : uint8_t {
    U_POD_INS, U_POD_ERA, U_MAP_INS, U_MAP_ERA, U_REL_INS, U_REL_ERA,   // a set insert / erase
    U_FLAGS,                                                            // flags[i] of runs_[r], with n_pods / n_maps
    U_RUN_ADD,                                                          // add_run appended a run
    U_RUN_ERA,                                                          // runs_[r] emptied and was erased: dead_runs_
    U_UID_MAX,                                                          // hash_uid_max_ was `uid`
    U_CLEAR,                                                            // clear(): the containers are in cleared_
  };
  struct Undo {
    UndoKind kind; uint8_t flags = 0; int node = 0; uint64_t uid = 0;
    size_t r = 0, i = 0, n_pods = 0, n_maps = 0;
  };
  struct Cleared {
    std::vector<Run> runs; std::unordered_set<NodeUid, NodeUidHash> pods; std::unordered_set<uint64_t> maps, released;
    uint64_t hash_uid_max;
  };

  void log(const Undo &u) { undo_.push_back(u); }
  void log_flags(size_t r, size_t i) {
    if (!journal_on_) return;
    const Run &R = runs_[r];
    Undo u{U_FLAGS, R.flags[i]}; u.r = r; u.i = i; u.n_pods = R.n_pods; u.n_maps = R.n_maps;
    log(u);
  }
  void erase_run(size_t r) {
    if (journal_on_) {
      dead_runs_.push_back(std::move(runs_[r]));
      Undo u{U_RUN_ERA}; u.r = r;
      log(u);
    }
    runs_.erase(runs_.begin() + (std::ptrdiff_t)r);
  }
  void raise_uid_max(uint64_t uid) {
    if (uid <= hash_uid_max_) return;
    if (journal_on_) log(Undo{U_UID_MAX, 0, 0, hash_uid_max_});
    hash_uid_max_ = uid;
  }
  template <class S, class K>
  bool set_insert(S &s, const K &k) {
    if (!s.insert(k).second) return false;
    if (journal_on_) log(undo_for(s, k, true));
    return true;
  }
  template <class S, class K>
  bool set_erase(S &s, const K &k) {
    if (!s.erase(k)) return false;
    if (journal_on_) log(undo_for(s, k, false));
    return true;
  }
  Undo undo_for(const std::unordered_set<NodeUid, NodeUidHash> &, const NodeUid &k, bool ins) const {
    return Undo{ins ? U_POD_INS : U_POD_ERA, 0, k.node, k.uid};
  }
  Undo undo_for(const std::unordered_set<uint64_t> &s, uint64_t uid, bool ins) const {
    const bool rel = &s == &released_;
    return Undo{rel ? (ins ? U_REL_INS : U_REL_ERA) : (ins ? U_MAP_INS : U_MAP_ERA), 0, 0, uid};
  }
  void clear_journal() { undo_.clear(); dead_runs_.clear(); cleared_.clear(); }

  std::vector<Run> runs_;                               // sorted by uid0, disjoint
  std::unordered_set<NodeUid, NodeUidHash> pods_;       // podsMap keys with no home in a run
  std::unordered_set<uint64_t> maps_, released_;        // podMaps uids with no home in a run; releasedPodMap
  uint64_t hash_uid_max_ = 0;                           // no uid above it was ever put in pods_ or maps_
  bool journal_on_ = false;                             // a checkpoint is open
  std::vector<Undo> undo_;                              // inverses of the changes since it, oldest first
  std::vector<Run> dead_runs_;                          // runs erased since it (U_RUN_ERA), oldest first
  std::vector<Cleared> cleared_;                        // books emptied by clear() since it (U_CLEAR), oldest first
};
