"""The rounds model (tests/rounds_model.py) with k_resolve_mw's PRE-INSTALL (csrc/egs_rounds.cuh, DESIGN.md §3.1).

Before a round's first pod the resolver tracks the round's likely winners: for rank r = 0 .. pre_h-1 and each shape
of the round set in order, the entry of merged rank r over the shape's shard lists, skipping nodes already chosen,
until pre_cap (< T) nodes.  Nothing is observed yet, so their NEW options stay NEW.  Installing a node early changes
no output -- the winner rule max(best tracked option, best untracked head) does not depend on which nodes are
tracked -- only where the rounds end.  `schedule_batch` below is RoundsModel.schedule_batch with that step added
(and the install of a node factored into `track`); with pre_h = 0 it is RoundsModel, which
tests/test_rounds_preinstall.py checks output for output.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import egs_oracle as po
from rounds_model import ABSENT, CACHED, MASK64, NEW, UNFIT, RoundsModel, fit_term, monotone, score_term


class PreinstallRoundsModel(RoundsModel):
    def __init__(self, policy: int, K: int = 32, T: int = 256, RS: int = 32, shards: int = 1, pre_h: int = 0,
                 pre_cap: Optional[int] = None):
        super().__init__(policy, K=K, T=T, RS=RS, shards=shards)
        self.pre_h, self.pre_cap = pre_h, min(T - 1 if pre_cap is None else pre_cap, T - 1)
        self.stats["pre"] = 0

    def schedule_batch(self, pods: Sequence[tuple]):
        out = []
        p0, P = 0, len(pods)
        N = len(self.nodes)
        bounds = [N * d // self.D for d in range(self.D + 1)]
        while p0 < P:
            # round set: distinct shapes in pod order
            shapes: List[tuple] = []
            plim = p0
            while plim < P:
                s = pods[plim]
                if s not in shapes:
                    if len(shapes) == self.RS:
                        break
                    shapes.append(s)
                plim += 1
            for s in shapes:
                self._table(s)
            mono = monotone(shapes)
            # ---- k_select per shard: evaluate ABSENT, convert NEW when observed since, aggregates, top-K
            lists = {s: [] for s in shapes}                      # per shape: per shard (keys, more)
            agg = {}
            for s in shapes:
                tab = self.tables[s]
                pend = self.obs_pending[s]
                fit, fd, sd = 0, 0, 0
                for d in range(self.D):
                    keys = []
                    for i in range(bounds[d], bounds[d + 1]):
                        e = tab[i]
                        if e.st == NEW and pend:
                            e.st = CACHED
                        if e.st == ABSENT:
                            opt = self._trade(self.nodes[i], s)
                            if opt is None:
                                e.st = UNFIT
                            else:
                                e.st, e.score, e.alloc = NEW, opt.score, opt.allocated
                        if e.st in (CACHED, NEW):
                            keys.append((-e.score, i))
                            fit += 1
                            fd = (fd + fit_term(i)) & MASK64
                            sd = (sd + score_term(i, e.score)) & MASK64
                    keys.sort()
                    lists[s].append((keys[:self.K], len(keys) > self.K))
                agg[s] = [fit, fd, sd]
                self.obs_pending[s] = False                       # consumed by this select (k_merge)
            # ---- k_resolve
            self.stats["rounds"] += 1
            tracked: Dict[int, dict] = {}                         # node -> {shape: [st, score, alloc]}, rows live in self.nodes copy
            rows_copy: Dict[int, List[po.GPU]] = {}
            dirty = set()
            observed = {s: False for s in shapes}
            cur = {s: [0] * self.D for s in shapes}

            def track(w):                                         # node w becomes tracked with its current options
                rows_copy[w] = self.nodes[w]                      # (the model mutates the node rows in place)
                ent = {}
                for s2 in shapes:
                    e = self.tables[s2][w]
                    st = e.st
                    if st == NEW and observed[s2]:
                        st = CACHED
                    ent[s2] = [st, e.score, e.alloc]
                tracked[w] = ent

            if self.pre_h > 0:                                    # nothing is observed yet: NEW options stay NEW
                merged = {s: sorted(k for keys, _ in lists[s] for k in keys) for s in shapes}
                for r in range(self.pre_h):
                    for s in shapes:
                        if len(tracked) < self.pre_cap and r < len(merged[s]) and merged[s][r][1] not in tracked:
                            track(merged[s][r][1])
                self.stats["pre"] += len(tracked)
            done = 0
            p = p0
            while p < plim:
                s = pods[p]
                if s not in lists:
                    self.stats["shape"] += 1
                    break
                pend = [n_ for n_, ent in tracked.items() if ent[s][0] == ABSENT]
                # device: k_resolve_mw's fast pod -- monotone round, single fractional container, every shape of the
                # round observed, at most one pending option (pu != -2); everything else goes through general_pod
                fast = (mono and len(s) == 1 and s[0][2] == 0 and s[0][0] >= 0 and s[0][1] >= 0
                        and all(observed.values()) and len(pend) <= 1)
                if not fast and len(tracked) >= self.T:           # general_pod: no free slot for a possible new winner
                    self.stats["full"] += 1
                    break
                # exact heads of the untracked candidate lists (entries that became tracked are skipped) and dbound =
                # the best last key of an exhausted TRUNCATED list: what such a list did not show is worse than that
                heads, dbound = [], None
                for d in range(self.D):
                    keys, more = lists[s][d]
                    c = cur[s][d]
                    while c < len(keys) and keys[c][1] in tracked:
                        c += 1
                    cur[s][d] = c
                    if c < len(keys):
                        heads.append(keys[c])
                    elif more and keys:
                        dbound = keys[-1] if dbound is None else min(dbound, keys[-1])
                if not fast and not observed[s]:
                    for n_, ent in tracked.items():
                        if ent[s][0] == NEW:
                            ent[s][0] = CACHED
                    observed[s] = True
                # this pod's filter Trades the absent options of tracked nodes.  general_pod records the results before
                # it decides whether the round goes on (the next round's first filter would do the same Trades on the
                # same rows); the fast pod Trades speculatively and records after the decision.
                traded = [(n_, self._trade(rows_copy[n_], s)) for n_ in pend]

                def record():
                    for n_, opt in traded:
                        e = tracked[n_][s]
                        if opt is None:
                            e[0] = UNFIT
                        else:
                            e[0], e[1], e[2] = CACHED, opt.score, opt.allocated
                            agg[s][0] += 1
                            agg[s][1] = (agg[s][1] + fit_term(n_)) & MASK64
                            agg[s][2] = (agg[s][2] + score_term(n_, opt.score)) & MASK64
                if not fast:
                    record()
                    traded_c = []
                else:
                    traded_c = [(-opt.score, n_) for n_, opt in traded if opt is not None]
                cands = [(-ent[s][1], n_) for n_, ent in tracked.items() if ent[s][0] in (CACHED, NEW)] + traded_c + heads
                win = min(cands) if cands else None
                # the exact stop rule: a truncated list ran dry AND what it hides could beat the winner
                if dbound is not None:
                    if win is None or dbound < win:
                        self.stats["dry"] += 1
                        break
                    self.stats["dry_harmless"] += 1
                if win is not None and win[1] not in tracked and len(tracked) >= self.T:   # (fast pods only get here)
                    self.stats["full"] += 1
                    break
                if fast:
                    record()
                    self.stats["fast"] += 1
                fitc, ofd, osd = agg[s]
                if win is None:
                    out.append(dict(node=-1, status=po.EGS_ERR_NOFIT, alloc=None, fit_count=fitc, fit_digest=ofd, score_digest=osd))
                    p += 1
                    done += 1
                    continue
                w = win[1]
                if w not in tracked:                              # head-win: the node becomes tracked
                    track(w)
                e = tracked[w][s]
                opt = po.GPUOption(request=list(s), allocated=e[2], score=e[1])
                # deferred delete + aggregates, Transact
                e[0] = ABSENT
                agg[s][0] -= 1
                agg[s][1] = (agg[s][1] - fit_term(w)) & MASK64
                agg[s][2] = (agg[s][2] - score_term(w, e[1])) & MASK64
                ok = po.transact(rows_copy[w], opt)
                dirty.add(w)
                all_obs = all(observed.values())
                if not mono or not all_obs:
                    for s2 in shapes:
                        if s2 == s:
                            continue
                        e2 = tracked[w][s2]
                        if e2[0] == UNFIT and not mono:
                            e2[0] = ABSENT
                        elif e2[0] == NEW and not observed[s2]:
                            e2[0] = ABSENT
                            agg[s2][0] -= 1
                            agg[s2][1] = (agg[s2][1] - fit_term(w)) & MASK64
                            agg[s2][2] = (agg[s2][2] - score_term(w, e2[1])) & MASK64
                out.append(dict(node=w, status=po.EGS_OK if ok else po.EGS_ERR_TRANSACT, alloc=opt.allocated if ok else None,
                                fit_count=fitc, fit_digest=ofd, score_digest=osd))
                p += 1
                done += 1
            assert done >= 1, "resolver made no progress"
            if p == plim and plim < P:
                self.stats["shape"] += 1                          # the next pod's shape is outside this round's set
            # ---- epilogue: write back
            for w, ent in tracked.items():
                for s2 in shapes:
                    e = self.tables[s2][w]
                    e.st, e.score, e.alloc = ent[s2]
                if w in dirty:
                    for s2, tab in self.tables.items():
                        if s2 in shapes:
                            continue
                        e = tab[w]
                        if e.st == UNFIT:
                            e.st = ABSENT
                        elif e.st == NEW:
                            e.st = CACHED if self.obs_pending[s2] else ABSENT
            for s2 in shapes:
                if observed[s2]:
                    self.obs_pending[s2] = True
            p0 += done
        # ---- finalize: no NEW outlives the batch
        for s2, tab in self.tables.items():
            for e in tab:
                if e.st == NEW:
                    e.st = CACHED if self.obs_pending[s2] else ABSENT
            self.obs_pending[s2] = False
        return out
