import sys, ctypes as C
sys.path.insert(0, "."); sys.path.insert(0, "oracle")
import numpy as np, egs_b200
n = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
cfg = int(sys.argv[2]) if len(sys.argv) > 2 else 4
w = egs_b200.workloads.config(cfg, n_pods=n)
e = egs_b200.Egs(w.policy, w.n_nodes)
e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
e.profile_reset(True)
e.schedule_batch(w.c_off, w.units, mode=2)
out = (C.c_longlong * 32)()
e.L.egs_debug_resolve_prof.argtypes = [C.c_void_p, C.c_void_p]
e.L.egs_debug_resolve_prof(e.h, out)
v = [int(x) for x in out]
print(e.rounds_stats(), "resolve ms", e.profile_get(3)[1], "select", e.profile_get(2)[1], "merge", e.profile_get(4)[1])
fast, gen, hw = max(v[6], 1), max(v[9], 1), max(v[11], 1)
print(f"pods: fast {v[6]} (head-wins {v[11]}), general {v[9]}; slots pre-installed in the round prologues {v[13]}")
npod = fast + gen
prep = v[22] + v[23] + v[24] + v[0]
print(f"  per-pod cycles (summed over owner warps / pods): prepare {prep/npod:.0f} (find the pod {v[22]/npod:.0f}, list heads {v[23]/npod:.0f},"
      f" payload prefetch {v[24]/npod:.0f}, best tracked + pending Trade {v[0]/npod:.0f})  wait {v[1]/npod:.0f}  post {v[3]/fast:.0f}")
print(f"  ticket: fast tracked-win {v[2]/max(fast-hw,1):.0f}  fast head-win {v[5]/hw:.0f}  general {v[4]/gen:.0f}")
tw = max(fast - hw, 1)
print(f"  tracked-win ticket split: rows+Trade {v[7]/tw:.0f}  winner {v[8]/tw:.0f}  transact {v[10]/tw:.0f}  stores+arrive {v[12]/tw:.0f}")
print(f"  pending Trade redone inside the ticket (rows changed since the preparation): {v[14]} of {fast} fast pods")
print(f"  total ticket Mcyc {(v[2]+v[5]+v[4])/1e6:.1f} = {(v[2]+v[5]+v[4])/1.965e6:.1f} ms at 1.965 GHz")
gaps = v[16] + v[18] + v[20]
print(f"  between tickets (release of pod p-1 -> start of pod p), Mcyc {gaps/1e6:.1f} = {gaps/1.965e6:.1f} ms at 1.965 GHz:")
print(f"    hand-over to a sleeping owner {v[17]} pods, {v[16]/max(v[17],1):.0f} cyc each;"
      f"  to an owner not yet ready {v[21]} pods, {v[20]/max(v[21],1):.0f} cyc each;"
      f"  ticket kept by its holder {v[19]} pods, {v[18]/max(v[19],1):.0f} cyc each")
