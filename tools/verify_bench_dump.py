"""Checks the per-pod outputs of a real benchmark run against the oracle, every pod of the batch.

    python bench.py --cfg N --dump-outputs DIR
    python tools/verify_bench_dump.py DIR --cfg N

DIR/<field>.npy are decoded as bench.py's dump_outputs wrote them (the 32- and 8-bit fields as float32, the 64-bit
digests as float64 (high 32 bits, low 32 bits) pairs) and compared with the indexed oracle driver
(egso_schedule_batch_indexed) on the same workload from a fresh cluster.  Exits 0 when every pod agrees on all six
fields, 1 naming the first differing pod and field otherwise."""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import oracle_c  # noqa: E402

DTYPES = {"node": np.int32, "status": np.int32, "alloc_mask": np.uint8, "fit_count": np.int32,
          "fit_digest": np.uint64, "score_digest": np.uint64}


def load_dump(path):
    out = {}
    for f, dt in DTYPES.items():
        a = np.load(os.path.join(path, f + ".npy"))
        if dt == np.uint64:
            if a.dtype != np.float64 or a.ndim != 2 or a.shape[1] != 2:
                raise ValueError(f"{f}: expected float64 [P, 2] (high, low), got {a.dtype} {a.shape}")
            out[f] = (a[:, 0].astype(np.uint64) << np.uint64(32)) | a[:, 1].astype(np.uint64)
        else:
            if a.dtype != np.float32:
                raise ValueError(f"{f}: expected float32, got {a.dtype}")
            out[f] = a.astype(np.int64).astype(dt)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("dir", help="the --dump-outputs directory of a bench.py run")
    ap.add_argument("--cfg", type=int, required=True, help="the config bench.py ran (its --cfg)")
    ap.add_argument("--pods", type=int, default=0, help="the pod prefix bench.py ran (its --pods), 0 = whole batch")
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    args = ap.parse_args(argv)
    import egs_b200
    w = egs_b200.workloads.config(args.cfg)
    if args.pods:
        w = w.prefix(args.pods)
    got = load_dump(args.dir)
    o = oracle_c.OracleC(w.policy)
    o.add_nodes(w.gpus, w.mem_total * w.gpus, w.core, w.mem)
    t0 = time.perf_counter()
    ref = o.schedule_batch_indexed(w.c_off, w.units64(), threads=args.threads)
    dt = time.perf_counter() - t0
    d = oracle_c.first_difference(ref, got)
    if d is not None:
        p, f = d
        have = got[f][p] if p < len(got[f]) else "missing"
        want = ref[f][p] if p < len(ref[f]) else "missing"
        print(f"cfg{args.cfg}: pod {p}: {f} differs: dump {have}, oracle {want}"
              f" ({len(got['node'])} pods dumped, {w.n_pods} in the batch)")
        return 1
    print(f"cfg{args.cfg}: all {w.n_pods} pods equal the oracle on all six fields (oracle {dt:.1f} s)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
