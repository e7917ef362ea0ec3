// rounds_geometry_on_host.cu -- the resolver geometry batch_rounds uses (mw_geometry in egs_rounds.cuh) behind a C
// call, so the CPU test suite can say which list depth, shared memory and pre-install a GPU case runs with
// (tests/test_shard_groups_host.py).  egs_rounds.cuh is compiled here as a translation unit of its own.  Not part of
// libegs.
#include "../egs_rounds.cuh"

extern "C" {
// ns: shapes of the round set (1..RSMAX), D: shards.  out[0..4] = rkm, rke, pre_h, pre_cap, smem bytes.
int egsrg_geometry(int ns, int D, long long *out) {
  if (ns < 1 || ns > RSMAX || D < 1 || D > RD || !out) return -1;
  const MwGeometry g = mw_geometry(ns, D);
  out[0] = g.rkm; out[1] = g.rke; out[2] = g.pre_h; out[3] = g.pre_cap; out[4] = (long long)g.smem;
  return 0;
}
int egsrg_smem_max() { return MW_SMEM_MAX; }
}
