/* shim_double.c -- C test double of integration/cuda_scheduler.go.
 *
 * The Go shim cannot be compiled in this repository (no Go toolchain); this program issues, per verb, exactly the C
 * calls the shim issues, in the same order, against libegs.so, driven by a line protocol on stdin
 * (tests/test_shim_double.py generates the scenario and checks every answer against the oracle):
 *
 *   NODE <name> <core_allocatable> <mem_allocatable>      getNodeID on first use: egs_node_set_allocatable
 *   ASSUME <npods-containers> {<core> <mem>}... | <node>...   predicate.go:26  -> egs_unit_from_requests, egs_filter
 *   SCORE  <C> {<core> <mem>}... | <node>...                 priority.go:33   -> egs_score
 *   BIND   <uid> <node> <C> {<core> <mem>}...                bind.go:51       -> egs_bind
 *   ADD    <uid> <node> <C> {<core> <mem> <n> <idx>*n}...    controller.go:330 -> egs_node_replay_pod (+ podMaps in the shim)
 *   FORGET <uid> <node|-> <C> {<core> <mem> <n> <idx>*n}...  controller.go:306 -> egs_pod_cancel (+ podMaps / released)
 *   KNOWN <uid> / RELEASED <uid>                             controller.go:314,322 (answered from the shim's own maps)
 *   STATUS                                                   routes.go:201    -> egs_state_dump
 *
 * argv: [policy [g_max [c_max]]] -- g_max is the widest node, EGS_MAX_GPUS by default; c_max the widest pod ASSUME /
 * SCORE / BIND place, EGS_MAX_CONTAINERS by default (egs_create_ex); masks are printed as the integer
 * EGS_MASK_BYTES(g_max) little-endian bytes hold, rows are dumped EGS_ROW_WIDTH(g_max) wide.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../include/egs.h"

#define MAXN 4096
static egs_handle *H;
static int G_MAX = EGS_MAX_GPUS, C_MAX = EGS_MAX_CONTAINERS;
static char names[MAXN][64];
static int n_nodes = 0;
static uint64_t known[65536], released[65536];
static int n_known = 0, n_released = 0;

static int node_id(const char *name) {
  for (int i = 0; i < n_nodes; i++) if (strcmp(names[i], name) == 0) return i;
  return -1;
}
static uint64_t uid_key(const char *uid) {           /* FNV-1a 64, as hash/fnv in the Go shim */
  uint64_t h = 0xcbf29ce484222325ull;
  for (const unsigned char *p = (const unsigned char *)uid; *p; p++) { h ^= *p; h *= 0x100000001b3ull; }
  return h;
}
static int mask_of(const uint8_t *masks, int c) {     /* maskToIDs: container c's mask, EGS_MASK_BYTES wide */
  int nb = EGS_MASK_BYTES(G_MAX), v = 0;
  for (int b = 0; b < nb; b++) v |= masks[c * nb + b] << (8 * b);
  return v;
}
static int has(uint64_t *set, int n, uint64_t k) { for (int i = 0; i < n; i++) if (set[i] == k) return 1; return 0; }
static void del(uint64_t *set, int *n, uint64_t k) { for (int i = 0; i < *n; i++) if (set[i] == k) { set[i] = set[--*n]; return; } }

static int read_units(char **tok, egs_unit *u) {     /* requestOf: NewGPURequest through egs_unit_from_requests */
  int C = atoi(strtok_r(NULL, " \n", tok));
  for (int i = 0; i < C; i++) {
    long long core = atoll(strtok_r(NULL, " \n", tok)), mem = atoll(strtok_r(NULL, " \n", tok));
    if (egs_unit_from_requests(core, mem, &u[i]) != EGS_OK) return -1;
  }
  return C;
}
static int read_units_alloc(char **tok, egs_unit *u, int32_t *off, int32_t *idx) {   /* + allocFromAnnotations */
  int C = atoi(strtok_r(NULL, " \n", tok)), k = 0;
  off[0] = 0;
  for (int i = 0; i < C; i++) {
    long long core = atoll(strtok_r(NULL, " \n", tok)), mem = atoll(strtok_r(NULL, " \n", tok));
    if (egs_unit_from_requests(core, mem, &u[i]) != EGS_OK) return -1;
    int n = atoi(strtok_r(NULL, " \n", tok));
    for (int j = 0; j < n; j++) idx[k++] = atoi(strtok_r(NULL, " \n", tok));
    off[i + 1] = k;
  }
  return C;
}

int main(int argc, char **argv) {
  int policy = argc > 1 ? atoi(argv[1]) : 0;
  if (argc > 2) G_MAX = atoi(argv[2]);
  if (argc > 3) C_MAX = atoi(argv[3]);
  if (egs_create_ex(policy, MAXN, G_MAX, C_MAX, 0, &H) != EGS_OK) { fprintf(stderr, "egs_create_ex failed\n"); return 2; }
  static char line[1 << 16];
  setvbuf(stdout, NULL, _IOLBF, 1 << 16);            /* every answer line reaches the driver at once */
  while (fgets(line, sizeof line, stdin)) {
    char *tok = NULL;
    char *cmd = strtok_r(line, " \n", &tok);
    if (!cmd) continue;
    egs_unit u[EGS_MAX_CONTAINERS_APPLY];
    int32_t off[EGS_MAX_CONTAINERS_APPLY + 1], idx[EGS_MAX_CONTAINERS_APPLY * EGS_MAX_GPUS_WIDE];
    if (!strcmp(cmd, "NODE")) {
      char *name = strtok_r(NULL, " \n", &tok);
      long long core = atoll(strtok_r(NULL, " \n", &tok)), mem = atoll(strtok_r(NULL, " \n", &tok));
      int st = egs_node_set_allocatable(H, n_nodes, core, mem);
      if (st == EGS_OK) { strncpy(names[n_nodes], name, 63); n_nodes++; }
      printf("NODE %d\n", st);
    } else if (!strcmp(cmd, "ASSUME") || !strcmp(cmd, "SCORE")) {
      int C = read_units(&tok, u);
      strtok_r(NULL, " \n", &tok);                                  /* the '|' */
      int32_t ids[MAXN]; int pos[MAXN]; int n = 0, m = 0;
      for (char *t; (t = strtok_r(NULL, " \n", &tok));) { int id = node_id(t); if (id >= 0) { ids[m] = id; pos[m++] = n; } n++; }
      if (!strcmp(cmd, "ASSUME")) {
        uint8_t fit[MAXN]; char ans[MAXN]; memset(ans, 'X', n);      /* X: "get node failed" */
        if (m && egs_filter(H, m, ids, C, u, fit) != EGS_OK) { printf("ASSUME error\n"); continue; }
        for (int k = 0; k < m; k++) ans[pos[k]] = fit[k] ? '1' : '0';
        printf("ASSUME %.*s\n", n, ans);
      } else {
        int32_t sc[MAXN]; long long out[MAXN]; memset(out, 0, sizeof(long long) * n);   /* ScoreMin for unknown nodes */
        int st = m ? egs_score(H, m, ids, C, u, sc) : EGS_OK;
        for (int k = 0; k < m; k++) out[pos[k]] = sc[k];
        /* EGS_ERR_PANIC: the Go shim panics like node.go:84 does; the double still prints what libegs computed so that
         * the driver can compare it with the oracle's view of the same call */
        printf(st == EGS_ERR_PANIC ? "SCORE! " : "SCORE");
        for (int i = 0; i < n; i++) printf(" %lld", out[i]);
        printf("\n");
      }
    } else if (!strcmp(cmd, "BIND")) {
      char *uid = strtok_r(NULL, " \n", &tok), *node = strtok_r(NULL, " \n", &tok);
      int C = read_units(&tok, u);
      uint8_t masks[2 * EGS_MAX_CONTAINERS_APPLY] = {0};
      int id = node_id(node);
      int st = id < 0 ? EGS_ERR_NO_NODE : egs_bind(H, id, C, u, uid_key(uid), masks);
      if (st == EGS_OK && !has(known, n_known, uid_key(uid))) known[n_known++] = uid_key(uid);   /* d.podMaps[pod.UID] = newPod */
      printf("BIND %d", st);
      for (int c = 0; c < C; c++) printf(" %d", st == EGS_OK ? mask_of(masks, c) : 0);
      printf("\n");
    } else if (!strcmp(cmd, "ADD")) {
      char *uid = strtok_r(NULL, " \n", &tok), *node = strtok_r(NULL, " \n", &tok);
      int C = read_units_alloc(&tok, u, off, idx);
      int id = node_id(node);
      if (id < 0) { printf("ADD nonode\n"); continue; }
      if (!has(known, n_known, uid_key(uid))) {                      /* scheduler.go:239-243 */
        egs_node_replay_pod(H, id, C, u, off, idx, uid_key(uid));
        known[n_known++] = uid_key(uid);
      }
      printf("ADD ok\n");
    } else if (!strcmp(cmd, "FORGET")) {
      char *uid = strtok_r(NULL, " \n", &tok), *node = strtok_r(NULL, " \n", &tok);
      int C = read_units_alloc(&tok, u, off, idx);
      if (strcmp(node, "-")) { int id = node_id(node); if (id >= 0) egs_pod_cancel(H, id, C, u, off, idx, uid_key(uid)); }
      if (has(known, n_known, uid_key(uid))) { del(known, &n_known, uid_key(uid)); if (!has(released, n_released, uid_key(uid))) released[n_released++] = uid_key(uid); }
      printf("FORGET ok\n");
    } else if (!strcmp(cmd, "KNOWN")) {
      printf("KNOWN %d\n", has(known, n_known, uid_key(strtok_r(NULL, " \n", &tok))));
    } else if (!strcmp(cmd, "RELEASED")) {
      printf("RELEASED %d\n", has(released, n_released, uid_key(strtok_r(NULL, " \n", &tok))));
    } else if (!strcmp(cmd, "ROWS")) {                                /* test support: synthetic prefill (egs_state_load) */
      int id = node_id(strtok_r(NULL, " \n", &tok)), G = atoi(strtok_r(NULL, " \n", &tok));
      if (G < 1 || G > EGS_MAX_GPUS_WIDE) { printf("ROWS %d\n", EGS_ERR_BAD_ARG); continue; }
      int32_t c[EGS_MAX_GPUS_WIDE], m[EGS_MAX_GPUS_WIDE];
      for (int g = 0; g < G; g++) c[g] = atoi(strtok_r(NULL, " \n", &tok));
      for (int g = 0; g < G; g++) m[g] = atoi(strtok_r(NULL, " \n", &tok));
      printf("ROWS %d\n", egs_state_load(H, id, c, m));
    } else if (!strcmp(cmd, "PEEK")) {                                /* test support: the option Assume cached (GPUIDs) */
      int id = node_id(strtok_r(NULL, " \n", &tok));
      int C = read_units(&tok, u);
      int32_t valid = 0, score = 0; uint8_t masks[2 * EGS_MAX_CONTAINERS_APPLY] = {0};
      egs_option_peek(H, id, C, u, &valid, &score, masks);
      printf("PEEK %d %d", valid, score);
      for (int c = 0; c < C; c++) printf(" %d", mask_of(masks, c));
      printf("\n");
    } else if (!strcmp(cmd, "STATUS")) {
      static int32_t core[MAXN * EGS_MAX_GPUS_WIDE], mem[MAXN * EGS_MAX_GPUS_WIDE], cnt[MAXN], tot[MAXN];
      const int W = EGS_ROW_WIDTH(G_MAX);
      if (n_nodes) egs_state_dump(H, 0, n_nodes, core, mem, cnt, tot);
      printf("STATUS");
      for (int i = 0; i < n_nodes; i++) {
        printf(" %s", names[i]);
        for (int g = 0; g < cnt[i]; g++) printf(":%d,%d", core[i * W + g], mem[i * W + g]);
      }
      printf("\n");
    }
    fflush(stdout);
  }
  egs_destroy(H);
  return 0;
}
