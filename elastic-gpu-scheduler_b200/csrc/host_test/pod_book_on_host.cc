// pod_book_on_host.cc -- PodBook (csrc/pod_book.h) behind a C API, so the CPU test suite can check the uid
// bookkeeping against a model of the reference's three maps (tests/test_pod_book_host.py) and its checkpoint journal
// (tests/test_pod_book_journal_host.py).  Not part of libegs.
#include "../pod_book.h"

static PodBook *B(void *b) { return (PodBook *)b; }

extern "C" {
void *egspb_create() { return new PodBook(); }
void egspb_free(void *b) { delete B(b); }
void egspb_add_run(void *b, uint64_t uid0, int n, const int32_t *node, const int32_t *status) {
  B(b)->add_run(uid0, n, node, status);
}
void egspb_add_batch(void *b, const uint64_t *uids, int n, const int32_t *node, const int32_t *status) {
  B(b)->add_batch(uids, n, node, status);
}
void egspb_record_bind(void *b, int node, uint64_t uid, int had_entry, int known, int status) {
  B(b)->record_bind(node, uid, had_entry != 0, known != 0, status);
}
// apply fails with EGS_ERR_BAD_ARG when fail_apply is set; the cancel argument of each apply call goes to
// cancels[*n_calls++] (room for 4)
int egspb_account(void *b, int kind, int node, uint64_t uid, int fail_apply, int *n_calls, int32_t *cancels) {
  *n_calls = 0;
  return B(b)->account(kind, node, uid, [&](int cancel) {
    if (*n_calls < 4) cancels[*n_calls] = cancel;
    ++*n_calls;
    return fail_apply ? EGS_ERR_BAD_ARG : EGS_OK;
  });
}
void egspb_drop_nodes(void *b, int node0, int n) { B(b)->drop_nodes(node0, n); }
void egspb_clear(void *b) { B(b)->clear(); }
void egspb_checkpoint(void *b) { B(b)->checkpoint(); }
void egspb_rollback(void *b) { B(b)->rollback(); }
void egspb_drop_checkpoint(void *b) { B(b)->drop_checkpoint(); }
uint64_t egspb_hash_uid_max(void *b) { return B(b)->hash_uid_max(); }
int egspb_in_pods_map(void *b, int node, uint64_t uid) { return B(b)->in_pods_map(node, uid) ? 1 : 0; }
int egspb_in_pod_maps(void *b, uint64_t uid) { return B(b)->in_pod_maps(uid) ? 1 : 0; }
int egspb_released(void *b, uint64_t uid) { return B(b)->released(uid) ? 1 : 0; }
}
