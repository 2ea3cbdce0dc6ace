/* Plain-C client of include/flmr_maxsim.h (compiled by tests/test_cabi_c_client.py with gcc -std=c99):
 * the boundary is a C ABI, not a C++/torch one.  Runs without a GPU: version, argument validation and
 * the host-only partition helper. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "flmr_maxsim.h"

int main(void) {
  if (flmr_abi_version() != FLMR_ABI_VERSION) return 10;
  flmr_corpus_t* corpus = NULL;
  int32_t doclens[3] = {4, 0, 8};
  unsigned short tokens[12 * FLMR_DIM];
  memset(tokens, 0, sizeof tokens);
  /* zero-length passage: rejected before any CUDA call, with a message */
  int rc = flmr_corpus_create(tokens, doclens, 3, FLMR_DIM, 0, 0, FLMR_CORPUS_COPY, &corpus);
  if (rc != FLMR_ERR_INVALID_ARG || corpus != NULL || strstr(flmr_last_error(), "zero-length") == NULL) return 11;
  rc = flmr_corpus_create(tokens, doclens, 3, 64, 0, 0, FLMR_CORPUS_COPY, &corpus);
  if (rc != FLMR_ERR_UNSUPPORTED) return 12;
  if (flmr_maxsim_topk(NULL, NULL, NULL, 1, 32, 5, 0, NULL, NULL, NULL) != FLMR_ERR_INVALID_ARG) return 13;
  if (flmr_topk_select(NULL, 1, 10, 5, 0, NULL, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 14;
  if (flmr_corpus_destroy(NULL) != FLMR_OK || flmr_workspace_destroy(NULL) != FLMR_OK) return 15;
  /* training / RAG entry points: argument validation happens before any CUDA call */
  if (flmr_maxsim_argmax(NULL, 1, 32, NULL, NULL, 1, 8, NULL, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 17;
  if (flmr_maxsim_backward(NULL, 1, 32, NULL, 1, 8, NULL, NULL, NULL, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 18;
  if (flmr_corpus_gather(NULL, NULL, 1, 8, NULL, NULL, NULL) != FLMR_ERR_INVALID_ARG) return 19;
  if (flmr_plaid_decode(NULL, NULL, 1, NULL, 1, NULL, 2, FLMR_DIM, 1, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 20;
  /* round-2 entry points: block-diagonal scoring, loss head, sharded search, streaming corpus builder */
  if (flmr_maxsim_argmax_grouped(NULL, 1, 32, NULL, NULL, 2, 8, NULL, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 21;
  if (flmr_maxsim_backward_grouped(NULL, 1, 32, NULL, 0, 8, NULL, NULL, NULL, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 22;
  if (flmr_ib_loss(NULL, 2, 4, 32, 2, 0, NULL, NULL, NULL, 0, NULL) != FLMR_ERR_INVALID_ARG) return 23;
  {
    flmr_comm_t* comm = NULL;
    char id[128];
    memset(id, 0, sizeof id);
    if (flmr_comm_create(id, 3, 2, 0, &comm) != FLMR_ERR_INVALID_ARG || comm != NULL) return 24; /* rank >= world */
    if (flmr_comm_destroy(NULL) != FLMR_OK) return 25;
    if (flmr_maxsim_topk_sharded(NULL, NULL, NULL, NULL, 1, 32, 5, 0, NULL, NULL, NULL) != FLMR_ERR_INVALID_ARG) return 26;
    if (flmr_topk_exchange(NULL, NULL, NULL, 1, 5, 5, NULL, NULL, NULL) != FLMR_ERR_INVALID_ARG) return 27;
  }
  {
    flmr_corpus_builder_t* b = NULL;
    rc = flmr_corpus_builder_create(doclens, 3, FLMR_DIM, 0, 0, &b);   /* zero-length passage again */
    if (rc != FLMR_ERR_INVALID_ARG || b != NULL) return 28;
    if (flmr_corpus_builder_append(NULL, tokens, 1) != FLMR_ERR_INVALID_ARG) return 29;
    if (flmr_corpus_builder_append_file(NULL, "x", 0, 1) != FLMR_ERR_INVALID_ARG) return 30;
    if (flmr_corpus_builder_finish(NULL, &corpus, NULL) != FLMR_ERR_INVALID_ARG) return 31;
    if (flmr_corpus_builder_destroy(NULL) != FLMR_OK) return 32;
  }
  if (flmr_debug_set_scan_variant(5) != FLMR_ERR_INVALID_ARG || flmr_debug_set_scan_variant(7) != FLMR_ERR_INVALID_ARG ||
      flmr_debug_set_scan_variant(0) != FLMR_OK)
    return 33;
  if (flmr_debug_set_argmax_path(7) != FLMR_ERR_INVALID_ARG || flmr_debug_set_argmax_path(0) != FLMR_OK) return 34;
  /* host-only helper: 5 passages over 2 CTAs */
  int32_t dl[5] = {100, 7, 96, 1, 50};
  int32_t row_begin[3];
  int64_t tile_base[3], n_tiles = 0;
  uint32_t mask[16];
  int32_t first_pid[16];
  rc = flmr_debug_build_partition(dl, 5, 2, row_begin, tile_base, mask, first_pid, 16, &n_tiles);
  if (rc != FLMR_OK || row_begin[0] != 0 || row_begin[2] != 100 + 8 + 96 + 4 + 52 || n_tiles < 3) return 16;
  printf("c_client ok: abi %d, %lld tiles, tile tokens %d\n", flmr_abi_version(), (long long)n_tiles, FLMR_TILE_TOKENS);
  return 0;
}
