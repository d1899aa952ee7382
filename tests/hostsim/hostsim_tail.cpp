/* tests/hostsim -- CPU emulation of the launches behind bk_tl_* (kernels_lines.cu: in_tail's `Parser` branch) as loops over the
 * same per-thread functions of dev_lines.cuh.  Part of tests/hostsim/libhostsim.so with hostsim.cpp; TEST INFRASTRUCTURE only. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include "../../fluent-bit_b200/csrc/flbgpu_prog.h"
#include "../../fluent-bit_b200/csrc/flbgpu_internal.h"
#include "../../fluent-bit_b200/csrc/dev_lines.cuh"

extern "C" {

int bk_tl_mid_size(bk_q *, const struct tl_env *t)
{
    for (uint32_t k = 0; k < t->ln.n_lines; k++) { t->msize[k] = tl_mid_size(t, k); if (t->msize[k]) t->ln.n_events[0]++; }

    return 0;
}
int bk_tl_mid_emit(bk_q *, const struct tl_env *t)
{
    uint64_t at = 0;
    for (uint32_t k = 0; k < t->ln.n_lines; k++) {
        if (k % BK_REC_BLOCK == 0) at = t->mbsum[k / BK_REC_BLOCK];
        if (t->msize[k]) tl_mid_emit(t, k, t->mid + at);
        at += t->msize[k];
    }
    return 0;
}
int bk_tl_sizes(bk_q *, const struct tl_env *t)
{
    uint64_t at = 0;
    for (uint32_t r = 0; r < t->n_rec; r++) {
        if (r % BK_REC_BLOCK == 0) at = t->r_bsum[r / BK_REC_BLOCK];
        t->r_out[r] = (uint32_t) at;
        at += t->r_size[r];
    }
    for (uint32_t k = 0; k < t->ln.n_lines; k++) {
        uint32_t r = TL_NONE, sz = 0;
        if (k % BK_REC_BLOCK == 0) at = t->mbsum[k / BK_REC_BLOCK];
        if (t->msize[k]) {
            r = tl_find(t, (uint32_t) at, t->msize[k]);
            if (r != TL_NONE) sz = tl_event(t, k, r, 0);
            if (!sz) t->bad[0]++;
        }
        t->rec[k] = sz ? r : TL_NONE;
        t->size[k] = sz;
        at += t->msize[k];
    }
    return 0;
}
int bk_tl_emit(bk_q *, const struct tl_env *t, const uint64_t *d_bsum, uint8_t *d_out)
{
    uint64_t at = 0;
    for (uint32_t k = 0; k < t->ln.n_lines; k++) {
        if (k % BK_REC_BLOCK == 0) at = d_bsum[k / BK_REC_BLOCK];
        if (t->size[k]) {
            uint32_t w = tl_event(t, k, t->rec[k], d_out + at);
            if (w != t->size[k]) {
                fprintf(stderr, "hostsim: line event size mismatch at line %u: %u vs %u\n", k, w, t->size[k]);
                return -1;
            }
        }
        at += t->size[k];
    }
    return 0;
}

}
