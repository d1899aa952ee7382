/* tests/hostsim -- CPU emulation of the launches behind bk_gf_* (kernels_tojson.cu: a chunk as GELF messages) as loops over the
 * same per-thread function of dev_gelf.cuh.  Part of tests/hostsim/libhostsim.so with hostsim.cpp; TEST INFRASTRUCTURE only. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include "../../fluent-bit_b200/csrc/flbgpu_prog.h"
#include "../../fluent-bit_b200/csrc/flbgpu_internal.h"
#include "../../fluent-bit_b200/csrc/dev_chain.cuh"
#include "../../fluent-bit_b200/csrc/dev_gelf.cuh"

extern "C" {

int bk_gf_sizes(bk_q *, const struct gf_env *e)
{
    for (uint32_t i = 0; i < e->n_rec; i++) e->size[i] = gf_event(e, i, 0);
    return 0;
}
int bk_gf_emit(bk_q *, const struct gf_env *e, const uint64_t *d_bsum, uint8_t *d_out)
{
    uint64_t at = 0;
    for (uint32_t i = 0; i < e->n_rec; i++) {
        if (i % BK_REC_BLOCK == 0) at = d_bsum[i / BK_REC_BLOCK];
        if (e->size[i]) {
            uint32_t w = gf_event(e, i, d_out + at);
            if (w != e->size[i]) {
                fprintf(stderr, "hostsim: GELF message size mismatch at event %u: %u vs %u\n", i, w, e->size[i]);
                return -1;
            }
        }
        at += e->size[i];
    }
    return 0;
}

}
