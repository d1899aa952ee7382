/* kernels_ml.cu -- filter_multiline on sm_90a: the launches behind bk_ml_plan / bk_ml_sizes / bk_ml_emit.
 *
 * All the work is in dev_ml.cuh (the same functions the CPU emulation of the tests loops over); a kernel here gives every
 * piece its thread:
 *   k_ml_feat ......... one lane per record: key_content, which rules' regexes match (the regex VM of dev_regex.cuh)
 *   k_ml_up1 .......... one lane per (block of ML_F1 records, state): the block as a function on automaton states (S bytes)
 *   k_ml_up2 .......... one lane per (ML_F2 blocks, state): composition
 *   k_ml_top .......... one lane: incoming state of every super-block (a few thousand dependent byte loads for 10 M records)
 *   k_ml_down2 ........ incoming state of every block
 *   k_ml_apply ........ the automaton over the records with the state known: actions, events and time marks per block
 *   k_ml_cnt_up2 / k_ml_cnt_top / k_ml_cnt_down2 .. the same tree for "events before this block" and "last time mark"
 *   k_ml_fill ......... the event list and the time mark of every record
 *   k_ml_size, k_ml_emit .. one lane per event (flush): the concatenated message
 * Byte-stream work: no tensor cores; the per-record pass is the regex VM's cost, everything else streams small arrays.
 * A translation unit of its own so that it compiles beside kernels.cu.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "flbgpu_internal.h"
#include "flbgpu_prog.h"
#include "rx_compile.h"
/* the device headers define their out-of-line functions (__noinline__: mp_canon, dt_strptime, ...) without `static`, and
 * kernels.cu has them too: here they get internal linkage.  The C types above are declared before the namespace opens. */
namespace {
#include "dev_ml.cuh"
}

#define CKM(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { bk_note_error(#call, cudaGetErrorString(e_)); return -1; } } while (0)
#define ML_BLOCK 128u

#define ML_KERNEL(name, fn, count) \
    __global__ void __launch_bounds__(ML_BLOCK) name(const __grid_constant__ ml_env e) \
    { const uint32_t t = blockIdx.x * ML_BLOCK + threadIdx.x; if (t < (count)) fn(&e, t); }
ML_KERNEL(k_ml_feat, ml_feat_record, e.n_rec)
ML_KERNEL(k_ml_up1, ml_up1, e.nt1 * e.S)
ML_KERNEL(k_ml_up2, ml_up2, e.nt2 * e.S)
ML_KERNEL(k_ml_down2, ml_down2, e.nt2)
ML_KERNEL(k_ml_apply, ml_apply, e.nt1)
ML_KERNEL(k_ml_cnt_up2, ml_cnt_up2, e.nt2)
ML_KERNEL(k_ml_cnt_down2, ml_cnt_down2, e.nt2)
ML_KERNEL(k_ml_fill, ml_fill, e.nt1)
__global__ void k_ml_top(const __grid_constant__ ml_env e) { ml_top(&e); }
__global__ void k_ml_cnt_top(const __grid_constant__ ml_env e) { ml_cnt_top(&e); }

__global__ void __launch_bounds__(ML_BLOCK) k_ml_size(const __grid_constant__ ml_env e, uint32_t n_ev)
{
    const uint32_t j = blockIdx.x * ML_BLOCK + threadIdx.x;
    if (j < n_ev) e.ev_size[j] = ml_event(&e, j, 0);
}

/* event j at bsum[its block of BK_REC_BLOCK events] + the sizes before it in the block */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_ml_emit(const __grid_constant__ ml_env e, uint32_t n_ev, const uint64_t *__restrict__ bsum,
                                                          uint8_t *__restrict__ out)
{
    __shared__ uint32_t wsum[BK_REC_BLOCK / 32];
    const uint32_t j = blockIdx.x * BK_REC_BLOCK + threadIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t sz = j < n_ev ? e.ev_size[j] : 0u;
    uint32_t x = sz, base = 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t) d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    for (uint32_t w = 0; w < warp; w++) base += wsum[w];
    if (sz) ml_event(&e, j, out + bsum[blockIdx.x] + base + x - sz);
}

static cudaStream_t st_of(bk_q *q) { return (cudaStream_t) bk_stream(q); }
#define GRID(n) (((n) + ML_BLOCK - 1) / ML_BLOCK)

extern "C" {

int bk_ml_plan(bk_q *q, const struct ml_env *e)
{
    cudaStream_t st = st_of(q);
    CKM(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 1);
    k_ml_feat<<<GRID(e->n_rec), ML_BLOCK, 0, st>>>(*e);
    k_ml_up1<<<GRID(e->nt1 * e->S), ML_BLOCK, 0, st>>>(*e);
    k_ml_up2<<<GRID(e->nt2 * e->S), ML_BLOCK, 0, st>>>(*e);
    k_ml_top<<<1, 1, 0, st>>>(*e);
    k_ml_down2<<<GRID(e->nt2), ML_BLOCK, 0, st>>>(*e);
    k_ml_apply<<<GRID(e->nt1), ML_BLOCK, 0, st>>>(*e);
    k_ml_cnt_up2<<<GRID(e->nt2), ML_BLOCK, 0, st>>>(*e);
    k_ml_cnt_top<<<1, 1, 0, st>>>(*e);
    k_ml_cnt_down2<<<GRID(e->nt2), ML_BLOCK, 0, st>>>(*e);
    k_ml_fill<<<GRID(e->nt1), ML_BLOCK, 0, st>>>(*e);
    bk_ev_end(q, 1);
    bk_note_launches(10);
    CKM(cudaGetLastError());
    return 0;
}

int bk_ml_sizes(bk_q *q, const struct ml_env *e, uint32_t n_ev)
{
    CKM(cudaSetDevice(bk_q_device(q)));
    if (!n_ev) return 0;
    bk_ev_begin(q, 2);
    k_ml_size<<<GRID(n_ev), ML_BLOCK, 0, st_of(q)>>>(*e, n_ev);
    bk_ev_end(q, 2);
    bk_note_launches(1);
    CKM(cudaGetLastError());
    return 0;
}

int bk_ml_emit(bk_q *q, const struct ml_env *e, uint32_t n_ev, const uint64_t *d_bsum, uint8_t *d_out)
{
    CKM(cudaSetDevice(bk_q_device(q)));
    if (!n_ev) return 0;
    bk_ev_begin(q, 2);
    k_ml_emit<<<(n_ev + BK_REC_BLOCK - 1) / BK_REC_BLOCK, BK_REC_BLOCK, 0, st_of(q)>>>(*e, n_ev, d_bsum, d_out);
    bk_ev_end(q, 2);
    bk_note_launches(1);
    CKM(cudaGetLastError());
    return 0;
}

}
