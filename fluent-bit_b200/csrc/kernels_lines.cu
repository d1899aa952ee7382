/* kernels_lines.cu -- raw text to log events on sm_90a (in_tail's line loop): the launches behind bk_ln_*.
 *
 *   k_ln_count ... one lane per tile of LN_TILE bytes: the line feeds of the tile (neighbouring lanes read neighbouring tiles)
 *   k_ln_fill .... the same lanes again: positions of the line feeds at the tile's offset (block offsets from the scan, the rest
 *                  by a shuffle scan inside the block)
 *   k_ln_size .... one lane per line: what the line keeps, the size of its event; lines that became events counted per block
 *   k_ln_emit .... one lane per line: the event at its offset
 * With a parser (flbgpu_lines_to_events_parsed):
 *   k_tl_mid_size / k_tl_mid_emit ... one lane per line: its event {"_": line} in the parser's input
 *   k_tl_roff .... one lane per record of the parser's chain: where its result starts
 *   k_tl_size .... one lane per line: its record (found by offset in the chain's index), the bytes of its event
 *   k_tl_emit .... one lane per line: the event at its offset, from the chain's result and the parser's report
 * Byte-stream work bounded by HBM traffic (text in once per pass, events out once): no tensor cores.  The functions are in
 * dev_lines.cuh, shared with the CPU emulation of the tests.  A translation unit of its own.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "flbgpu_internal.h"
#include "flbgpu_prog.h"
namespace {
#include "dev_lines.cuh"
}

#define CKL(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { bk_note_error(#call, cudaGetErrorString(e_)); return -1; } } while (0)

/* exclusive prefix of v over the block's lanes (BK_REC_BLOCK of them) */
__device__ __forceinline__ uint32_t ln_block_excl(uint32_t v)
{
    __shared__ uint32_t wsum[BK_REC_BLOCK / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t x = v, base = 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t) d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    for (uint32_t w = 0; w < warp; w++) base += wsum[w];
    return base + x - v;
}

__global__ void __launch_bounds__(BK_REC_BLOCK) k_ln_count(const __grid_constant__ ln_env e)
{
    const uint32_t t = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    if (t < e.n_tiles) e.cnt[t] = ln_count(&e, t);
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_ln_fill(const __grid_constant__ ln_env e, const uint64_t *__restrict__ bsum)
{
    const uint32_t t = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t c = t < e.n_tiles ? e.cnt[t] : 0u;
    const uint32_t ex = ln_block_excl(c);
    if (c) ln_fill(&e, t, bsum[blockIdx.x] + ex);
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_ln_size(const __grid_constant__ ln_env e)
{
    const uint32_t k = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    uint32_t a, b, sz = 0;
    if (k < e.n_lines) { sz = ln_line(&e, k, &a, &b); e.size[k] = sz; }
    const int made = __syncthreads_count(sz != 0);
    if (threadIdx.x == 0 && made) atomicAdd(e.n_events, (unsigned long long) made);
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_ln_emit(const __grid_constant__ ln_env e, const uint64_t *__restrict__ bsum, uint8_t *__restrict__ out)
{
    const uint32_t k = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = k < e.n_lines ? e.size[k] : 0u;
    const uint32_t ex = ln_block_excl(sz);
    if (sz) ln_emit(&e, k, out + bsum[blockIdx.x] + ex);
}

/* with a parser (tl_*): the parser's input, the result offsets of the chain's records, the events */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_tl_mid_size(const __grid_constant__ tl_env t)
{
    const uint32_t k = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    uint32_t sz = 0;
    if (k < t.ln.n_lines) { sz = tl_mid_size(&t, k); t.msize[k] = sz; }
    const int made = __syncthreads_count(sz != 0);
    if (threadIdx.x == 0 && made) atomicAdd(t.ln.n_events, (unsigned long long) made);
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_tl_mid_emit(const __grid_constant__ tl_env t)
{
    const uint32_t k = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = k < t.ln.n_lines ? t.msize[k] : 0u;
    const uint32_t ex = ln_block_excl(sz);
    if (sz) tl_mid_emit(&t, k, t.mid + t.mbsum[blockIdx.x] + ex);
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_tl_roff(const __grid_constant__ tl_env t)
{
    const uint32_t r = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = r < t.n_rec ? t.r_size[r] : 0u;
    const uint32_t ex = ln_block_excl(sz);
    if (r < t.n_rec) t.r_out[r] = (uint32_t) (t.r_bsum[blockIdx.x] + ex);
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_tl_size(const __grid_constant__ tl_env t)
{
    const uint32_t k = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t ms = k < t.ln.n_lines ? t.msize[k] : 0u;
    const uint32_t ex = ln_block_excl(ms);
    if (k < t.ln.n_lines) {
        uint32_t r = TL_NONE, sz = 0;
        if (ms) {
            r = tl_find(&t, (uint32_t) (t.mbsum[blockIdx.x] + ex), ms);
            if (r != TL_NONE) sz = tl_event(&t, k, r, 0);
            if (!sz) atomicAdd(t.bad, 1u);
        }
        t.rec[k] = sz ? r : TL_NONE;
        t.size[k] = sz;
    }
}
__global__ void __launch_bounds__(BK_REC_BLOCK) k_tl_emit(const __grid_constant__ tl_env t, const uint64_t *__restrict__ bsum, uint8_t *__restrict__ out)
{
    const uint32_t k = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = k < t.ln.n_lines ? t.size[k] : 0u;
    const uint32_t ex = ln_block_excl(sz);
    if (sz) tl_event(&t, k, t.rec[k], out + bsum[blockIdx.x] + ex);
}

#define LN_GRID(n) (((n) + BK_REC_BLOCK - 1) / BK_REC_BLOCK)
#define LN_ST(q) ((cudaStream_t) bk_stream(q))

extern "C" {

int bk_ln_count(bk_q *q, const struct ln_env *e)
{
    CKL(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 0);
    k_ln_count<<<LN_GRID(e->n_tiles), BK_REC_BLOCK, 0, LN_ST(q)>>>(*e);
    bk_ev_end(q, 0);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}
int bk_ln_fill(bk_q *q, const struct ln_env *e, const uint64_t *d_bsum)
{
    CKL(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 0);
    k_ln_fill<<<LN_GRID(e->n_tiles), BK_REC_BLOCK, 0, LN_ST(q)>>>(*e, d_bsum);
    bk_ev_end(q, 0);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}
int bk_ln_sizes(bk_q *q, const struct ln_env *e)
{
    CKL(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 1);
    k_ln_size<<<LN_GRID(e->n_lines), BK_REC_BLOCK, 0, LN_ST(q)>>>(*e);
    bk_ev_end(q, 1);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}
int bk_ln_emit(bk_q *q, const struct ln_env *e, const uint64_t *d_bsum, uint8_t *d_out)
{
    CKL(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 2);
    k_ln_emit<<<LN_GRID(e->n_lines), BK_REC_BLOCK, 0, LN_ST(q)>>>(*e, d_bsum, d_out);
    bk_ev_end(q, 2);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}

int bk_tl_mid_size(bk_q *q, const struct tl_env *t)
{
    if (!t->ln.n_lines) return 0;
    CKL(cudaSetDevice(bk_q_device(q)));
    k_tl_mid_size<<<LN_GRID(t->ln.n_lines), BK_REC_BLOCK, 0, LN_ST(q)>>>(*t);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}
int bk_tl_mid_emit(bk_q *q, const struct tl_env *t)
{
    if (!t->ln.n_lines) return 0;
    CKL(cudaSetDevice(bk_q_device(q)));
    k_tl_mid_emit<<<LN_GRID(t->ln.n_lines), BK_REC_BLOCK, 0, LN_ST(q)>>>(*t);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}
int bk_tl_sizes(bk_q *q, const struct tl_env *t)
{
    CKL(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 2);
    if (t->n_rec) k_tl_roff<<<LN_GRID(t->n_rec), BK_REC_BLOCK, 0, LN_ST(q)>>>(*t);
    if (t->ln.n_lines) k_tl_size<<<LN_GRID(t->ln.n_lines), BK_REC_BLOCK, 0, LN_ST(q)>>>(*t);
    bk_ev_end(q, 2);
    bk_note_launches(2);
    CKL(cudaGetLastError());
    return 0;
}
int bk_tl_emit(bk_q *q, const struct tl_env *t, const uint64_t *d_bsum, uint8_t *d_out)
{
    if (!t->ln.n_lines) return 0;
    CKL(cudaSetDevice(bk_q_device(q)));
    bk_ev_begin(q, 2);
    k_tl_emit<<<LN_GRID(t->ln.n_lines), BK_REC_BLOCK, 0, LN_ST(q)>>>(*t, d_bsum, d_out);
    bk_ev_end(q, 2);
    bk_note_launches(1);
    CKL(cudaGetLastError());
    return 0;
}

}
