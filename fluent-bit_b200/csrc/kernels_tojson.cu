/* kernels_tojson.cu -- a chunk of log events as JSON text on sm_90a: the launches behind bk_tj_sizes / bk_tj_emit, and the
 * same two passes for GELF messages (dev_gelf.cuh) behind bk_gf_sizes / bk_gf_emit.
 *
 * One lane per event, two passes over dev_tojson.cuh's tj_event(): the sizing pass packs the event as one msgpack map into its
 * scratch slice (what the reference converts from) and measures the text; after the scan over the sizes the emission pass
 * converts again and writes at the event's offset.  Byte-stream work: no tensor cores; neighbouring lanes read neighbouring
 * events, each lane writes its own run of the result.  A translation unit of its own (compiles beside kernels.cu).
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "flbgpu_internal.h"
#include "flbgpu_prog.h"
#include "rx_compile.h"
namespace {                     /* the device headers' out-of-line functions get internal linkage here (kernels.cu has them too) */
#include "dev_chain.cuh"
#include "dev_tojson.cuh"
#include "dev_gelf.cuh"
}

#define CKT(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { bk_note_error(#call, cudaGetErrorString(e_)); return -1; } } while (0)
#define TJ_BLOCK 128u

/* (left alone the converter takes 228 registers per lane, one block of 256 lanes per SM: bounded to 128 so that two to four blocks fit) */
__global__ void __launch_bounds__(TJ_BLOCK, 4) k_tj_size(const __grid_constant__ tj_env e)
{
    const uint32_t i = blockIdx.x * TJ_BLOCK + threadIdx.x;
    if (i < e.n_rec) e.size[i] = tj_event(&e, i, 0);
}

/* event i at bsum[its block of BK_REC_BLOCK events] + the sizes before it in the block */
__global__ void __launch_bounds__(BK_REC_BLOCK, 2) k_tj_emit(const __grid_constant__ tj_env e, const uint64_t *__restrict__ bsum, uint8_t *__restrict__ out)
{
    __shared__ uint32_t wsum[BK_REC_BLOCK / 32];
    const uint32_t i = blockIdx.x * BK_REC_BLOCK + threadIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t sz = i < e.n_rec ? e.size[i] : 0u;
    uint32_t x = sz, base = 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t) d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    for (uint32_t w = 0; w < warp; w++) base += wsum[w];
    if (sz) tj_event(&e, i, out + bsum[blockIdx.x] + base + x - sz);
}

/* GELF: the same shape -- the sizing pass (which also re-packs an event with its tag), then the emission at the scanned offsets */
__global__ void __launch_bounds__(TJ_BLOCK, 4) k_gf_size(const __grid_constant__ gf_env e)
{
    const uint32_t i = blockIdx.x * TJ_BLOCK + threadIdx.x;
    if (i < e.n_rec) e.size[i] = gf_event(&e, i, 0);
}

__global__ void __launch_bounds__(BK_REC_BLOCK, 2) k_gf_emit(const __grid_constant__ gf_env e, const uint64_t *__restrict__ bsum, uint8_t *__restrict__ out)
{
    __shared__ uint32_t wsum[BK_REC_BLOCK / 32];
    const uint32_t i = blockIdx.x * BK_REC_BLOCK + threadIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t sz = i < e.n_rec ? e.size[i] : 0u;
    uint32_t x = sz, base = 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t) d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    for (uint32_t w = 0; w < warp; w++) base += wsum[w];
    if (sz) gf_event(&e, i, out + bsum[blockIdx.x] + base + x - sz);
}

extern "C" {

int bk_tj_sizes(bk_q *q, const struct tj_env *e)
{
    CKT(cudaSetDevice(bk_q_device(q)));
    if (!e->n_rec) return 0;
    bk_ev_begin(q, 1);
    k_tj_size<<<(e->n_rec + TJ_BLOCK - 1) / TJ_BLOCK, TJ_BLOCK, 0, (cudaStream_t) bk_stream(q)>>>(*e);
    bk_ev_end(q, 1);
    bk_note_launches(1);
    CKT(cudaGetLastError());
    return 0;
}

int bk_tj_emit(bk_q *q, const struct tj_env *e, const uint64_t *d_bsum, uint8_t *d_out)
{
    CKT(cudaSetDevice(bk_q_device(q)));
    if (!e->n_rec) return 0;
    bk_ev_begin(q, 2);
    k_tj_emit<<<(e->n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK, BK_REC_BLOCK, 0, (cudaStream_t) bk_stream(q)>>>(*e, d_bsum, d_out);
    bk_ev_end(q, 2);
    bk_note_launches(1);
    CKT(cudaGetLastError());
    return 0;
}

int bk_gf_sizes(bk_q *q, const struct gf_env *e)
{
    CKT(cudaSetDevice(bk_q_device(q)));
    if (!e->n_rec) return 0;
    bk_ev_begin(q, 1);
    k_gf_size<<<(e->n_rec + TJ_BLOCK - 1) / TJ_BLOCK, TJ_BLOCK, 0, (cudaStream_t) bk_stream(q)>>>(*e);
    bk_ev_end(q, 1);
    bk_note_launches(1);
    CKT(cudaGetLastError());
    return 0;
}

int bk_gf_emit(bk_q *q, const struct gf_env *e, const uint64_t *d_bsum, uint8_t *d_out)
{
    CKT(cudaSetDevice(bk_q_device(q)));
    if (!e->n_rec) return 0;
    bk_ev_begin(q, 2);
    k_gf_emit<<<(e->n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK, BK_REC_BLOCK, 0, (cudaStream_t) bk_stream(q)>>>(*e, d_bsum, d_out);
    bk_ev_end(q, 2);
    bk_note_launches(1);
    CKT(cudaGetLastError());
    return 0;
}

}
