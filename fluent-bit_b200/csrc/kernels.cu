/* kernels.cu -- sm_90a kernels and the CUDA implementation of the bk_* seam.
 *
 *   k_index<FILL> ..... K1 record index: every 0x92 byte is a record candidate; a
 *                       candidate is kept when a complete, well-formed log event
 *                       ([[ts, meta], body] or [ts, body]) starts there
 *                       (reference framing rules: src/flb_log_event_decoder.c:214-297).
 *                       Two passes (count -> prefix sum -> fill) keep file order.
 *   k_index_check ..... the kept candidates must tile the chunk; the first gap ends
 *                       the decodable prefix (the reference decoder stops there too).
 *   k_index_repair .... walks the record chain across the (few) broken links;
 *   k_link_* .......... the same by pointer doubling when a slice has more broken links than
 *                       the one-CTA walk holds (records with nested [int, {map}] values).
 *   k_scan_top ........ exclusive prefix sum over per-block totals (one CTA).
 *   k_chain_eval ...... one lane = one record through the filter-chain interpreter
 *                       (dev_chain.cuh): sizes, verdict evidence, final field list.
 *   k_chain_emit_list . encodes the surviving records at their offsets.
 *   k_small_* ......... glue of the small-chunk form: every count stays on the device.
 *
 * This is byte-stream work bounded by HBM traffic and instruction issue; there is no
 * contraction here, so no tensor-core path.  Loads of chunk bytes are 128-bit and
 * coalesced in k_index; k_chain lanes walk adjacent records (L1/L2 resident lines).
 *
 * Host side: all state is per queue (struct bk_q, flbgpu_internal.h); nothing here is
 * process-global except the launch counter and the thread-local error text.
 */
#include <cuda_runtime.h>
#include <atomic>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <vector>
#include <new>
#include <string.h>
#include <stdlib.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <dlfcn.h>
#include <nccl.h>
#include "flbgpu_internal.h"
#include "dev_chain.cuh"

static thread_local char g_err[256];
static std::atomic<unsigned long long> g_launches;

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    snprintf(g_err, sizeof(g_err), "%s: %s", #call, cudaGetErrorString(e_)); return -1; } } while (0)

/* 4 resident blocks per SM (64 registers per lane): the interpreter is bound by instruction fetch and load
 * latency, which more resident warps hide better than fewer spills do */
#ifndef BK_EVAL_MIN_BLOCKS
#define BK_EVAL_MIN_BLOCKS 4
#endif

/* ---------------------------------------------------------------- helpers */
/* exclusive scan of one value per thread over a 256-thread block */
template <typename T>
__device__ __forceinline__ T block_excl_scan_t(T v, T *total)
{
    __shared__ T wsum[8];
    __shared__ T tot;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (unsigned) d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        T s = lane < 8 ? wsum[lane] : 0;
#pragma unroll
        for (int d = 1; d < 8; d <<= 1) {
            T y = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= (unsigned) d) s += y;
        }
        if (lane < 8) wsum[lane] = s;
        if (lane == 7) tot = s;
    }
    __syncthreads();
    T base = warp ? wsum[warp - 1] : 0;
    *total = tot;
    __syncthreads();
    return base + x - v;
}
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *total)
{
    return block_excl_scan_t<uint32_t>(v, total);
}

/* what the kernels of the small-chunk form hand each other (device memory; copied to the host once) */
struct bk_mail {
    unsigned long long n_cand64;     /* candidates counted (k_small_tiles) */
    unsigned long long total;        /* result bytes */
    unsigned long long n_out;        /* surviving records */
    uint32_t n_breaks, n_valid, tiled, end_off;     /* k_index_check / k_index_repair (same order as the sliced form) */
    uint32_t n_cand;                 /* candidates the arrays hold (0 on overflow) */
    uint32_t overflow;               /* 1: more candidates than the arrays hold; 2: more broken links than the walk holds */
    uint32_t emitted;                /* the result fits the output buffer and was written */
    uint32_t pad;
};

/* ------------------------------------------------------------------ index */
/* The counting pass leaves what it validated in a staging row per tile -- word 0: records kept, then one word per record
 * (position in the tile, kind, length) -- so that the filling pass, which runs once the offsets are known, only copies: it does
 * not read the chunk again and does not frame a record twice.  A tile with more records than a row holds (events of a few
 * bytes) is validated again by the filling pass, as before. */
#define BK_STAGE_ROW 256u                           /* 64-bit words per tile: 2 KB for 8 KB of input */
#define BK_STAGE_PACK(rel, kind, rlen) (((unsigned long long) (rel) << 48) | ((unsigned long long) (kind) << 40) | (unsigned long long) (rlen))
template <bool FILL>
__global__ void __launch_bounds__(256) k_index(const uint8_t *__restrict__ in, uint32_t len, uint32_t skip, uint32_t abs_base,
                                               uint32_t *__restrict__ tile, uint32_t *__restrict__ o_off,
                                               uint32_t *__restrict__ o_len, uint8_t *__restrict__ o_kind,
                                               const struct bk_mail *__restrict__ mail, unsigned long long *__restrict__ stage)
{
    __shared__ uint16_t cand[BK_INDEX_TILE];
    __shared__ uint32_t v2ok[BK_INDEX_TILE / 32];   /* bit per tile byte: a valid v2 frame starts here */
    __shared__ uint32_t s_ncand;
    const uint32_t base = blockIdx.x * BK_INDEX_TILE;
    uint32_t ncand = 0;
    if (FILL && mail && mail->overflow) return;      /* small form: the arrays cannot hold the candidates */
    if (FILL && stage) {
        const unsigned long long *row = stage + (size_t) blockIdx.x * BK_STAGE_ROW;
        const uint32_t n = (uint32_t) row[0];
        if (n < BK_STAGE_ROW) {
            const uint32_t tb = tile[blockIdx.x];
            for (uint32_t j = threadIdx.x; j < n; j += 256) {
                const unsigned long long e = row[1 + j];
                o_off[tb + j] = abs_base + base + (uint32_t) (e >> 48);
                o_len[tb + j] = (uint32_t) (e & 0xffffffffull);
                o_kind[tb + j] = (uint8_t) ((e >> 40) & 0xff);
            }
            return;
        }
    }

    /* phase 1: ordered list of candidate positions in this tile */
    for (uint32_t it = 0; it < BK_INDEX_TILE / (256 * 16); it++) {
        const uint32_t rel = (it * 256 + threadIdx.x) * 16;
        const uint32_t pos = base + rel;
        uint32_t mask = 0;
        if (pos + 16 <= len) {
            const uint4 v = *reinterpret_cast<const uint4 *>(in + pos);   /* 128-bit coalesced load */
            const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
            for (int k = 0; k < 16; k++) if (((w[k >> 2] >> (8 * (k & 3))) & 0xff) == 0x92) mask |= 1u << k;
        }
        else {
            for (int k = 0; k < 16; k++) if (pos + k < len && in[pos + k] == 0x92) mask |= 1u << k;
        }
        /* `in` is the slice start rounded down to 16 bytes: bytes before `skip` belong to the previous slice */
        if (pos < skip) mask &= (pos + 16 <= skip) ? 0u : (0xffffu << (skip - pos));
        uint32_t tot;
        uint32_t at = block_excl_scan(__popc(mask), &tot) + ncand;
        while (mask) {
            int k = __ffs(mask) - 1;
            mask &= mask - 1;
            cand[at++] = (uint16_t) (rel + k);
        }
        ncand += tot;
    }
    if (threadIdx.x == 0) s_ncand = ncand;
    v2ok[threadIdx.x] = 0;
    __syncthreads();
    ncand = s_ncand;

    /* phase 2: validate candidates, 256 at a time, keeping order.  A candidate whose
     * predecessor byte starts a valid v2 frame is that frame's header array, not a
     * record (rec_is_shadowed); within a tile the predecessor's verdict is read from
     * shared memory (it belongs to an earlier or the same round: positions ascend). */
    uint32_t kept = 0;
    const uint32_t tile_base = FILL ? tile[blockIdx.x] : 0;
    for (uint32_t r = 0; r < ncand; r += 256) {
        const uint32_t j = r + threadIdx.x;
        uint32_t ok = 0, rlen = 0;
        int kind = 0;
        uint32_t pos = 0, rel = 0;
        if (j < ncand) {
            rel = cand[j];
            pos = base + rel;
            const uint8_t *e = rec_frame(in + pos, in + len, &kind);
            if (e) {
                ok = 1; rlen = (uint32_t) (e - (in + pos));
                if (in[pos + 1] == 0x92) atomicOr(&v2ok[rel >> 5], 1u << (rel & 31));
            }
        }
        __syncthreads();
        if (ok && pos > 0 && in[pos - 1] == 0x92) {
            if (rel > 0) { if ((v2ok[(rel - 1) >> 5] >> ((rel - 1) & 31)) & 1) ok = 0; }
            else if (rec_is_shadowed(in, in + pos, in + len)) ok = 0;      /* predecessor lives in the previous tile */
        }
        uint32_t tot;
        uint32_t at = block_excl_scan(ok, &tot);
        if (FILL && ok) {
            const uint32_t o = tile_base + kept + at;
            o_off[o] = abs_base + pos; o_len[o] = rlen; o_kind[o] = (uint8_t) kind;
        }
        if (!FILL && ok && stage && kept + at + 1 < BK_STAGE_ROW)
            stage[(size_t) blockIdx.x * BK_STAGE_ROW + 1 + kept + at] = BK_STAGE_PACK(rel, kind, rlen);
        kept += tot;
    }
    if (!FILL && threadIdx.x == 0) {
        tile[blockIdx.x] = kept;
        if (stage) stage[(size_t) blockIdx.x * BK_STAGE_ROW] = kept;
    }
}

/* exclusive scan of a[0..n) in place, one CTA; total in *out_total (and added to *accum) */
template <typename T>
__global__ void __launch_bounds__(256) k_scan_top(T *a, uint32_t n, unsigned long long *out_total, unsigned long long *accum)
{
    unsigned long long carry = 0;
    for (uint32_t b = 0; b < n; b += 256) {
        const uint32_t i = b + threadIdx.x;
        unsigned long long v = i < n ? (unsigned long long) a[i] : 0, tot;
        unsigned long long ex = block_excl_scan_t<unsigned long long>(v, &tot);
        if (i < n) a[i] = (T) (carry + ex);
        carry += tot;
    }
    if (threadIdx.x == 0) { *out_total = carry; if (accum) *accum += carry; }
}

#define BK_MAX_BREAKS 8192u

/* Links of the candidate list: candidate i must end where candidate i+1 starts (the
 * last one at the end of the chunk).  Broken links are rare -- a false candidate is a
 * byte run inside a real record that happens to frame as an event, e.g. the timestamp
 * bytes `.. 92 ce 00 00 01 a6 | 80` read as the legacy event [422, {}] -- and are
 * collected for k_index_repair. */
__global__ void k_index_check(const uint32_t *__restrict__ off, const uint32_t *__restrict__ rlen, uint32_t n_host,
                              const uint32_t *__restrict__ n_dev,
                              uint32_t total /* absolute end of the slice */, uint32_t *n_breaks, uint32_t *breaks)
{
    const uint32_t n = n_dev ? *n_dev : n_host;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t next = (i + 1 < n) ? off[i + 1] : total;
    if (off[i] + rlen[i] != next) {
        const uint32_t at = atomicAdd(n_breaks, 1u);
        if (at < BK_MAX_BREAKS) breaks[at] = i;
    }
}

/* One CTA: sort the broken links, then follow the record chain across them.  At a
 * break the chain jumps to the candidate that starts exactly where the current record
 * ends; the candidates jumped over were false and get kind 2 (ignored by k_chain).
 * If nothing starts there the decodable prefix ends (the reference decoder stops at
 * the first undecodable byte too).  res[0] = records in the prefix, res[1] = tiled,
 * res[2] = where the chain ends.  More than BK_MAX_BREAKS broken links: *ovf = 2, nothing
 * is touched (the pointer-doubling form below decides). */
__global__ void __launch_bounds__(1024) k_index_repair(const uint32_t *__restrict__ off, const uint32_t *__restrict__ rlen,
                                                        uint8_t *kind, uint32_t n_host, const uint32_t *__restrict__ n_dev,
                                                        uint32_t base, uint32_t total,
                                                        const uint32_t *n_breaks, const uint32_t *breaks, uint32_t *res, uint32_t *ovf)
{
    __shared__ uint32_t sorted[BK_MAX_BREAKS];
    const uint32_t n = n_dev ? *n_dev : n_host;
    const uint32_t m = *n_breaks;
    if (m > BK_MAX_BREAKS) {
        if (threadIdx.x == 0) { res[0] = 0; res[1] = 0; res[2] = base; if (ovf) *ovf = 2; }
        return;
    }
    if (n == 0) {
        if (threadIdx.x == 0) { res[0] = 0; res[1] = (base == total); res[2] = base; }
        return;
    }
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {          /* rank sort: values are distinct */
        const uint32_t v = breaks[i];
        uint32_t r = 0;
        for (uint32_t j = 0; j < m; j++) r += breaks[j] < v;
        sorted[r] = v;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    uint32_t n_valid = n, tiled = 1, skip_until = 0;
    if (off[0] != base) { res[0] = 0; res[1] = 0; res[2] = base; return; }
    for (uint32_t q = 0; q < m; q++) {
        const uint32_t b = sorted[q];
        if (b < skip_until) continue;                                  /* a candidate already ruled out */
        const uint32_t target = off[b] + rlen[b];
        uint32_t k = b + 1;
        while (k < n && off[k] < target) { kind[k] = 2; k++; }
        if (k < n && off[k] == target) { skip_until = k; continue; }
        if (k == n && target == total) { skip_until = n; continue; }
        n_valid = b + 1; tiled = 0;                                    /* nothing decodable starts at `target` */
        break;
    }
    res[0] = n_valid; res[1] = tiled;
    /* where the chain ends: the next slice starts here */
    {
        uint32_t last = n_valid;
        while (last > 0 && kind[last - 1] == 2) last--;
        res[2] = last ? off[last - 1] + rlen[last - 1] : base;
    }
}

/* ---- the same decision by pointer doubling (any number of broken links) ----
 * next[i] = the candidate that starts where candidate i ends (n = "the slice ends there",
 * 0xffffffff = nothing starts there).  The records are the candidates on the path from
 * candidate 0; after k rounds `mark` holds the first 2^k of them and jump = next^(2^k). */
#define LINK_NONE 0xffffffffu
__global__ void k_link_next(const uint32_t *__restrict__ off, const uint32_t *__restrict__ rlen, uint32_t n, uint32_t base,
                            uint32_t total, uint32_t *__restrict__ next, uint8_t *__restrict__ mark)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t target = off[i] + rlen[i];
    uint32_t lo = i + 1, hi = n;                       /* first candidate at or behind target */
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (off[mid] < target) lo = mid + 1; else hi = mid; }
    next[i] = (lo < n && off[lo] == target) ? lo : (lo == n && target == total) ? n : LINK_NONE;
    mark[i] = (i == 0 && off[0] == base) ? 1 : 0;
}
__global__ void k_link_step(const uint32_t *__restrict__ jump, uint32_t *__restrict__ jump2, uint8_t *mark, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t j = jump[i];
    if (j < n) { if (mark[i]) mark[j] = 1; jump2[i] = jump[j]; }
    else jump2[i] = j;
}
/* kind 2 for the candidates off the path; res as k_index_repair leaves it */
__global__ void k_link_finish(const uint32_t *__restrict__ off, const uint32_t *__restrict__ rlen, const uint32_t *__restrict__ next,
                              const uint8_t *__restrict__ mark, uint8_t *kind, uint32_t n, uint32_t base, uint32_t *res)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!mark[i]) { kind[i] = 2; return; }
    if (next[i] >= n) {                                /* the last record of the path: the prefix ends behind it */
        res[0] = i + 1; res[1] = next[i] == n; res[2] = off[i] + rlen[i];
    }
}

/* ------------------------------------------------------------------ chain */
struct k_chain_params {
    struct ch_env env;
    const uint32_t *off, *len;
    const uint8_t *kind;
    uint32_t r0;                 /* first record / first block of this launch */
    uint32_t bm_words;           /* JSON stage 1: 32-bit words of string-event bitmap per warp in shared memory, 0 = none */
    uint32_t *defer_list;        /* records put off by the stage-2 walker (CH_DEFER), and how many */
    unsigned long long *defer_cnt;
    uint32_t *tlist, *tn;        /* split evaluation: the records the head launch left for the tail launch, and how many */
    uint32_t n_rec;
    const uint32_t *n_dev;       /* small form: the record count lives on the device */
    uint32_t *size;
    uint64_t *bsum;
    uint8_t *out;
};

/* chains with a rewrite_tag filter: where the bytes the reference's decoder consumed for record i begin -- behind the previous
 * decoded record (the events it steps over in between, kind 1, are handed to the emitter with the record: rewrite_tag.c:462-470) */
__device__ __forceinline__ uint32_t raw_lo_of(const k_chain_params &p, uint32_t i)
{
    uint32_t j = i;
    while (j > 0 && p.kind[j - 1] != 0) j--;
    return j ? p.off[j - 1] + p.len[j - 1] : 0u;
}

/* evaluation: record r0 + global thread id.  No barrier: a warp retires as soon as its
 * 32 records are done (block-level reductions happen in k_bsum). */

/* Optional staging (stage_bytes > 0, FLBGPU_STAGE_KB): the 32 records of a warp are adjacent in the
 * chunk, so the warp first copies their bytes to its own slice of shared memory with coalesced 128-bit
 * loads and the lanes then scan from there; `in` is rebased so that input offsets keep their meaning.
 * A warp whose records span more than its slice reads global memory as before. */
/* Stage 1 of the JSON tokenizer (chains with a JSON parser): the warp's 32 records are adjacent in the chunk, so the
 * warp reads their whole byte range once with coalesced 128-bit loads and leaves one bit per byte in shared memory --
 * set where a string scan has to stop and look ('"', '\\', control, >= 0x80).  Stage 2 (djf_record_bm, one lane per record)
 * then finds the end of a plain string with a bit scan.  A range longer than BM_BYTES is scanned the old way. */
#define BM_BYTES 8192u                               /* per warp: 256 words = 1 KB of shared memory */
__device__ __forceinline__ uint32_t bm_mask4(uint32_t w)
{
    /* bit 7 of each byte of the result: byte is '"', '\\', < 0x20 or >= 0x80 */
    uint32_t t, m;
    t = w ^ 0x22222222u; m = (t - 0x01010101u) & ~t;
    t = w ^ 0x5c5c5c5cu; m |= (t - 0x01010101u) & ~t;
    m |= (w - 0x20202020u) & ~w;
    m |= w;
    m &= 0x80808080u;
    return ((m >> 7) * 0x00204081u) >> 21 & 0xfu;        /* gather the four flags into bits 0..3 */
}

/* PH: CH_PH_ALL = the whole chain in one launch.  Split form (chains `parser, then other filters`): a CH_PH_HEAD launch
 * decodes and parses and leaves the field lists in the capture cache, a CH_PH_TAIL launch runs the other filters from there.
 * Each half has roughly half the interpreter's code, which is what the single launch is bound by (instruction cache misses,
 * the interpreter's hot code does not fit an SM's instruction cache). */
template <int PH>
__global__ void __launch_bounds__(1024, 1) k_chain_eval_t(const __grid_constant__ k_chain_params p)       /* 64 registers per lane; block size chosen at launch.
                                                                                                             (5 or 6 resident blocks of 256 lanes with 48 / 40 registers were slower) */
{
    extern __shared__ __align__(16) uint8_t dsm[];
    const uint32_t n_rec = p.n_dev ? *p.n_dev : p.n_rec;
    uint32_t i = p.r0 + blockIdx.x * blockDim.x + threadIdx.x;
    bool valid = i < n_rec;
    if (PH == CH_PH_TAIL) {
        /* dense: lane t takes the t-th record the head launch left.  The tail reads nothing of a record that is not on the
         * list: the follow-up launch beside it writes the size and the cache row of the records the head put off. */
        const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
        valid = t < *p.tn;
        i = valid ? p.tlist[t] : 0;
    }
    const uint32_t my_off = valid ? p.off[i] : 0, my_len = valid ? p.len[i] : 0;
    const bool live = valid && p.kind[i] == 0;
    const uint8_t *in = p.env.in;
    const uint32_t *bm = 0;
    uint32_t bm_base = 0, bm_end = 0;
    if (PH != CH_PH_TAIL && p.bm_words) {
        const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t lo = __reduce_min_sync(0xffffffffu, live ? my_off : 0xffffffffu);
        const uint32_t hi = __reduce_max_sync(0xffffffffu, live ? my_off + my_len : 0u);
        if (hi > lo) {
            lo -= (uint32_t) ((uintptr_t) (in + lo) & 15u);           /* 16-byte aligned in the address space */
            if (hi - lo <= BM_BYTES) {
                uint32_t *w = reinterpret_cast<uint32_t *>(dsm) + (size_t) warp * p.bm_words;
                for (uint32_t o0 = 0; o0 < hi - lo; o0 += 2048) {                        /* the same trip count in every lane: the shuffle below pairs them */
                    uint4 v[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {                                        /* four 512-byte rows in flight: the range is read once, from DRAM */
                        const uint32_t o = o0 + (uint32_t) u * 512 + lane * 16;
                        v[u] = make_uint4(0, 0, 0, 0);
                        if (o < hi - lo) v[u] = *reinterpret_cast<const uint4 *>(in + lo + o);   /* reads past `hi` stay inside the padded buffer */
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const uint32_t o = o0 + (uint32_t) u * 512 + lane * 16;
                        const uint32_t m16 = bm_mask4(v[u].x) | (bm_mask4(v[u].y) << 4) | (bm_mask4(v[u].z) << 8) | (bm_mask4(v[u].w) << 12);
                        const uint32_t other = __shfl_xor_sync(0xffffffffu, m16, 1);
                        if (!(lane & 1) && o < hi - lo) w[o >> 5] = m16 | (other << 16);
                    }
                }
                __syncwarp();
                bm = w; bm_base = lo; bm_end = hi;
            }
        }
    }
    if (!valid) return;
    uint32_t sz = 0;
    if (PH != CH_PH_TAIL && !live && p.env.esize) p.env.esize[i] = 0;      /* an event the decoder steps over has no entry of its own */
    if (live) {
        /* the environment is read where the kernel parameters live (__grid_constant__: no per-lane copy); what differs per
         * lane travels in a few words */
        struct ch_lane ln;
        ln.bm = bm; ln.bm_base = bm_base; ln.bm_end = bm_end;
        ln.defer_ok = (bm && p.defer_list) ? 1u : 0u; ln.l2m_probe = 0; ln.l2m_forced = 0;
        ln.raw_lo = p.env.esize ? raw_lo_of(p, i) : my_off;
        sz = chain_record<false, PH>(&p.env, &ln, i, my_off, my_len, 0);
        if (sz == CH_DEFER) {                          /* the follow-up launch evaluates it whole, with the byte scanner */
            p.defer_list[atomicAdd(p.defer_cnt, 1ull)] = i;
            if (PH != CH_PH_HEAD) return;
            sz = 0;                                    /* kept off the tail launch's list */
        }
    }
    if (PH == CH_PH_HEAD) {
        /* the survivors of the warp go to the tail launch's list side by side (one atomic per warp; the order of the warps in
         * the list does not matter: every record owns its slots) */
        const unsigned lanes = __activemask();
        const unsigned alive = __ballot_sync(lanes, sz != 0);
        if (sz) {
            const unsigned lane = threadIdx.x & 31u, leader = (unsigned) __ffs((int) alive) - 1u;
            uint32_t base = 0;
            if (lane == leader) base = atomicAdd(p.tn, (uint32_t) __popc(alive));
            base = __shfl_sync(alive, base, (int) leader);
            p.tlist[base + (uint32_t) __popc(alive & ((1u << lane) - 1u))] = i;
        }
    }
    __stcs(&p.size[i], sz);
}
#define k_chain_eval k_chain_eval_t<CH_PH_ALL>

/* The records the stage-2 walker put off (nested values, odd spacing, lines that are not JSON ...: a few per cent): dense,
 * so that the byte scanner and the exact transcoder run with full warps instead of inside warps whose other lanes wait. */
__global__ void __launch_bounds__(1024, 1) k_chain_eval_deferred(const __grid_constant__ k_chain_params p)
{
    const unsigned long long n = *p.defer_cnt;
    for (unsigned long long t = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (unsigned long long) gridDim.x * blockDim.x) {
        const uint32_t i = p.defer_list[t];
        struct ch_lane ln;
        ln.bm = 0; ln.bm_base = ln.bm_end = 0; ln.defer_ok = 0; ln.l2m_probe = 0; ln.l2m_forced = 0;
        ln.raw_lo = p.env.esize ? raw_lo_of(p, i) : p.off[i];
        __stcs(&p.size[i], chain_record<false>(&p.env, &ln, i, p.off[i], p.len[i], 0));
    }
}

/* Chains with a log_to_metrics filter only: the events the decoder steps over (kind 1: group markers, negative
 * timestamps) are counted by that filter as long as nothing before it rewrote the chunk (chain_skipped_record).
 * A kernel of its own so that k_chain_eval stays what it is for every other chain. */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_chain_skipped(const __grid_constant__ k_chain_params p)
{
    const uint32_t n_rec = p.n_dev ? *p.n_dev : p.n_rec;
    const uint32_t i = p.r0 + blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    if (i >= n_rec || p.kind[i] != 1) return;
    chain_skipped_record(&p.env, i, p.off[i], p.len[i]);
}

/* The re-tagged stream of a rewrite_tag filter: one entry per matched record (RT_ENTRY_HDR, tag, record as the filter saw it),
 * in record order.  p.size = the entry sizes of the evaluation pass, p.bsum = exclusive offset per block, p.out = the stream. */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_rtag_emit(const __grid_constant__ k_chain_params p)
{
    const uint32_t i = p.r0 + blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = i < p.n_rec ? p.size[i] : 0;
    uint32_t tot;
    const uint32_t ex = block_excl_scan(sz, &tot);
    if (!sz) return;
    struct ch_lane ln;
    ln.bm = 0; ln.bm_base = ln.bm_end = 0; ln.defer_ok = 0; ln.l2m_probe = 0; ln.l2m_forced = 0;
    ln.raw_lo = raw_lo_of(p, i);
    chain_record<true, CH_PH_RTAG>(&p.env, &ln, i, p.off[i], p.len[i], p.out + p.bsum[blockIdx.x] + ex);
}

/* log_to_metrics, gauge / histogram: the records the evaluation listed because their value text converts nothing
 * (dev_chain.cuh: l2m_fixup_record).  A handful per call at most; entries [done, listed) are new since the last launch.
 * ONE entry per warp, worked on by lane 0 while the other lanes have left: the interpreter's reconvergence points (full-mask
 * __syncwarp) pair up only among lanes that are in step or gone, and the entries of a warp would neither start together nor
 * walk back equally far (a launch that gave every lane an entry and met at a block barrier afterwards hung on the device). */
__global__ void __launch_bounds__(1024) k_l2m_fixup(const __grid_constant__ k_chain_params p)
{
    if (threadIdx.x & 31u) return;
    const unsigned long long n = p.env.l2m.pending_n[0], d = p.env.l2m.pending_n[1];
    const unsigned long long lim = n < p.env.l2m.pending_cap ? n : p.env.l2m.pending_cap;
    for (unsigned long long t = d + (threadIdx.x >> 5); t < lim; t += blockDim.x >> 5)
        l2m_fixup_record(&p.env, p.env.l2m.pending[t], p.off, p.len, p.kind);
}
/* ... and, behind it in the stream, what has been observed so far */
__global__ void k_l2m_fixup_done(const __grid_constant__ k_chain_params p)
{
    p.env.l2m.pending_n[1] = p.env.l2m.pending_n[0];
}

/* per-block sums of the record sizes */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_bsum(const uint32_t *__restrict__ size, uint32_t n, uint64_t *__restrict__ bsum)
{
    const uint32_t i = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    uint32_t tot;
    block_excl_scan(i < n ? size[i] : 0, &tot);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

/* ---- emission over a dense list of survivors ----
 * After a selective grep most records of a block are gone; packing the survivors of the whole range
 * (not just of one block) keeps every warp of the emission kernel full.
 *   k_surv_count: survivors per block            k_scan_top<uint32_t>: rank base per block
 *   k_surv_fill : (record, output offset) at its rank      k_chain_emit_list: one lane per rank */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_surv_count(const uint32_t *__restrict__ size, uint32_t n, uint32_t *__restrict__ cnt)
{
    const uint32_t i = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    uint32_t tot;
    block_excl_scan((i < n && size[i]) ? 1u : 0u, &tot);
    if (threadIdx.x == 0) cnt[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(BK_REC_BLOCK) k_surv_fill(const uint32_t *__restrict__ size, uint32_t n_host, const uint32_t *__restrict__ n_dev,
                                                            uint32_t rec0, const uint32_t *__restrict__ base, const uint64_t *__restrict__ bsum,
                                                            uint32_t *__restrict__ l_rec, uint64_t *__restrict__ l_off)
{
    const uint32_t n = n_dev ? *n_dev : n_host;
    const uint32_t i = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = i < n ? size[i] : 0;
    uint32_t tot, nsurv;
    const uint32_t local = block_excl_scan(sz, &tot);
    const uint32_t rank = block_excl_scan(sz ? 1u : 0u, &nsurv);
    if (sz) {
        l_rec[base[blockIdx.x] + rank] = rec0 + i;
        l_off[base[blockIdx.x] + rank] = bsum[blockIdx.x] + local;
    }
}

/* One lane encodes one surviving record.  The survivors of a warp are consecutive in the result (the list is in
 * record order and the offsets are a running sum), so the warp first encodes its 32 records into a slice of shared
 * memory laid out like the result, then copies the whole range out with coalesced 16-byte stores: the result leaves
 * the SM in full sectors instead of byte-sized partial writes (about one DRAM write byte per result byte).
 * A warp whose range does not fit its slice writes directly, as before. */
#define EMIT_BLOCK 128u
#define EMIT_STAGE 8192u          /* bytes of result per warp that can be staged (+16 of alignment slack) */
__global__ void __launch_bounds__(EMIT_BLOCK, 6) k_chain_emit_list(const __grid_constant__ k_chain_params p, const uint32_t *__restrict__ l_rec,
                                                                   const uint64_t *__restrict__ l_off,
                                                                   const unsigned long long *__restrict__ n_list,
                                                                   const uint32_t *__restrict__ go)
{
    extern __shared__ __align__(16) uint8_t emit_stage[];
    const uint32_t t = blockIdx.x * EMIT_BLOCK + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (go && !*go) return;
    const bool valid = t < (uint32_t) *n_list;
    const uint32_t r = valid ? l_rec[t] : 0;
    const unsigned long long off = valid ? l_off[t] : 0ull;
    const uint32_t sz = valid ? p.size[r] : 0u;
    const unsigned vmask = __ballot_sync(0xffffffffu, valid);
    if (!vmask) return;
    /* valid lanes are a prefix of the warp: lane 0 holds the start of the range, the last valid lane its end */
    const int last = 31 - __clz((int) vmask);
    const unsigned long long base = __shfl_sync(0xffffffffu, off, 0);
    const unsigned long long end = __shfl_sync(0xffffffffu, off + sz, last);
    const uint32_t total = (uint32_t) (end - base), mis = (uint32_t) ((uintptr_t) (p.out + base) & 15u);
    /* A record whose field list did not fit the cache row is re-run through the whole chain, reconvergence points
     * (full-mask __syncwarp) included: those pair up only among lanes that all take that path or have exited.  A warp
     * holding such a record therefore emits the old way -- finished lanes exit, nothing waits at a warp barrier. */
    const bool rerun = valid && p.env.capcache[(size_t) (p.env.cap_stride - RC_CACHE_INTS) * p.env.cap_n + r] == RC_CACHE_NONE;
    if (!__any_sync(0xffffffffu, rerun) && total + mis <= EMIT_STAGE) {
        uint8_t *sb = emit_stage + (size_t) warp * (EMIT_STAGE + 16);
        if (valid) { struct ch_lane ln; ln.bm = 0; ln.bm_base = ln.bm_end = 0; ln.defer_ok = 0; ln.l2m_probe = 0; ln.l2m_forced = 0; ln.raw_lo = p.off[r]; chain_record<true>(&p.env, &ln, r, p.off[r], p.len[r], sb + mis + (uint32_t) (off - base)); }   /* cached field list: encode only */
        __syncwarp();
        {
            /* shared byte i corresponds to result byte (base - mis + i): 16-byte chunks are aligned on both sides */
            uint8_t *g = p.out + base - mis;
            const uint32_t lo = mis, hi = mis + total;
            const uint32_t body_lo = (lo + 15u) & ~15u, body_hi = hi & ~15u;
            if (body_lo >= body_hi) { for (uint32_t i = lo + lane; i < hi; i += 32) g[i] = sb[i]; }
            else {
                for (uint32_t i = lo + lane; i < body_lo; i += 32) g[i] = sb[i];
                for (uint32_t i = body_lo + lane * 16; i < body_hi; i += 512) __stcs(reinterpret_cast<uint4 *>(g + i), *reinterpret_cast<const uint4 *>(sb + i));
                for (uint32_t i = body_hi + lane; i < hi; i += 32) g[i] = sb[i];
            }
        }
        return;
    }
    if (!valid) return;
    { struct ch_lane ln; ln.bm = 0; ln.bm_base = ln.bm_end = 0; ln.defer_ok = 0; ln.l2m_probe = 0; ln.l2m_forced = 0; ln.raw_lo = p.off[r]; chain_record<true>(&p.env, &ln, r, p.off[r], p.len[r], p.out + off); }
}

/* ---- glue of the small-chunk form ---- */
/* exclusive scan of the tile counts; n_cand = total, or 0 + overflow when the record arrays are too small */
__global__ void __launch_bounds__(256) k_small_tiles(uint32_t *tile, uint32_t n_tiles, uint32_t cap, struct bk_mail *mail)
{
    unsigned long long carry = 0;
    for (uint32_t b = 0; b < n_tiles; b += 256) {
        const uint32_t i = b + threadIdx.x;
        unsigned long long v = i < n_tiles ? (unsigned long long) tile[i] : 0, tot;
        unsigned long long ex = block_excl_scan_t<unsigned long long>(v, &tot);
        if (i < n_tiles) tile[i] = (uint32_t) (carry + ex);
        carry += tot;
    }
    if (threadIdx.x == 0) {
        mail->n_cand64 = carry;
        mail->overflow = carry > cap ? 1u : 0u;
        mail->n_cand = carry > cap ? 0u : (uint32_t) carry;
    }
}

/* per-block output bytes and survivors of size[0, n_valid) (zero for the blocks behind) */
__global__ void __launch_bounds__(BK_REC_BLOCK) k_small_sizes(const uint32_t *__restrict__ size, const struct bk_mail *__restrict__ mail,
                                                              uint64_t *__restrict__ bsum, uint32_t *__restrict__ cnt)
{
    const uint32_t n = mail->n_valid;
    const uint32_t i = blockIdx.x * BK_REC_BLOCK + threadIdx.x;
    const uint32_t sz = i < n ? size[i] : 0;
    uint32_t tot, ns;
    block_excl_scan(sz, &tot);
    block_excl_scan(sz ? 1u : 0u, &ns);
    if (threadIdx.x == 0) { bsum[blockIdx.x] = tot; cnt[blockIdx.x] = ns; }
}

/* exclusive scans of both; totals and the "fits the output buffer" decision into the mail */
__global__ void __launch_bounds__(256) k_small_scan2(uint64_t *bsum, uint32_t *cnt, uint32_t nb, unsigned long long cap_out, struct bk_mail *mail)
{
    unsigned long long cb = 0, cc = 0;
    for (uint32_t b = 0; b < nb; b += 256) {
        const uint32_t i = b + threadIdx.x;
        unsigned long long v = i < nb ? (unsigned long long) bsum[i] : 0, w = i < nb ? (unsigned long long) cnt[i] : 0, tv, tw;
        unsigned long long ev = block_excl_scan_t<unsigned long long>(v, &tv);
        unsigned long long ew = block_excl_scan_t<unsigned long long>(w, &tw);
        if (i < nb) { bsum[i] = cb + ev; cnt[i] = (uint32_t) (cc + ew); }
        cb += tv; cc += tw;
    }
    if (threadIdx.x == 0) { mail->total = cb; mail->n_out = cc; mail->emitted = (cb <= cap_out && !mail->overflow) ? 1u : 0u; }
}

/* ---- streaming JSON packer: one lane per stream buffer (dev_jsmn.cuh) ---- */
__global__ void __launch_bounds__(64) k_jsmn_scan(const struct bk_jsmn_args a)
{
    const uint32_t i = blockIdx.x * 64 + threadIdx.x;
    if (i >= a.n) return;
    const uint8_t *js = a.d_js + a.d_off[i];
    struct jm_tok *tok = a.d_tok + a.d_tok_off[i];
    uint32_t toknext = 0;
    const int tret = jm_tokenise(js, a.d_len[i], tok, a.d_tok_cap[i], &toknext);
    struct jm_result r;
    r.tret = tret; r.pad = 0;
    if (tret == JM_NOMEM) { r.status = JM_NOMEM; r.last_byte = 0; r.tokens_count = 0; r.records = 0; r.out_size = 0; r.toknext = toknext; }
    else jm_pack(js, a.d_len[i], tok, toknext, tret, 0, a.d_tmp + a.d_off[i] + i, &r);
    a.d_res[i] = r;
}

__global__ void __launch_bounds__(64) k_jsmn_emit(const struct bk_jsmn_args a)
{
    const uint32_t i = blockIdx.x * 64 + threadIdx.x;
    if (i >= a.n) return;
    struct jm_result r = a.d_res[i];
    if (r.status != JM_OK || r.out_size == 0) return;
    jm_pack(a.d_js + a.d_off[i], a.d_len[i], a.d_tok + a.d_tok_off[i], r.toknext, r.tret, a.d_out + a.d_out_off[i], a.d_tmp + a.d_off[i] + i, &r);
}

/* ------------------------------------------------------------ bk_* seam */
/* persistent worker threads of a queue: idle on a condition variable, woken for one job at a time */
struct bk_pool {
    std::mutex m;
    std::condition_variable cv, cv_done;
    std::vector<std::thread> th;
    long gen = 0;
    int running = 0;
    bool quit = false;
    void (*fn)(void *, int) = 0;
    void *arg = 0;
    int device = 0;

    void loop(int t)
    {
        long seen = 0;
        cudaSetDevice(device);
        for (;;) {
            void (*f)(void *, int); void *a;
            {
                std::unique_lock<std::mutex> lk(m);
                cv.wait(lk, [&] { return quit || gen != seen; });
                if (quit) return;
                seen = gen; f = fn; a = arg;
            }
            f(a, t);
            {
                std::lock_guard<std::mutex> lk(m);
                if (--running == 0) cv_done.notify_all();
            }
        }
    }
    void ensure(int n, int dev)
    {
        device = dev;
        while ((int) th.size() < n) { const int t = (int) th.size(); th.emplace_back([this, t] { loop(t); }); }
    }
    void run(void (*f)(void *, int), void *a)        /* every thread calls f(a, t) once */
    {
        std::lock_guard<std::mutex> lk(m);
        fn = f; arg = a; running = (int) th.size(); gen++;
        cv.notify_all();
    }
    void wait()
    {
        std::unique_lock<std::mutex> lk(m);
        cv_done.wait(lk, [&] { return running == 0; });
    }
    ~bk_pool()
    {
        { std::lock_guard<std::mutex> lk(m); quit = true; cv.notify_all(); }
        for (auto &t : th) t.join();
    }
};

#define EV_MAX 1024
#define UP_PIECE ((size_t) 32 << 20)
#define UP_MAX_EV 256
#define UP_THREADS_MAX 16
#define UP_STAGE_SLOTS_MAX 32
static int UP_THREADS = 6, UP_STAGE_SLOTS = 12;      /* FLBGPU_UP_THREADS: host threads staging a pageable chunk (slots = 2 x threads) */
#define XF_MAX_SLOTS 32
#define XF_MAX_RANGES 512

struct bk_q {
    int device;
    cudaStream_t stream, istream, h2d, copy;
    cudaStream_t dstream;                  /* split evaluation: the follow-up launch over the records put off runs beside the tail launch */
    cudaEvent_t d_ev[2];
    /* CUDA-event timing of the kernel groups of the last call: one event pair per launch
     * (0 = index, 1 = evaluate, 2 = emit); bk_kernel_ms() sums the pairs of a group. */
    cudaEvent_t evp[3][EV_MAX][2];
    int ev_made[3], ev_used[3];
    /* small device scratch */
    unsigned long long *dtotal;            /* [0] totals, [1..] index results, [8] records emitted */
    uint32_t *dbreaks;
    uint32_t *d_cnt, *d_lrec; uint64_t *d_loff; unsigned long long *d_nlist; size_t cap_b, cap_r;
    uint32_t *d_link[2]; uint8_t *d_mark; size_t cap_link;
    unsigned long long *h_word;            /* pinned: a few words read back per call */
    struct bk_mail *d_mail, *h_mail;       /* small form */
    uint32_t *h_flags;                     /* pinned copy of the evidence words */
    uint8_t *h_sin, *h_sout; size_t cap_sin, cap_sout;    /* small form: pinned staging for the chunk and its result */
    cudaEvent_t ev_small;
    int json_bm;                           /* FLBGPU_JSON_BM=1: two-stage JSON tokenizer (stage-1 bitmap + bit-scan walker + deferral).
                                              Off by default in the single launch: slower there than the byte scanner
                                              -- the walker's lanes diverge on the value type */
    int eval_block;                        /* FLBGPU_EVAL_BLOCK: threads per evaluation block */
    int n_sm;                              /* multiprocessors of the device: the grid of the grid-stride launches */
    uint8_t *d_tag; size_t cap_tag;        /* rewrite_tag: the tag of the call; the re-tagged stream before it goes to the host */
    uint8_t *d_eout; size_t cap_eout;
    unsigned long long *d_stage; size_t cap_stage;   /* index: what the counting pass validated, one row per tile */
    uint32_t *d_tlist; size_t cap_tlist;   /* split evaluation: the records the head launch left for the tail launch */
    uint32_t *d_defer; size_t cap_defer;   /* records the JSON stage-2 walker put off to the follow-up launch */
    /* upload */
    cudaEvent_t up_ev[UP_MAX_EV]; int up_ev_made;
    size_t up_total, up_piece; int up_active, up_staged;
    uint8_t *up_stage[UP_STAGE_SLOTS_MAX]; int up_stage_ready;
    std::atomic<int> up_recorded[UP_MAX_EV];
    std::atomic<long> up_next_issue;
    std::atomic<int> up_failed;
    uint8_t *up_dst; const uint8_t *up_src; size_t up_n, up_np;
    bk_pool *up_pool; int up_running;
    /* download: ring geometry FLBGPU_XF_SLOTS staging buffers (one copy-out thread each) of FLBGPU_XF_MB MiB */
    int xf_slots; size_t xf_slice;
    cudaEvent_t xf_rev[XF_MAX_RANGES];
    int xf_rev_made;
    uint8_t *xf_ring[XF_MAX_SLOTS];
    cudaEvent_t xf_ev[XF_MAX_SLOTS];
    int xf_ready;
    uint8_t *xf_dst; const uint8_t *xf_src;
    std::atomic<long> xf_issued[XF_MAX_SLOTS], xf_done[XF_MAX_SLOTS];
    size_t xf_off[XF_MAX_SLOTS], xf_len[XF_MAX_SLOTS];
    std::atomic<long> xf_n_issued;          /* ring slices issued so far */
    std::atomic<int> xf_closed, xf_failed;
    /* byte ranges handed over by bk_download_push(); the issuer thread turns them into ring slices so
     * that the caller (which also drives indexing and evaluation of the next slice) never blocks on a
     * full ring.  The range slots are a ring themselves. */
    size_t xf_lo[XF_MAX_RANGES], xf_hi[XF_MAX_RANGES];
    std::atomic<long> xf_n_pushed, xf_n_taken;
    std::atomic<int> xf_push_closed;
    bk_pool *xf_pool; int xf_open;
    /* metric-table exchange */
    ncclComm_t comm; int comm_ranks, comm_rank;
};

static inline void use(bk_q *q) { cudaSetDevice(q->device); }

/* Waiting for another thread: a few yields, then short sleeps.  A thread that spins through a whole staging wait burns
 * a core for nothing -- and an agent running under a CPU quota (cgroup cpu.max) pays for that with throttling of the
 * threads that do have work.  The hand-offs here are milliseconds apart; 50 us of extra latency is nothing. */
#include <time.h>
struct bk_backoff {
    int n = 0;
    void wait() { if (n++ < 32) sched_yield(); else { struct timespec ts = { 0, 50000 }; nanosleep(&ts, 0); } }
};

/* ---- NCCL, resolved at run time ---- */
static struct {
    void *dso;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *);
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int);
    ncclResult_t (*CommDestroy)(ncclComm_t);
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
    const char *(*GetErrorString)(ncclResult_t);
} N;
static std::mutex g_nccl_lock;

static int nccl_load(void)
{
    std::lock_guard<std::mutex> lk(g_nccl_lock);
    if (N.dso) return 0;
    const char *path = getenv("FLBGPU_NCCL_LIB");
    void *h = dlopen(path && *path ? path : "libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { snprintf(g_err, sizeof(g_err), "cannot open libnccl.so.2 (%s): the metric-table exchange needs NCCL", dlerror()); return -1; }
#define NSYM(f) do { *(void **) &N.f = dlsym(h, "nccl" #f); if (!N.f) { snprintf(g_err, sizeof(g_err), "libnccl lacks nccl" #f); dlclose(h); return -1; } } while (0)
    NSYM(GetUniqueId); NSYM(CommInitRank); NSYM(CommDestroy); NSYM(AllGather); NSYM(AllReduce); NSYM(GetErrorString);
#undef NSYM
    N.dso = h;
    return 0;
}
#define NK(call) do { ncclResult_t r_ = (call); if (r_ != ncclSuccess) { \
    snprintf(g_err, sizeof(g_err), "%s: %s", #call, N.GetErrorString(r_)); return -1; } } while (0)



static void ev_begin_on(bk_q *q, int k, cudaStream_t st)
{
    if (q->ev_used[k] >= EV_MAX) return;
    if (q->ev_used[k] >= q->ev_made[k]) {
        cudaEventCreate(&q->evp[k][q->ev_made[k]][0]); cudaEventCreate(&q->evp[k][q->ev_made[k]][1]);
        q->ev_made[k]++;
    }
    cudaEventRecord(q->evp[k][q->ev_used[k]][0], st);
}
static void ev_end_on(bk_q *q, int k, cudaStream_t st)
{
    if (q->ev_used[k] >= EV_MAX) return;
    cudaEventRecord(q->evp[k][q->ev_used[k]][1], st);
    q->ev_used[k]++;
}

extern "C" {

const char *bk_name(void) { return "cuda-sm_90a"; }
const char *bk_last_error(void) { return g_err; }
uint64_t bk_launch_count(void) { return g_launches.load(); }
/* for the other translation units of the back end (kernels_ml.cu): the launch counter and the calling thread's error text */
void bk_note_launches(unsigned n) { g_launches += n; }
void bk_note_error(const char *what, const char *detail) { snprintf(g_err, sizeof(g_err), "%s: %s", what, detail); }
void bk_ev_begin(bk_q *q, int k) { ev_begin_on(q, k, q->stream); }
void bk_ev_end(bk_q *q, int k) { ev_end_on(q, k, q->stream); }

int bk_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

/* Keep this process's host side next to its GPU: the threads that stage, copy out and allocate the
 * pinned rings run on the CPUs local to the device's PCIe root (sysfs local_cpulist), so first-touch
 * places those buffers on that NUMA node.  Opt-in (FLBGPU_NUMA_BIND=1): on the bench box, with four
 * GPUs behind one socket, confining four processes to that socket lost 15 % end to end. */
static void bind_near_device(int device)
{
    char bus[32], path[128], line[1024];
    const char *e = getenv("FLBGPU_NUMA_BIND");
    FILE *f;
    cpu_set_t set;
    int any = 0;
    if (!(e && e[0] == '1')) return;
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return; }
    for (char *c = bus; *c; c++) if (*c >= 'A' && *c <= 'F') *c = (char) (*c + 32);
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", bus);
    f = fopen(path, "r");
    if (!f) return;
    if (!fgets(line, sizeof(line), f)) { fclose(f); return; }
    fclose(f);
    CPU_ZERO(&set);
    for (char *p = line; *p && *p != '\n'; ) {            /* "0-31,64-95" */
        char *end;
        long a = strtol(p, &end, 10), b = a;
        if (end == p) break;
        if (*end == '-') { p = end + 1; b = strtol(p, &end, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET((int) c, &set); any = 1; }
        p = (*end == ',') ? end + 1 : end;
    }
    if (any) sched_setaffinity(0, sizeof(set), &set);
}

static int func_attrs_once(void)
{
    /* The interpreter keeps its field list and backtrack stack in local memory: as much L1 as possible -- but the JSON
     * stage-1 bitmaps need 9 KB of shared memory per 256-lane block, and four blocks have to stay resident per SM (a
     * carve-out sized for one block would cost three quarters of the occupancy): 20 % of the unified array. */
    const char *e = getenv("FLBGPU_EVAL_CARVEOUT");
    int pct = e ? atoi(e) : 20;
    if (pct < 0 || pct > 100) pct = 20;
    CK(cudaFuncSetAttribute(k_chain_eval, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    CK(cudaFuncSetAttribute(k_chain_eval_t<CH_PH_HEAD>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    CK(cudaFuncSetAttribute(k_chain_eval_t<CH_PH_TAIL>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
    /* the emission kernel stages a warp's result range in shared memory (6 blocks x 32 KB per SM) */
    CK(cudaFuncSetAttribute(k_chain_emit_list, cudaFuncAttributePreferredSharedMemoryCarveout, 80));
    cudaGetLastError();
    return 0;
}

void bk_q_free(bk_q *q)
{
    if (!q) return;
    use(q);
    if (q->stream) cudaStreamSynchronize(q->stream);
    if (q->comm && N.CommDestroy) N.CommDestroy(q->comm);
    delete q->up_pool; delete q->xf_pool;
    for (int k = 0; k < 3; k++) for (int i = 0; i < q->ev_made[k]; i++) { cudaEventDestroy(q->evp[k][i][0]); cudaEventDestroy(q->evp[k][i][1]); }
    for (int i = 0; i < q->up_ev_made; i++) cudaEventDestroy(q->up_ev[i]);
    for (int i = 0; i < q->xf_rev_made; i++) cudaEventDestroy(q->xf_rev[i]);
    for (int i = 0; i < UP_STAGE_SLOTS_MAX; i++) cudaFreeHost(q->up_stage[i]);
    if (q->xf_ready) for (int i = 0; i < q->xf_slots; i++) { cudaFreeHost(q->xf_ring[i]); cudaEventDestroy(q->xf_ev[i]); }
    cudaFree(q->dtotal); cudaFree(q->dbreaks); cudaFree(q->d_cnt); cudaFree(q->d_lrec); cudaFree(q->d_loff); cudaFree(q->d_nlist);
    cudaFree(q->d_link[0]); cudaFree(q->d_link[1]); cudaFree(q->d_mark); cudaFree(q->d_mail); cudaFree(q->d_defer); cudaFree(q->d_tlist); cudaFree(q->d_stage); cudaFree(q->d_tag); cudaFree(q->d_eout);
    cudaFreeHost(q->h_word); cudaFreeHost(q->h_mail); cudaFreeHost(q->h_flags); cudaFreeHost(q->h_sin); cudaFreeHost(q->h_sout);
    if (q->ev_small) cudaEventDestroy(q->ev_small);
    if (q->stream) cudaStreamDestroy(q->stream);
    if (q->istream) cudaStreamDestroy(q->istream);
    if (q->h2d) cudaStreamDestroy(q->h2d);
    if (q->copy) cudaStreamDestroy(q->copy);
    if (q->dstream) cudaStreamDestroy(q->dstream);
    if (q->d_ev[0]) cudaEventDestroy(q->d_ev[0]);
    if (q->d_ev[1]) cudaEventDestroy(q->d_ev[1]);
    cudaGetLastError();
    q->~bk_q();
    free(q);
}

static int q_setup(bk_q *q)
{
    int lo = 0, hi = 0;
    CK(cudaSetDevice(q->device));
    if (func_attrs_once()) return -1;
    CK(cudaDeviceGetAttribute(&q->n_sm, cudaDevAttrMultiProcessorCount, q->device));
    CK(cudaStreamCreateWithFlags(&q->stream, cudaStreamNonBlocking));
    /* the index kernels of the next slice are short and the host waits for their result: let their
     * blocks go ahead of the thousands of queued evaluation blocks of the previous slice */
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CK(cudaStreamCreateWithPriority(&q->istream, cudaStreamNonBlocking, hi));
    CK(cudaStreamCreateWithFlags(&q->h2d, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&q->copy, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&q->dstream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&q->d_ev[0], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&q->d_ev[1], cudaEventDisableTiming));
    CK(cudaMalloc((void **) &q->dtotal, 128));
    CK(cudaMemset(q->dtotal, 0, 128));
    CK(cudaMalloc((void **) &q->dbreaks, sizeof(uint32_t) * BK_MAX_BREAKS));
    CK(cudaMalloc((void **) &q->d_nlist, 64));
    CK(cudaMalloc((void **) &q->d_mail, sizeof(struct bk_mail)));
    CK(cudaMallocHost((void **) &q->h_word, 128));
    CK(cudaMallocHost((void **) &q->h_mail, sizeof(struct bk_mail)));
    CK(cudaMallocHost((void **) &q->h_flags, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1)));
    {
        const char *eb = getenv("FLBGPU_EVAL_BLOCK");
        q->eval_block = eb ? atoi(eb) : (int) BK_REC_BLOCK;
        if (q->eval_block != 128 && q->eval_block != 256 && q->eval_block != 512 && q->eval_block != 1024) q->eval_block = (int) BK_REC_BLOCK;
    }
    {
        const char *e = getenv("FLBGPU_JSON_BM");
        q->json_bm = e ? (e[0] == '1') : -1;           /* unset: with the split evaluation only (measured: faster there, slower in the single launch) */
    }
    return 0;
}

bk_q *bk_q_new(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    void *mem;
    bk_q *q;
    if (e != cudaSuccess || n <= 0) {
        snprintf(g_err, sizeof(g_err), "no CUDA device available (%s); libflbgpu has no CPU path",
                 e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
        return 0;
    }
    if (device < 0 || device >= n) { snprintf(g_err, sizeof(g_err), "device %d out of range (0..%d)", device, n - 1); return 0; }
    {
        static int once;
        const char *e = getenv("FLBGPU_UP_THREADS");
        if (!once && e && atoi(e) >= 1 && atoi(e) <= UP_THREADS_MAX) { UP_THREADS = atoi(e); UP_STAGE_SLOTS = 2 * UP_THREADS; }
        once = 1;
    }
    mem = calloc(1, sizeof(bk_q));
    if (!mem) { snprintf(g_err, sizeof(g_err), "out of memory"); return 0; }
    q = new (mem) bk_q;
    q->device = device;
    q->xf_slots = 16;                 /* 16 x 8 MiB; FLBGPU_XF_SLOTS / FLBGPU_XF_MB */
    q->xf_slice = (size_t) 8 << 20;
    if (cudaSetDevice(device) != cudaSuccess) { snprintf(g_err, sizeof(g_err), "cudaSetDevice(%d) failed", device); q->~bk_q(); free(q); return 0; }
    bind_near_device(device);
    if (q_setup(q)) { bk_q_free(q); return 0; }
    return q;
}

int bk_q_device(bk_q *q) { return q->device; }

/* 64 bytes of slack: djf_scan_plain reads whole aligned 8-byte words */
void *bk_alloc(bk_q *q, size_t n) { void *p = 0; use(q); if (cudaMalloc(&p, n + 64) != cudaSuccess) { cudaGetLastError(); snprintf(g_err, sizeof(g_err), "cudaMalloc(%zu) failed", n); return 0; } return p; }
void bk_free(bk_q *q, void *p) { if (p) { use(q); cudaFree(p); } }
void *bk_alloc_host(bk_q *q, size_t n) { void *p = 0; use(q); if (cudaMallocHost(&p, n ? n : 16) != cudaSuccess) { cudaGetLastError(); return 0; } return p; }
void bk_free_host(bk_q *q, void *p) { if (p) { use(q); cudaFreeHost(p); } }
int bk_h2d(bk_q *q, void *d, const void *h, size_t n) { use(q); CK(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, q->stream)); return 0; }
int bk_d2h(bk_q *q, void *h, const void *d, size_t n) { use(q); CK(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, q->stream)); return 0; }
int bk_zero(bk_q *q, void *d, size_t n) { use(q); CK(cudaMemsetAsync(d, 0, n, q->stream)); return 0; }
int bk_sync(bk_q *q) { use(q); CK(cudaStreamSynchronize(q->stream)); return 0; }
void *bk_stream(bk_q *q) { return (void *) q->stream; }

/* milliseconds of [index, evaluate (last pass), emit] of the last call; needs a prior bk_sync() */
int bk_kernel_ms(bk_q *q, float out[3])
{
    use(q);
    for (int k = 0; k < 3; k++) {
        out[k] = 0.f;
        for (int i = 0; i < q->ev_used[k]; i++) {
            float ms = 0.f;
            if (cudaEventSynchronize(q->evp[k][i][1]) == cudaSuccess &&
                cudaEventElapsedTime(&ms, q->evp[k][i][0], q->evp[k][i][1]) == cudaSuccess) out[k] += ms;
        }
    }
    return 0;
}

/* ---- upload: pieces with events ----
 * Pageable input (a chunk that lives in ordinary malloc()ed memory, as Fluent Bit's do): the driver
 * would stage every cudaMemcpyAsync itself, synchronously and single-threaded.  Instead UP_THREADS host
 * threads copy the pieces into pinned staging buffers in parallel and enqueue the H2D copies in piece
 * order; up_recorded[i] tells the indexing side when piece i's event exists. */
static void up_worker(void *arg, int t)
{
    bk_q *q = (bk_q *) arg;
    const size_t n = q->up_n, piece = q->up_piece, np = q->up_np;
    for (size_t i = (size_t) t; i < np; i += UP_THREADS) {
        const int slot = (int) (i % UP_STAGE_SLOTS);
        const size_t off = i * piece, sz = (off + piece <= n) ? piece : n - off;
        /* the slot was last used by piece i - UP_STAGE_SLOTS: its H2D must have left the buffer */
        if (i >= UP_STAGE_SLOTS) {
            for (bk_backoff b; !q->up_recorded[i - UP_STAGE_SLOTS].load(std::memory_order_acquire); b.wait()) if (q->up_failed.load()) return;
            if (cudaEventSynchronize(q->up_ev[i - UP_STAGE_SLOTS]) != cudaSuccess) { q->up_failed.store(1); return; }
        }
        if (!q->up_stage[slot] && cudaMallocHost((void **) &q->up_stage[slot], UP_PIECE) != cudaSuccess) { q->up_failed.store(1); q->up_next_issue.store((long) i + 1); return; }
        memcpy(q->up_stage[slot], q->up_src + off, sz);
        for (bk_backoff b; q->up_next_issue.load(std::memory_order_acquire) != (long) i; b.wait()) if (q->up_failed.load()) return;
        if (cudaMemcpyAsync(q->up_dst + off, q->up_stage[slot], sz, cudaMemcpyHostToDevice, q->h2d) != cudaSuccess ||
            cudaEventRecord(q->up_ev[i], q->h2d) != cudaSuccess) { q->up_failed.store(1); q->up_next_issue.store((long) i + 1); return; }
        q->up_recorded[i].store(1, std::memory_order_release);
        q->up_next_issue.store((long) i + 1, std::memory_order_release);
    }
}

void bk_upload_end(bk_q *q)
{
    if (q->up_running) { q->up_pool->wait(); q->up_running = 0; }
}

int bk_upload_start(bk_q *q, void *d_dst, const void *h_src, size_t n)
{
    use(q);
    bk_upload_end(q);
    q->up_piece = UP_PIECE;
    while ((n + q->up_piece - 1) / q->up_piece > UP_MAX_EV) q->up_piece *= 2;
    const size_t np = (n + q->up_piece - 1) / q->up_piece;
    for (; q->up_ev_made < (int) np; q->up_ev_made++) CK(cudaEventCreateWithFlags(&q->up_ev[q->up_ev_made], cudaEventDisableTiming | cudaEventBlockingSync));
    q->up_total = n; q->up_active = 1; q->up_staged = 0;
    {
        cudaPointerAttributes at;
        const int pinned = cudaPointerGetAttributes(&at, h_src) == cudaSuccess && (at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged);
        cudaGetLastError();
        if (!pinned && q->up_piece == UP_PIECE && !getenv("FLBGPU_NO_STAGING")) {
            q->up_stage_ready = 1;                 /* the pinned staging slots are allocated by the thread that first uses them */
            if (!q->up_pool) { q->up_pool = new bk_pool; q->up_pool->ensure(UP_THREADS, q->device); }
            for (size_t i = 0; i < np; i++) q->up_recorded[i].store(0);
            q->up_next_issue.store(0); q->up_failed.store(0);
            q->up_staged = 1;
            q->up_dst = (uint8_t *) d_dst; q->up_src = (const uint8_t *) h_src; q->up_n = n; q->up_np = np;
            q->up_pool->run(up_worker, q);
            q->up_running = 1;
            return 0;
        }
    }
    for (size_t i = 0; i < np; i++) {
        const size_t off = i * q->up_piece, sz = (off + q->up_piece <= n) ? q->up_piece : n - off;
        CK(cudaMemcpyAsync((uint8_t *) d_dst + off, (const uint8_t *) h_src + off, sz, cudaMemcpyHostToDevice, q->h2d));
        CK(cudaEventRecord(q->up_ev[i], q->h2d));
    }
    return 0;
}
void bk_upload_none(bk_q *q) { bk_upload_end(q); q->up_active = 0; }
int bk_upload_wait_index(bk_q *q, size_t upto)
{
    use(q);
    if (!q->up_active || upto == 0) return 0;
    if (upto > q->up_total) upto = q->up_total;
    const size_t last = (upto - 1) / q->up_piece;
    if (q->up_staged) {
        for (bk_backoff b; !q->up_recorded[last].load(std::memory_order_acquire); b.wait())
            if (q->up_failed.load()) { snprintf(g_err, sizeof(g_err), "host->device staging failed"); return -1; }
    }
    CK(cudaStreamWaitEvent(q->istream, q->up_ev[last], 0));
    return 0;
}

/* ---- download session: pinned ring + one persistent host thread per slot + the issuer ---- */
static int xf_init(bk_q *q)
{
    if (q->xf_ready) return 0;
    {
        const char *es = getenv("FLBGPU_XF_SLOTS"), *em = getenv("FLBGPU_XF_MB");
        if (es && atoi(es) >= 2 && atoi(es) <= XF_MAX_SLOTS) q->xf_slots = atoi(es);
        if (em && atoi(em) >= 1 && atoi(em) <= 256) q->xf_slice = (size_t) atoi(em) << 20;
    }
    for (int i = 0; i < q->xf_slots; i++) CK(cudaEventCreateWithFlags(&q->xf_ev[i], cudaEventDisableTiming | cudaEventBlockingSync));   /* ring buffers: on first use */
    q->xf_pool = new bk_pool;
    q->xf_pool->ensure(q->xf_slots + 1, q->device);
    q->xf_ready = 1;
    return 0;
}

static void xf_copy_out(bk_q *q, int s)
{
    for (long i = s;; i += q->xf_slots) {
        for (bk_backoff b; q->xf_issued[s].load(std::memory_order_acquire) < i; b.wait()) {
            if (q->xf_failed.load()) return;
            if (q->xf_closed.load() && q->xf_n_issued.load() <= i) return;
        }
        if (cudaEventSynchronize(q->xf_ev[s]) != cudaSuccess) { q->xf_failed.store(1); return; }
        flbgpu_stream_copy(q->xf_dst + q->xf_off[s], q->xf_ring[s], q->xf_len[s]);
        q->xf_done[s].store(i, std::memory_order_release);
    }
}

static void xf_issue(bk_q *q)
{
    for (long r = 0;; r++) {
        for (bk_backoff b; q->xf_n_pushed.load(std::memory_order_acquire) <= r; b.wait()) {
            if (q->xf_failed.load() || q->xf_push_closed.load()) {
                if (q->xf_n_pushed.load(std::memory_order_acquire) > r) break;
                q->xf_closed.store(1);
                return;
            }
        }
        const int rs = (int) (r % XF_MAX_RANGES);
        const size_t lo = q->xf_lo[rs], hi = q->xf_hi[rs];
        /* bytes [lo,hi) exist once the emission recorded in xf_rev[rs] is done */
        if (cudaStreamWaitEvent(q->copy, q->xf_rev[rs], 0) != cudaSuccess) { q->xf_failed.store(1); q->xf_closed.store(1); return; }
        q->xf_n_taken.store(r + 1, std::memory_order_release);          /* the range slot may be used again */
        for (size_t off = lo; off < hi && !q->xf_failed.load(); off += q->xf_slice) {
            const long i = q->xf_n_issued.load();
            const int s = (int) (i % q->xf_slots);
            const size_t sz = (off + q->xf_slice <= hi) ? q->xf_slice : hi - off;
            if (i >= q->xf_slots) for (bk_backoff b; q->xf_done[s].load(std::memory_order_acquire) < i - q->xf_slots; b.wait()) if (q->xf_failed.load()) break;
            q->xf_off[s] = off; q->xf_len[s] = sz;
            if (!q->xf_ring[s] && cudaMallocHost((void **) &q->xf_ring[s], q->xf_slice) != cudaSuccess) { q->xf_failed.store(1); break; }
            if (cudaMemcpyAsync(q->xf_ring[s], q->xf_src + off, sz, cudaMemcpyDeviceToHost, q->copy) != cudaSuccess ||
                cudaEventRecord(q->xf_ev[s], q->copy) != cudaSuccess) { q->xf_failed.store(1); break; }
            q->xf_issued[s].store(i, std::memory_order_release);
            q->xf_n_issued.store(i + 1);
        }
    }
}

static void xf_worker(void *arg, int t)
{
    bk_q *q = (bk_q *) arg;
    if (t == q->xf_slots) xf_issue(q); else xf_copy_out(q, t);
}

int bk_download_begin(bk_q *q, void *h_dst, const void *d_out)
{
    use(q);
    if (xf_init(q)) return -1;
    q->xf_dst = (uint8_t *) h_dst; q->xf_src = (const uint8_t *) d_out;
    for (int s = 0; s < q->xf_slots; s++) { q->xf_issued[s].store(-1); q->xf_done[s].store(-1); }
    q->xf_n_issued.store(0); q->xf_closed.store(0); q->xf_failed.store(0);
    q->xf_n_pushed.store(0); q->xf_n_taken.store(0); q->xf_push_closed.store(0);
    q->xf_pool->run(xf_worker, q);
    q->xf_open = 1;
    return 0;
}

int bk_download_push(bk_q *q, size_t lo, size_t hi)
{
    use(q);
    if (!q->xf_open) return -1;
    if (hi <= lo) return 0;
    const long r = q->xf_n_pushed.load();
    for (bk_backoff b; r - q->xf_n_taken.load(std::memory_order_acquire) >= XF_MAX_RANGES; b.wait()) if (q->xf_failed.load()) return -1;
    const int rs = (int) (r % XF_MAX_RANGES);
    for (; q->xf_rev_made <= rs; q->xf_rev_made++) CK(cudaEventCreateWithFlags(&q->xf_rev[q->xf_rev_made], cudaEventDisableTiming));
    CK(cudaEventRecord(q->xf_rev[rs], q->stream));
    q->xf_lo[rs] = lo; q->xf_hi[rs] = hi;
    q->xf_n_pushed.store(r + 1, std::memory_order_release);
    return q->xf_failed.load() ? -1 : 0;
}

int bk_download_end(bk_q *q)
{
    int rc = 0;
    if (!q->xf_open) return -1;
    q->xf_push_closed.store(1);
    q->xf_pool->wait();
    q->xf_open = 0;
    if (q->xf_failed.load()) { use(q); snprintf(g_err, sizeof(g_err), "device->host transfer failed: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
    return rc;
}

int bk_d2d_2d(bk_q *q, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows)
{
    use(q);
    CK(cudaMemcpy2D(dst, dpitch, src, spitch, width, rows, cudaMemcpyDeviceToDevice));
    return 0;
}

int bk_rx_search_host(const void *prog, const uint8_t *s, int n, int *caps)
{
    uint32_t stk[1024], budget = CH_RX_BUDGET;
    return rx_search((const struct rx_prog *) prog, s, n, caps, stk, 1024, &budget);
}

int bk_d2d(bk_q *q, void *dst, const void *src, size_t n)
{
    use(q);
    CK(cudaMemcpy(dst, src, n, cudaMemcpyDeviceToDevice));
    return 0;
}

/* staging rows of the index for n_tiles tiles (k_index) */
static int stage_setup(bk_q *q, uint32_t n_tiles)
{
    if (q->cap_stage >= (size_t) n_tiles) return 0;
    CK(cudaStreamSynchronize(q->istream));
    CK(cudaStreamSynchronize(q->stream));
    cudaFree(q->d_stage); q->d_stage = 0; q->cap_stage = 0;
    CK(cudaMalloc((void **) &q->d_stage, sizeof(unsigned long long) * BK_STAGE_ROW * ((size_t) n_tiles + n_tiles / 4 + 16)));
    q->cap_stage = (size_t) n_tiles + n_tiles / 4 + 16;
    return 0;
}

int bk_index_count(bk_q *q, const uint8_t *d_in, size_t slice_off, uint32_t slice_len, uint32_t *d_tile, uint32_t n_tiles,
                   uint32_t *n_cand)
{
    use(q);
    *n_cand = 0;
    if (n_tiles == 0) return 0;
    ev_begin_on(q, 0, q->istream);
    {
        const uint32_t skip = (uint32_t) ((uintptr_t) (d_in + slice_off) & 15);      /* tiles start at a 16-byte boundary of the address space */
        if (stage_setup(q, n_tiles)) return -1;
        k_index<false><<<n_tiles, 256, 0, q->istream>>>(d_in + slice_off - skip, slice_len + skip, skip, (uint32_t) (slice_off - skip), d_tile, 0, 0, 0, 0, q->d_stage);
    }
    k_scan_top<uint32_t><<<1, 256, 0, q->istream>>>(d_tile, n_tiles, q->dtotal, 0);
    ev_end_on(q, 0, q->istream);
    g_launches += 2;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&q->h_word[0], q->dtotal, sizeof(unsigned long long), cudaMemcpyDeviceToHost, q->istream));
    CK(cudaStreamSynchronize(q->istream));
    *n_cand = (uint32_t) q->h_word[0];
    return 0;
}

int bk_index_fill(bk_q *q, const uint8_t *d_in, size_t slice_off, uint32_t slice_len, const uint32_t *d_tile, uint32_t n_tiles,
                  uint32_t n_cand, uint32_t *d_off, uint32_t *d_len, uint8_t *d_kind,
                  uint32_t *n_valid, uint64_t *end_off, int *tiled)
{
    uint32_t *h = (uint32_t *) &q->h_word[2];
    uint32_t *d_w = (uint32_t *) (q->dtotal + 1);          /* [0] n_breaks, [1] n_valid, [2] tiled, [3] end offset, [4] overflow */
    use(q);
    *n_valid = 0; *tiled = (slice_len == 0); *end_off = slice_off;
    if (n_cand == 0) return 0;
    ev_begin_on(q, 0, q->istream);
    {
        const uint32_t skip = (uint32_t) ((uintptr_t) (d_in + slice_off) & 15);      /* tiles start at a 16-byte boundary of the address space */
        k_index<true><<<n_tiles, 256, 0, q->istream>>>(d_in + slice_off - skip, slice_len + skip, skip, (uint32_t) (slice_off - skip), (uint32_t *) d_tile, d_off, d_len, d_kind, 0,
                                                       q->cap_stage >= (size_t) n_tiles ? q->d_stage : 0);
    }
    CK(cudaMemsetAsync(d_w, 0, 32, q->istream));
    k_index_check<<<(n_cand + 255) / 256, 256, 0, q->istream>>>(d_off, d_len, n_cand, 0, (uint32_t) (slice_off + slice_len), d_w, q->dbreaks);
    k_index_repair<<<1, 1024, 0, q->istream>>>(d_off, d_len, d_kind, n_cand, 0, (uint32_t) slice_off, (uint32_t) (slice_off + slice_len), d_w, q->dbreaks, d_w + 1, d_w + 4);
    ev_end_on(q, 0, q->istream);
    g_launches += 3;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h, d_w, 32, cudaMemcpyDeviceToHost, q->istream));
    CK(cudaStreamSynchronize(q->istream));
    if (h[4] == 2) {
        /* more broken links than the one-CTA walk holds (e.g. every record carries a nested [int, {map}]
         * value, which frames as a legacy event): decide the chain by pointer doubling instead */
        const uint32_t nb = (n_cand + 255) / 256, base = (uint32_t) slice_off, total = (uint32_t) (slice_off + slice_len);
        uint32_t steps = 1, cur = 0;
        if (q->cap_link < n_cand) {
            const size_t want = (size_t) n_cand + n_cand / 2 + 1024;
            cudaFree(q->d_link[0]); cudaFree(q->d_link[1]); cudaFree(q->d_mark);
            q->d_link[0] = q->d_link[1] = 0; q->d_mark = 0; q->cap_link = 0;
            CK(cudaMalloc((void **) &q->d_link[0], sizeof(uint32_t) * want));
            CK(cudaMalloc((void **) &q->d_link[1], sizeof(uint32_t) * want));
            CK(cudaMalloc((void **) &q->d_mark, want));
            q->cap_link = want;
        }
        while ((1ull << steps) < (unsigned long long) n_cand + 1) steps++;
        {
            const uint32_t none[3] = { 0, 0, base };    /* candidate 0 does not start the slice: nothing decodable */
            CK(cudaMemcpyAsync(d_w + 1, none, sizeof(none), cudaMemcpyHostToDevice, q->istream));
        }
        ev_begin_on(q, 0, q->istream);
        k_link_next<<<nb, 256, 0, q->istream>>>(d_off, d_len, n_cand, base, total, q->d_link[0], q->d_mark);
        for (uint32_t s = 0; s < steps; s++) {
            k_link_step<<<nb, 256, 0, q->istream>>>(q->d_link[cur], q->d_link[cur ^ 1], q->d_mark, n_cand);
            cur ^= 1;
        }
        /* the jump arrays are spent: recompute next[] (mark untouched: a scratch byte array takes the second output) */
        k_link_next<<<nb, 256, 0, q->istream>>>(d_off, d_len, n_cand, 0xffffffffu, total, q->d_link[0], (uint8_t *) q->d_link[1]);
        k_link_finish<<<nb, 256, 0, q->istream>>>(d_off, d_len, q->d_link[0], q->d_mark, d_kind, n_cand, base, d_w + 1);
        ev_end_on(q, 0, q->istream);
        g_launches += steps + 3;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(h, d_w, 32, cudaMemcpyDeviceToHost, q->istream));
        CK(cudaStreamSynchronize(q->istream));
    }
    *n_valid = h[1];
    *tiled = (int) h[2];
    *end_off = h[3];
    return 0;
}

static void fill_params(const struct bk_chain_args *a, k_chain_params *p, uint8_t *d_out, uint32_t r0)
{
    p->env.in = a->d_in; p->env.in_len = a->in_len; p->env.blob = a->d_blob; p->env.scr = a->d_scr; p->env.scr_mul = a->scr_mul ? a->scr_mul : 4;
    p->env.capcache = a->d_capcache; p->env.cap_stride = a->cap_stride; p->env.cap_n = a->cap_n; p->env.now = a->now;
    p->env.assume = a->assume; p->env.active = a->active; p->env.fl_flags = a->d_flags; p->env.err = a->d_flags + FLBGPU_MAX_FILTERS;
    p->env.l2m = a->l2m; p->env.prep = a->d_prep;
    p->env.esize = a->d_esize; p->env.tag = a->d_tag; p->env.tag_len = a->tag_len;
    p->off = a->d_off; p->len = a->d_len; p->kind = a->d_kind; p->r0 = r0; p->n_rec = a->n_rec; p->bm_words = 0;
    p->n_dev = 0; p->defer_list = 0; p->defer_cnt = 0; p->tlist = 0; p->tn = 0;
    p->size = a->d_size; p->bsum = a->d_bsum; p->out = d_out;
}

int bk_flags_clear(bk_q *q, uint32_t *d_flags)
{
    use(q);
    CK(cudaMemsetAsync(d_flags, 0, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1), q->stream));
    CK(cudaMemsetAsync(q->dtotal + 8, 0, sizeof(unsigned long long), q->stream));      /* records emitted */
    q->ev_used[0] = q->ev_used[1] = q->ev_used[2] = 0;
    return 0;
}

/* The slice of input the next evaluation reads is touched once: mark it as streaming in L2 (access
 * policy window of the stream) so that it does not evict the lanes' local-memory lines (field lists,
 * regex stacks), which are re-used by every block.  It had no measurable effect, so it
 * is opt-in: FLBGPU_L2_WINDOW=1. */
int bk_hint_streaming(bk_q *q, const void *base, size_t bytes)
{
    static int max_win = -1, enabled = -1;
    cudaStreamAttrValue v;
    if (enabled < 0) { const char *e = getenv("FLBGPU_L2_WINDOW"); enabled = (e && e[0] == '1'); }   /* off by default: see above */
    if (!enabled) return 0;
    use(q);
    if (max_win < 0) {
        if (cudaDeviceGetAttribute(&max_win, cudaDevAttrMaxAccessPolicyWindowSize, q->device) != cudaSuccess) max_win = 0;
    }
    if (max_win <= 0 || !base || !bytes) return 0;
    memset(&v, 0, sizeof(v));
    v.accessPolicyWindow.base_ptr = (void *) base;
    v.accessPolicyWindow.num_bytes = bytes < (size_t) max_win ? bytes : (size_t) max_win;
    v.accessPolicyWindow.hitRatio = 1.0f;
    v.accessPolicyWindow.hitProp = cudaAccessPropertyStreaming;
    v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    if (cudaStreamSetAttribute(q->stream, cudaStreamAttributeAccessPolicyWindow, &v) != cudaSuccess) cudaGetLastError();
    return 0;
}

/* deferral list for up to n records; the counter lives in dtotal[9] and is zeroed on `st` */
static int defer_setup(bk_q *q, k_chain_params *p, const struct bk_chain_args *a, size_t n, cudaStream_t st)
{
    p->defer_list = 0; p->defer_cnt = 0;
    if (!(p->bm_words && a->defer_ok) && !a->split) return 0;
    if (q->cap_defer < n) {
        CK(cudaStreamSynchronize(q->stream));           /* a follow-up launch still running reads the old list */
        cudaFree(q->d_defer); q->d_defer = 0; q->cap_defer = 0;
        CK(cudaMalloc((void **) &q->d_defer, sizeof(uint32_t) * (n + n / 4 + 1024)));
        q->cap_defer = n + n / 4 + 1024;
    }
    CK(cudaMemsetAsync(q->dtotal + 9, 0, sizeof(unsigned long long) * 2, st));       /* [9] records put off, [10] records left for the tail launch */
    p->defer_list = q->d_defer; p->defer_cnt = q->dtotal + 9;
    if (a->split) {
        if (q->cap_tlist < n) {
            CK(cudaStreamSynchronize(q->stream));
            cudaFree(q->d_tlist); q->d_tlist = 0; q->cap_tlist = 0;
            CK(cudaMalloc((void **) &q->d_tlist, sizeof(uint32_t) * (n + n / 4 + 1024)));
            q->cap_tlist = n + n / 4 + 1024;
        }
        p->tlist = q->d_tlist; p->tn = (uint32_t *) (q->dtotal + 10);
    }
    return 0;
}

int bk_chain_eval(bk_q *q, const struct bk_chain_args *a, uint32_t r0, uint32_t r1)
{
    k_chain_params p;
    if (r1 <= r0) return 0;
    use(q);
    fill_params(a, &p, 0, r0);
    p.n_rec = r1;
    p.bm_words = (a->d_scr && (q->json_bm > 0 || (q->json_bm < 0 && a->split))) ? BM_BYTES / 32 : 0;          /* a JSON parser is in the chain */
    if (defer_setup(q, &p, a, r1 - r0, q->stream)) return -1;
    ev_begin_on(q, 1, q->stream);
    if (a->split) {
        const unsigned grid = (r1 - r0 + q->eval_block - 1) / q->eval_block;
        k_chain_eval_t<CH_PH_HEAD><<<grid, q->eval_block, (size_t) p.bm_words * 4 * (q->eval_block / 32), q->stream>>>(p);
        /* the records the head put off (a few per cent, one long lane each: ~200 us per slice with most of the GPU idle) are
         * evaluated BESIDE the tail launch -- the two touch different records: the tail only those on the head's list */
        CK(cudaEventRecord(q->d_ev[0], q->stream));
        CK(cudaStreamWaitEvent(q->dstream, q->d_ev[0], 0));
        k_chain_eval_deferred<<<q->n_sm * 4, BK_REC_BLOCK, 0, q->dstream>>>(p);
        CK(cudaEventRecord(q->d_ev[1], q->dstream));
        k_chain_eval_t<CH_PH_TAIL><<<grid, q->eval_block, 0, q->stream>>>(p);
        CK(cudaStreamWaitEvent(q->stream, q->d_ev[1], 0));
        g_launches += 2;
    }
    else {
        k_chain_eval<<<(r1 - r0 + q->eval_block - 1) / q->eval_block, q->eval_block, (size_t) p.bm_words * 4 * (q->eval_block / 32), q->stream>>>(p);
        if (p.defer_list) { k_chain_eval_deferred<<<q->n_sm * 4, BK_REC_BLOCK, 0, q->stream>>>(p); g_launches += 1; }
    }
    if (p.env.l2m.hash) {
        k_chain_skipped<<<(r1 - r0 + BK_REC_BLOCK - 1) / BK_REC_BLOCK, BK_REC_BLOCK, 0, q->stream>>>(p);
        g_launches += 1;
        if (p.env.l2m.pending) { k_l2m_fixup<<<1, 1024, 0, q->stream>>>(p); k_l2m_fixup_done<<<1, 1, 0, q->stream>>>(p); g_launches += 2; }
    }
    ev_end_on(q, 1, q->stream);
    g_launches += 1;
    CK(cudaGetLastError());
    return 0;
}

int bk_flags_fetch(bk_q *q, const uint32_t *d_flags, uint32_t *h_flags)
{
    use(q);
    CK(cudaMemcpyAsync(q->h_flags, d_flags, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1), cudaMemcpyDeviceToHost, q->stream));
    CK(cudaStreamSynchronize(q->stream));
    memcpy(h_flags, q->h_flags, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1));
    return 0;
}

int bk_sizes_scan(bk_q *q, const uint32_t *d_size, uint32_t n_rec, uint64_t *d_bsum, uint64_t *h_bsum)
{
    const uint32_t nb = (n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    use(q);
    h_bsum[0] = 0;
    q->h_word[0] = 0;
    if (nb) {
        k_bsum<<<nb, BK_REC_BLOCK, 0, q->stream>>>(d_size, n_rec, d_bsum);
        k_scan_top<uint64_t><<<1, 256, 0, q->stream>>>(d_bsum, nb, q->dtotal, 0);
        g_launches += 2;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(&q->h_word[0], q->dtotal, sizeof(unsigned long long), cudaMemcpyDeviceToHost, q->stream));
        CK(cudaMemcpyAsync(h_bsum, d_bsum, sizeof(uint64_t) * nb, cudaMemcpyDeviceToHost, q->stream));
    }
    CK(cudaStreamSynchronize(q->stream));
    h_bsum[nb] = q->h_word[0];
    return 0;
}

/* ---- rewrite_tag: the tag of the call on the device, and the re-tagged stream ---- */
int bk_tag_upload(bk_q *q, const char *tag, uint32_t tag_len, const uint8_t **d_tag)
{
    use(q);
    if (q->cap_tag < (size_t) tag_len + 1) {
        CK(cudaStreamSynchronize(q->stream));
        cudaFree(q->d_tag); q->d_tag = 0; q->cap_tag = 0;
        CK(cudaMalloc((void **) &q->d_tag, (size_t) tag_len + 256));
        q->cap_tag = (size_t) tag_len + 256;
    }
    if (tag_len) CK(cudaMemcpyAsync(q->d_tag, tag, tag_len, cudaMemcpyHostToDevice, q->stream));     /* pageable source: staged before the call returns */
    *d_tag = q->d_tag;
    return 0;
}

/* entries of records [0, n_rec): a->d_esize holds their sizes; *h_out = malloc()ed stream of *bytes bytes (NULL when empty) */
int bk_rtag_emit(bk_q *q, const struct bk_chain_args *a, uint32_t n_rec, uint64_t *d_bsum, uint64_t *h_bsum, void **h_out, size_t *bytes)
{
    const uint32_t nb = (n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    k_chain_params p;
    uint64_t total;
    void *out;
    *h_out = 0; *bytes = 0;
    if (!nb) return 0;
    if (bk_sizes_scan(q, a->d_esize, n_rec, d_bsum, h_bsum)) return -1;
    total = h_bsum[nb];
    if (!total) return 0;
    if (total >= 0xfff00000ull) { snprintf(g_err, sizeof(g_err), "re-tagged records larger than 4 GiB"); return -1; }
    if (q->cap_eout < total) {
        cudaFree(q->d_eout); q->d_eout = 0; q->cap_eout = 0;
        CK(cudaMalloc((void **) &q->d_eout, (size_t) total + (size_t) total / 4 + 4096));
        q->cap_eout = (size_t) total + (size_t) total / 4 + 4096;
    }
    fill_params(a, &p, q->d_eout, 0);
    p.n_rec = n_rec; p.size = a->d_esize; p.bsum = d_bsum;
    p.env.esize = 0;                                   /* (the entry sizes are read as p.size; nothing is sized here) */
    k_rtag_emit<<<nb, BK_REC_BLOCK, 0, q->stream>>>(p);
    g_launches += 1;
    CK(cudaGetLastError());
    out = malloc((size_t) total);
    if (!out) { snprintf(g_err, sizeof(g_err), "out of memory"); return -1; }
    if (cudaMemcpyAsync(out, q->d_eout, (size_t) total, cudaMemcpyDeviceToHost, q->stream) != cudaSuccess ||
        cudaStreamSynchronize(q->stream) != cudaSuccess) { free(out); CK(cudaGetLastError()); snprintf(g_err, sizeof(g_err), "copy of the re-tagged records failed"); return -1; }
    *h_out = out; *bytes = (size_t) total;
    return 0;
}

/* Offsets of blocks [b0, b1) when everything before them is already placed: block sums, exclusive
 * scan continued from carry_in, host copy of the new entries; h_bsum[b1] = bytes placed so far. */
__global__ void __launch_bounds__(256) k_scan_carry(uint64_t *a, uint32_t n, unsigned long long *carry_io)
{
    unsigned long long carry = *carry_io;
    for (uint32_t b = 0; b < n; b += 256) {
        const uint32_t i = b + threadIdx.x;
        unsigned long long v = i < n ? (unsigned long long) a[i] : 0, tot;
        unsigned long long ex = block_excl_scan_t<unsigned long long>(v, &tot);
        if (i < n) a[i] = carry + ex;
        carry += tot;
    }
    __syncthreads();
    if (threadIdx.x == 0) *carry_io = carry;
}

int bk_sizes_scan_range(bk_q *q, const uint32_t *d_size, uint32_t n_rec, uint32_t b0, uint32_t b1, uint64_t *d_bsum, uint64_t *h_bsum,
                        uint64_t carry_in)
{
    use(q);
    h_bsum[b0] = carry_in;
    q->h_word[0] = carry_in;
    if (b1 > b0) {
        const uint32_t nb = b1 - b0;
        q->h_word[1] = carry_in;
        CK(cudaMemcpyAsync(q->dtotal, &q->h_word[1], sizeof(unsigned long long), cudaMemcpyHostToDevice, q->stream));
        k_bsum<<<nb, BK_REC_BLOCK, 0, q->stream>>>(d_size + (size_t) b0 * BK_REC_BLOCK, n_rec - b0 * BK_REC_BLOCK, d_bsum + b0);
        k_scan_carry<<<1, 256, 0, q->stream>>>(d_bsum + b0, nb, q->dtotal);
        g_launches += 2;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(&q->h_word[0], q->dtotal, sizeof(unsigned long long), cudaMemcpyDeviceToHost, q->stream));
        CK(cudaMemcpyAsync(h_bsum + b0, d_bsum + b0, sizeof(uint64_t) * nb, cudaMemcpyDeviceToHost, q->stream));
    }
    CK(cudaStreamSynchronize(q->stream));
    h_bsum[b1] = q->h_word[0];
    return 0;
}

/* records emitted since the last bk_flags_clear(); synchronises the library stream */
int bk_records_out(bk_q *q, uint64_t *n)
{
    use(q);
    CK(cudaMemcpyAsync(&q->h_word[0], q->dtotal + 8, sizeof(unsigned long long), cudaMemcpyDeviceToHost, q->stream));
    CK(cudaStreamSynchronize(q->stream));
    *n = q->h_word[0];
    return 0;
}

/* survivor lists for nb blocks */
static int ensure_lists(bk_q *q, uint32_t nb)
{
    if (q->cap_b < nb) { cudaFree(q->d_cnt); q->d_cnt = 0; q->cap_b = 0; CK(cudaMalloc((void **) &q->d_cnt, sizeof(uint32_t) * (nb + nb / 2 + 64))); q->cap_b = nb + nb / 2 + 64; }
    if (q->cap_r < (size_t) nb * BK_REC_BLOCK) {
        const size_t want = (size_t) (nb + nb / 2 + 64) * BK_REC_BLOCK;
        CK(cudaStreamSynchronize(q->stream));           /* an emission still running reads the old lists */
        cudaFree(q->d_lrec); cudaFree(q->d_loff); q->d_lrec = 0; q->d_loff = 0; q->cap_r = 0;
        CK(cudaMalloc((void **) &q->d_lrec, sizeof(uint32_t) * want));
        CK(cudaMalloc((void **) &q->d_loff, sizeof(uint64_t) * want));
        q->cap_r = want;
    }
    return 0;
}

int bk_chain_emit(bk_q *q, const struct bk_chain_args *a, uint8_t *d_out, uint32_t b0, uint32_t b1)
{
    k_chain_params p;
    if (b1 <= b0) return 0;
    use(q);
    fill_params(a, &p, d_out, b0 * BK_REC_BLOCK);
    {
        const uint32_t nb = b1 - b0, rec0 = b0 * BK_REC_BLOCK;
        const uint32_t n = (a->n_rec > rec0) ? ((a->n_rec - rec0 < nb * BK_REC_BLOCK) ? a->n_rec - rec0 : nb * BK_REC_BLOCK) : 0;
        if (ensure_lists(q, nb)) return -1;
        ev_begin_on(q, 2, q->stream);
        k_surv_count<<<nb, BK_REC_BLOCK, 0, q->stream>>>(a->d_size + rec0, n, q->d_cnt);
        k_scan_top<uint32_t><<<1, 256, 0, q->stream>>>(q->d_cnt, nb, q->d_nlist, q->dtotal + 8);
        k_surv_fill<<<nb, BK_REC_BLOCK, 0, q->stream>>>(a->d_size + rec0, n, 0, rec0, q->d_cnt, a->d_bsum + b0, q->d_lrec, q->d_loff);
        k_chain_emit_list<<<nb * (BK_REC_BLOCK / EMIT_BLOCK), EMIT_BLOCK, (EMIT_BLOCK / 32) * (EMIT_STAGE + 16), q->stream>>>(p, q->d_lrec, q->d_loff, q->d_nlist, 0);
        ev_end_on(q, 2, q->stream);
        g_launches += 4;
    }
    CK(cudaGetLastError());
    return 0;
}

/* ---- the small-chunk form: one stream, no host synchronisation until the mail is read ---- */
int bk_small_run(bk_q *q, const struct bk_chain_args *a, const void *h_in, uint8_t *d_in, size_t bytes, uint32_t cap_rec,
                 uint32_t *d_tile, uint32_t n_tiles, uint8_t *d_out, size_t cap_out, struct bk_small_res *res)
{
    k_chain_params p;
    cudaStream_t st = q->stream;
    const uint32_t nb_cap = (cap_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    struct bk_mail *m = q->d_mail;
    use(q);
    memset(res, 0, sizeof(*res));
    if (ensure_lists(q, nb_cap)) return -1;
    bk_upload_none(q);
    if (h_in) {
        /* A pageable source makes cudaMemcpyAsync stage inside the driver, one copy at a time for the whole process;
         * with several instances calling at once that is the bottleneck.  Each queue stages through its own pinned
         * buffer instead, piece by piece so that the DMA of one piece runs while the next is being copied. */
        cudaPointerAttributes at;
        const int pinned = cudaPointerGetAttributes(&at, h_in) == cudaSuccess && (at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged);
        cudaGetLastError();
        if (pinned || bytes < 4096) CK(cudaMemcpyAsync(d_in, h_in, bytes, cudaMemcpyHostToDevice, st));
        else {
            const size_t piece = (size_t) 256 << 10;
            if (q->cap_sin < bytes) {
                cudaFreeHost(q->h_sin); q->h_sin = 0; q->cap_sin = 0;
                CK(cudaMallocHost((void **) &q->h_sin, bytes + bytes / 4 + 65536));
                q->cap_sin = bytes + bytes / 4 + 65536;
            }
            for (size_t off = 0; off < bytes; off += piece) {
                const size_t sz = off + piece <= bytes ? piece : bytes - off;
                memcpy(q->h_sin + off, (const uint8_t *) h_in + off, sz);
                CK(cudaMemcpyAsync(d_in + off, q->h_sin + off, sz, cudaMemcpyHostToDevice, st));
            }
        }
    }
    CK(cudaMemsetAsync(m, 0, sizeof(*m), st));
    /* record index */
    ev_begin_on(q, 0, st);
    if (stage_setup(q, n_tiles)) return -1;
    k_index<false><<<n_tiles, 256, 0, st>>>(d_in, (uint32_t) bytes, 0, 0, d_tile, 0, 0, 0, 0, q->d_stage);
    k_small_tiles<<<1, 256, 0, st>>>(d_tile, n_tiles, cap_rec, m);
    k_index<true><<<n_tiles, 256, 0, st>>>(d_in, (uint32_t) bytes, 0, 0, d_tile, (uint32_t *) a->d_off, (uint32_t *) a->d_len, (uint8_t *) a->d_kind, m, q->d_stage);
    k_index_check<<<nb_cap, 256, 0, st>>>(a->d_off, a->d_len, 0, &m->n_cand, (uint32_t) bytes, &m->n_breaks, q->dbreaks);
    k_index_repair<<<1, 1024, 0, st>>>(a->d_off, a->d_len, (uint8_t *) a->d_kind, 0, &m->n_cand, 0, (uint32_t) bytes, &m->n_breaks, q->dbreaks, &m->n_valid, &m->overflow);
    ev_end_on(q, 0, st);
    /* evaluation of records [0, n_valid) */
    /* A call this small is the latency of its launches one behind the other: the split evaluation and the follow-up launch of the
     * two-stage tokenizer, which pay off per byte, cost a serial pass each here (64 KB JSON calls: 330 us against 260 us).
     * They start where a call is about throughput. */
    struct bk_chain_args a_small = *a;
    if (bytes < ((size_t) 3 << 20)) a_small.split = 0;
    a = &a_small;
    fill_params(a, &p, d_out, 0);
    p.n_rec = 0; p.n_dev = &m->n_valid;
    p.bm_words = (a->d_scr && (q->json_bm > 0 || (q->json_bm < 0 && a->split))) ? BM_BYTES / 32 : 0;
    if (defer_setup(q, &p, a, cap_rec, st)) return -1;
    ev_begin_on(q, 1, st);
    if (a->split) {
        k_chain_eval_t<CH_PH_HEAD><<<nb_cap, BK_REC_BLOCK, (size_t) p.bm_words * 4 * (BK_REC_BLOCK / 32), st>>>(p);
        k_chain_eval_t<CH_PH_TAIL><<<nb_cap, BK_REC_BLOCK, 0, st>>>(p);
        g_launches += 1;
    }
    else
        k_chain_eval<<<nb_cap, BK_REC_BLOCK, (size_t) p.bm_words * 4 * (BK_REC_BLOCK / 32), st>>>(p);
    if (p.defer_list) { k_chain_eval_deferred<<<q->n_sm, BK_REC_BLOCK, 0, st>>>(p); g_launches += 1; }
    if (p.env.l2m.hash) {
        k_chain_skipped<<<nb_cap, BK_REC_BLOCK, 0, st>>>(p); g_launches += 1;
        if (p.env.l2m.pending) { k_l2m_fixup<<<1, 1024, 0, st>>>(p); k_l2m_fixup_done<<<1, 1, 0, st>>>(p); g_launches += 2; }
    }
    ev_end_on(q, 1, st);
    /* sizes, survivor lists, emission under the speculated verdicts */
    ev_begin_on(q, 2, st);
    k_small_sizes<<<nb_cap, BK_REC_BLOCK, 0, st>>>(a->d_size, m, a->d_bsum, q->d_cnt);
    k_small_scan2<<<1, 256, 0, st>>>(a->d_bsum, q->d_cnt, nb_cap, (unsigned long long) cap_out, m);
    k_surv_fill<<<nb_cap, BK_REC_BLOCK, 0, st>>>(a->d_size, 0, &m->n_valid, 0, q->d_cnt, a->d_bsum, q->d_lrec, q->d_loff);
    p.bm_words = 0;
    k_chain_emit_list<<<nb_cap * (BK_REC_BLOCK / EMIT_BLOCK), EMIT_BLOCK, (EMIT_BLOCK / 32) * (EMIT_STAGE + 16), st>>>(p, q->d_lrec, q->d_loff, &m->n_out, &m->emitted);
    ev_end_on(q, 2, st);
    g_launches += 10;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(q->h_mail, m, sizeof(*m), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(q->h_flags, a->d_flags, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    res->n_cand = (uint32_t) (q->h_mail->n_cand64 > 0xffffffffull ? 0xffffffffu : q->h_mail->n_cand64);
    res->n_valid = q->h_mail->n_valid; res->tiled = q->h_mail->tiled; res->overflow = q->h_mail->overflow;
    res->end_off = q->h_mail->end_off; res->total = q->h_mail->total; res->n_out = q->h_mail->n_out;
    res->emitted = q->h_mail->emitted;
    memcpy(res->flags, q->h_flags, sizeof(res->flags));
    return 0;
}

int bk_comm_unique_id(uint8_t id[128])
{
    ncclUniqueId u;
    if (nccl_load()) return -1;
    NK(N.GetUniqueId(&u));
    memcpy(id, u.internal, 128);
    return 0;
}

int bk_comm_init(bk_q *q, int nranks, int rank, const uint8_t id[128])
{
    ncclUniqueId u;
    if (nccl_load()) return -1;
    use(q);
    if (q->comm) { N.CommDestroy(q->comm); q->comm = 0; }
    memcpy(u.internal, id, 128);
    NK(N.CommInitRank(&q->comm, nranks, u, rank));
    q->comm_ranks = nranks; q->comm_rank = rank;
    return 0;
}

int bk_comm_info(bk_q *q, int *nranks, int *rank)
{
    if (!q->comm) return -1;
    *nranks = q->comm_ranks; *rank = q->comm_rank;
    return 0;
}

int bk_comm_allgather(bk_q *q, const void *d_send, void *d_recv, size_t bytes_per_rank)
{
    use(q);
    if (!q->comm) { snprintf(g_err, sizeof(g_err), "no communicator: call flbgpu_comm_init first"); return -1; }
    NK(N.AllGather(d_send, d_recv, bytes_per_rank, ncclUint8, q->comm, q->stream));
    CK(cudaStreamSynchronize(q->stream));
    return 0;
}

int bk_comm_allreduce_u64(bk_q *q, void *d_buf, size_t count)
{
    use(q);
    if (!q->comm) { snprintf(g_err, sizeof(g_err), "no communicator: call flbgpu_comm_init first"); return -1; }
    NK(N.AllReduce(d_buf, d_buf, count, ncclUint64, ncclSum, q->comm, q->stream));
    CK(cudaStreamSynchronize(q->stream));
    return 0;
}

int bk_comm_allreduce_f64(bk_q *q, void *d_buf, size_t count)
{
    use(q);
    if (!q->comm) { snprintf(g_err, sizeof(g_err), "no communicator: call flbgpu_comm_init first"); return -1; }
    NK(N.AllReduce(d_buf, d_buf, count, ncclFloat64, ncclSum, q->comm, q->stream));
    CK(cudaStreamSynchronize(q->stream));
    return 0;
}

int bk_jsmn_scan(bk_q *q, const struct bk_jsmn_args *a)
{
    use(q);
    if (!a->n) return 0;
    k_jsmn_scan<<<(a->n + 63) / 64, 64, 0, q->stream>>>(*a);
    g_launches += 1;
    CK(cudaGetLastError());
    return 0;
}

int bk_jsmn_emit(bk_q *q, const struct bk_jsmn_args *a)
{
    use(q);
    if (!a->n) return 0;
    k_jsmn_emit<<<(a->n + 63) / 64, 64, 0, q->stream>>>(*a);
    g_launches += 1;
    CK(cudaGetLastError());
    return 0;
}

int bk_small_fetch(bk_q *q, void *h_dst, const uint8_t *d_out, size_t n)
{
    use(q);
    if (!n) return 0;
    if (n < 4096) {
        CK(cudaMemcpyAsync(h_dst, d_out, n, cudaMemcpyDeviceToHost, q->stream));
        CK(cudaStreamSynchronize(q->stream));
        return 0;
    }
    /* through the queue's pinned buffer, in two halves: the first is copied out while the second arrives */
    if (q->cap_sout < n) {
        cudaFreeHost(q->h_sout); q->h_sout = 0; q->cap_sout = 0;
        CK(cudaMallocHost((void **) &q->h_sout, n + n / 4 + 65536));
        q->cap_sout = n + n / 4 + 65536;
    }
    if (!q->ev_small) CK(cudaEventCreateWithFlags(&q->ev_small, cudaEventDisableTiming));
    {
        const size_t half = n >= ((size_t) 512 << 10) ? (n / 2) & ~(size_t) 4095 : n;
        CK(cudaMemcpyAsync(q->h_sout, d_out, half, cudaMemcpyDeviceToHost, q->stream));
        CK(cudaEventRecord(q->ev_small, q->stream));
        if (half < n) CK(cudaMemcpyAsync(q->h_sout + half, d_out + half, n - half, cudaMemcpyDeviceToHost, q->stream));
        CK(cudaEventSynchronize(q->ev_small));
        memcpy(h_dst, q->h_sout, half);
        if (half < n) {
            CK(cudaStreamSynchronize(q->stream));
            memcpy((uint8_t *) h_dst + half, q->h_sout + half, n - half);
        }
    }
    return 0;
}

}
