/* tests/hostsim -- CPU-only emulation of the DEVICE code paths.
 *
 * The .cuh files under fluent-bit_b200/csrc are written as host+device functions.
 * This file compiles them with g++ so the `-m "not gpu"` tests can check the exact
 * device algorithms (regex VM, msgpack walkers, chain interpreter) against the
 * oracle on a box without a GPU.  It is TEST INFRASTRUCTURE: libflbgpu.so (the
 * product) never links or loads it and has no CPU path of any kind.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../../fluent-bit_b200/csrc/flbgpu_prog.h"
#include "../../fluent-bit_b200/csrc/rx_compile.h"
#include "../../fluent-bit_b200/csrc/dev_regex.cuh"

extern "C" {

void *sim_rx_compile(const char *pattern, char *err, int errcap)
{
    struct rx_compiled *c = (struct rx_compiled *) calloc(1, sizeof(*c));
    if (rx_compile(pattern, c) != 0) {
        if (err) { strncpy(err, c->err, errcap - 1); err[errcap - 1] = 0; }
        free(c);
        return NULL;
    }
    return c;
}

void sim_rx_free(void *h) { if (h) { rx_compiled_free((struct rx_compiled *) h); free(h); } }

int sim_rx_ngroups(void *h) { return (int) ((struct rx_compiled *) h)->prog->n_groups; }
int sim_rx_ncode(void *h) { return (int) ((struct rx_compiled *) h)->prog->n_code; }
const uint32_t *sim_rx_code(void *h)
{
    struct rx_prog *p = ((struct rx_compiled *) h)->prog;
    return (const uint32_t *) ((const char *) p + p->code_off);
}

int sim_rx_names(void *h, char *out, int cap)
{
    struct rx_compiled *c = (struct rx_compiled *) h;
    int i, len = 0;
    for (i = 0; i < c->n_names; i++) {
        int l = (int) strlen(c->names[i].name);
        if (len + l + 1 >= cap) break;
        memcpy(out + len, c->names[i].name, l);
        len += l;
        out[len++] = '\n';
    }
    out[len] = 0;
    return c->n_names;
}

/* returns RX_R_*; caps gets 2*(ngroups+1) ints */
int sim_rx_search(void *h, const char *s, int len, int *caps, int stack_words, unsigned budget)
{
    struct rx_compiled *c = (struct rx_compiled *) h;
    uint32_t *stk = (uint32_t *) malloc(sizeof(uint32_t) * (stack_words > 0 ? stack_words : 1));
    uint32_t b = budget;
    int r = rx_search(c->prog, (const uint8_t *) s, len, caps, stk, stack_words, &b);
    free(stk);
    return r;
}

}

/* ------------------------------------------------------------------------
 * CPU implementation of the bk_* seam (flbgpu_internal.h) so that runtime.c --
 * the real host logic -- and dev_chain.cuh -- the real device algorithms -- can be
 * exercised without a GPU.  Linked ONLY into tests/hostsim/libhostsim.so.
 * ---------------------------------------------------------------------- */
#include <stdio.h>
#include "../../fluent-bit_b200/csrc/flbgpu_internal.h"
#include "../../fluent-bit_b200/csrc/dev_chain.cuh"
#include "../../fluent-bit_b200/csrc/dev_ml.cuh"
#include "../../fluent-bit_b200/csrc/dev_tojson.cuh"
#include "../../fluent-bit_b200/csrc/dev_lines.cuh"

static thread_local char hs_err[256];
static uint64_t hs_launches;

struct sim_comm;
struct bk_q { int device; uint64_t records_out; uint8_t *dl_dst; const uint8_t *dl_src; struct sim_comm *comm; int comm_ranks, comm_rank; uint8_t *tag; };

extern "C" {

const char *bk_name(void) { return "hostsim-cpu-emulation(TEST ONLY)"; }
const char *bk_last_error(void) { return hs_err; }
uint64_t bk_launch_count(void) { return hs_launches; }
int bk_device_count(void) { return 1; }
bk_q *bk_q_new(int device) { bk_q *q = (bk_q *) calloc(1, sizeof(bk_q)); q->device = device; return q; }
void bk_q_free(bk_q *q) { if (q) free(q->tag); free(q); }
int bk_q_device(bk_q *q) { return q->device; }
#ifdef HS_POISON        /* device memory is not zero when it is handed out: a build of the emulation that makes the same point */
void *bk_alloc(bk_q *, size_t n) { void *p = malloc(n + 64); if (p) memset(p, HS_POISON, n + 64); return p; }
#else
void *bk_alloc(bk_q *, size_t n) { return malloc(n + 64); }
#endif
void bk_free(bk_q *, void *p) { free(p); }
void *bk_alloc_host(bk_q *, size_t n) { return malloc(n ? n : 16); }
void bk_free_host(bk_q *, void *p) { free(p); }
int bk_h2d(bk_q *, void *d, const void *h, size_t n) { memcpy(d, h, n); return 0; }
int bk_d2h(bk_q *, void *h, const void *d, size_t n) { memcpy(h, d, n); return 0; }
int bk_zero(bk_q *, void *d, size_t n) { memset(d, 0, n); return 0; }
int bk_sync(bk_q *) { return 0; }
void *bk_stream(bk_q *) { return 0; }
int bk_kernel_ms(bk_q *, float out[3]) { out[0] = out[1] = out[2] = 0.f; return 0; }

int bk_d2d_2d(bk_q *, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows)
{
    for (size_t r = 0; r < rows; r++) memcpy((uint8_t *) dst + r * dpitch, (const uint8_t *) src + r * spitch, width);
    return 0;
}
int bk_rx_search_host(const void *prog, const uint8_t *s, int n, int *caps)
{
    uint32_t stk[1024], budget = CH_RX_BUDGET;
    return rx_search((const struct rx_prog *) prog, s, n, caps, stk, 1024, &budget);
}
int bk_d2d(bk_q *, void *dst, const void *src, size_t n) { memcpy(dst, src, n); return 0; }
int bk_upload_start(bk_q *, void *d_dst, const void *h_src, size_t n) { memcpy(d_dst, h_src, n); return 0; }
int bk_upload_wait_index(bk_q *, size_t upto) { (void) upto; return 0; }
void bk_upload_none(bk_q *) {}
void bk_upload_end(bk_q *) {}
int bk_hint_streaming(bk_q *, const void *base, size_t bytes) { (void) base; (void) bytes; return 0; }

int bk_index_count(bk_q *, const uint8_t *d_in, size_t slice_off, uint32_t len, uint32_t *d_tile, uint32_t n_tiles, uint32_t *n_cand)
{
    const uint8_t *in = d_in + slice_off;
    const uint32_t skip = (uint32_t) ((uintptr_t) (d_in + slice_off) & 15);
    uint32_t t, run = 0;
    for (t = 0; t < n_tiles; t++) {
        /* tile t covers bytes [t*TILE - skip, (t+1)*TILE - skip) of the slice, like the CUDA kernel */
        uint32_t b = t * BK_INDEX_TILE > skip ? t * BK_INDEX_TILE - skip : 0, e = (t + 1) * BK_INDEX_TILE - skip, i, cnt = 0;
        if (e > len) e = len;
        for (i = b; i < e; i++) {
            int kind;
            if (in[i] == 0x92 && rec_frame(in + i, in + len, &kind) && !rec_is_shadowed(in, in + i, in + len)) cnt++;
        }
        d_tile[t] = run;
        run += cnt;
    }
    *n_cand = run;
    hs_launches += 2;
    return 0;
}

int bk_index_fill(bk_q *, const uint8_t *d_in, size_t slice_off, uint32_t len, const uint32_t *d_tile, uint32_t n_tiles, uint32_t n_cand,
                  uint32_t *d_off, uint32_t *d_len, uint8_t *d_kind, uint32_t *n_valid, uint64_t *end_off, int *tiled)
{
    const uint8_t *in = d_in + slice_off;
    const uint32_t base = (uint32_t) slice_off, total = base + len, skip = (uint32_t) ((uintptr_t) (d_in + slice_off) & 15);
    uint32_t t, i;
    *n_valid = 0; *tiled = (len == 0); *end_off = slice_off;
    if (n_cand == 0) return 0;
    for (t = 0; t < n_tiles; t++) {
        uint32_t b = t * BK_INDEX_TILE > skip ? t * BK_INDEX_TILE - skip : 0, e = (t + 1) * BK_INDEX_TILE - skip, o = d_tile[t];
        if (e > len) e = len;
        for (i = b; i < e; i++) {
            int kind = 0;
            const uint8_t *q;
            if (in[i] == 0x92 && (q = rec_frame(in + i, in + len, &kind)) && !rec_is_shadowed(in, in + i, in + len)) {
                d_off[o] = base + i; d_len[o] = (uint32_t) (q - (in + i)); d_kind[o] = (uint8_t) kind; o++;
            }
        }
    }
    hs_launches += 3;
    {
        /* same walk as k_index_repair: breaks visited in ascending order */
        uint32_t skip_until = 0, nv = n_cand, til = 1, last;
        if (d_off[0] != base) { *n_valid = 0; *tiled = 0; return 0; }
        for (i = 0; i < n_cand; i++) {
            uint32_t next = (i + 1 < n_cand) ? d_off[i + 1] : total, target, k;
            if (d_off[i] + d_len[i] == next) continue;
            if (i < skip_until) continue;
            target = d_off[i] + d_len[i];
            k = i + 1;
            while (k < n_cand && d_off[k] < target) { d_kind[k] = 2; k++; }
            if (k < n_cand && d_off[k] == target) { skip_until = k; continue; }
            if (k == n_cand && target == total) { skip_until = n_cand; continue; }
            nv = i + 1; til = 0;
            break;
        }
        last = nv;
        while (last > 0 && d_kind[last - 1] == 2) last--;
        *end_off = last ? d_off[last - 1] + d_len[last - 1] : base;
        *n_valid = nv; *tiled = (int) til;
    }
    return 0;
}

static void hs_env(const struct bk_chain_args *a, struct ch_env *e)
{
    e->in = a->d_in; e->in_len = a->in_len; e->blob = a->d_blob; e->scr = a->d_scr; e->scr_mul = a->scr_mul ? a->scr_mul : 4;
    e->capcache = a->d_capcache; e->cap_stride = a->cap_stride; e->cap_n = a->cap_n; e->now = a->now; e->assume = a->assume; e->active = a->active;
    e->fl_flags = a->d_flags; e->err = a->d_flags + FLBGPU_MAX_FILTERS;
    e->l2m = a->l2m; e->prep = a->d_prep;
    e->esize = a->d_esize; e->tag = a->d_tag; e->tag_len = a->tag_len;
}
/* where the bytes the reference's decoder consumed for record i begin (kernels.cu: raw_lo_of) */
static uint32_t hs_raw_lo(const struct bk_chain_args *a, uint32_t i)
{
    uint32_t j = i;
    while (j > 0 && a->d_kind[j - 1] != 0) j--;
    return j ? a->d_off[j - 1] + a->d_len[j - 1] : 0u;
}

int bk_flags_clear(bk_q *q, uint32_t *d_flags) { memset(d_flags, 0, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1)); q->records_out = 0; return 0; }
int bk_flags_fetch(bk_q *, const uint32_t *d_flags, uint32_t *h_flags) { memcpy(h_flags, d_flags, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1)); return 0; }

/* FLBGPU_SIM_ORDER=reverse: every record loop of an evaluation runs from its last entry to its first.  The kernels give no
 * order among a launch's records; this is the emulation's other extreme, for results that must not depend on it. */
static int hs_reverse(void)
{
    const char *e = getenv("FLBGPU_SIM_ORDER");
    return e && !strcmp(e, "reverse");
}
/* entry t of a loop over n entries, in the emulation's order */
static inline uint32_t hs_at(uint32_t t, uint32_t n, int rev) { return rev ? n - 1 - t : t; }

int bk_chain_eval(bk_q *, const struct bk_chain_args *a, uint32_t r0, uint32_t r1)
{
    const int rev = hs_reverse();
    struct ch_env e;
    uint32_t i;
    uint32_t *bm = 0;
    struct ch_lane ln;
    memset(&ln, 0, sizeof(ln));
    hs_env(a, &e);
    if (a->d_scr && r1 > r0 && !getenv("FLBGPU_JSON_BM_OFF")) {
        /* stage 1 of the JSON tokenizer as the CUDA kernel leaves it: one bit per byte that a string scan has to look at.
         * (Here over the records' whole byte range at once; the kernel does it per warp.) */
        const uint32_t lo = a->d_off[r0], hi = a->d_off[r1 - 1] + a->d_len[r1 - 1];
        bm = (uint32_t *) calloc((hi - lo + 31) / 32 + 1, 4);
        for (uint32_t b = lo; b < hi; b++) {
            const uint8_t c = a->d_in[b];
            if (c == '"' || c == 0x5c || c < 0x20 || c >= 0x80) bm[(b - lo) >> 5] |= 1u << ((b - lo) & 31);
        }
        ln.bm = bm; ln.bm_base = lo; ln.bm_end = hi;
        ln.defer_ok = a->defer_ok && !getenv("FLBGPU_SIM_NODEFER");     /* as the kernel: records the walker cannot take go to a follow-up pass */
    }
    if (a->d_esize) for (i = r0; i < r1; i++) if (a->d_kind[i] != 0) a->d_esize[i] = 0;
    if (a->split) {
        /* the three launches of the split form: the head over all records, which lists the records it keeps for the tail
         * and those it puts off; the tail over its list; the put-off records, whole.  The kernel runs the last two side by
         * side on two streams, so either may finish first: FLBGPU_SIM_DEFER_FIRST=1 runs the put-off records before the tail. */
        const int defer_first = getenv("FLBGPU_SIM_DEFER_FIRST") && getenv("FLBGPU_SIM_DEFER_FIRST")[0] == '1';
        uint32_t *tlist = (uint32_t *) malloc(sizeof(uint32_t) * (r1 - r0 + 1)), *dlist = (uint32_t *) malloc(sizeof(uint32_t) * (r1 - r0 + 1));
        uint32_t tn = 0, dn = 0, t;
        /* (the lists fill in the head's order: under FLBGPU_SIM_ORDER=reverse the tail and the put-off records run backwards too) */
        for (t = 0; t < r1 - r0; t++) {
            uint32_t sz = 0;
            i = r0 + hs_at(t, r1 - r0, rev);
            if (a->d_kind[i] == 0) ln.raw_lo = hs_raw_lo(a, i), sz = chain_record<false, CH_PH_HEAD>(&e, &ln, i, a->d_off[i], a->d_len[i], 0);
            if (sz == CH_DEFER) { dlist[dn++] = i; sz = 0; }
            if (sz) tlist[tn++] = i;
            a->d_size[i] = sz;
        }
        for (int pass = 0; pass < 2; pass++) {
            if (pass == (defer_first ? 1 : 0))
                for (t = 0; t < tn; t++) i = tlist[t], a->d_size[i] = chain_record<false, CH_PH_TAIL>(&e, &ln, i, a->d_off[i], a->d_len[i], 0);
            else for (t = 0; t < dn; t++) {
                struct ch_lane plain;
                memset(&plain, 0, sizeof(plain));
                i = dlist[t];
                plain.raw_lo = hs_raw_lo(a, i);
                a->d_size[i] = chain_record<false>(&e, &plain, i, a->d_off[i], a->d_len[i], 0);
            }
        }
        for (t = 0; t < r1 - r0; t++)
            if (i = r0 + hs_at(t, r1 - r0, rev), a->d_kind[i] == 1 && e.l2m.hash) chain_skipped_record(&e, i, a->d_off[i], a->d_len[i]);
        free(tlist); free(dlist);
        hs_launches += 1;
    }
    else {
        uint8_t *put_off = (uint8_t *) calloc(r1 - r0 + 1, 1);
        struct ch_lane plain;
        memset(&plain, 0, sizeof(plain));
        uint32_t t;
        for (t = 0; t < r1 - r0; t++) {
            uint32_t sz = 0;
            i = r0 + hs_at(t, r1 - r0, rev);
            if (a->d_kind[i] == 0) ln.raw_lo = hs_raw_lo(a, i), sz = chain_record<false>(&e, &ln, i, a->d_off[i], a->d_len[i], 0);
            else if (a->d_kind[i] == 1 && e.l2m.hash) chain_skipped_record(&e, i, a->d_off[i], a->d_len[i]);
            if (sz == CH_DEFER) { put_off[i - r0] = 1; sz = 0; }
            a->d_size[i] = sz;
        }
        for (t = 0; t < r1 - r0; t++)
            if (i = r0 + hs_at(t, r1 - r0, rev), put_off[i - r0]) { plain.raw_lo = hs_raw_lo(a, i); a->d_size[i] = chain_record<false>(&e, &plain, i, a->d_off[i], a->d_len[i], 0); }
        free(put_off);
    }
    free(bm);
    if (e.l2m.hash && e.l2m.pending) {             /* k_l2m_fixup: the records whose value text converts nothing, in the list's
                                                    * order (backwards under FLBGPU_SIM_ORDER=reverse, as the evaluation filled it) */
        unsigned long long n = e.l2m.pending_n[0], d = e.l2m.pending_n[1], t;
        if (n > e.l2m.pending_cap) n = e.l2m.pending_cap;
        for (t = d; t < n; t++) l2m_fixup_record(&e, e.l2m.pending[t], a->d_off, a->d_len, a->d_kind);
        e.l2m.pending_n[1] = e.l2m.pending_n[0];
        hs_launches += 1;
    }
    hs_launches += 1;
    return 0;
}

int bk_sizes_scan(bk_q *, const uint32_t *d_size, uint32_t n_rec, uint64_t *d_bsum, uint64_t *h_bsum)
{
    uint32_t nb = (n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK, b, i;
    uint64_t run = 0;
    for (b = 0; b < nb; b++) {
        d_bsum[b] = run; h_bsum[b] = run;
        for (i = b * BK_REC_BLOCK; i < n_rec && i < (b + 1) * BK_REC_BLOCK; i++) run += d_size[i];
    }
    h_bsum[nb] = run;
    hs_launches += 2;
    return 0;
}

int bk_sizes_scan_range(bk_q *, const uint32_t *d_size, uint32_t n_rec, uint32_t b0, uint32_t b1, uint64_t *d_bsum, uint64_t *h_bsum,
                        uint64_t carry_in)
{
    uint32_t b, i;
    uint64_t run = carry_in;
    for (b = b0; b < b1; b++) {
        d_bsum[b] = run; h_bsum[b] = run;
        for (i = b * BK_REC_BLOCK; i < n_rec && i < (b + 1) * BK_REC_BLOCK; i++) run += d_size[i];
    }
    h_bsum[b0] = carry_in;
    h_bsum[b1] = run;
    hs_launches += 2;
    return 0;
}

int bk_records_out(bk_q *q, uint64_t *n) { *n = q->records_out; return 0; }

int bk_chain_emit(bk_q *q, const struct bk_chain_args *a, uint8_t *d_out, uint32_t b0, uint32_t b1)
{
    struct ch_env e;
    uint32_t i, b;
    hs_env(a, &e);
    for (b = b0; b < b1; b++) {
        uint64_t at = a->d_bsum[b];
        for (i = b * BK_REC_BLOCK; i < a->n_rec && i < (b + 1) * BK_REC_BLOCK; i++) {
            if (a->d_size[i]) {
                struct ch_lane ln;
                memset(&ln, 0, sizeof(ln));
                uint32_t w = chain_record<true>(&e, &ln, i, a->d_off[i], a->d_len[i], d_out + at);
                q->records_out++;
                if (w != a->d_size[i]) { snprintf(hs_err, sizeof(hs_err), "emit size mismatch at record %u: %u vs %u", i, w, a->d_size[i]); return -1; }
                at += w;
            }
        }
    }
    hs_launches += 1;
    return 0;
}

/* ---- rewrite_tag ---- */
int bk_tag_upload(bk_q *q, const char *tag, uint32_t tag_len, const uint8_t **d_tag)
{
    free(q->tag);
    q->tag = (uint8_t *) malloc(tag_len + 1);
    if (tag_len) memcpy(q->tag, tag, tag_len);
    *d_tag = q->tag;
    return 0;
}
int bk_rtag_emit(bk_q *q, const struct bk_chain_args *a, uint32_t n_rec, uint64_t *, uint64_t *, void **h_out, size_t *bytes)
{
    struct ch_env e;
    size_t total = 0, at = 0;
    uint32_t i;
    uint8_t *out;
    *h_out = 0; *bytes = 0;
    for (i = 0; i < n_rec; i++) total += a->d_esize[i];
    if (!total) return 0;
    out = (uint8_t *) malloc(total);
    hs_env(a, &e);
    e.esize = 0;
    for (i = 0; i < n_rec; i++) {
        struct ch_lane ln;
        uint32_t w;
        if (!a->d_esize[i]) continue;
        memset(&ln, 0, sizeof(ln));
        ln.raw_lo = hs_raw_lo(a, i);
        w = chain_record<true, CH_PH_RTAG>(&e, &ln, i, a->d_off[i], a->d_len[i], out + at);
        if (w != a->d_esize[i]) { snprintf(hs_err, sizeof(hs_err), "re-tagged entry size mismatch at record %u: %u vs %u", i, w, a->d_esize[i]); free(out); return -1; }
        at += w;
    }
    hs_launches += 1;
    (void) q;
    *h_out = out; *bytes = total;
    return 0;
}

int bk_download_begin(bk_q *q, void *h_dst, const void *d_out) { q->dl_dst = (uint8_t *) h_dst; q->dl_src = (const uint8_t *) d_out; return 0; }
int bk_download_push(bk_q *q, size_t lo, size_t hi) { memcpy(q->dl_dst + lo, q->dl_src + lo, hi - lo); return 0; }
int bk_download_end(bk_q *) { return 0; }

/* the small-chunk form: the same steps in sequence, with the same "does it fit" decisions the device takes */
int bk_small_run(bk_q *q, const struct bk_chain_args *a, const void *h_in, uint8_t *d_in, size_t bytes, uint32_t cap_rec,
                 uint32_t *d_tile, uint32_t n_tiles, uint8_t *d_out, size_t cap_out, struct bk_small_res *res)
{
    struct bk_chain_args b = *a;
    uint32_t n_cand = 0, n_valid = 0, nb, i;
    uint64_t end_off = 0;
    int tiled = 0;
    memset(res, 0, sizeof(*res));
    if (h_in) memcpy(d_in, h_in, bytes);
    if (bk_index_count(q, d_in, 0, (uint32_t) bytes, d_tile, n_tiles, &n_cand)) return -1;
    res->n_cand = n_cand;
    if (n_cand > cap_rec) { res->overflow = 1; return 0; }
    if (bk_index_fill(q, d_in, 0, (uint32_t) bytes, d_tile, n_tiles, n_cand, (uint32_t *) a->d_off, (uint32_t *) a->d_len, (uint8_t *) a->d_kind,
                      &n_valid, &end_off, &tiled)) return -1;
    res->n_valid = n_valid; res->tiled = (uint32_t) tiled; res->end_off = end_off;
    b.n_rec = n_valid;
    if (bk_chain_eval(q, &b, 0, n_valid)) return -1;
    nb = (n_valid + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    {
        uint64_t *h_bsum = (uint64_t *) malloc(sizeof(uint64_t) * (nb + 2));
        if (bk_sizes_scan(q, a->d_size, n_valid, a->d_bsum, h_bsum)) { free(h_bsum); return -1; }
        res->total = h_bsum[nb];
        free(h_bsum);
    }
    for (i = 0; i < n_valid; i++) if (a->d_size[i]) res->n_out++;
    res->emitted = res->total <= cap_out;
    if (res->emitted && bk_chain_emit(q, &b, d_out, 0, nb)) return -1;
    memcpy(res->flags, a->d_flags, sizeof(res->flags));
    return 0;
}
/* ---- the collectives of the metric-table exchange between PROCESSES on this host, through a POSIX shared-memory
 * segment named by the "unique id" (test infrastructure for the world-size-2 CPU tests of the product's merge logic) ---- */
}
#include <atomic>
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>
#include <sched.h>
#define SIM_SLOT ((size_t) 8 << 20)
struct sim_comm { std::atomic<int> arrived; std::atomic<int> phase; char pad[56]; };
static void sim_barrier(bk_q *q)
{
    struct sim_comm *c = q->comm;
    const int ph = c->phase.load();
    if (c->arrived.fetch_add(1) + 1 == q->comm_ranks) { c->arrived.store(0); c->phase.store(ph + 1); }
    else while (c->phase.load() == ph) sched_yield();
}
static uint8_t *sim_slot(bk_q *q, int r) { return (uint8_t *) q->comm + 4096 + (size_t) r * SIM_SLOT; }
extern "C" {
int bk_comm_unique_id(uint8_t id[128])
{
    static int n;
    memset(id, 0, 128);
    snprintf((char *) id, 128, "/flbgpu_sim_%d_%d", (int) getpid(), n++);
    return 0;
}
int bk_comm_init(bk_q *q, int nranks, int rank, const uint8_t id[128])
{
    const size_t size = 4096 + (size_t) nranks * SIM_SLOT;
    int fd = shm_open((const char *) id, O_CREAT | O_RDWR, 0600);
    void *m;
    if (fd < 0 || ftruncate(fd, (off_t) size) != 0) { snprintf(hs_err, sizeof(hs_err), "shm_open(%s) failed", (const char *) id); return -1; }
    m = mmap(0, size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (m == MAP_FAILED) return -1;
    q->comm = (struct sim_comm *) m; q->comm_ranks = nranks; q->comm_rank = rank;
    sim_barrier(q);
    if (rank == 0) shm_unlink((const char *) id);
    return 0;
}
int bk_comm_info(bk_q *q, int *nranks, int *rank) { if (!q->comm) return -1; *nranks = q->comm_ranks; *rank = q->comm_rank; return 0; }
int bk_comm_allgather(bk_q *q, const void *d_send, void *d_recv, size_t n)
{
    if (!q->comm || n > SIM_SLOT) return -1;
    memcpy(sim_slot(q, q->comm_rank), d_send, n);
    sim_barrier(q);
    for (int r = 0; r < q->comm_ranks; r++) memcpy((uint8_t *) d_recv + (size_t) r * n, sim_slot(q, r), n);
    sim_barrier(q);
    return 0;
}
int bk_comm_allreduce_u64(bk_q *q, void *d_buf, size_t count)
{
    if (!q->comm || count * 8 > SIM_SLOT) return -1;
    memcpy(sim_slot(q, q->comm_rank), d_buf, count * 8);
    sim_barrier(q);
    for (size_t i = 0; i < count; i++) { uint64_t v = 0; for (int r = 0; r < q->comm_ranks; r++) v += ((const uint64_t *) sim_slot(q, r))[i]; ((uint64_t *) d_buf)[i] = v; }
    sim_barrier(q);
    return 0;
}
int bk_comm_allreduce_f64(bk_q *q, void *d_buf, size_t count)
{
    if (!q->comm || count * 8 > SIM_SLOT) return -1;
    memcpy(sim_slot(q, q->comm_rank), d_buf, count * 8);
    sim_barrier(q);
    for (size_t i = 0; i < count; i++) { double v = 0; for (int r = 0; r < q->comm_ranks; r++) v += ((const double *) sim_slot(q, r))[i]; ((double *) d_buf)[i] = v; }
    sim_barrier(q);
    return 0;
}

int bk_jsmn_scan(bk_q *, const struct bk_jsmn_args *a)
{
    for (uint32_t i = 0; i < a->n; i++) {
        const uint8_t *js = a->d_js + a->d_off[i];
        struct jm_tok *tok = a->d_tok + a->d_tok_off[i];
        uint32_t toknext = 0;
        const int tret = jm_tokenise(js, a->d_len[i], tok, a->d_tok_cap[i], &toknext);
        struct jm_result r;
        memset(&r, 0, sizeof(r));
        r.tret = tret;
        if (tret == JM_NOMEM) { r.status = JM_NOMEM; r.toknext = toknext; }
        else jm_pack(js, a->d_len[i], tok, toknext, tret, 0, a->d_tmp + a->d_off[i] + i, &r);
        a->d_res[i] = r;
    }
    hs_launches += 1;
    return 0;
}
int bk_jsmn_emit(bk_q *, const struct bk_jsmn_args *a)
{
    for (uint32_t i = 0; i < a->n; i++) {
        struct jm_result r = a->d_res[i];
        if (r.status != JM_OK || r.out_size == 0) continue;
        jm_pack(a->d_js + a->d_off[i], a->d_len[i], a->d_tok + a->d_tok_off[i], r.toknext, r.tret, a->d_out + a->d_out_off[i], a->d_tmp + a->d_off[i] + i, &r);
    }
    hs_launches += 1;
    return 0;
}
int bk_small_fetch(bk_q *, void *h_dst, const uint8_t *d_out, size_t n) { memcpy(h_dst, d_out, n); return 0; }

/* raw text -> log events: the launches of kernels_lines.cu as loops */
int bk_ln_count(bk_q *, const struct ln_env *e)
{
    for (uint32_t t = 0; t < e->n_tiles; t++) e->cnt[t] = ln_count(e, t);
    hs_launches += 1;
    return 0;
}
int bk_ln_fill(bk_q *, const struct ln_env *e, const uint64_t *d_bsum)
{
    uint64_t at = 0;
    for (uint32_t t = 0; t < e->n_tiles; t++) {
        if (t % BK_REC_BLOCK == 0) at = d_bsum[t / BK_REC_BLOCK];
        ln_fill(e, t, at);
        at += e->cnt[t];
    }
    hs_launches += 1;
    return 0;
}
int bk_ln_sizes(bk_q *, const struct ln_env *e)
{
    for (uint32_t k = 0; k < e->n_lines; k++) { uint32_t a, b; e->size[k] = ln_line(e, k, &a, &b); if (e->size[k]) e->n_events[0]++; }
    hs_launches += 1;
    return 0;
}
int bk_ln_emit(bk_q *, const struct ln_env *e, const uint64_t *d_bsum, uint8_t *d_out)
{
    uint64_t at = 0;
    for (uint32_t k = 0; k < e->n_lines; k++) {
        if (k % BK_REC_BLOCK == 0) at = d_bsum[k / BK_REC_BLOCK];
        if (e->size[k]) ln_emit(e, k, d_out + at);
        at += e->size[k];
    }
    hs_launches += 1;
    return 0;
}

/* chunk -> JSON text: the launches of kernels_tojson.cu as loops */
int bk_tj_sizes(bk_q *, const struct tj_env *e)
{
    for (uint32_t i = 0; i < e->n_rec; i++) e->size[i] = tj_event(e, i, 0);
    hs_launches += 1;
    return 0;
}
int bk_tj_emit(bk_q *, const struct tj_env *e, const uint64_t *d_bsum, uint8_t *d_out)
{
    uint64_t at = 0;
    for (uint32_t i = 0; i < e->n_rec; i++) {
        if (i % BK_REC_BLOCK == 0) at = d_bsum[i / BK_REC_BLOCK];
        if (e->size[i]) tj_event(e, i, d_out + at);
        at += e->size[i];
    }
    hs_launches += 1;
    return 0;
}

/* filter_multiline: the launches of kernels_ml.cu as loops over the same per-thread functions (dev_ml.cuh) */
int bk_ml_plan(bk_q *, const struct ml_env *e)
{
    uint32_t i;
    for (i = 0; i < e->n_rec; i++) ml_feat_record(e, i);
    for (i = 0; i < e->nt1 * e->S; i++) ml_up1(e, i);
    for (i = 0; i < e->nt2 * e->S; i++) ml_up2(e, i);
    ml_top(e);
    for (i = 0; i < e->nt2; i++) ml_down2(e, i);
    for (i = 0; i < e->nt1; i++) ml_apply(e, i);
    for (i = 0; i < e->nt2; i++) ml_cnt_up2(e, i);
    ml_cnt_top(e);
    for (i = 0; i < e->nt2; i++) ml_cnt_down2(e, i);
    for (i = 0; i < e->nt1; i++) ml_fill(e, i);
    hs_launches += 10;
    return 0;
}
int bk_ml_sizes(bk_q *, const struct ml_env *e, uint32_t n_ev)
{
    for (uint32_t j = 0; j < n_ev; j++) e->ev_size[j] = ml_event(e, j, 0);
    hs_launches += 1;
    return 0;
}
int bk_ml_emit(bk_q *, const struct ml_env *e, uint32_t n_ev, const uint64_t *d_bsum, uint8_t *d_out)
{
    uint64_t at = 0;
    for (uint32_t j = 0; j < n_ev; j++) {
        if (j % BK_REC_BLOCK == 0) at = d_bsum[j / BK_REC_BLOCK];
        if (e->ev_size[j]) ml_event(e, j, d_out + at);
        at += e->ev_size[j];
    }
    hs_launches += 1;
    return 0;
}

}
