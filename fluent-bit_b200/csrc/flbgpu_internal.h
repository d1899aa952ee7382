/* flbgpu_internal.h -- seam between the host runtime (C) and the device back end.
 *
 * The product library links runtime.c + kernels.cu (CUDA, sm_90a) and nothing
 * else: there is no CPU implementation of bk_* in libflbgpu.so, so every entry
 * point fails loudly when no CUDA device is present.  tests/hostsim provides a
 * second implementation of the same functions for CPU-only CI of the host logic
 * and of the device algorithms; it is never linked into the product.
 *
 * All mutable back-end state lives in a QUEUE (bk_q): the device ordinal, the
 * streams, the timing events, the pinned staging rings with their persistent
 * worker threads and the small device scratch.  One filter instance / fused chain
 * owns one queue, so two instances may run on different threads (and different
 * devices) at the same time -- what flb_processor_run() does to filters
 * (/root/reference/src/flb_processor.c:1352-1378).  A queue itself is not
 * re-entrant; runtime.c serialises the calls of one chain.
 */
#ifndef FLBGPU_INTERNAL_H
#define FLBGPU_INTERNAL_H

#include <stddef.h>
#include <stdint.h>
#include "flbgpu_prog.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BK_INDEX_TILE   8192u     /* input bytes per index block */
#define BK_REC_BLOCK    256u      /* records per chain block */

typedef struct bk_q bk_q;

struct bk_chain_args {
    const uint8_t *d_in;          /* input chunk (device) */
    uint32_t in_len;
    const uint8_t *d_blob;        /* chain program (device) */
    uint8_t *d_scr;               /* scratch or NULL */
    uint32_t scr_mul;             /* scratch bytes per record byte: 4, or 8 when a parser has field decoders */
    int32_t *d_capcache;          /* capture cache or NULL: word w of record r at [w * cap_n + r] */
    uint32_t cap_stride;
    uint32_t cap_n;               /* records per column of the capture cache (= capacity of the record arrays) */
    int64_t now;
    uint32_t assume;
    uint32_t active;              /* bit k: filter k sees this call's chunk (Match routing) */
    uint32_t defer_ok;            /* a record may be put off to the follow-up launch before the first JSON parser runs (nothing
                                     with side effects -- log_to_metrics -- comes earlier in the chain) */
    uint32_t split;               /* evaluate as two launches: filter 0 (the parser) and the grep filters right behind it, then
                                     the rest over the list of records the first left (the capture cache has RC_CACHE_MAXF
                                     columns more than cap_stride) */
    const uint32_t *d_off;        /* record index */
    const uint32_t *d_len;
    const uint8_t *d_kind;
    uint32_t n_rec;               /* records indexed so far */
    uint32_t *d_size;             /* [n_rec] output size per record */
    uint64_t *d_bsum;             /* [ceil(n_rec/BK_REC_BLOCK)+1] exclusive output offset per block */
    uint32_t *d_flags;            /* [FLBGPU_MAX_FILTERS + 1]: CHF_* per filter, last = error word */
    struct l2m_table l2m;         /* device pointers of the log_to_metrics delta table (hash NULL = none) */
    int32_t *d_prep;              /* parser report, 6 ints per record (dev_chain.cuh: ch_env.prep), or NULL */
    uint32_t *d_esize;            /* chains with a rewrite_tag filter: [n_rec] bytes of each record's entry in the re-tagged stream */
    const uint8_t *d_tag;         /* the tag of the call on the device (bk_tag_upload) */
    uint32_t tag_len;
};

int   bk_tag_upload(bk_q *q, const char *tag, uint32_t tag_len, const uint8_t **d_tag);
/* the re-tagged stream of records [0, n_rec) (sizes in a->d_esize): *h_out = malloc()ed, *bytes long, NULL when empty */
int   bk_rtag_emit(bk_q *q, const struct bk_chain_args *a, uint32_t n_rec, uint64_t *d_bsum, uint64_t *h_bsum, void **h_out, size_t *bytes);
const char *bk_name(void);
int   bk_device_count(void);
const char *bk_last_error(void);                 /* of the calling thread */
uint64_t bk_launch_count(void);                  /* kernels launched by this library so far (all queues) */
void bk_note_launches(unsigned n);               /* (between the translation units of a back end) */
void bk_note_error(const char *what, const char *detail);
void bk_ev_begin(bk_q *q, int k);                /* CUDA-event pair of kernel group k (0 index, 1 evaluate, 2 emit) on the queue's stream */
void bk_ev_end(bk_q *q, int k);

bk_q *bk_q_new(int device);                      /* NULL: no usable device (bk_last_error) */
void  bk_q_free(bk_q *q);
int   bk_q_device(bk_q *q);
void *bk_alloc(bk_q *q, size_t n);
void  bk_free(bk_q *q, void *p);
void *bk_alloc_host(bk_q *q, size_t n);          /* pinned host memory */
void  bk_free_host(bk_q *q, void *p);
int   bk_h2d(bk_q *q, void *d, const void *h, size_t n);
int   bk_d2h(bk_q *q, void *h, const void *d, size_t n);
int   bk_zero(bk_q *q, void *d, size_t n);
int   bk_sync(bk_q *q);
void *bk_stream(bk_q *q);
int   bk_kernel_ms(bk_q *q, float out[3]);       /* CUDA-event ms of index / evaluate / emit in the last call */
int   bk_d2d(bk_q *q, void *dst, const void *src, size_t n);   /* synchronous device copy (buffer growth) */
/* the same for `rows` rows of `width` bytes with different pitches (re-laying the capture-cache columns) */
int   bk_d2d_2d(bk_q *q, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows);
/* the regex VM on the host, for control-plane decisions on tags (Match_Regex); caps has 2 * (RX_MAX_GROUPS + 1) ints */
int   bk_rx_search_host(const void *prog, const uint8_t *s, int n, int *caps);

/* ---- the per-call pipeline ----------------------------------------------------
 * A chunk is processed in SLICES (byte ranges that start at a record boundary):
 *
 *   upload stream :  H2D piece 0 | piece 1 | piece 2 | ...
 *   index stream  :        index(slice 0) | index(slice 1) | ...      (waits for its pieces)
 *   compute stream:               eval(slice 0) | eval(slice 1) | ... | sizes scan |
 *                                  emit(range 0) | emit(range 1) | ...
 *   download strm :                                       D2H(range 0) | D2H(range 1) ...
 *   host threads  :                                          pinned ring -> malloc()ed result
 *
 * so host->device copy, evaluation, emission and device->host copy overlap. */

/* start the asynchronous upload of a whole chunk (pieces + one event per piece) */
int bk_upload_start(bk_q *q, void *d_dst, const void *h_src, size_t n);
/* the index stream may not read beyond bytes that have arrived: wait (on the device) for [0,upto) */
int bk_upload_wait_index(bk_q *q, size_t upto);
/* device-resident input: nothing to wait for */
void bk_upload_none(bk_q *q);
/* waits for the staging threads of a pageable upload: the caller's buffer is not read after this */
void bk_upload_end(bk_q *q);

/* Record index (K1) of one slice d_in[slice_off, slice_off+slice_len).  Pass 1 counts
 * validated candidates per tile (exclusive tile offsets left in d_tile) and returns the
 * total (synchronises the index stream only). */
int bk_index_count(bk_q *q, const uint8_t *d_in, size_t slice_off, uint32_t slice_len, uint32_t *d_tile, uint32_t n_tiles,
                   uint32_t *n_cand);
/* Pass 2 writes (absolute offset, length, kind) of the slice's candidates at d_off/d_len/
 * d_kind (already advanced to the slice's first record), repairs the candidate chain and
 * reports: *n_valid records that chain from the slice start, *end_off = absolute offset
 * where the last of them ends, *tiled = 1 when that is the slice end. */
int bk_index_fill(bk_q *q, const uint8_t *d_in, size_t slice_off, uint32_t slice_len, const uint32_t *d_tile, uint32_t n_tiles,
                  uint32_t n_cand, uint32_t *d_off, uint32_t *d_len, uint8_t *d_kind,
                  uint32_t *n_valid, uint64_t *end_off, int *tiled);

int bk_flags_clear(bk_q *q, uint32_t *d_flags);
/* L2 hint: [base, base+bytes) is read once by the next evaluation launches */
int bk_hint_streaming(bk_q *q, const void *base, size_t bytes);
/* evaluation pass over records [r0, r1): asynchronous on the compute stream */
int bk_chain_eval(bk_q *q, const struct bk_chain_args *a, uint32_t r0, uint32_t r1);
/* evidence + error word (synchronises the compute stream) */
int bk_flags_fetch(bk_q *q, const uint32_t *d_flags, uint32_t *h_flags);
/* per-block sums of d_size[0,n_rec) -> exclusive offsets in d_bsum, copied to h_bsum
 * (n_blocks+1 entries, last = total).  Synchronises. */
int bk_sizes_scan(bk_q *q, const uint32_t *d_size, uint32_t n_rec, uint64_t *d_bsum, uint64_t *h_bsum);
/* the same for blocks [b0, b1) only, continuing from carry_in bytes already placed; fills
 * d_bsum[b0..b1), h_bsum[b0..b1] (h_bsum[b1] = bytes placed after these blocks).  Synchronous. */
int bk_sizes_scan_range(bk_q *q, const uint32_t *d_size, uint32_t n_rec, uint32_t b0, uint32_t b1, uint64_t *d_bsum, uint64_t *h_bsum,
                        uint64_t carry_in);
/* emission of blocks [b0, b1) into d_out: asynchronous on the compute stream */
int bk_chain_emit(bk_q *q, const struct bk_chain_args *a, uint8_t *d_out, uint32_t b0, uint32_t b1);
/* records emitted since the last bk_flags_clear() */
int bk_records_out(bk_q *q, uint64_t *n);

/* result download session: bytes [lo,hi) of d_out become valid after the emission just
 * enqueued; they are DMA'd into a pinned ring and moved into h_dst by host threads. */
/* memcpy for write-once destinations (runtime.c): non-temporal stores where available */
void flbgpu_stream_copy(void *dst, const void *src, size_t n);
int bk_download_begin(bk_q *q, void *h_dst, const void *d_out);
int bk_download_push(bk_q *q, size_t lo, size_t hi);
int bk_download_end(bk_q *q);

/* ---- the small-chunk form -------------------------------------------------------
 * What flb_filter_do() hands a filter is one append: tens of KB to a few MB.  For such a chunk the
 * pipeline above is all overhead, so the whole call is enqueued on ONE stream without a host
 * synchronisation in between -- upload, record index, evaluation, sizes, emission under the
 * speculated verdict vector -- with every count the later kernels need (records, candidates, result
 * bytes) staying in device memory; the host waits once, reads the mail below, and fetches the result.
 * a->d_off/d_len/d_kind/d_size hold cap_rec records, a->d_bsum ceil(cap_rec/BK_REC_BLOCK)+2 entries. */
struct bk_small_res {
    uint32_t n_cand, n_valid, tiled, overflow;   /* overflow: more candidates than cap_rec, nothing after the index is valid */
    uint64_t end_off;                            /* where the decodable prefix ends */
    uint64_t total;                              /* result bytes */
    uint64_t n_out;                              /* records in the result */
    uint32_t emitted;                            /* 0: the result did not fit cap_out, nothing was written */
    uint32_t flags[FLBGPU_MAX_FILTERS + 1];
};
int bk_small_run(bk_q *q, const struct bk_chain_args *a, const void *h_in, uint8_t *d_in, size_t bytes, uint32_t cap_rec,
                 uint32_t *d_tile, uint32_t n_tiles, uint8_t *d_out, size_t cap_out, struct bk_small_res *res);
/* result bytes [0,n) of d_out into the caller's (pageable) buffer; synchronises */
int bk_small_fetch(bk_q *q, void *h_dst, const uint8_t *d_out, size_t n);

/* ---- the one exchange of the path: metric tables of filter_log_to_metrics over NCCL (NVLink / NVSwitch) ----
 * One communicator per context (its default queue).  libnccl is opened at run time, so a single-GPU deployment needs
 * no NCCL at all.  d_* are device buffers; the calls are synchronous (the tables are a few KB). */
int bk_comm_unique_id(uint8_t id[128]);
int bk_comm_init(bk_q *q, int nranks, int rank, const uint8_t id[128]);
int bk_comm_info(bk_q *q, int *nranks, int *rank);          /* 0 when a communicator exists */
int bk_comm_allgather(bk_q *q, const void *d_send, void *d_recv, size_t bytes_per_rank);
int bk_comm_allreduce_u64(bk_q *q, void *d_buf, size_t count);            /* sum */
int bk_comm_allreduce_f64(bk_q *q, void *d_buf, size_t count);            /* sum */

/* ---- streaming JSON packer (flb_pack_json_state over a batch of stream buffers): one lane per buffer ----
 * d_js holds the buffers back to back, buffer i = d_js[d_off[i], d_off[i] + d_len[i]); its tokens live at
 * d_tok[d_tok_off[i] .. + d_tok_cap[i]), its unescape scratch at d_tmp[d_off[i] + i ..) (d_len[i] + 1 bytes).
 * scan: tokenise, decide what is whole, measure (d_res[i]); emit: pack buffer i at d_out + d_out_off[i].
 * Both are asynchronous on the queue's stream. */
struct bk_jsmn_args {
    const uint8_t *d_js; const uint32_t *d_off, *d_len; uint32_t n;
    struct jm_tok *d_tok; const uint32_t *d_tok_off, *d_tok_cap;
    uint8_t *d_tmp; struct jm_result *d_res;
    uint8_t *d_out; const uint32_t *d_out_off;
};
int bk_jsmn_scan(bk_q *q, const struct bk_jsmn_args *a);
int bk_jsmn_emit(bk_q *q, const struct bk_jsmn_args *a);

/* filter_multiline (dev_ml.cuh), asynchronous on the queue's stream.  plan: per-record pass, automaton tree, action and
 * event lists (e->res: events, final state, the group's time); sizes: ev_size[] of the n_ev events; emit: event j at
 * d_out + d_bsum[j / BK_REC_BLOCK] + (sum of the sizes before it in its block). */
int bk_ml_plan(bk_q *q, const struct ml_env *e);
int bk_ml_sizes(bk_q *q, const struct ml_env *e, uint32_t n_ev);
int bk_ml_emit(bk_q *q, const struct ml_env *e, uint32_t n_ev, const uint64_t *d_bsum, uint8_t *d_out);

/* chunk -> JSON text (dev_tojson.cuh), asynchronous on the queue's stream.  sizes: every event packed as one map in its scratch
 * slice, e->size[i] = bytes of its text; emit: event i at d_out + d_bsum[i / BK_REC_BLOCK] + (sizes before it in its block). */
int bk_tj_sizes(bk_q *q, const struct tj_env *e);
int bk_tj_emit(bk_q *q, const struct tj_env *e, const uint64_t *d_bsum, uint8_t *d_out);
/* chunk -> GELF messages (dev_gelf.cuh), asynchronous on the queue's stream.  sizes: e->size[i] = bytes of event i's message
 * and separator, 0 for an event left out (counted in e->failed when the reference returns NULL for it); emit: event i at
 * d_out + d_bsum[i / BK_REC_BLOCK] + (sizes before it in its block). */
int bk_gf_sizes(bk_q *q, const struct gf_env *e);
int bk_gf_emit(bk_q *q, const struct gf_env *e, const uint64_t *d_bsum, uint8_t *d_out);

/* raw text -> log events (dev_lines.cuh), asynchronous on the queue's stream.  count: e->cnt[t] per tile; fill: e->nl[] from the
 * tile offsets (d_bsum per BK_REC_BLOCK tiles); sizes: e->size[k] per line; emit: line k's event at d_out + d_bsum[k / BK_REC_BLOCK]
 * + (sizes before it in its block). */
int bk_ln_count(bk_q *q, const struct ln_env *e);
int bk_ln_fill(bk_q *q, const struct ln_env *e, const uint64_t *d_bsum);
int bk_ln_sizes(bk_q *q, const struct ln_env *e);
int bk_ln_emit(bk_q *q, const struct ln_env *e, const uint64_t *d_bsum, uint8_t *d_out);
/* ... with a parser, asynchronous on the queue's stream.  mid_size: t->msize[k] per line, kept lines counted in t->ln.n_events;
 * mid_emit: line k's event of the parser's input at t->mid + t->mbsum[k / BK_REC_BLOCK] + (sizes before it in its block);
 * sizes (after the parser's chain has run): t->r_out[] per record, then t->rec[k] and t->size[k] per line (*t->bad counts the
 * lines without a record); emit: line k's event at d_out + d_bsum[k / BK_REC_BLOCK] + (sizes before it in its block). */
int bk_tl_mid_size(bk_q *q, const struct tl_env *t);
int bk_tl_mid_emit(bk_q *q, const struct tl_env *t);
int bk_tl_sizes(bk_q *q, const struct tl_env *t);
int bk_tl_emit(bk_q *q, const struct tl_env *t, const uint64_t *d_bsum, uint8_t *d_out);

#ifdef __cplusplus
}
#endif
#endif
