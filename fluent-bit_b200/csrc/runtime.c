/* runtime.c -- host side of libflbgpu (plain C): contexts, parser definitions,
 * filter instances (property lists, cb_init-time validation), chain compilation
 * into the device program blob, and the per-call driver
 *   upload -> record index -> evaluation pass (-> revise chunk-level assumptions)
 *          -> prefix sum -> emission pass -> download.
 *
 * Reference behaviour mirrored here (paths in /root/reference):
 *   flb_parser_create ............ src/flb_parser.c:148-348
 *   flb_filter_set_property ...... src/flb_filter.c:325-410
 *   filter_parser cb_init ........ plugins/filter_parser/filter_parser.c:60-172
 *   filter_grep set_rules ........ plugins/filter_grep/grep.c:56-165,196-248
 *   filter_modify setup .......... plugins/filter_modify/modify.c:141-513
 *   record_modifier configure .... plugins/filter_record_modifier/filter_modifier.c:36-160
 *   record accessor text ......... src/flb_record_accessor.c:64-232, src/record_accessor/ra.l,ra.y
 *   chunk-level MODIFIED/NOTOUCH . each plugin's cb_filter epilogue (see dev_chain.cuh header)
 */
#define _GNU_SOURCE
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <ctype.h>
#include <time.h>
#include <sys/mman.h>
#include <pthread.h>
#include "../../include/flbgpu.h"
#include "flbgpu_internal.h"
#include "rx_compile.h"

static __thread char g_rt_err[1024];
static void set_err(const char *fmt, const char *a, const char *b)
{
    snprintf(g_rt_err, sizeof(g_rt_err), fmt, a ? a : "", b ? b : "");
}
const char *flbgpu_last_error(void)
{
    if (g_rt_err[0]) return g_rt_err;
    return bk_last_error();
}
const char *flbgpu_backend_name(void) { return bk_name(); }
int flbgpu_device_count(void) { return bk_device_count(); }

/* ------------------------------------------------------------------ blob */
struct blob { uint8_t *p; size_t n, cap; };

static uint32_t blob_reserve(struct blob *b, size_t n, size_t align)
{
    size_t off = (b->n + align - 1) & ~(align - 1);
    if (off + n > b->cap) {
        size_t nc = b->cap ? b->cap * 2 : 4096;
        while (nc < off + n) nc *= 2;
        {
            uint8_t *np_ = realloc(b->p, nc);
            if (!np_) { fprintf(stderr, "libflbgpu: out of memory while building a chain program\n"); abort(); }   /* (configuration time, a few KB) */
            b->p = np_;
        }
        memset(b->p + b->cap, 0, nc - b->cap);
        b->cap = nc;
    }
    memset(b->p + b->n, 0, off - b->n);
    b->n = off + n;
    return (uint32_t) off;
}
static uint32_t blob_add(struct blob *b, const void *d, size_t n, size_t align)
{
    uint32_t off = blob_reserve(b, n ? n : 1, align);
    if (n) memcpy(b->p + off, d, n);
    return off;
}
/* msgpack str (pack_template.h:762-780) */
static uint32_t blob_add_mpstr(struct blob *b, const char *s, uint32_t n, uint32_t *out_len)
{
    uint8_t h[5];
    uint32_t hl, off;
    if (n < 32) { h[0] = 0xa0 | n; hl = 1; }
    else if (n < 256) { h[0] = 0xd9; h[1] = (uint8_t) n; hl = 2; }
    else if (n < 65536) { h[0] = 0xda; h[1] = n >> 8; h[2] = n & 0xff; hl = 3; }
    else { h[0] = 0xdb; h[1] = n >> 24; h[2] = n >> 16; h[3] = n >> 8; h[4] = n; hl = 5; }
    off = blob_reserve(b, hl + n, 1);
    memcpy(b->p + off, h, hl);
    memcpy(b->p + off + hl, s, n);
    *out_len = hl + n;
    return off;
}

/* --------------------------------------------------------------- objects */
struct flbgpu_parser {
    flbgpu_ctx *ctx;
    char *name;
    int type;
    struct rx_compiled rx;
    int has_rx;
    int skip_empty, time_keep, time_strict, logfmt_no_bare_keys;
    char *time_fmt;          /* format up to %L, already "%Y "-prefixed when the format has no year */
    char *time_frac;         /* format after %L or NULL */
    char *time_key;
    int time_with_year, time_with_tz, time_offset, has_time;
    struct flbgpu_parser_types *types;
    int types_len;
    struct flbgpu_parser *next;
    struct pdec *decs; int n_decs;     /* field decoders, one entry per decoded key in order of first appearance */
    flbgpu_chain *solo;      /* lazily built chain behind flbgpu_parser_do() */
    flbgpu_filter *solo_filter;
};

struct pdec_rule { int type, backend, action; };
struct pdec { char *key; int add_extra_keys; struct pdec_rule *rules; int n_rules; };

struct kv { char *k, *v; struct kv *next; };
static void rtag_release(flbgpu_filter *f);
static uint32_t key_hash(const char *s, size_t n);

/* host-side cumulative state of one filter_log_to_metrics instance: what the reference
 * keeps in its struct cmt (lib/cmetrics): one metric per label set, first-seen order */
struct l2m_set {
    uint64_t hash;
    char *labels;            /* n_labels strings, each L2M_LABEL_BYTES: length byte + bytes */
    uint64_t count;          /* counter value / histogram _count */
    double sum;
    uint64_t *buckets;       /* n_buckets + 1 */
    uint64_t call_last;      /* gauge: last record index + 1 seen for this set in the call being folded in */
    /* histogram: a bound on |sum| while the sum is an integer reached by exact additions only (L2M_NOT_EXACT: no longer).
     * While bound + count x max |value| of a call stays <= 2^53, any order of adding gives the record-order sum. */
    uint64_t bound;
    uint64_t call_n, call_amax;  /* histogram: observations of the call being folded in, and their amax */
    double call_sum;             /* ... their atomic sum */
};
struct l2m_state {
    int mode, n_labels, n_buckets, discard;
    char *label_keys[L2M_MAX_LABELS];
    double *bounds;
    char *ns, *subsystem, *name, *desc;
    struct l2m_set *sets;
    int n_sets, cap_sets;
};

struct flbgpu_filter {
    flbgpu_ctx *ctx;
    int kind;
    struct kv *props, *props_tail;
    int inited;
    int needs_scratch;       /* a JSON parser transcodes into per-record scratch */
    flbgpu_chain *solo;
    struct l2m_state *l2m;   /* cumulative metrics of a log_to_metrics filter */
    /* routing (struct flb_filter_instance: match, match_regex; the `active` property): consulted by the fused chain,
     * like flb_filter_do() does per filter (src/flb_filter.c:180-190) */
    char *match;
    struct rx_compiled match_rx; int has_match_rx;
    int inactive;
    /* rewrite_tag: what the last call handed to the emitter, grouped by new tag (flbgpu_filter_emitted) */
    struct flbgpu_emit_group *rt_groups;
    size_t rt_n;
    void *rt_stream;         /* the entries as the device left them: the tags of rt_groups point in here */
    void **rt_bufs;          /* one record buffer per group */
    /* multiline: what the parser instance keeps from chunk to chunk (everything pending is flushed at the end of a call):
     * the rule the group is in (struct flb_ml_stream_group: rule_to_state) and its mp_time */
    uint32_t ml_state;
    int64_t ml_time[2];
};

struct flbgpu_ctx {
    int device;
    struct flbgpu_parser *parsers;
    bk_q *q0;                /* queue of the context-level helpers (flbgpu_dev_*, flbgpu_stream) */
    bk_q *last_q;            /* queue of the most recent chain call: flbgpu_kernel_ms() reads its events */
    struct flbgpu_ml_parser *ml_parsers;      /* multiline parser definitions (config->multiline_parsers) */
    size_t ml_limit; int ml_limit_set;        /* config->multiline_buffer_limit */
    flbgpu_chain *util;                       /* queue and buffers of the context-level conversions (flbgpu_msgpack_to_json_format) */
};
static void ml_parsers_free(flbgpu_ctx *ctx);

struct flbgpu_chain {
    flbgpu_ctx *ctx;
    bk_q *q;                                  /* this instance's device queue: streams, staging rings, worker threads */
    pthread_mutex_t lock;                     /* one call at a time per instance (the reference never re-enters one either) */
    flbgpu_filter *f[FLBGPU_MAX_FILTERS];
    int nf;
    int inited;
    struct blob blob;
    uint8_t *d_blob;
    uint32_t cap_stride;
    int needs_scratch;
    uint32_t scr_mul;
    int split;                                /* evaluation in two launches: the parser (filter 0), then the other filters */
    int defer_ok;                             /* no log_to_metrics filter in front of a parser filter: records may be re-evaluated from scratch */
    uint8_t *d_scr; size_t cap_scr;
    int l2m_index;                            /* filter index of the log_to_metrics filter, or -1 */
    int ml_index;                             /* filter index of the multiline filter, or -1 (it runs on its own: ml_run) */
    uint32_t ml_cfg_off;
    uint8_t *d_mlw; size_t cap_mlw;           /* multiline: work arrays of a call */
    /* `multiline, then other filters` (the shape of BASELINE configs[4]): the multiline filter runs as a chain of its own and
     * hands its result to a chain of the filters behind it on the device -- no trip through host memory in between */
    flbgpu_chain *ml_solo, *ml_post;
    /* flbgpu_chain_set_result_buffer(): results that fit go here instead of into a fresh malloc() */
    uint8_t *res_buf; size_t res_cap;
    int rtag_index;                           /* filter index of the rewrite_tag filter, or -1; -2 = several: the chain runs filter by filter */
    uint32_t *d_esize;                        /* rewrite_tag: bytes of each record's entry in the re-tagged stream */
    uint64_t *d_ebsum, *h_ebsum; size_t cap_ebsum;   /* ... and the scan over them */
    const uint8_t *d_tag; uint32_t tag_len;   /* the tag of the call on the device */
    struct l2m_table l2m;                     /* device table (per-call delta) */
    size_t l2m_slots;
    uint64_t *h_hash, *h_chash, *h_cnt, *h_bkt; uint32_t *h_first; double *h_sum;    /* host mirror */
    uint64_t *h_amax; int32_t *h_setof;       /* histogram: the slots' amax, and the set each slot of a call folds into */
    uint32_t *h_obs_slot; double *h_obs_val; size_t cap_hobs;   /* histogram: the observations of a call, when one set needs them */
    int l2m_record;                           /* histogram: the evaluation writes its observations (from the first call that needed them on) */
    /* device buffers, grown on demand */
    uint8_t *d_in;  size_t cap_in;
    uint8_t *d_out; size_t cap_out;
    uint32_t *d_tile; size_t cap_tile;
    uint32_t *d_off, *d_len, *d_size; uint8_t *d_kind; size_t cap_rec;
    uint64_t *d_bsum; size_t cap_bsum;
    int32_t *d_cap; size_t cap_cap;
    uint32_t *d_flags;
    uint64_t *h_bsum; size_t cap_hbsum;      /* host copy of the per-block output offsets */
    uint32_t spec_assume; int spec_valid;     /* verdict vector of the previous call: what the streaming path speculates on */
    int want_report;                          /* the chain behind flbgpu_parser_do(): the parser also reports position and time per record */
    int32_t *d_prep; size_t cap_prep; int32_t *h_prep; size_t cap_hprep;
    uint32_t active;                          /* bit k: filter k is routed this call's tag (Match / Match_Regex / active) */
    uint32_t spec_active;                     /* the routing the speculation belongs to */
    uint32_t small_cap_rec; size_t small_cap_out;   /* what the small-chunk form learnt about this instance's chunks */
    int keep_result;                          /* the device-output form without a caller's buffer: the result stays in d_out */
    /* flbgpu_lines_to_events_parsed() on a parser's chain: the text, the lines and the parser's input live apart from every
     * buffer chain_run() grows, since growing one frees memory queued kernels may still read */
    uint8_t *d_tl_text, *d_tl_mid, *d_tl_out; uint32_t *d_tl_line, *d_tl_rec; uint64_t *d_tl_bsum, *h_tl_bsum;
    size_t cap_tl_text, cap_tl_mid, cap_tl_out, cap_tl_line, cap_tl_rec, cap_tl_bsum, cap_tl_hbsum;
    struct flbgpu_stats st;
};

/* ---------------------------------------------------------------- context */
flbgpu_ctx *flbgpu_init(int device)
{
    flbgpu_ctx *c;
    g_rt_err[0] = 0;
    {
        bk_q *q0 = bk_q_new(device);
        if (!q0) return NULL;
        c = calloc(1, sizeof(*c));
        if (!c) { bk_q_free(q0); set_err("out of memory%s%s", NULL, NULL); return NULL; }
        c->device = device;
        c->q0 = q0;
    }
    return c;
}

void flbgpu_parser_destroy(flbgpu_parser *p);

void flbgpu_shutdown(flbgpu_ctx *ctx)
{
    if (!ctx) return;
    while (ctx->parsers) flbgpu_parser_destroy(ctx->parsers);
    ml_parsers_free(ctx);
    if (ctx->util) flbgpu_chain_destroy(ctx->util);
    bk_q_free(ctx->q0);
    free(ctx);
}

void *flbgpu_dev_alloc(flbgpu_ctx *ctx, size_t n) { return bk_alloc(ctx->q0, n); }
void  flbgpu_dev_free(flbgpu_ctx *ctx, void *p) { bk_free(ctx->q0, p); }
int   flbgpu_dev_upload(flbgpu_ctx *ctx, void *d, const void *h, size_t n) { if (bk_h2d(ctx->q0, d, h, n)) return -1; return bk_sync(ctx->q0); }
int   flbgpu_dev_download(flbgpu_ctx *ctx, void *h, const void *d, size_t n) { if (bk_d2h(ctx->q0, h, d, n)) return -1; return bk_sync(ctx->q0); }
void *flbgpu_host_alloc(flbgpu_ctx *ctx, size_t n) { return bk_alloc_host(ctx->q0, n); }
void  flbgpu_host_free(flbgpu_ctx *ctx, void *p) { bk_free_host(ctx->q0, p); }
void *flbgpu_stream(flbgpu_ctx *ctx) { return bk_stream(ctx->q0); }

/* ---------------------------------------------------------------- parsers */
static int tzone_offset(const char *str, int len, int *tmdiff)
{
    /* flb_parser_tzone_offset(), src/flb_parser.c:1069-1127 */
    int neg;
    long hour, min;
    const char *end, *p = str;
    if (*p == 'Z') { *tmdiff = 0; return 0; }
    if (*p != '+' && *p != '-') { *tmdiff = 0; return -1; }
    if (len < 4) { *tmdiff = 0; return -1; }
    neg = (*p++ == '-');
    end = str + len;
    hour = ((p[0] - '0') * 10) + (p[1] - '0');
    if (end - p == 5 && p[2] == ':') {
        if (len < 5) { *tmdiff = 0; return -1; }
        min = ((p[3] - '0') * 10) + (p[4] - '0');
    }
    else min = ((p[2] - '0') * 10) + (p[3] - '0');
    if (hour < 0 || hour > 59 || min < 0 || min > 59) return -1;
    *tmdiff = (int) ((hour * 3600) + (min * 60));
    if (neg) *tmdiff = -*tmdiff;
    return 0;
}

/* conversions dev_time.cuh implements */
static int time_fmt_supported(const char *f, char *bad)
{
    for (; *f; f++) {
        if (*f != '%') continue;
        f++;
        while (*f == 'E' || *f == 'O') f++;
        if (!*f) return 1;
        /* conversions flb_strptime() has and the device restatement has not (locale formats); a letter neither knows
         * makes every parse fail at run time, there (src/flb_strptime.c: default -> NULL) and here (dt_strptime) */
        if (strchr("cxX+", *f)) { *bad = *f; return 0; }
    }
    return 1;
}

flbgpu_parser *flbgpu_parser_get(flbgpu_ctx *ctx, const char *name)
{
    struct flbgpu_parser *p;
    for (p = ctx->parsers; p; p = p->next) if (p->name && strcmp(p->name, name) == 0) return p;
    return NULL;
}

static int split_tokens(const char *str, int max_split, char **out, int max_out);
static void free_toks(char **t, int n);

/* flb_parser_decoder_list_create(), src/flb_parser_decoder.c:594-745 */
static int parser_decoders(struct flbgpu_parser *p, const struct flbgpu_parser_decoder *d)
{
    for (; d->property; d++) {
        char *tok[4];
        int nt, type, backend, action = PDEC_ACT_NONE, i;
        struct pdec *dec = NULL;
        if (!strcasecmp(d->property, "decode_field")) type = PDEC_DEFAULT;
        else if (!strcasecmp(d->property, "decode_field_as")) type = PDEC_AS;
        else continue;
        nt = split_tokens(d->value ? d->value : "", 3, tok, 4);
        if (nt < 2) { free_toks(tok, nt); set_err("[parser] invalid number of parameters in decoder%s%s", NULL, NULL); return -1; }
        if (!strcasecmp(tok[0], "json")) backend = PDEC_JSON;
        else if (!strcasecmp(tok[0], "escaped")) backend = PDEC_ESCAPED;
        else if (!strcasecmp(tok[0], "escaped_utf8")) backend = PDEC_ESCAPED_UTF8;
        else if (!strcasecmp(tok[0], "mysql_quoted")) backend = PDEC_MYSQL_QUOTED;
        else { set_err("[parser] field decoder '%s' unknown%s", tok[0], NULL); free_toks(tok, nt); return -1; }
        if (nt >= 3) {
            if (!strcasecmp(tok[2], "try_next")) action = PDEC_ACT_TRY_NEXT;
            else if (!strcasecmp(tok[2], "do_next")) action = PDEC_ACT_DO_NEXT;
        }
        for (i = 0; i < p->n_decs; i++) if (!strcmp(p->decs[i].key, tok[1])) { dec = &p->decs[i]; break; }
        if (!dec) {
            struct pdec *nd = realloc(p->decs, sizeof(*nd) * (size_t) (p->n_decs + 1));
            if (!nd) { free_toks(tok, nt); set_err("out of memory%s%s", NULL, NULL); return -1; }
            p->decs = nd;
            dec = &p->decs[p->n_decs++];
            memset(dec, 0, sizeof(*dec));
            dec->key = strdup(tok[1]);
        }
        {
            struct pdec_rule *nr = realloc(dec->rules, sizeof(*nr) * (size_t) (dec->n_rules + 1));
            if (!nr) { free_toks(tok, nt); set_err("out of memory%s%s", NULL, NULL); return -1; }
            dec->rules = nr;
            nr[dec->n_rules].type = type; nr[dec->n_rules].backend = backend; nr[dec->n_rules].action = action;
            dec->n_rules++;
        }
        if (type == PDEC_DEFAULT) dec->add_extra_keys = 1;
        free_toks(tok, nt);
    }
    return 0;
}

flbgpu_parser *flbgpu_parser_create(flbgpu_ctx *ctx, const char *name, const char *format,
                                    const char *p_regex, int skip_empty,
                                    const char *time_fmt, const char *time_key,
                                    const char *time_offset, int time_keep, int time_strict,
                                    int time_system_timezone, int logfmt_no_bare_keys,
                                    struct flbgpu_parser_types *types, int types_len, void *decoders)
{
    struct flbgpu_parser *p;
    int i;
    g_rt_err[0] = 0;
    if (!ctx || !name || !format) { set_err("parser: missing argument%s%s", NULL, NULL); return NULL; }
    if (flbgpu_parser_get(ctx, name)) { set_err("[parser] parser named '%s' already exists, skip.%s", name, NULL); return NULL; }
    if (time_system_timezone) { set_err("[parser:%s] Time_System_Timezone is not supported on the GPU path%s", name, NULL); return NULL; }
    p = calloc(1, sizeof(*p));
    if (!p) { set_err("out of memory%s%s", NULL, NULL); return NULL; }
    p->ctx = ctx;
    if (!strcasecmp(format, "regex")) p->type = FLBGPU_PARSER_REGEX;
    else if (!strcasecmp(format, "json")) p->type = FLBGPU_PARSER_JSON;
    else if (!strcasecmp(format, "ltsv")) p->type = FLBGPU_PARSER_LTSV;
    else if (!strcasecmp(format, "logfmt")) p->type = FLBGPU_PARSER_LOGFMT;
    else { set_err("[parser:%s] Invalid format %s", name, format); free(p); return NULL; }

    if (p->type == FLBGPU_PARSER_REGEX) {
        if (!p_regex) { set_err("[parser:%s] Invalid regex pattern%s", name, NULL); free(p); return NULL; }
        if (rx_compile(p_regex, &p->rx) != 0) {
            char tmp[300];
            snprintf(tmp, sizeof(tmp), "%s (%s)", p_regex, p->rx.err);
            set_err("[parser:%s] Invalid regex pattern %s", name, tmp);
            free(p);
            return NULL;
        }
        p->has_rx = 1;
        p->skip_empty = skip_empty;
    }
    p->name = strdup(name);
    if (time_fmt) {
        char *fmt, *l;
        char bad = 0;
        p->has_time = 1;
        if (strstr(time_fmt, "%Y") || strstr(time_fmt, "%y") || strstr(time_fmt, "%s")) {
            p->time_with_year = 1;
            fmt = strdup(time_fmt);
        }
        else {
            p->time_with_year = 0;
            fmt = malloc(strlen(time_fmt) + 4);
            sprintf(fmt, "%%Y %s", time_fmt);
        }
        if (strstr(time_fmt, "%z") || strstr(time_fmt, "%Z") || strstr(time_fmt, "%SZ") || strstr(time_fmt, "%S.%LZ"))
            p->time_with_tz = 1;
        l = strstr(fmt, "%L");
        if (l) { l[0] = 0; p->time_frac = strdup(l + 2); }
        p->time_fmt = fmt;
        if (!time_fmt_supported(p->time_fmt, &bad) || (p->time_frac && !time_fmt_supported(p->time_frac, &bad))) {
            char b[2] = { bad, 0 };
            set_err("[parser:%s] time conversion %%%s is not supported on the GPU path", name, b);
            flbgpu_parser_destroy(p);
            return NULL;
        }
        if (time_offset) {
            int diff = 0;
            if (tzone_offset(time_offset, (int) strlen(time_offset), &diff) == -1) {
                set_err("[parser:%s] invalid Time_Offset '%s'", name, time_offset);
                flbgpu_parser_destroy(p);
                return NULL;
            }
            p->time_offset = diff;
        }
    }
    if (time_key) p->time_key = strdup(time_key);
    p->time_keep = time_keep;
    p->time_strict = time_strict;
    p->logfmt_no_bare_keys = logfmt_no_bare_keys;
    if (types_len > 0) {
        p->types = calloc(types_len, sizeof(*types));
        for (i = 0; i < types_len; i++) {
            p->types[i].key = types[i].key ? strndup(types[i].key, types[i].key_len) : NULL;
            p->types[i].key_len = types[i].key_len;
            p->types[i].type = types[i].type;
        }
        p->types_len = types_len;
    }
    if (decoders && parser_decoders(p, (const struct flbgpu_parser_decoder *) decoders) != 0) { flbgpu_parser_destroy(p); return NULL; }
    p->next = ctx->parsers;
    ctx->parsers = p;
    return p;
}

void flbgpu_parser_destroy(flbgpu_parser *p)
{
    struct flbgpu_parser **pp;
    int i;
    if (!p) return;
    for (pp = &p->ctx->parsers; *pp; pp = &(*pp)->next) if (*pp == p) { *pp = p->next; break; }
    if (p->solo) flbgpu_chain_destroy(p->solo);
    if (p->solo_filter) flbgpu_filter_destroy(p->solo_filter);
    if (p->has_rx) rx_compiled_free(&p->rx);
    for (i = 0; i < p->n_decs; i++) { free(p->decs[i].key); free(p->decs[i].rules); }
    free(p->decs);
    for (i = 0; i < p->types_len; i++) free(p->types[i].key);
    free(p->types); free(p->name); free(p->time_fmt); free(p->time_frac); free(p->time_key);
    free(p);
}

/* emit the device view of a parser; returns its offset */
/* Compile "fmt [%L frac_fmt]" into TF_* ops (flbgpu_prog.h) when it only uses directives with a fixed
 * shape; 0 when it does not (the general interpreter handles everything anyway). */
static int time_fast_compile(const char *fmt, const char *frac_fmt, uint8_t *out, int cap)
{
    int n = 0, part;
    int seen_year = 0;
    for (part = 0; part < 2; part++) {
        const char *f = part == 0 ? fmt : frac_fmt;
        if (part == 1) {
            if (!frac_fmt) break;
            if (n + 1 >= cap) return 0;
            out[n++] = TF_FRAC;
        }
        for (; f && *f; f++) {
            if (n + 4 >= cap) return 0;
            if (*f == ' ') { out[n++] = TF_SPACE; continue; }
            if (isspace((unsigned char) *f)) return 0;
            if (*f != '%') { out[n++] = TF_LIT; out[n++] = (uint8_t) *f; continue; }
            f++;
            switch (*f) {
            case 'd': out[n++] = TF_D2; out[n++] = TFF_MDAY; out[n++] = 1; out[n++] = 31; break;
            case 'm': out[n++] = TF_D2; out[n++] = TFF_MON; out[n++] = 1; out[n++] = 12; break;
            case 'H': out[n++] = TF_D2; out[n++] = TFF_HOUR; out[n++] = 0; out[n++] = 23; break;
            case 'M': out[n++] = TF_D2; out[n++] = TFF_MIN; out[n++] = 0; out[n++] = 59; break;
            case 'S': out[n++] = TF_D2; out[n++] = TFF_SEC; out[n++] = 0; out[n++] = 60; break;
            case 'Y': out[n++] = TF_Y4; seen_year = 1; break;
            case 'b': case 'h': out[n++] = TF_MON3; break;
            case 'z': out[n++] = TF_TZ; break;
            case '%': out[n++] = TF_LIT; out[n++] = '%'; break;
            case 'T':
                out[n++] = TF_D2; out[n++] = TFF_HOUR; out[n++] = 0; out[n++] = 23; out[n++] = TF_LIT; out[n++] = ':';
                if (n + 12 >= cap) return 0;
                out[n++] = TF_D2; out[n++] = TFF_MIN; out[n++] = 0; out[n++] = 59; out[n++] = TF_LIT; out[n++] = ':';
                out[n++] = TF_D2; out[n++] = TFF_SEC; out[n++] = 0; out[n++] = 60;
                break;
            default: return 0;           /* %y %e %j %s %Z %F ...: general path only */
            }
        }
    }
    if (!seen_year || n + 1 >= cap) return 0;
    out[n++] = TF_END;
    return n;
}

static uint32_t emit_pdef(struct blob *b, struct flbgpu_parser *p)
{
    struct cf_pdef d;
    uint32_t off, i, nn = 0;
    memset(&d, 0, sizeof(d));
    d.type = p->type;
    d.skip_empty = p->skip_empty; d.time_keep = p->time_keep; d.time_strict = p->time_strict;
    d.has_time = p->has_time; d.time_with_year = p->time_with_year; d.time_with_tz = p->time_with_tz;
    /* bit 1: the access-log format, for which the device has a direct path (dt_fast_apache) */
    if (p->has_time && p->time_fmt && !p->time_frac && !strcmp(p->time_fmt, "%d/%b/%Y:%H:%M:%S %z")) d.has_time |= 2;
    d.time_offset = p->time_offset; d.logfmt_no_bare_keys = p->logfmt_no_bare_keys;
    if (p->has_time && p->time_with_year) {
        uint8_t prog[128];
        int n = time_fast_compile(p->time_fmt, p->time_frac, prog, (int) sizeof(prog));
        if (n > 0) d.tfast_off = blob_add(b, prog, (size_t) n, 1);
    }
    if (p->has_time) {
        d.fmt_off = blob_add(b, p->time_fmt, strlen(p->time_fmt) + 1, 1);
        if (p->time_frac) { d.has_frac = 1; d.frac_off = blob_add(b, p->time_frac, strlen(p->time_frac) + 1, 1); }
    }
    if (p->has_rx) {
        const char *tk = p->time_key ? p->time_key : "time";
        struct cf_pname *nm;
        int ni, g;
        d.rx_off = blob_add(b, p->rx.prog, p->rx.prog->total_bytes, 16);
        d.n_groups = p->rx.prog->n_groups;
        for (ni = 0; ni < p->rx.n_names; ni++) nn += p->rx.names[ni].n_groups;
        nm = calloc(nn ? nn : 1, sizeof(*nm));
        i = 0;
        for (ni = 0; ni < p->rx.n_names; ni++) {
            const char *name = p->rx.names[ni].name;
            uint32_t len = (uint32_t) strlen(name);
            for (g = 0; g < p->rx.names[ni].n_groups; g++, i++) {
                int t;
                nm[i].kmp_off = blob_add_mpstr(b, name, len, &nm[i].kmp_len);
                nm[i].raw_off = blob_add(b, name, len, 1);
                nm[i].raw_len = len;
                nm[i].hash = key_hash(name, len);
                nm[i].group = p->rx.names[ni].groups[g];
                nm[i].is_time = p->has_time && strcmp(name, tk) == 0;
                for (t = 0; t < p->types_len; t++) {
                    if (p->types[t].key && (uint32_t) p->types[t].key_len == len && !strncmp(name, p->types[t].key, len)) {
                        nm[i].cast = p->types[t].type;
                        break;
                    }
                }
            }
        }
        d.n_names = nn;
        d.names_off = blob_add(b, nm, sizeof(*nm) * (nn ? nn : 1), 8);
        free(nm);
    }
    {
        const char *tk = p->time_key ? p->time_key : "time";
        d.time_key_off = blob_add(b, tk, strlen(tk), 1);
        d.time_key_hash = key_hash(tk, strlen(tk));
        d.time_key_len = (uint32_t) strlen(tk);
    }
    if (p->types_len > 0 && !p->has_rx) {
        struct cf_ptype *ty = calloc(p->types_len, sizeof(*ty));
        int t, nt = 0;
        for (t = 0; t < p->types_len; t++) {
            if (!p->types[t].key) continue;
            ty[nt].key_off = blob_add(b, p->types[t].key, p->types[t].key_len, 1);
            ty[nt].key_len = (uint32_t) p->types[t].key_len;
            ty[nt].type = (uint32_t) p->types[t].type;
            nt++;
        }
        d.n_types = nt;
        d.types_off = blob_add(b, ty, sizeof(*ty) * (nt ? nt : 1), 8);
        free(ty);
    }
    if (p->n_decs > 0) {
        struct cf_pdec *dc = calloc((size_t) p->n_decs, sizeof(*dc));
        int k;
        for (k = 0; k < p->n_decs; k++) {
            struct cf_pdec_rule *rl = calloc((size_t) p->decs[k].n_rules, sizeof(*rl));
            int r;
            for (r = 0; r < p->decs[k].n_rules; r++) {
                rl[r].type = (uint32_t) p->decs[k].rules[r].type; rl[r].backend = (uint32_t) p->decs[k].rules[r].backend;
                rl[r].action = (uint32_t) p->decs[k].rules[r].action;
            }
            dc[k].key_off = blob_add(b, p->decs[k].key, strlen(p->decs[k].key), 1);
            dc[k].key_len = (uint32_t) strlen(p->decs[k].key);
            dc[k].add_extra_keys = (uint32_t) p->decs[k].add_extra_keys;
            dc[k].n_rules = (uint32_t) p->decs[k].n_rules;
            dc[k].rules_off = blob_add(b, rl, sizeof(*rl) * (size_t) p->decs[k].n_rules, 8);
            free(rl);
        }
        d.n_dec = (uint32_t) p->n_decs;
        d.dec_off = blob_add(b, dc, sizeof(*dc) * (size_t) p->n_decs, 8);
        free(dc);
    }
    off = blob_add(b, &d, sizeof(d), 8);
    return off;
}

/* ----------------------------------------------------------------- filters */
static int plugin_kind(const char *name)
{
    if (!strcasecmp(name, "parser")) return FLBGPU_F_PARSER;
    if (!strcasecmp(name, "grep")) return FLBGPU_F_GREP;
    if (!strcasecmp(name, "modify")) return FLBGPU_F_MODIFY;
    if (!strcasecmp(name, "record_modifier")) return FLBGPU_F_RECORD_MODIFIER;
    if (!strcasecmp(name, "log_to_metrics")) return FLBGPU_F_LOG_TO_METRICS;
    if (!strcasecmp(name, "rewrite_tag")) return FLBGPU_F_REWRITE_TAG;
    if (!strcasecmp(name, "multiline")) return FLBGPU_F_MULTILINE;
    return 0;
}

flbgpu_filter *flbgpu_filter_new(flbgpu_ctx *ctx, const char *plugin)
{
    flbgpu_filter *f;
    int kind = plugin ? plugin_kind(plugin) : 0;
    g_rt_err[0] = 0;
    if (!ctx || !kind) { set_err("unknown filter plugin '%s'%s", plugin, NULL); return NULL; }
    f = calloc(1, sizeof(*f));
    if (!f) { set_err("out of memory%s%s", NULL, NULL); return NULL; }
    f->ctx = ctx;
    f->kind = kind;
    return f;
}

int flbgpu_filter_set_property(flbgpu_filter *f, const char *k, const char *v)
{
    struct kv *n;
    if (!f || !k || !v) return -1;
    /* instance-level keys are consumed by the framework, not by the plugin
     * (src/flb_filter.c:346-395) */
    if (!strcasecmp(k, "match")) { free(f->match); f->match = strdup(v); return f->match ? 0 : -1; }
    if (!strcasecmp(k, "match_regex")) {
        if (f->has_match_rx) { rx_compiled_free(&f->match_rx); f->has_match_rx = 0; }
        if (rx_compile(v, &f->match_rx) != 0) { set_err("could not compile Match_Regex '%s' (%s)", v, f->match_rx.err); return -1; }
        f->has_match_rx = 1;
        return 0;
    }
    if (!strcasecmp(k, "alias") || !strcasecmp(k, "log_level") || !strcasecmp(k, "log_suppress_interval")) return 0;
    if (!strcasecmp(k, "active")) {                   /* is_active(), src/flb_filter.c:90-105; the property stays in the list there too */
        if (!strcasecmp(v, "FALSE") || !strcmp(v, "0")) f->inactive = 1;
        return 0;
    }
    n = calloc(1, sizeof(*n));
    if (!n) { set_err("out of memory%s%s", NULL, NULL); return -1; }
    n->k = strdup(k);
    n->v = strdup(v);
    if (!n->k || !n->v) { free(n->k); free(n->v); free(n); set_err("out of memory%s%s", NULL, NULL); return -1; }
    if (f->props_tail) f->props_tail->next = n; else f->props = n;
    f->props_tail = n;
    return 0;
}

static void l2m_state_free(struct l2m_state *st);
/* 64-bit words per slot of the device table's bkt array: cumulative buckets + Inf, or the gauge's (last record + 1, value bits) */
#define L2M_NBK(st) ((st)->mode == L2M_GAUGE ? (size_t) 2 : (size_t) (st)->n_buckets + 1)

void flbgpu_filter_destroy(flbgpu_filter *f)
{
    struct kv *n, *nx;
    if (!f) return;
    if (f->solo) flbgpu_chain_destroy(f->solo);
    l2m_state_free(f->l2m);
    rtag_release(f);
    free(f->match);
    if (f->has_match_rx) rx_compiled_free(&f->match_rx);
    for (n = f->props; n; n = nx) { nx = n->next; free(n->k); free(n->v); free(n); }
    free(f);
}

static void rtag_release(flbgpu_filter *f)
{
    size_t i;
    for (i = 0; i < f->rt_n; i++) free(f->rt_bufs[i]);
    free(f->rt_bufs); free(f->rt_groups); free(f->rt_stream);
    f->rt_bufs = NULL; f->rt_groups = NULL; f->rt_stream = NULL; f->rt_n = 0;
}

static int parse_bool(const char *v)
{
    /* flb_utils_bool() */
    if (!strcasecmp(v, "true") || !strcasecmp(v, "on") || !strcasecmp(v, "yes")) return 1;
    if (!strcasecmp(v, "false") || !strcasecmp(v, "off") || !strcasecmp(v, "no")) return 0;
    return -1;
}

/* record accessor text -> struct cf_ra in the blob.  Supported shapes: "$key",
 * "$key['a'][0]...", and a plain string (taken as the key name).  Returns 0 on error. */
static uint32_t emit_ra(struct blob *b, const char *s)
{
    struct cf_ra ra;
    struct cf_ra_sub subs[32];
    uint32_t ns = 0;
    memset(&ra, 0, sizeof(ra));
    if (!s || !*s) return 0;
    if (s[0] != '$') {
        if (strchr(s, '$')) { set_err("unsupported record accessor '%s'%s", s, NULL); return 0; }
        ra.key_off = blob_add(b, s, strlen(s), 1);
        ra.key_len = (uint32_t) strlen(s);
        return blob_add(b, &ra, sizeof(ra), 8);
    }
    {
        const char *p = s + 1, *st = p;
        if (!(isalpha((unsigned char) *p) || *p == '_')) { set_err("invalid record accessor? '%s'%s", s, NULL); return 0; }
        while (isalnum((unsigned char) *p) || *p == '_' || *p == '.' || *p == '-' || *p == '/') {
            /* src/flb_record_accessor.c:170-182: '.', ' ', ',' and '"' end the accessor text */
            if (*p == '.') break;
            p++;
        }
        ra.key_off = blob_add(b, st, (size_t) (p - st), 1);
        ra.key_len = (uint32_t) (p - st);
        while (*p == '[') {
            p++;
            if (ns >= 32) { set_err("record accessor too deep '%s'%s", s, NULL); return 0; }
            if (*p == '\'') {
                char *tmp = malloc(strlen(p) + 1);
                size_t n = 0;
                p++;
                for (;;) {
                    if (!*p) { free(tmp); set_err("invalid record accessor? '%s'%s", s, NULL); return 0; }
                    if (*p == '\'') { if (p[1] == '\'') { tmp[n++] = '\''; p += 2; continue; } break; }
                    tmp[n++] = *p++;
                }
                p++;
                subs[ns].is_index = 0; subs[ns].index = 0;
                subs[ns].str_off = blob_add(b, tmp, n, 1);
                subs[ns].str_len = (uint32_t) n;
                free(tmp);
            }
            else if (isdigit((unsigned char) *p)) {
                subs[ns].is_index = 1; subs[ns].index = (uint32_t) atoi(p);
                subs[ns].str_off = 0; subs[ns].str_len = 0;
                while (isdigit((unsigned char) *p)) p++;
            }
            else { set_err("invalid record accessor? '%s'%s", s, NULL); return 0; }
            if (*p != ']') { set_err("invalid record accessor? '%s'%s", s, NULL); return 0; }
            p++;
            ns++;
        }
        if (*p && *p != '.' && *p != ' ' && *p != ',' && *p != '"') { set_err("invalid record accessor? '%s'%s", s, NULL); return 0; }
        if (*p) { set_err("unsupported record accessor '%s' (text after the key)%s", s, NULL); return 0; }
        ra.n_sub = ns;
        if (ns) ra.sub_off = blob_add(b, subs, sizeof(subs[0]) * ns, 8);
        return blob_add(b, &ra, sizeof(ra), 8);
    }
}

static uint32_t emit_rx(struct blob *b, const char *pattern, uint32_t *max_groups)
{
    struct rx_compiled c;
    uint32_t off;
    if (rx_compile(pattern, &c) != 0) {
        set_err("could not compile regex pattern '%s' (%s)", pattern, c.err);
        return 0;
    }
    off = blob_add(b, c.prog, c.prog->total_bytes, 16);
    if (max_groups && c.prog->n_groups > *max_groups) *max_groups = c.prog->n_groups;
    rx_compiled_free(&c);
    return off;
}

/* flb_utils_split(line, ' ', max_split): leading separators skipped per token, at most
 * max_split tokens then the rest verbatim (src/flb_utils.c:321-456), unquoted */
static int split_plain(const char *line, int max_split, char **out, int max_out)
{
    int n = 0, i = 0, len = (int) strlen(line);
    while (i < len && n < max_out) {
        const char *t = line + i;
        int tl;
        const char *sp;
        while (*t == ' ') t++;
        sp = strchr(t, ' ');
        tl = (sp && sp > t) ? (int) (sp - t) : (int) strlen(t);
        out[n++] = strndup(t, tl);
        i = (int) (t - line) + tl;
        i++;
        if (n >= max_split && max_split > 0 && i < len) {
            if (n < max_out) out[n++] = strdup(line + i);
            break;
        }
    }
    return n;
}

/* flb_utils_split_quoted(line, ' ', max_split) */
static int split_quoted(const char *line, int max_split, char **out, int max_out)
{
    int n = 0, i = 0, len = (int) strlen(line);
    while (i < len && n < max_out) {
        const char *t = line + i;
        while (*t == ' ') t++;
        if (*t != '"' && *t != '\'') {
            const char *sp = strchr(t, ' ');
            int tl = (sp && sp > t) ? (int) (sp - t) : (int) strlen(t);
            out[n++] = strndup(t, tl);
            i = (int) (t - line) + tl;
        }
        else {
            char q = *t;
            const char *p = t + 1;
            char *tok = malloc(strlen(t) + 1);
            int tl = 0;
            while (*p && *p != q) {
                if (*p == '\\' && (p[1] == q || p[1] == '\\')) p++;
                tok[tl++] = *p++;
            }
            if (!*p) { free(tok); return -1; }      /* unterminated quote */
            tok[tl] = 0;
            out[n++] = tok;
            i = (int) (p - line);                    /* at the closing quote */
        }
        i++;
        if (n >= max_split && max_split > 0 && i < len) {
            if (n < max_out) out[n++] = strdup(line + i);
            break;
        }
    }
    return n;
}

/* token_retrieve() loop of flb_slist_split_tokens() for SLIST_2 ("Record k v") */
static int split_tokens(const char *str, int max_split, char **out, int max_out)
{
    const char *p = str;
    int n = 0;
    while (n < max_out) {
        const char *start;
        char *tok;
        int quoted = 0, tl;
        while (*p == ' ') p++;
        if (!*p) break;
        start = p;
        if (*p == '"') {
            quoted = 1; p++; start = p;
            for (;;) {
                while (*p && *p != '"') p++;
                if (!*p) break;
                if (p[-1] == '\\') { p++; continue; }
                break;
            }
        }
        else while (*p && *p != ' ') p++;
        tl = (int) (p - start);
        tok = strndup(start, tl);
        if (quoted) {
            char *in = tok, *o = tok;
            while (*in) { if (in[0] == '\\' && in[1] == '"') { *o++ = '"'; in += 2; } else *o++ = *in++; }
            *o = 0;
            if (*p == '"') p++;
        }
        out[n++] = tok;
        if (!*p) break;
        if (n >= max_split && max_split > 0) {
            while (*p == ' ') p++;
            if (*p && n < max_out) out[n++] = strdup(p);
            break;
        }
    }
    return n;
}

static void free_toks(char **t, int n) { int i; for (i = 0; i < n; i++) free(t[i]); }

/* ---- per-plugin configuration -> blob ---- */
static uint32_t emit_parser_filter(flbgpu_filter *f, struct blob *b, uint32_t *cap_need)
{
    struct cf_parser cf;
    struct kv *p;
    const char *key_name = NULL;
    memset(&cf, 0, sizeof(cf));
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "key_name")) key_name = p->v;
        else if (!strcasecmp(p->k, "parser")) {
            struct flbgpu_parser *ps = flbgpu_parser_get(f->ctx, p->v);
            if (!ps) { set_err("requested parser '%s' not found%s", p->v, NULL); return 0; }
            if (cf.n_parsers >= 8) { set_err("too many parsers in one filter%s%s", NULL, NULL); return 0; }
            cf.pdef_off[cf.n_parsers++] = emit_pdef(b, ps);
            /* no per-record capture slots any more: the emission pass encodes from the cached final
             * field list (RC_CACHE_INTS); only records with more than RC_CACHE_MAXF fields re-run the
             * chain there, and then they re-run the parser too */
            if (ps->type == FLBGPU_PARSER_JSON || ps->type == FLBGPU_PARSER_LOGFMT) f->needs_scratch |= 1;   /* transcoded JSON / decoded logfmt escapes */
            if (ps->n_decs) f->needs_scratch |= 3;                                                        /* + the decoders' own half of the region */
        }
        else if (!strcasecmp(p->k, "preserve_key")) { int v = parse_bool(p->v); if (v < 0) { set_err("invalid boolean '%s'%s", p->v, NULL); return 0; } cf.preserve_key = v; }
        else if (!strcasecmp(p->k, "reserve_data")) { int v = parse_bool(p->v); if (v < 0) { set_err("invalid boolean '%s'%s", p->v, NULL); return 0; } cf.reserve_data = v; }
        else if (!strcasecmp(p->k, "unescape_key")) { /* deprecated, ignored */ }
        else { set_err("[filter parser] unknown configuration property '%s'%s", p->k, NULL); return 0; }
    }
    if (!key_name) { set_err("Key name is required%s%s", NULL, NULL); return 0; }
    if (cf.n_parsers == 0) { set_err("Invalid 'parser'%s%s", NULL, NULL); return 0; }
    cf.key_off = blob_add(b, key_name, strlen(key_name), 1);
    cf.key_len = (uint32_t) strlen(key_name);
    if (key_name[0] == '$') { cf.ra_off = emit_ra(b, key_name); if (!cf.ra_off) return 0; }
    return blob_add(b, &cf, sizeof(cf), 8);
}

static uint32_t emit_grep_filter(flbgpu_filter *f, struct blob *b)
{
    struct cf_grep cf;
    struct cf_grep_rule rules[64];
    struct kv *p;
    int first_rule = 0;
    memset(&cf, 0, sizeof(cf));
    cf.op = GREP_OP_LEGACY;
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "logical_op")) {
            if (!strcasecmp(p->v, "AND")) cf.op = GREP_OP_AND;
            else if (!strcasecmp(p->v, "OR")) cf.op = GREP_OP_OR;
            else if (!strcasecmp(p->v, "legacy")) cf.op = GREP_OP_LEGACY;
        }
    }
    for (p = f->props; p; p = p->next) {
        char *tok[3];
        char field[512];
        int nt, type;
        if (!strcasecmp(p->k, "regex")) type = GREP_REGEX;
        else if (!strcasecmp(p->k, "exclude")) type = GREP_EXCLUDE;
        else if (!strcasecmp(p->k, "logical_op")) continue;
        else { set_err("[filter grep] unknown configuration property '%s'%s", p->k, NULL); return 0; }
        if (cf.op != GREP_OP_LEGACY && first_rule != 0 && first_rule != type) { set_err("Both 'regex' and 'exclude' are set.%s%s", NULL, NULL); return 0; }
        first_rule = type;
        nt = split_plain(p->v, 1, tok, 3);
        if (nt != 2) { free_toks(tok, nt); set_err("invalid regex, expected field and regular expression%s%s", NULL, NULL); return 0; }
        if (cf.n_rules >= 64) { free_toks(tok, nt); set_err("too many grep rules%s%s", NULL, NULL); return 0; }
        if (tok[0][0] == '$') snprintf(field, sizeof(field), "%s", tok[0]);
        else snprintf(field, sizeof(field), "$%s", tok[0]);
        rules[cf.n_rules].type = type;
        rules[cf.n_rules].pad = 0;
        rules[cf.n_rules].ra_off = emit_ra(b, field);
        if (!rules[cf.n_rules].ra_off) { free_toks(tok, nt); return 0; }
        rules[cf.n_rules].rx_off = emit_rx(b, tok[1], NULL);
        free_toks(tok, nt);
        if (!rules[cf.n_rules].rx_off) return 0;
        cf.n_rules++;
    }
    cf.rules_off = blob_add(b, rules, sizeof(rules[0]) * (cf.n_rules ? cf.n_rules : 1), 8);
    return blob_add(b, &cf, sizeof(cf), 8);
}

/* ch_khash() of dev_chain.cuh: length, first, middle and last byte; never 0 */
static uint32_t key_hash(const char *s, size_t n)
{
    uint32_t h = (uint32_t) n * 2654435761u;
    if (n) h ^= (uint32_t) (unsigned char) s[0] ^ ((uint32_t) (unsigned char) s[n - 1] << 8) ^ ((uint32_t) (unsigned char) s[n >> 1] << 16);
    return h | 1u;
}

/* modify.c:468-507 builds a regex from the key AND the value text of EVERY rule, regex rule or not, and refuses
 * the configuration when Onigmo rejects either (tests/runtime/filter_modify.c issue_7368: `remove_wildcard *s3`).
 * Nothing is emitted here; a construct this compiler merely does not cover is not a syntax error. */
static int rule_text_is_a_regex(const char *text)
{
    struct rx_compiled rc;
    memset(&rc, 0, sizeof(rc));
    if (rx_compile(text, &rc) == 0) { rx_compiled_free(&rc); return 1; }
    rx_compiled_free(&rc);
    return strstr(rc.err, "not supported") != NULL;
}

static uint32_t emit_modify_filter(flbgpu_filter *f, struct blob *b)
{
    struct cf_modify cf;
    struct cf_mod_cond *conds = calloc(64, sizeof(*conds));
    struct cf_mod_rule *rules = calloc(256, sizeof(*rules));
    struct kv *p;
    uint32_t ret = 0;
    memset(&cf, 0, sizeof(cf));
    for (p = f->props; p; p = p->next) {
        char *tok[4];
        int nt = split_quoted(p->v, 3, tok, 4);
        if (nt <= 0 || nt > 3) { if (nt > 0) free_toks(tok, nt); set_err("Invalid config for %s%s", p->k, NULL); goto out; }
        if (!strcasecmp(p->k, "condition")) {
            struct cf_mod_cond *c = &conds[cf.n_conds];
            static const struct { const char *n; int t, a_rx, b_rx; } ct[] = {
                { "key_exists", MODC_KEY_EXISTS, 0, 0 }, { "key_does_not_exist", MODC_KEY_DOES_NOT_EXIST, 0, 0 },
                { "a_key_matches", MODC_A_KEY_MATCHES, 1, 0 }, { "no_key_matches", MODC_NO_KEY_MATCHES, 1, 0 },
                { "key_value_equals", MODC_KEY_VALUE_EQUALS, 0, 0 }, { "key_value_does_not_equal", MODC_KEY_VALUE_DOES_NOT_EQUAL, 0, 0 },
                { "key_value_matches", MODC_KEY_VALUE_MATCHES, 0, 1 }, { "key_value_does_not_match", MODC_KEY_VALUE_DOES_NOT_MATCH, 0, 1 },
                { "matching_keys_have_matching_values", MODC_MATCHING_KEYS_HAVE_MATCHING_VALUES, 1, 1 },
                { "matching_keys_do_not_have_matching_values", MODC_MATCHING_KEYS_DO_NOT_HAVE_MATCHING_VALUES, 1, 1 } };
            int i, found = -1;
            if (cf.n_conds >= 64 || nt < 2) { free_toks(tok, nt); set_err("Invalid config for %s : %s", p->k, p->v); goto out; }
            for (i = 0; i < 10; i++) if (!strcasecmp(tok[0], ct[i].n)) found = i;
            if (found < 0) { free_toks(tok, nt); set_err("Invalid config for %s : %s", p->k, p->v); goto out; }
            c->type = ct[found].t;
            if (!ct[found].a_rx) {
                c->ra_off = emit_ra(b, tok[1]);
                if (!c->ra_off) { free_toks(tok, nt); goto out; }
            }
            else {
                if (!*tok[1]) { free_toks(tok, nt); set_err("Unable to create regex for condition %s %s", p->k, p->v); goto out; }
                c->a_rx = emit_rx(b, tok[1], NULL);
                if (!c->a_rx) { free_toks(tok, nt); goto out; }
            }
            if (nt == 3) { c->b_off = blob_add(b, tok[2], strlen(tok[2]), 1); c->b_len = (uint32_t) strlen(tok[2]); }
            if (ct[found].b_rx) {
                if (nt < 3 || !*tok[2]) { free_toks(tok, nt); set_err("Unable to create regex for condition %s %s", p->k, p->v); goto out; }
                c->b_rx = emit_rx(b, tok[2], NULL);
                if (!c->b_rx) { free_toks(tok, nt); goto out; }
            }
            cf.n_conds++;
        }
        else {
            struct cf_mod_rule *r = &rules[cf.n_rules];
            const char *key = tok[0], *val = tok[nt - 1];
            int type = 0;
            if (cf.n_rules >= 256) { free_toks(tok, nt); set_err("too many modify rules%s%s", NULL, NULL); goto out; }
            if (nt == 1) {
                if (!strcasecmp(p->k, "remove")) type = MOD_REMOVE;
                else if (!strcasecmp(p->k, "remove_wildcard")) type = MOD_REMOVE_WILDCARD;
                else if (!strcasecmp(p->k, "remove_regex")) type = MOD_REMOVE_REGEX;
                else if (!strcasecmp(p->k, "move_to_start")) type = MOD_MOVE_TO_START;
                else if (!strcasecmp(p->k, "move_to_end")) type = MOD_MOVE_TO_END;
            }
            else if (nt == 2) {
                if (!strcasecmp(p->k, "rename")) type = MOD_RENAME;
                else if (!strcasecmp(p->k, "hard_rename")) type = MOD_HARD_RENAME;
                else if (!strcasecmp(p->k, "add")) type = MOD_ADD;       /* (add_if_not_present is handled in setup() but absent from the config map: flb_start() refuses it) */
                else if (!strcasecmp(p->k, "set")) type = MOD_SET;
                else if (!strcasecmp(p->k, "copy")) type = MOD_COPY;
                else if (!strcasecmp(p->k, "hard_copy")) type = MOD_HARD_COPY;
            }
            else if (nt == 3) {
                /* modify.c:412-466 only names a rule type for one or two words; with three the calloc()ed rule keeps
                 * type 0 = RENAME, key = first word, value = last word -- whatever the property was called */
                static const char *known[] = { "set", "add", "remove", "remove_wildcard", "remove_regex", "rename",
                                               "hard_rename", "copy", "hard_copy", "move_to_start", "move_to_end" };
                size_t q;
                for (q = 0; q < sizeof(known) / sizeof(known[0]); q++) if (!strcasecmp(p->k, known[q])) type = MOD_RENAME;
            }
            if (!type) { free_toks(tok, nt); set_err("Invalid operation %s : %s in configuration", p->k, p->v); goto out; }
            if ((type == MOD_HARD_COPY || type == MOD_HARD_RENAME) && !strcmp(key, val)) {
                /* modify.c:1142-1160 / :1010-1040 size the new map for "one conflicting key goes, one copy comes" and then
                 * skip (or keep) the one key that is both: the header and the pairs that follow disagree and every
                 * record after it is read out of step.  There is no result to be identical to. */
                set_err("%s %s: source and target are the same key; the reference writes a malformed map for it -- refused", p->k, p->v);
                free_toks(tok, nt); goto out;
            }
            r->type = type;
            r->key_off = blob_add(b, key, strlen(key), 1); r->key_len = (uint32_t) strlen(key);
            r->kmp_off = blob_add_mpstr(b, key, (uint32_t) strlen(key), &r->kmp_len);
            r->val_off = blob_add(b, val, strlen(val), 1); r->val_len = (uint32_t) strlen(val);
            r->vmp_off = blob_add_mpstr(b, val, (uint32_t) strlen(val), &r->vmp_len);
            r->key_hash = key_hash(key, strlen(key)); r->val_hash = key_hash(val, strlen(val));
            if (type != MOD_REMOVE_REGEX && !rule_text_is_a_regex(key)) { set_err("Unable to create regex(key) from %s%s", key, NULL); free_toks(tok, nt); goto out; }
            if (!rule_text_is_a_regex(val)) { set_err("Unable to create regex(val) from %s%s", val, NULL); free_toks(tok, nt); goto out; }
            if (type == MOD_REMOVE_REGEX) {
                if (!*key) { free_toks(tok, nt); set_err("Unable to create regex for rule %s %s", p->k, p->v); goto out; }
                r->key_rx = emit_rx(b, key, NULL);
                if (!r->key_rx) { free_toks(tok, nt); goto out; }
            }
            cf.n_rules++;
        }
        free_toks(tok, nt);
    }
    cf.conds_off = blob_add(b, conds, sizeof(*conds) * (cf.n_conds ? cf.n_conds : 1), 8);
    cf.rules_off = blob_add(b, rules, sizeof(*rules) * (cf.n_rules ? cf.n_rules : 1), 8);
    ret = blob_add(b, &cf, sizeof(cf), 8);
out:
    free(conds);
    free(rules);
    return ret;
}

static uint32_t emit_recmod_filter(flbgpu_filter *f, struct blob *b)
{
    struct cf_recmod cf;
    struct cf_rm_rec recs[64];
    struct cf_rm_key rem[64], allow[64];
    struct kv *p;
    int pass;
    memset(&cf, 0, sizeof(cf));
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "record")) {
            char *tok[4];
            int nt = split_tokens(p->v, 2, tok, 4);
            if (nt < 2) { free_toks(tok, nt); set_err("[filter record_modifier] invalid value for 'record': %s%s", p->v, NULL); return 0; }
            if (nt != 2) { free_toks(tok, nt); continue; }          /* "invalid record parameters": entry skipped */
            if (cf.n_records >= 64) { free_toks(tok, nt); set_err("too many Record entries%s%s", NULL, NULL); return 0; }
            recs[cf.n_records].kmp_off = blob_add_mpstr(b, tok[0], (uint32_t) strlen(tok[0]), &recs[cf.n_records].kmp_len);
            recs[cf.n_records].vmp_off = blob_add_mpstr(b, tok[1], (uint32_t) strlen(tok[1]), &recs[cf.n_records].vmp_len);
            cf.n_records++;
            free_toks(tok, nt);
        }
        else if (!strcasecmp(p->k, "remove_key")) {
            uint32_t l = (uint32_t) strlen(p->v);
            if (cf.n_remove >= 64) { set_err("too many Remove_key entries%s%s", NULL, NULL); return 0; }
            rem[cf.n_remove].dynamic = l > 0 && p->v[l - 1] == '*';
            if (rem[cf.n_remove].dynamic) l--;
            rem[cf.n_remove].off = blob_add(b, p->v, l, 1); rem[cf.n_remove].len = l; rem[cf.n_remove].pad = 0;
            cf.n_remove++;
        }
        else if (!strcasecmp(p->k, "allowlist_key") || !strcasecmp(p->k, "whitelist_key")) { /* second pass: allowlist first, then whitelist */ }
        else if (!strcasecmp(p->k, "uuid_key")) { set_err("Uuid_key draws random numbers and cannot be reproduced; not supported on the GPU path%s%s", NULL, NULL); return 0; }
        else { set_err("[filter record_modifier] unknown configuration property '%s'%s", p->k, NULL); return 0; }
    }
    for (pass = 0; pass < 2; pass++) {
        for (p = f->props; p; p = p->next) {
            uint32_t l;
            if (strcasecmp(p->k, pass == 0 ? "allowlist_key" : "whitelist_key")) continue;
            l = (uint32_t) strlen(p->v);
            if (cf.n_allow >= 64) { set_err("too many Allowlist_key entries%s%s", NULL, NULL); return 0; }
            allow[cf.n_allow].dynamic = l > 0 && p->v[l - 1] == '*';
            if (allow[cf.n_allow].dynamic) l--;
            allow[cf.n_allow].off = blob_add(b, p->v, l, 1); allow[cf.n_allow].len = l; allow[cf.n_allow].pad = 0;
            cf.n_allow++;
        }
    }
    if (cf.n_remove > 0 && cf.n_allow > 0) { set_err("remove_keys and allowlist_keys are exclusive with each other.%s%s", NULL, NULL); return 0; }
    cf.records_off = blob_add(b, recs, sizeof(recs[0]) * (cf.n_records ? cf.n_records : 1), 8);
    cf.remove_off = blob_add(b, rem, sizeof(rem[0]) * (cf.n_remove ? cf.n_remove : 1), 8);
    cf.allow_off = blob_add(b, allow, sizeof(allow[0]) * (cf.n_allow ? cf.n_allow : 1), 8);
    return blob_add(b, &cf, sizeof(cf), 8);
}

static void l2m_state_free(struct l2m_state *st)
{
    int i;
    if (!st) return;
    for (i = 0; i < st->n_labels; i++) free(st->label_keys[i]);
    for (i = 0; i < st->n_sets; i++) { free(st->sets[i].labels); free(st->sets[i].buckets); }
    free(st->sets); free(st->bounds); free(st->ns); free(st->subsystem); free(st->name); free(st->desc);
    free(st);
}

static int cmp_double(const void *a, const void *b)
{
    double x = *(const double *) a, y = *(const double *) b;
    return x < y ? -1 : x > y;
}

/* cb_log_to_metrics_init(), plugins/filter_log_to_metrics/log_to_metrics.c:649-962 */
static uint32_t emit_l2m_filter(flbgpu_filter *f, struct blob *b)
{
    struct cf_l2m cf;
    struct l2m_state *st;
    struct kv *p;
    const char *mode = "counter", *value_field = NULL, *name = "a", *ns = "log_metric", *subsystem = NULL,
               *desc = NULL, *tag = NULL;
    double bounds[64];
    static const double def_bounds[11] = { 0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, 5.0, 10.0 };
    int nb = 0, i;
    flbgpu_filter g;

    memset(&cf, 0, sizeof(cf));
    st = calloc(1, sizeof(*st));
    /* Regex / Exclude rules: same text and legacy semantics as filter_grep */
    memset(&g, 0, sizeof(g));
    g.ctx = f->ctx; g.kind = FLBGPU_F_GREP;
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "regex") || !strcasecmp(p->k, "exclude")) {
            struct kv *n;
            const char *q = p->v;
            /* log_to_metrics.c:318 creates the accessor from the field text as written (no '$' is
             * prepended like grep.c does): identical for plain key names, which is what we accept */
            if (*q != '$') {
                for (; *q && *q != ' '; q++) {
                    if (!(isalnum((unsigned char) *q) || *q == '_' || *q == '-')) {
                        set_err("log_to_metrics rule field '%s' must be a plain key or a $accessor%s", p->v, NULL);
                        l2m_state_free(st); return 0;
                    }
                }
            }
            n = calloc(1, sizeof(*n));
            n->k = p->k; n->v = p->v;
            if (g.props_tail) g.props_tail->next = n; else g.props = n;
            g.props_tail = n;
        }
    }
    if (g.props) {
        cf.grep_off = emit_grep_filter(&g, b);
        while (g.props) { struct kv *n = g.props->next; free(g.props); g.props = n; }
        if (!cf.grep_off) { l2m_state_free(st); return 0; }
    }
    /* kubernetes_mode: five fixed labels in front of the user's (log_to_metrics.c:43-50, 148-156, 422-438) */
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "kubernetes_mode") && parse_bool(p->v) < 0) { set_err("invalid boolean '%s'%s", p->v, NULL); l2m_state_free(st); return 0; }
        if (!strcasecmp(p->k, "kubernetes_mode") && parse_bool(p->v) == 1 && st->n_labels == 0) {
            static const char *k8s[5] = { "namespace_name", "pod_name", "container_name", "docker_id", "pod_id" };
            int q;
            for (q = 0; q < 5; q++) {
                char acc[64];
                snprintf(acc, sizeof(acc), "$kubernetes['%s']", k8s[q]);
                st->label_keys[st->n_labels] = strdup(k8s[q]);
                cf.label_ra_off[st->n_labels] = emit_ra(b, acc);
                if (!cf.label_ra_off[st->n_labels]) { st->n_labels++; l2m_state_free(st); return 0; }
                st->n_labels++;
            }
        }
    }
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "regex") || !strcasecmp(p->k, "exclude")) continue;
        else if (!strcasecmp(p->k, "metric_mode")) mode = p->v;
        else if (!strcasecmp(p->k, "value_field")) value_field = p->v;
        else if (!strcasecmp(p->k, "metric_name")) name = p->v;
        else if (!strcasecmp(p->k, "metric_namespace")) ns = p->v;
        else if (!strcasecmp(p->k, "metric_subsystem")) subsystem = p->v;
        else if (!strcasecmp(p->k, "metric_description")) desc = p->v;
        else if (!strcasecmp(p->k, "tag")) tag = p->v;
        else if (!strcasecmp(p->k, "kubernetes_mode")) { /* handled before the loop: its labels come first */ }
        else if (!strcasecmp(p->k, "discard_logs")) { int v = parse_bool(p->v); if (v < 0) { set_err("invalid boolean '%s'%s", p->v, NULL); l2m_state_free(st); return 0; } cf.discard = v; }
        else if (!strcasecmp(p->k, "bucket")) {
            char *end = NULL;
            double d = strtod(p->v, &end);
            if (end == p->v || nb >= 64) { set_err("Setting buckets failed (%s)%s", p->v, NULL); l2m_state_free(st); return 0; }
            bounds[nb++] = d;
        }
        else if (!strcasecmp(p->k, "label_field") || !strcasecmp(p->k, "add_label")) {
            char *tok[3];
            const char *key, *acc;
            int nt = 0;
            if (st->n_labels >= L2M_MAX_LABELS) { set_err("too many labels%s%s", NULL, NULL); l2m_state_free(st); return 0; }
            if (!strcasecmp(p->k, "label_field")) { key = p->v; acc = p->v; }
            else {
                nt = split_plain(p->v, 1, tok, 3);
                if (nt != 2) { free_toks(tok, nt); set_err("invalid label, expected name and key%s%s", NULL, NULL); l2m_state_free(st); return 0; }
                key = tok[0]; acc = tok[1];
            }
            st->label_keys[st->n_labels] = strdup(key);
            cf.label_ra_off[st->n_labels] = emit_ra(b, acc);
            if (nt) free_toks(tok, nt);
            if (!cf.label_ra_off[st->n_labels]) { st->n_labels++; l2m_state_free(st); return 0; }
            st->n_labels++;
        }
        else if (!strcasecmp(p->k, "emitter_name") || !strcasecmp(p->k, "emitter_mem_buf_limit") ||
                 !strcasecmp(p->k, "flush_interval_sec") || !strcasecmp(p->k, "flush_interval_nsec")) { /* delivery side: host concern */ }
        else { set_err("[filter log_to_metrics] unknown configuration property '%s'%s", p->k, NULL); l2m_state_free(st); return 0; }
    }
    if (!tag || !*tag) { set_err("Metric tag is not set%s%s", NULL, NULL); l2m_state_free(st); return 0; }
    if (!strcasecmp(mode, "counter")) cf.mode = L2M_COUNTER;
    else if (!strcasecmp(mode, "histogram")) cf.mode = L2M_HISTOGRAM;
    else if (!strcasecmp(mode, "gauge")) cf.mode = L2M_GAUGE;
    else { set_err("invalid 'mode' value. Only 'counter', 'gauge' or 'histogram' types are allowed%s%s", NULL, NULL); l2m_state_free(st); return 0; }
    if (!desc || !*desc) { set_err("metric_description is not set%s%s", NULL, NULL); l2m_state_free(st); return 0; }
    if (cf.mode != L2M_COUNTER) {
        if (!value_field || !*value_field) { set_err("value_field is not set%s%s", NULL, NULL); l2m_state_free(st); return 0; }
        cf.value_ra_off = emit_ra(b, value_field);
        if (!cf.value_ra_off) { l2m_state_free(st); return 0; }
    }
    if (cf.mode == L2M_HISTOGRAM) {
        if (nb == 0) { memcpy(bounds, def_bounds, sizeof(def_bounds)); nb = 11; }
        else qsort(bounds, nb, sizeof(double), cmp_double);
        cf.n_buckets = nb;
        cf.buckets_off = blob_add(b, bounds, sizeof(double) * nb, 8);
        st->bounds = malloc(sizeof(double) * nb);
        memcpy(st->bounds, bounds, sizeof(double) * nb);
    }
    cf.n_labels = st->n_labels;
    st->mode = cf.mode; st->n_buckets = cf.n_buckets; st->discard = cf.discard;
    st->ns = strdup(ns); st->name = strdup(name); st->desc = strdup(desc);
    st->subsystem = strdup(subsystem && *subsystem ? subsystem : mode);
    for (i = 0; i < st->n_labels; i++) (void) i;
    if (f->l2m) {                       /* re-emission for a chain: keep accumulated values */
        l2m_state_free(st);
    }
    else f->l2m = st;
    return blob_add(b, &cf, sizeof(cf), 8);
}

/* ---- filter_rewrite_tag ---- */
/* ra_parse_buffer() (src/flb_record_accessor.c:75-214) on a tag template: the text is cut at every '$' into literal text,
 * $0..$9, $TAG, $TAG[n] and $key['sub'] parts -- with the cutting rules of that loop, oddities included (the character behind
 * `$TAG` or behind a key is never looked at as a '$'; a one-character tail behind a key is dropped; a '$' at the very end too). */
struct rt_parts { struct cf_rt_part p[64]; int n; };
static int rt_add(struct rt_parts *ps, uint32_t type, uint32_t a, uint32_t b2)
{
    if (ps->n >= 64) { set_err("[filter rewrite_tag] tag template with too many parts%s%s", NULL, NULL); return -1; }
    ps->p[ps->n].type = type; ps->p[ps->n].a = a; ps->p[ps->n].b = b2; ps->p[ps->n].pad = 0;
    ps->n++;
    return 0;
}
static int rt_add_string(struct rt_parts *ps, struct blob *b, const char *s, int len)
{
    return rt_add(ps, RT_STRING, len > 0 ? blob_add(b, s, (size_t) len, 1) : 0, (uint32_t) (len > 0 ? len : 0));
}
static int rt_parse_template(struct blob *b, const char *buf, struct rt_parts *ps)
{
    const int len = (int) strlen(buf);
    int i, n, pre = 0, end = 0;
    ps->n = 0;
    for (i = 0; i < len; i++) {
        if (buf[i] != '$') continue;
        if (i > pre && rt_add_string(ps, b, buf + pre, i - pre)) return -1;
        pre = i;
        n = i + 1;
        if (n >= len) break;
        if (isdigit((unsigned char) buf[n])) {
            if (rt_add(ps, RT_REGEX_ID, (uint32_t) atoi(buf + n), 0)) return -1;
            i++;
            pre = i + 1;
            continue;
        }
        if (n + 2 < len && strncmp(buf + n, "TAG", 3) == 0) {
            if (n + 4 < len) {
                end = -1;
                if (buf[n + 3] == '[') {
                    const int t = n + 3;
                    const char *br = memchr(buf + t, ']', (size_t) (len - t));
                    end = br ? (int) (br - (buf + t)) : -1;
                    if (end == 0) end = -1;
                    if (rt_add(ps, RT_TAG_PART, (uint32_t) atoi(buf + t + 1), 0)) return -1;
                    i = t + end + 1;
                    pre = i;
                    continue;
                }
            }
            if (rt_add(ps, RT_TAG, 0, 0)) return -1;
            i = n + 3;
            pre = n + 3;
            continue;
        }
        {
            int quote_cnt = 0;
            char *key;
            uint32_t ra;
            for (end = i + 1; end < len; end++) {
                if (buf[end] == '\'') ++quote_cnt;
                else if (buf[end] == '.' && (quote_cnt & 1)) continue;
                else if (buf[end] == '.' || buf[end] == ' ' || buf[end] == ',' || buf[end] == '"') break;
            }
            key = strndup(buf + i, (size_t) (end - i));
            if (!key) return -1;
            ra = emit_ra(b, key);
            free(key);
            if (!ra) return -1;
            if (rt_add(ps, RT_KEYMAP, ra, 0)) return -1;
            pre = end;
            i = end;
        }
    }
    if ((i - 1 > end && pre < i) || i == 1) {
        if (pre <= len && rt_add_string(ps, b, buf + (pre < len ? pre : len), pre < len ? len - pre : 0)) return -1;
    }
    return 0;
}

static uint32_t emit_rtag_filter(flbgpu_filter *f, struct blob *b)
{
    struct cf_rtag cf;
    struct cf_rt_rule rules[32];
    struct kv *p;
    memset(&cf, 0, sizeof(cf));
    memset(rules, 0, sizeof(rules));
    for (p = f->props; p; p = p->next) {
        char *tok[6];
        struct rt_parts parts;
        struct cf_rt_rule *r;
        int nt;
        if (!strcasecmp(p->k, "emitter_name") || !strcasecmp(p->k, "emitter_mem_buf_limit")) continue;      /* the emitter is the caller's */
        if (!strcasecmp(p->k, "emitter_storage.type")) {
            if (strcasecmp(p->v, "memory") && strcasecmp(p->v, "filesystem")) {
                set_err("invalid 'emitter_storage.type' value. Only 'memory' or 'filesystem' types are allowed%s%s", NULL, NULL);
                return 0;
            }
            continue;
        }
        if (strcasecmp(p->k, "rule")) { set_err("[filter rewrite_tag] unknown configuration property '%s'%s", p->k, NULL); return 0; }
        nt = split_tokens(p->v, 4, tok, 6);                        /* FLB_CONFIG_MAP_SLIST_4: at least four entries (flb_config_map.c:51-55) */
        if (nt < 4) { free_toks(tok, nt); set_err("[config map] rule: four values expected (key, regex, tag, keep): '%s'%s", p->v, NULL); return 0; }
        if (cf.n_rules >= 32) { free_toks(tok, nt); set_err("[filter rewrite_tag] too many rules%s%s", NULL, NULL); return 0; }
        r = &rules[cf.n_rules];
        /* the key: the FIRST part of the accessor text decides (flb_ra_regex_match: mk_list_entry_first) -- a key name with or
         * without '$'; a part without a key ($TAG, $0) never matches */
        if (rt_parse_template(b, tok[0], &parts)) { free_toks(tok, nt); if (!g_rt_err[0]) set_err("invalid record accessor key ? '%s'%s", tok[0], NULL); return 0; }
        if (parts.n == 0) { free_toks(tok, nt); set_err("invalid record accessor key ? '%s'%s", tok[0], NULL); return 0; }
        if (parts.p[0].type == RT_KEYMAP) r->ra_off = parts.p[0].a;
        else if (parts.p[0].type == RT_STRING && parts.p[0].b) {
            char *name = strndup((const char *) b->p + parts.p[0].a, parts.p[0].b);
            r->ra_off = name ? emit_ra(b, name) : 0;
            free(name);
            if (!r->ra_off) { free_toks(tok, nt); return 0; }
        }
        else r->ra_off = 0;
        r->rx_off = emit_rx(b, tok[1], NULL);
        if (!r->rx_off) { free_toks(tok, nt); return 0; }
        if (rt_parse_template(b, tok[2], &parts)) { free_toks(tok, nt); if (!g_rt_err[0]) set_err("could not compose tag: %s%s", tok[2], NULL); return 0; }
        r->n_parts = (uint32_t) parts.n;
        r->parts_off = blob_add(b, parts.p, sizeof(parts.p[0]) * (size_t) (parts.n ? parts.n : 1), 8);
        r->keep = parse_bool(tok[3]) == 1;                          /* flb_utils_bool(): anything that is not true keeps nothing */
        free_toks(tok, nt);
        cf.n_rules++;
    }
    cf.rules_off = blob_add(b, rules, sizeof(rules[0]) * (cf.n_rules ? cf.n_rules : 1), 8);
    return blob_add(b, &cf, sizeof(cf), 8);
}

static uint32_t emit_ml_filter(flbgpu_filter *f, struct blob *b);
static uint32_t emit_filter(flbgpu_filter *f, struct blob *b, uint32_t *cap_need)
{
    switch (f->kind) {
    case FLBGPU_F_PARSER: return emit_parser_filter(f, b, cap_need);
    case FLBGPU_F_GREP: return emit_grep_filter(f, b);
    case FLBGPU_F_MODIFY: return emit_modify_filter(f, b);
    case FLBGPU_F_RECORD_MODIFIER: return emit_recmod_filter(f, b);
    case FLBGPU_F_LOG_TO_METRICS: return emit_l2m_filter(f, b);
    case FLBGPU_F_REWRITE_TAG: return emit_rtag_filter(f, b);
    case FLBGPU_F_MULTILINE: return emit_ml_filter(f, b);
    }
    return 0;
}

/* flb_config_map_properties_check() (src/flb_config_map.c:523-530): a property whose config map entry is not
 * FLB_CONFIG_MAP_MULT may be set once.  The names below are the MULT entries of the five plugins' maps. */
static int single_valued_set_twice(flbgpu_filter *f)
{
    static const char *mult[] = { "regex", "exclude",                                   /* grep, log_to_metrics */
                                  "parser",                                             /* parser */
                                  "record", "remove_key", "allowlist_key", "whitelist_key",   /* record_modifier */
                                  "set", "add", "remove", "remove_wildcard", "remove_regex", "move_to_start", "move_to_end", "rename",
                                  "hard_rename", "copy", "hard_copy", "condition",            /* modify */
                                  "add_label", "label_field", "bucket",                       /* log_to_metrics */
                                  "rule",                                                     /* rewrite_tag */
                                  "multiline.parser" };                                       /* multiline */
    struct kv *p, *q;
    for (p = f->props; p; p = p->next) {
        size_t m;
        int is_mult = 0, n = 0;
        for (m = 0; m < sizeof(mult) / sizeof(mult[0]); m++) if (!strcasecmp(p->k, mult[m])) is_mult = 1;
        if (is_mult) continue;
        for (q = f->props; q; q = q->next) if (!strcasecmp(p->k, q->k)) n++;
        if (n > 1) { set_err("configuration property '%s' is set more than once%s", p->k, NULL); return 1; }
    }
    return 0;
}

int flbgpu_filter_init(flbgpu_filter *f)
{
    struct blob b;
    uint32_t cap = 0, off;
    if (!f) return -1;
    g_rt_err[0] = 0;
    if (single_valued_set_twice(f)) return -1;
    memset(&b, 0, sizeof(b));
    blob_reserve(&b, sizeof(struct chain_hdr), 16);
    off = emit_filter(f, &b, &cap);         /* validation pass; the chain re-emits */
    free(b.p);
    if (!off) return -1;
    f->inited = 1;
    return 0;
}

/* ------------------------------------------------------------------ chain */
flbgpu_chain *flbgpu_chain_new(flbgpu_ctx *ctx)
{
    flbgpu_chain *c;
    if (!ctx) return NULL;
    c = calloc(1, sizeof(*c));
    if (!c) { set_err("out of memory%s%s", NULL, NULL); return NULL; }
    c->ctx = ctx;
    c->q = bk_q_new(ctx->device);
    if (!c->q) { free(c); return NULL; }
    pthread_mutex_init(&c->lock, NULL);
    return c;
}

int flbgpu_chain_add(flbgpu_chain *c, flbgpu_filter *f)
{
    if (!c || !f || !f->inited || c->inited || c->nf >= FLBGPU_MAX_FILTERS) return -1;
    c->f[c->nf++] = f;
    return 0;
}

int flbgpu_chain_init(flbgpu_chain *c)
{
    struct chain_hdr h;
    struct chain_filter cf[FLBGPU_MAX_FILTERS];
    uint32_t cap = 0, i;
    uint8_t empty = 0x80;
    if (!c || c->inited) return -1;
    g_rt_err[0] = 0;
    memset(&h, 0, sizeof(h));
    blob_reserve(&c->blob, sizeof(h), 16);
    h.empty_map_off = blob_add(&c->blob, &empty, 1, 1);
    for (i = 0; i < (uint32_t) c->nf; i++) {
        cf[i].kind = c->f[i]->kind;
        cf[i].cfg_off = emit_filter(c->f[i], &c->blob, &cap);
        if (!cf[i].cfg_off) return -1;
    }
    c->l2m_index = -1;
    for (i = 0; i < (uint32_t) c->nf; i++) {
        if (c->f[i]->kind != FLBGPU_F_LOG_TO_METRICS) continue;
        if (c->l2m_index >= 0) { set_err("only one log_to_metrics filter per fused chain%s%s", NULL, NULL); return -1; }
        c->l2m_index = (int) i;
    }
    c->ml_index = -1;
    for (i = 0; i < (uint32_t) c->nf; i++) if (c->f[i]->kind == FLBGPU_F_MULTILINE) { c->ml_index = (int) i; c->ml_cfg_off = cf[i].cfg_off; }
    c->rtag_index = -1;
    for (i = 0; i < (uint32_t) c->nf; i++) {
        if (c->f[i]->kind != FLBGPU_F_REWRITE_TAG) continue;
        c->rtag_index = c->rtag_index == -1 ? (int) i : -2;
    }
    for (i = 0; i < (uint32_t) c->nf; i++) h.needs_scratch |= (uint32_t) c->f[i]->needs_scratch;
    c->needs_scratch = (int) h.needs_scratch;
    c->scr_mul = (h.needs_scratch & 2) ? 8 : 4;           /* scratch bytes per record byte */
    {
        int last_parser = -1, k2;
        c->defer_ok = 1;
        for (k2 = 0; k2 < c->nf; k2++) if (c->f[k2]->kind == FLBGPU_F_PARSER) last_parser = k2;
        for (k2 = 0; k2 < last_parser; k2++) if (c->f[k2]->kind == FLBGPU_F_LOG_TO_METRICS) c->defer_ok = 0;
        /* `parser, then filters that are not parsers`: the evaluation runs as two launches (kernels.cu: k_chain_eval_t) */
        {
            /* The split pays when the parser is the JSON transcoder (the largest piece of code) and costs when it is a regex
             * parser (two launches re-load what one keeps) -- so by default only the former.  FLBGPU_EVAL_SPLIT=1 / 0 forces it. */
            const char *e = getenv("FLBGPU_EVAL_SPLIT");
            const int want = e ? e[0] != '0' : (c->f[0]->needs_scratch & 1);
            c->split = c->nf >= 2 && last_parser == 0 && want;
            /* the grep filters right behind the parser only look at the record: they run in the head launch, and what they drop
             * is never handed over */
            h.split_at = 1;
            if (c->split) while ((int) h.split_at < c->nf && c->f[h.split_at]->kind == FLBGPU_F_GREP) h.split_at++;
        }
    }
    h.n_filters = c->nf;
    h.filters_off = blob_add(&c->blob, cf, sizeof(cf[0]) * (c->nf ? c->nf : 1), 8);
    cap += RC_CACHE_INTS;                 /* every chain: the final field list for the emission pass */
    h.cap_stride = cap;
    blob_reserve(&c->blob, 16, 16);
    h.total_bytes = (uint32_t) c->blob.n;
    memcpy(c->blob.p, &h, sizeof(h));
    c->cap_stride = cap;
    c->d_blob = bk_alloc(c->q, c->blob.n);
    c->d_flags = bk_alloc(c->q, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1));
    if (!c->d_blob || !c->d_flags) return -1;
    if (c->l2m_index >= 0) {
        struct l2m_state *st = c->f[c->l2m_index]->l2m;
        size_t n = (size_t) 1 << L2M_SLOTS_LOG2, nbk = L2M_NBK(st);
        c->l2m_slots = n;
        c->l2m.hash = bk_alloc(c->q, n * 8); c->l2m.chash = bk_alloc(c->q, n * 8); c->l2m.first = bk_alloc(c->q, n * 4); c->l2m.cnt = bk_alloc(c->q, n * 8);
        c->l2m.sum = bk_alloc(c->q, n * 8); c->l2m.bkt = bk_alloc(c->q, n * nbk * 8);
        c->l2m.str = bk_alloc(c->q, n * (st->n_labels ? st->n_labels : 1) * L2M_LABEL_BYTES);
        c->l2m.mask = (uint32_t) (n - 1);
        if (st->mode != L2M_COUNTER) {               /* the list of records whose value text converts nothing (flbgpu_prog.h: struct l2m_table) */
            c->l2m.pending = bk_alloc(c->q, sizeof(uint32_t) * L2M_PENDING_CAP);
            c->l2m.pending_n = bk_alloc(c->q, 16);
            c->l2m.pending_cap = L2M_PENDING_CAP;
            if (!c->l2m.pending || !c->l2m.pending_n) return -1;
        }
        c->h_hash = malloc(n * 8); c->h_chash = malloc(n * 8); c->h_first = malloc(n * 4); c->h_cnt = malloc(n * 8); c->h_sum = malloc(n * 8);
        c->h_bkt = malloc(n * nbk * 8);
        if (st->mode == L2M_HISTOGRAM) {
            c->l2m.amax = bk_alloc(c->q, n * 8);
            c->h_amax = malloc(n * 8); c->h_setof = malloc(n * sizeof(int32_t));
            if (!c->l2m.amax || !c->h_amax || !c->h_setof) return -1;
        }
        if (!c->l2m.hash || !c->l2m.chash || !c->l2m.first || !c->l2m.cnt || !c->l2m.sum || !c->l2m.bkt || !c->l2m.str) return -1;
    }
    if (bk_h2d(c->q, c->d_blob, c->blob.p, c->blob.n) || bk_sync(c->q)) return -1;
    if (c->ml_index == 0 && c->nf > 1) {
        int has_special = 0, k2;
        for (k2 = 1; k2 < c->nf; k2++) if (c->f[k2]->kind == FLBGPU_F_REWRITE_TAG || c->f[k2]->kind == FLBGPU_F_MULTILINE) has_special = 1;
        if (!has_special) {                       /* (a re-tagged stream or a second multiline filter: filter by filter) */
            c->ml_solo = flbgpu_chain_new(c->ctx);
            c->ml_post = flbgpu_chain_new(c->ctx);
            if (!c->ml_solo || !c->ml_post || flbgpu_chain_add(c->ml_solo, c->f[0]) || flbgpu_chain_init(c->ml_solo)) return -1;
            for (k2 = 1; k2 < c->nf; k2++) if (flbgpu_chain_add(c->ml_post, c->f[k2])) return -1;
            if (flbgpu_chain_init(c->ml_post)) return -1;
        }
    }
    c->inited = 1;
    return 0;
}

void flbgpu_chain_destroy(flbgpu_chain *c)
{
    if (!c) return;
    flbgpu_chain_destroy(c->ml_solo); flbgpu_chain_destroy(c->ml_post);
    bk_free(c->q, c->d_blob); bk_free(c->q, c->d_in); bk_free(c->q, c->d_out); bk_free(c->q, c->d_tile); bk_free(c->q, c->d_off);
    bk_free(c->q, c->d_len); bk_free(c->q, c->d_size); bk_free(c->q, c->d_kind); bk_free(c->q, c->d_bsum); bk_free(c->q, c->d_cap);
    bk_free(c->q, c->d_flags); bk_free(c->q, c->d_scr); free(c->h_bsum); bk_free(c->q, c->d_mlw);
    bk_free(c->q, c->d_prep); free(c->h_prep);
    bk_free(c->q, c->d_tl_text); bk_free(c->q, c->d_tl_mid); bk_free(c->q, c->d_tl_out); bk_free(c->q, c->d_tl_line); bk_free(c->q, c->d_tl_rec);
    bk_free(c->q, c->d_tl_bsum); free(c->h_tl_bsum);
    bk_free(c->q, c->d_esize); bk_free(c->q, c->d_ebsum); free(c->h_ebsum);
    bk_free(c->q, c->l2m.hash); bk_free(c->q, c->l2m.chash); bk_free(c->q, c->l2m.first); bk_free(c->q, c->l2m.cnt); bk_free(c->q, c->l2m.sum); bk_free(c->q, c->l2m.bkt); bk_free(c->q, c->l2m.str); bk_free(c->q, c->l2m.pending); bk_free(c->q, c->l2m.pending_n);
    bk_free(c->q, c->l2m.amax); bk_free(c->q, c->l2m.obs_slot); bk_free(c->q, c->l2m.obs_val);
    free(c->h_hash); free(c->h_chash); free(c->h_first); free(c->h_cnt); free(c->h_sum); free(c->h_bkt);
    free(c->h_amax); free(c->h_setof); free(c->h_obs_slot); free(c->h_obs_val);
    free(c->blob.p);
    if (c->ctx && c->ctx->last_q == c->q) c->ctx->last_q = NULL;
    bk_q_free(c->q);
    pthread_mutex_destroy(&c->lock);
    free(c);
}

void flbgpu_chain_stats(flbgpu_chain *c, struct flbgpu_stats *out) { if (c && out) *out = c->st; }
int flbgpu_chain_set_result_buffer(flbgpu_chain *c, void *buf, size_t cap)
{
    if (!c) return -1;
    pthread_mutex_lock(&c->lock);
    c->res_buf = buf; c->res_cap = buf ? cap : 0;
    pthread_mutex_unlock(&c->lock);
    return 0;
}
void *flbgpu_chain_stream(flbgpu_chain *c) { return c ? bk_stream(c->q) : NULL; }
int flbgpu_kernel_ms(flbgpu_ctx *ctx, float out[3])
{
    bk_q *q = ctx && ctx->last_q ? ctx->last_q : (ctx ? ctx->q0 : NULL);
    if (!q || bk_sync(q)) return -1;
    return bk_kernel_ms(q, out);
}

/* grow a device buffer of `elem`-byte elements to hold n of them (n + n/4 + 64, and bk_alloc's tail), keeping its first
 * `keep` elements.  The queue drains first: kernels queued on it may still read the old buffer. */
static int dev_grow(flbgpu_chain *c, void **p, size_t *cap, size_t n, size_t elem, size_t keep)
{
    size_t nc = n + n / 4 + 64;
    void *np;
    if (*cap >= n) return 0;
    if (bk_sync(c->q)) return -1;
    np = bk_alloc(c->q, nc * elem);
    if (!np || (keep && bk_d2d(c->q, np, *p, keep * elem))) { bk_free(c->q, np); return -1; }
    bk_free(c->q, *p);
    *p = np; *cap = nc;
    return 0;
}

/* the same for a host array, whose contents never need to move */
static int host_grow(void **p, size_t *cap, size_t n, size_t elem)
{
    size_t nc = n + n / 4 + 64;
    if (*cap >= n) return 0;
    free(*p);
    *p = malloc(nc * elem);
    *cap = *p ? nc : 0;
    if (!*p) { set_err("out of memory%s%s", NULL, NULL); return -1; }
    return 0;
}

/* per-record sizes -> block offsets, on the device (d_bsum) and the host (h_bsum); *total = the sum of the n sizes.  NULL
 * arrays: the chain's own, grown to fit.  A total of 4 GiB or more fails the call with the text `too_big`. */
static int sizes_to_offsets(flbgpu_chain *c, const uint32_t *d_size, uint32_t n, uint64_t *d_bsum, uint64_t *h_bsum,
                            const char *too_big, uint64_t *total)
{
    const size_t nb = ((size_t) n + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    if (!d_bsum) {
        if (dev_grow(c, (void **) &c->d_bsum, &c->cap_bsum, nb + 2, sizeof(uint64_t), 0) ||
            host_grow((void **) &c->h_bsum, &c->cap_hbsum, nb + 2, sizeof(uint64_t))) return -1;
        d_bsum = c->d_bsum; h_bsum = c->h_bsum;
    }
    if (bk_sizes_scan(c->q, d_size, n, d_bsum, h_bsum)) return -1;
    *total = h_bsum[nb];
    if (*total >= 0xfff00000ull) { set_err("%s%s", too_big, NULL); return -1; }
    return 0;
}

/* chunk-level verdict of filter k from the evidence word (see dev_chain.cuh).
 * `clean`: the filter's input decodes to its very end.  grep and modify return
 * NOTOUCH (after logging an encoder error) when the decoder stopped early
 * (plugins/filter_grep/grep.c:355-384, plugins/filter_modify/modify.c:1547-1566);
 * filter_parser and record_modifier hand back whatever they encoded. */
static int verdict(int kind, uint32_t fl, int clean)
{
    switch (kind) {
    case FLBGPU_F_PARSER: return (fl & CHF_EMITTED) != 0;
    case FLBGPU_F_GREP: return (fl & CHF_CAUSE) != 0 && clean;
    case FLBGPU_F_MODIFY: return (fl & CHF_CAUSE) != 0 && clean;
    case FLBGPU_F_RECORD_MODIFIER: return (fl & CHF_CAUSE) && (fl & CHF_EMITTED);
    case FLBGPU_F_REWRITE_TAG: return (fl & CHF_CAUSE) != 0 && clean;       /* emitted_num > 0 (rewrite_tag.c:500-531) */
    }
    return 0;
}
/* log_to_metrics: MODIFIED (empty) iff discard_logs, whatever the records were */
#define L2M_VERDICT(c, k) ((c)->f[k]->l2m->discard ? 1 : 0)

/* the chunk-level verdicts of a call from its evidence words, front to back.  Returns the first filter whose verdict differs
 * from `assume` (the filters behind it saw the wrong input), or -1.  *settled = `assume` with that verdict in place, which is
 * also what the next call speculates on. */
static int settle(flbgpu_chain *c, uint32_t assume, const uint32_t *flags, int clean, uint32_t *settled)
{
    int k;
    for (k = 0; k < c->nf; k++) {
        const int v = !((c->active >> k) & 1) ? 0 : c->f[k]->kind == FLBGPU_F_LOG_TO_METRICS ? L2M_VERDICT(c, k) : verdict(c->f[k]->kind, flags[k], clean);
        if (v) clean = 1;                    /* a MODIFIED filter hands a well-formed chunk on */
        if (v != (int) ((assume >> k) & 1)) { assume ^= 1u << k; break; }
    }
    *settled = assume;
    c->spec_assume = assume; c->spec_valid = 1; c->spec_active = c->active;
    return k < c->nf ? k : -1;
}

/* grow the per-record arrays to hold `need` records, keeping the first `keep` */
static int ensure_rec_cap(flbgpu_chain *c, size_t need, size_t keep)
{
    size_t nc;
    uint32_t *o, *l, *z;
    uint8_t *k;
    int32_t *cp = NULL;
    if (c->cap_rec >= need) return 0;
    nc = need + need / 2 + 1024;
    o = bk_alloc(c->q, nc * 4); l = bk_alloc(c->q, nc * 4); z = bk_alloc(c->q, nc * 4); k = bk_alloc(c->q, nc);
    /* split evaluation: RC_CACHE_MAXF more columns behind the rows carry the key fingerprints from the head to the tail launch */
    if (c->cap_stride) cp = bk_alloc(c->q, nc * (c->cap_stride + (c->split ? RC_CACHE_MAXF : 0)) * sizeof(int32_t));
    if (!o || !l || !z || !k || (c->cap_stride && !cp)) return -1;
    if (c->rtag_index >= 0) {                          /* sized anew by every evaluation: nothing to keep */
        uint32_t *ne = bk_alloc(c->q, nc * 4);
        if (!ne) return -1;
        if (keep && (bk_sync(c->q) || bk_d2d(c->q, ne, c->d_esize, keep * 4))) return -1;
        bk_free(c->q, c->d_esize);
        c->d_esize = ne;
    }
    if (c->want_report) {
        int32_t *np_ = bk_alloc(c->q, nc * 6 * sizeof(int32_t));
        if (!np_ || bk_zero(c->q, np_, nc * 6 * sizeof(int32_t))) return -1;
        if (keep && (bk_sync(c->q) || bk_d2d(c->q, np_, c->d_prep, keep * 6 * sizeof(int32_t)))) return -1;
        bk_free(c->q, c->d_prep);
        c->d_prep = np_;
    }
    if (c->l2m.amax) {                                 /* histogram observations, "none" for the new records */
        uint32_t *ns_ = bk_alloc(c->q, nc * 4);
        double *nv = bk_alloc(c->q, nc * 8);
        if (!ns_ || !nv || bk_zero(c->q, ns_, nc * 4)) return -1;
        if (keep && (bk_sync(c->q) || bk_d2d(c->q, ns_, c->l2m.obs_slot, keep * 4) || bk_d2d(c->q, nv, c->l2m.obs_val, keep * 8))) return -1;
        bk_free(c->q, c->l2m.obs_slot); bk_free(c->q, c->l2m.obs_val);
        c->l2m.obs_slot = ns_; c->l2m.obs_val = nv;
    }
    if (keep) {
        if (bk_sync(c->q)) return -1;                 /* running kernels still read the old arrays */
        if (bk_d2d(c->q, o, c->d_off, keep * 4) || bk_d2d(c->q, l, c->d_len, keep * 4) || bk_d2d(c->q, z, c->d_size, keep * 4) ||
            bk_d2d(c->q, k, c->d_kind, keep)) return -1;
        /* the capture cache is laid out in columns of cap_rec records: every column moves to its new pitch */
        if (cp && bk_d2d_2d(c->q, cp, nc * sizeof(int32_t), c->d_cap, c->cap_rec * sizeof(int32_t), keep * sizeof(int32_t), c->cap_stride)) return -1;
    }
    bk_free(c->q, c->d_off); bk_free(c->q, c->d_len); bk_free(c->q, c->d_size); bk_free(c->q, c->d_kind); bk_free(c->q, c->d_cap);
    c->d_off = o; c->d_len = l; c->d_size = z; c->d_kind = k; c->d_cap = cp;
    c->cap_rec = nc;
    return 0;
}

static size_t slice_bytes(void)
{
    const char *e = getenv("FLBGPU_SLICE_MB");
    size_t mb = e ? (size_t) atol(e) : 128;       /* not re-tuned on H100: FLBGPU_SLICE_MB */
    if (mb < 1) mb = 1;
    if (mb > 2048) mb = 2048;
    return mb << 20;
}

/* the record index of the slice [off, off + len) of a chunk, behind the n_rec records indexed so far: *n_valid more records,
 * and the slice's decodable part ends at *end_off */
static int index_slice(flbgpu_chain *c, const uint8_t *d_in, size_t off, size_t len, uint32_t n_rec, uint32_t *n_valid, uint64_t *end_off)
{
    /* tiles start at the address rounded down to 16 B */
    const uint32_t n_tiles = (uint32_t) ((len + ((uintptr_t) (d_in + off) & 15) + BK_INDEX_TILE - 1) / BK_INDEX_TILE);
    uint32_t n_cand = 0;
    int tiled = 0;
    *n_valid = 0; *end_off = off;
    if (bk_upload_wait_index(c->q, off + len)) return -1;
    if (dev_grow(c, (void **) &c->d_tile, &c->cap_tile, n_tiles + 1, sizeof(uint32_t), 0)) return -1;
    if (bk_index_count(c->q, d_in, off, (uint32_t) len, c->d_tile, n_tiles, &n_cand)) return -1;
    if (ensure_rec_cap(c, (size_t) n_rec + n_cand, n_rec)) return -1;
    if (bk_index_fill(c->q, d_in, off, (uint32_t) len, c->d_tile, n_tiles, n_cand, c->d_off + n_rec, c->d_len + n_rec,
                      c->d_kind + n_rec, n_valid, end_off, &tiled)) {
        c->st.error_bits = FLBGPU_E_INDEX;
        return -1;
    }
    return 0;
}

/* the record index of a whole chunk, slice by slice: *n_rec records, whose decodable prefix ends at *off */
static int index_chunk(flbgpu_chain *c, const uint8_t *d_in, size_t bytes, uint32_t *n_rec, size_t *off)
{
    size_t S = slice_bytes();
    *n_rec = 0; *off = 0;
    while (*off < bytes) {
        size_t len = bytes - *off < S ? bytes - *off : S;
        uint32_t n_valid;
        uint64_t end_off;
        if (index_slice(c, d_in, *off, len, *n_rec, &n_valid, &end_off)) return -1;
        if (n_valid == 0) {
            if (*off + len < bytes) { S *= 2; continue; }     /* a record longer than the slice: widen it */
            break;                                           /* nothing decodable from here to the end */
        }
        *n_rec += n_valid;
        *off = (size_t) end_off;
    }
    return 0;
}

static void fill_args(flbgpu_chain *c, struct bk_chain_args *a, const uint8_t *d_in, size_t bytes, uint32_t n_rec)
{
    a->d_in = d_in; a->in_len = (uint32_t) bytes; a->d_blob = c->d_blob; a->d_scr = c->needs_scratch ? c->d_scr : NULL;
    a->d_capcache = c->cap_stride ? c->d_cap : NULL; a->cap_stride = c->cap_stride; a->cap_n = (uint32_t) c->cap_rec;
    a->d_off = c->d_off; a->d_len = c->d_len; a->d_kind = c->d_kind; a->n_rec = n_rec;
    a->d_size = c->d_size; a->d_bsum = c->d_bsum; a->d_flags = c->d_flags;
    if (c->l2m_index >= 0 && ((c->active >> c->l2m_index) & 1)) a->l2m = c->l2m; else memset(&a->l2m, 0, sizeof(a->l2m));
    if (!c->l2m_record) a->l2m.obs_slot = NULL, a->l2m.obs_val = NULL;
    a->active = c->active;
    a->scr_mul = c->scr_mul ? c->scr_mul : 4;
    a->defer_ok = (uint32_t) c->defer_ok;
    a->split = (uint32_t) c->split;
    a->d_esize = (c->rtag_index >= 0 && ((c->active >> c->rtag_index) & 1)) ? c->d_esize : NULL;
    a->d_tag = c->d_tag; a->tag_len = c->tag_len;
    a->d_prep = c->want_report ? c->d_prep : NULL;
}

/* the interpreter's error word of a call: 0 = nothing that stops the call */
static int refused(flbgpu_chain *c, uint32_t bits)
{
    if (c->nf == 1) bits &= ~FLBGPU_E_DEEP;          /* nothing behind the parser decodes its result in this call */
    if (!bits) return 0;
    c->st.error_bits = bits;
    snprintf(g_rt_err, sizeof(g_rt_err), "device interpreter refused some records (error bits 0x%x: "
             "1=too many keys 2=regex stack 4=regex budget 8=float text not restated (hex float, nan(payload)) 32=logfmt escapes "
             "64=log_to_metrics value/label outside the device path 128=a pattern with POSIX brackets, \\b or case-insensitivity met a non-ASCII value "
             "256=a parsed value nested to msgpack-c's unpack limit inside a fused chain "
             "1024=a multiline message reached the buffer limit 2048=multiline: an event with non-empty metadata "
             "8192=to-JSON: more group markers than the list holds)", bits);
    return 1;
}

/* parser report of the previous call: flags back to "not parsed" */
static int report_clear(flbgpu_chain *c)
{
    if (!c->want_report || !c->d_prep || !c->cap_rec) return 0;
    return bk_zero(c->q, c->d_prep, c->cap_rec * 6 * sizeof(int32_t));
}

/* zero the per-call metrics table (before every evaluation pass) */
static int l2m_clear(flbgpu_chain *c)
{
    struct l2m_state *st;
    size_t n = c->l2m_slots;
    if (c->l2m_index < 0 || !((c->active >> c->l2m_index) & 1)) return 0;
    st = c->f[c->l2m_index]->l2m;
    if (bk_zero(c->q, c->l2m.hash, n * 8) || bk_zero(c->q, c->l2m.first, n * 4) || bk_zero(c->q, c->l2m.cnt, n * 8) ||
        bk_zero(c->q, c->l2m.sum, n * 8) || bk_zero(c->q, c->l2m.bkt, n * L2M_NBK(st) * 8)) return -1;
    if (c->l2m.pending_n && bk_zero(c->q, c->l2m.pending_n, 16)) return -1;
    if (c->l2m.amax && bk_zero(c->q, c->l2m.amax, n * 8)) return -1;
    if (c->l2m_record && c->l2m.obs_slot && bk_zero(c->q, c->l2m.obs_slot, c->cap_rec * 4)) return -1;
    return 0;
}

/* histogram: 1 when the settled table holds a set whose sum has to be added up in record order (l2m_fold_sums) while this
 * call's evaluation did not write its observations -- from now on it does, and the call evaluates again.  Conservative: any
 * set that left the exact path, any observation that is not an exact integer, or all observations against the largest bound. */
static int l2m_want_observations(flbgpu_chain *c)
{
    struct l2m_state *st;
    size_t n = c->l2m_slots, i;
    uint64_t maxb = 0, amax = 0, cnt = 0;
    int need = 0, j;
    if (c->l2m_record || !c->l2m.amax || c->l2m_index < 0 || !((c->active >> c->l2m_index) & 1)) return 0;
    st = c->f[c->l2m_index]->l2m;
    if (bk_d2h(c->q, c->h_hash, c->l2m.hash, n * 8) || bk_d2h(c->q, c->h_cnt, c->l2m.cnt, n * 8) ||
        bk_d2h(c->q, c->h_amax, c->l2m.amax, n * 8) || bk_sync(c->q)) return -1;
    for (j = 0; j < st->n_sets; j++) if (st->sets[j].bound > maxb) maxb = st->sets[j].bound;
    for (i = 0; i < n; i++) {
        if (!c->h_hash[i]) continue;
        cnt += c->h_cnt[i];
        if (c->h_amax[i] > amax) amax = c->h_amax[i];
    }
    if (cnt) need = maxb == L2M_NOT_EXACT || amax == L2M_NOT_EXACT || (amax && cnt > (L2M_EXACT_MAX - maxb) / amax);
    if (need) c->l2m_record = 1;
    return need;
}

/* the bound (struct l2m_set) a histogram sum starts from: |sum| when it is an integer of at most 2^53 other than -0.0 */
static uint64_t l2m_sum_bound(double sum)
{
    const double a = sum < 0 ? -sum : sum;
    uint64_t bits;
    memcpy(&bits, &sum, 8);
    if (!(a <= (double) L2M_EXACT_MAX) || (double) (uint64_t) a != a || bits == 0x8000000000000000ull) return L2M_NOT_EXACT;
    return (uint64_t) a;
}

/* histogram: the sums of the sets the call observed.  A set keeps the atomic sum while it provably equals the record-order
 * sum; otherwise its observations are added to its previous sum one by one, in record order, as cmt_metric_hist_sum_add()
 * does (new = old + val). */
static int l2m_fold_sums(flbgpu_chain *c, struct l2m_state *st, uint32_t n_rec)
{
    int i, any = 0;
    uint32_t r;
    for (i = 0; i < st->n_sets; i++) {
        struct l2m_set *s = &st->sets[i];
        if (!s->call_n) continue;
        if (s->bound != L2M_NOT_EXACT && s->call_amax != L2M_NOT_EXACT &&
            (s->call_amax == 0 || s->call_n <= (L2M_EXACT_MAX - s->bound) / s->call_amax)) {
            s->sum += s->call_sum;
            s->bound += s->call_n * s->call_amax;
            s->call_n = 0;
        }
        else { s->bound = L2M_NOT_EXACT; any = 1; }
    }
    if (!any) return 0;
    if (!c->l2m_record) { set_err("log_to_metrics: histogram observations were not recorded%s%s", NULL, NULL); return -1; }
    if (c->cap_hobs < n_rec) {
        free(c->h_obs_slot); free(c->h_obs_val);
        c->cap_hobs = (size_t) n_rec + n_rec / 4 + 64;
        c->h_obs_slot = malloc(c->cap_hobs * sizeof(uint32_t)); c->h_obs_val = malloc(c->cap_hobs * sizeof(double));
        if (!c->h_obs_slot || !c->h_obs_val) { c->cap_hobs = 0; set_err("out of memory%s%s", NULL, NULL); return -1; }
    }
    if (n_rec && (bk_d2h(c->q, c->h_obs_slot, c->l2m.obs_slot, (size_t) n_rec * 4) ||
                  bk_d2h(c->q, c->h_obs_val, c->l2m.obs_val, (size_t) n_rec * 8) || bk_sync(c->q))) return -1;
    for (r = 0; r < n_rec; r++) {
        struct l2m_set *s;
        if (!c->h_obs_slot[r]) continue;
        s = &st->sets[c->h_setof[c->h_obs_slot[r] - 1]];
        if (s->call_n) s->sum += c->h_obs_val[r];
    }
    return 0;
}

static int cmp_first(const void *a, const void *b, void *arg)
{
    const uint32_t *first = arg;
    uint32_t x = first[*(const uint32_t *) a], y = first[*(const uint32_t *) b];
    return x > y ? -1 : x < y;             /* stored as 0xffffffff - index: larger = seen earlier */
}

/* fold the settled per-call table into the filter's cumulative state, new label sets in
 * first-seen (record) order -- the order cmetrics appends them (cmt_map.c:209-243) */
static int l2m_merge(flbgpu_chain *c, uint32_t n_rec)
{
    struct l2m_state *st;
    size_t n = c->l2m_slots, nbk, i, m = 0;
    uint32_t *order;
    if (c->l2m_index < 0 || !((c->active >> c->l2m_index) & 1)) return 0;
    st = c->f[c->l2m_index]->l2m;
    nbk = L2M_NBK(st);
    if (bk_d2h(c->q, c->h_hash, c->l2m.hash, n * 8) || bk_d2h(c->q, c->h_chash, c->l2m.chash, n * 8) || bk_d2h(c->q, c->h_first, c->l2m.first, n * 4) || bk_d2h(c->q, c->h_cnt, c->l2m.cnt, n * 8) ||
        bk_d2h(c->q, c->h_sum, c->l2m.sum, n * 8) || bk_d2h(c->q, c->h_bkt, c->l2m.bkt, n * nbk * 8) ||
        (c->l2m.amax && bk_d2h(c->q, c->h_amax, c->l2m.amax, n * 8)) || bk_sync(c->q)) return -1;
    order = malloc(sizeof(uint32_t) * (n ? n : 1));
    if (!order) { set_err("out of memory%s%s", NULL, NULL); return -1; }
    for (i = 0; i < (size_t) st->n_sets; i++) { st->sets[i].call_last = 0; st->sets[i].call_n = st->sets[i].call_amax = 0; st->sets[i].call_sum = 0; }
    for (i = 0; i < n; i++) if (c->h_hash[i]) order[m++] = (uint32_t) i;
    qsort_r(order, m, sizeof(uint32_t), cmp_first, c->h_first);
    for (i = 0; i < m; i++) {
        uint32_t slot = order[i];
        struct l2m_set *set = NULL;
        size_t lb = (size_t) (st->n_labels ? st->n_labels : 1) * L2M_LABEL_BYTES, k;
        int j;
        char *labels = NULL;
        /* cmetrics finds a metric by the hash of its label values run together: tuples that concatenate alike are one
         * metric, shown with the labels of whichever came first (this loop runs in first-seen order) */
        for (j = 0; j < st->n_sets; j++) if (st->sets[j].hash == c->h_chash[slot]) { set = &st->sets[j]; break; }
        if (!set) {
            labels = calloc(1, lb);
            if (!labels) { free(order); set_err("out of memory%s%s", NULL, NULL); return -1; }
            if (st->n_labels && (bk_d2h(c->q, labels, c->l2m.str + (size_t) slot * lb, lb) || bk_sync(c->q))) { free(labels); free(order); return -1; }
            if (st->n_sets == st->cap_sets) {
                struct l2m_set *ns_ = realloc(st->sets, sizeof(*st->sets) * (size_t) (st->cap_sets ? st->cap_sets * 2 : 64));
                if (!ns_) { free(labels); free(order); set_err("out of memory%s%s", NULL, NULL); return -1; }
                st->sets = ns_;
                st->cap_sets = st->cap_sets ? st->cap_sets * 2 : 64;
            }
            set = &st->sets[st->n_sets++];
            memset(set, 0, sizeof(*set));
            set->hash = c->h_chash[slot];
            set->labels = labels;
            set->buckets = calloc((size_t) st->n_buckets + 1, sizeof(uint64_t));
            if (!set->buckets) { st->n_sets--; free(labels); free(order); set_err("out of memory%s%s", NULL, NULL); return -1; }
        }
        set->count += c->h_cnt[slot];
        if (st->mode == L2M_GAUGE) {             /* the call's last record of this set overwrites what earlier calls left */
            if (c->h_bkt[slot * 2] > set->call_last) { set->call_last = c->h_bkt[slot * 2]; memcpy(&set->sum, &c->h_bkt[slot * 2 + 1], 8); }
            continue;
        }
        for (k = 0; k < nbk; k++) set->buckets[k] += c->h_bkt[slot * nbk + k];
        if (st->mode != L2M_HISTOGRAM) continue;
        c->h_setof[slot] = (int32_t) (set - st->sets);
        set->call_n += c->h_cnt[slot];
        set->call_sum += c->h_sum[slot];
        if (c->h_amax[slot] > set->call_amax) set->call_amax = c->h_amax[slot];
    }
    free(order);
    return st->mode == L2M_HISTOGRAM ? l2m_fold_sums(c, st, n_rec) : 0;
}


/* msgpack-c's streaming parser (lib/msgpack-c/include/msgpack/unpack_template.h: template_execute) on the bytes
 * behind the last whole event: it eats a header byte, then that header's fixed-size part (length field or scalar)
 * only if all of it is there, then a payload only if all of it is there.  When the buffer runs out exactly at one
 * of those points, inside the first unfinished object, msgpack_unpack_next() reports CONTINUE with the offset at
 * the end of the buffer -- which flb_log_event_decoder_next() turns into INSUFFICIENT_DATA and the filters
 * (grep.c:357-360, modify.c) accept as a clean end when `offset == bytes`.  1 = that is the case for b[0..n). */
static int msgpack_tail_runs_out_cleanly(const uint8_t *b, size_t n)
{
    size_t p = 0;
    uint64_t open[64];                  /* elements still owed per open container */
    int depth = 0;
    if (n == 0) return 1;
    for (;;) {
        uint32_t c, fixed = 0, is_len = 0, items = 0, is_container = 0;
        uint64_t payload = 0;
        if (p == n) return 1;                                   /* ran out between two objects of an open container */
        c = b[p++];
        if (c <= 0x7f || c >= 0xe0 || c == 0xc0 || c == 0xc2 || c == 0xc3) { }
        else if (c >= 0xa0 && c <= 0xbf) payload = c & 31;
        else if (c >= 0x90 && c <= 0x9f) { is_container = 1; items = c & 15; }
        else if (c >= 0x80 && c <= 0x8f) { is_container = 1; items = 2 * (c & 15); }
        else switch (c) {
        case 0xcc: case 0xd0: fixed = 1; break;
        case 0xcd: case 0xd1: fixed = 2; break;
        case 0xce: case 0xd2: case 0xca: fixed = 4; break;
        case 0xcf: case 0xd3: case 0xcb: fixed = 8; break;
        case 0xd4: fixed = 2; break; case 0xd5: fixed = 3; break; case 0xd6: fixed = 5; break;
        case 0xd7: fixed = 9; break; case 0xd8: fixed = 17; break;
        case 0xd9: case 0xc4: fixed = 1; is_len = 1; break;
        case 0xda: case 0xc5: fixed = 2; is_len = 1; break;
        case 0xdb: case 0xc6: fixed = 4; is_len = 1; break;
        case 0xc7: fixed = 1; is_len = 2; break;
        case 0xc8: fixed = 2; is_len = 2; break;
        case 0xc9: fixed = 4; is_len = 2; break;
        case 0xdc: fixed = 2; is_len = 3; break;
        case 0xdd: fixed = 4; is_len = 3; break;
        case 0xde: fixed = 2; is_len = 4; break;
        case 0xdf: fixed = 4; is_len = 4; break;
        default: return 0;                                      /* 0xc1: a parse error, not a shortage */
        }
        if (fixed) {
            uint64_t v = 0;
            uint32_t i;
            if (n - p < fixed) return p == n;                   /* stops behind the header byte */
            for (i = 0; i < fixed; i++) v = (v << 8) | b[p + i];
            p += fixed;
            if (is_len == 1) payload = v;
            else if (is_len == 2) payload = v + 1;              /* ext: type byte + data */
            else if (is_len == 3) { is_container = 1; items = (uint32_t) v; if (v > 0x7fffffffu) return 0; }
            else if (is_len == 4) { is_container = 1; if (v > 0x3fffffffu) return 0; items = (uint32_t) (2 * v); }
        }
        if (payload) {
            if (n - p < payload) return p == n;                 /* stops where the payload begins */
            p += (size_t) payload;
        }
        if (is_container) {
            if (depth >= 32) return 0;                          /* MSGPACK_EMBED_STACK_SIZE: a failure, not a shortage (dev_msgpack.cuh: mp_skip_lim) */
            if (items) { open[depth++] = items; continue; }
        }
        /* one object done: pay it to the containers it closes */
        for (;;) {
            if (depth == 0) return 0;                           /* a whole top-level object fits: not a shortage */
            if (--open[depth - 1]) break;
            depth--;
        }
    }
}

/* `clean`: the decodable prefix is the whole chunk, or what follows it is an event cut short at a point where the
 * reference's decoder still reports `offset == bytes` (see above) */
static int ends_cleanly(bk_q *q, const uint8_t *h_in, const uint8_t *d_in, size_t off, size_t bytes)
{
    uint8_t *tmp;
    int r;
    if (off == bytes) return 1;
    if (h_in) return msgpack_tail_runs_out_cleanly(h_in + off, bytes - off);
    tmp = malloc(bytes - off);
    if (!tmp) return 0;
    r = (bk_d2h(q, tmp, d_in + off, bytes - off) || bk_sync(q)) ? 0 : msgpack_tail_runs_out_cleanly(tmp, bytes - off);
    free(tmp);
    return r;
}

/* The record index frames events whose root and header arrays are fixarrays (0x92), which is all msgpack-c's
 * packer ever writes for two elements.  The reference's decoder would also take the same arrays spelled as
 * array16 / array32: when the decodable prefix [0, off) stops at such a spelling the call is refused, not cut short.
 * Nonzero = refused (FLBGPU_E_INDEX and the error text are set). */
static int refuse_wide_arrays(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in, size_t off, size_t bytes)
{
    uint8_t b[8] = { 0 };
    size_t n = bytes - off < sizeof(b) ? bytes - off : sizeof(b), i = 0;
    int wide = 0;
    if (n == 0) return 0;
    if (h_in) memcpy(b, h_in + off, n);
    else if (bk_d2h(c->q, b, d_in + off, n) || bk_sync(c->q)) return 0;
    if (b[0] == 0x92) i = 1;                                   /* [ [ts, meta], body ] with a wide header array */
    if (b[i] == 0xdc) wide = b[i + 1] == 0 && b[i + 2] == 2;
    if (b[i] == 0xdd) wide = b[i + 1] == 0 && b[i + 2] == 0 && b[i + 3] == 0 && b[i + 4] == 2;
    if (!wide) return 0;
    c->st.error_bits = FLBGPU_E_INDEX;
    snprintf(g_rt_err, sizeof(g_rt_err), "event framed with an array16/array32 header at byte %zu: not decoded on the GPU path", off);
    return 1;
}

/* the start of a chain call: fresh stats, no result yet, the call's clock (t0, when given) running.  A chunk of 4 GiB or
 * more is refused: record offsets are 32-bit. */
static int call_start(flbgpu_chain *c, size_t bytes, size_t *out_size, struct timespec *t0)
{
    memset(&c->st, 0, sizeof(c->st));
    c->st.bytes_in = bytes;
    *out_size = 0;
    if (t0) clock_gettime(CLOCK_MONOTONIC, t0);
    if (bytes >= 0xfff00000ull) { set_err("chunk larger than 4 GiB: split the append%s%s", NULL, NULL); return -1; }
    return 0;
}

/* the chunk on the device: h_in uploaded in pieces into the chain's input buffer (the index waits for each piece), or the
 * caller's d_in_ext as it is.  NULL on failure. */
static const uint8_t *place_input(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in_ext, size_t bytes)
{
    if (d_in_ext) { bk_upload_none(c->q); return d_in_ext; }
    if (dev_grow(c, (void **) &c->d_in, &c->cap_in, bytes + 64, 1, 0) || bk_upload_start(c->q, c->d_in, h_in, bytes)) return NULL;
    return c->d_in;
}

/* the scratch a call needs, its arguments before the first evaluation (fill_args() adds the buffers once they have grown)
 * and the per-call evidence, metrics and parser report cleared */
static int call_args(flbgpu_chain *c, struct bk_chain_args *a, size_t bytes, uint32_t assume)
{
    if (c->needs_scratch && dev_grow(c, (void **) &c->d_scr, &c->cap_scr, (size_t) c->scr_mul * bytes + 64, 1, 0)) return -1;
    memset(a, 0, sizeof(*a));
    a->now = (int64_t) time(NULL);
    a->assume = assume;
    return (bk_flags_clear(c->q, c->d_flags) || l2m_clear(c) || report_clear(c)) ? -1 : 0;
}

#include "runtime_ml.h"
#include "runtime_tojson.h"
#include "runtime_lines.h"

/* flb_router_match() (src/flb_router.c:37-128): Match_Regex first -- onig_match() at the start of the tag with a match of
 * positive length -- then the Match pattern, where '*' stands for any run of characters. */
static int wildcard_match(const char *tag, size_t n, const char *m)
{
    while (*m) {
        if (*m == '*') {
            while (*++m == '*') { }
            if (!*m) return 1;
            {
                size_t i;
                for (i = 0; i < n; i++) if (tag[i] == *m && wildcard_match(tag + i, n - i, m)) return 1;
            }
            return 0;
        }
        if (n == 0 || *tag != *m) return 0;
        tag++; n--; m++;
    }
    return n == 0;
}

static int filter_routes(const flbgpu_filter *f, const char *tag, int tag_len)
{
    if (f->inactive) return 0;
    if (tag_len < 0) return 0;
    if (!tag) { if (tag_len) return 0; tag = ""; }
    if (f->has_match_rx) {
        int caps[2 * (RX_MAX_GROUPS + 1)];
        if (bk_rx_search_host(f->match_rx.prog, (const uint8_t *) tag, tag_len, caps) == RX_R_MATCH && caps[0] == 0 && caps[1] > 0) return 1;
    }
    if (!f->match) return !f->has_match_rx;           /* no rule given at all: every chunk (the engine refuses such an instance) */
    return wildcard_match(tag, (size_t) tag_len, f->match);
}

static uint32_t chain_active_mask(flbgpu_chain *c, const char *tag, int tag_len)
{
    uint32_t m = 0;
    int k;
    for (k = 0; k < c->nf; k++) if (filter_routes(c->f[k], tag, tag_len)) m |= 1u << k;
    return m;
}

/* the verdict vector a call starts from: every routed filter modifies (log_to_metrics only when it discards) */
static uint32_t initial_assume(flbgpu_chain *c)
{
    uint32_t a = c->active;
    if (c->l2m_index >= 0 && !c->f[c->l2m_index]->l2m->discard) a &= ~(1u << c->l2m_index);
    return a;
}

/* the verdict vector the speculating forms emit under: the one the previous call settled on, if it had the same routing */
static uint32_t speculated_assume(flbgpu_chain *c)
{
    return (c->spec_valid && c->spec_active == c->active) ? c->spec_assume : initial_assume(c);
}

/* One call.  Input: h_in (host, uploaded in pieces) or d_in_ext (already in HBM).
 * Result: host_out != NULL -> malloc()ed host buffer; else ext_out (device, capacity ext_cap). */
/* rewrite_tag: fetch the re-tagged stream of this call and group it by new tag, in order of first appearance -- what the
 * reference's per-record in_emitter_add_record() calls leave in the emitter (one chunk per tag, records in order). */
static int rtag_collect(flbgpu_chain *c, const struct bk_chain_args *a, uint32_t n_rec, int any)
{
    flbgpu_filter *f = c->f[c->rtag_index];
    uint8_t *stream = NULL;
    size_t bytes = 0, at, g, ng = 0, cap = 0;
    struct flbgpu_emit_group *gr = NULL;
    size_t *fill = NULL;
    rtag_release(f);
    if (!any) return 0;
    {
        const size_t nb = ((size_t) n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK + 2;
        if (c->cap_ebsum < nb) {
            bk_free(c->q, c->d_ebsum); free(c->h_ebsum);
            c->cap_ebsum = 0;
            c->d_ebsum = bk_alloc(c->q, (nb + nb / 4 + 64) * sizeof(uint64_t));
            c->h_ebsum = malloc((nb + nb / 4 + 64) * sizeof(uint64_t));
            if (!c->d_ebsum || !c->h_ebsum) { set_err("out of memory%s%s", NULL, NULL); return -1; }
            c->cap_ebsum = nb + nb / 4 + 64;
        }
    }
    if (bk_rtag_emit(c->q, a, n_rec, c->d_ebsum, c->h_ebsum, (void **) &stream, &bytes)) { set_err("%s%s", bk_last_error(), NULL); return -1; }
    if (!stream) return 0;
    /* pass 1: the groups and their sizes */
    for (at = 0; at + RT_ENTRY_HDR <= bytes; ) {
        uint32_t tl, rl;
        memcpy(&tl, stream + at, 4); memcpy(&rl, stream + at + 4, 4);
        if (at + RT_ENTRY_HDR + tl + rl > bytes) break;
        for (g = 0; g < ng; g++) if (gr[g].tag_len == tl && !memcmp(gr[g].tag, stream + at + RT_ENTRY_HDR, tl)) break;
        if (g == ng) {
            if (ng == cap) {
                struct flbgpu_emit_group *n2 = realloc(gr, sizeof(*gr) * (cap ? cap * 2 : 16));
                if (!n2) { free(gr); free(stream); set_err("out of memory%s%s", NULL, NULL); return -1; }
                gr = n2; cap = cap ? cap * 2 : 16;
            }
            memset(&gr[ng], 0, sizeof(gr[ng]));
            gr[ng].tag = (const char *) stream + at + RT_ENTRY_HDR; gr[ng].tag_len = tl;
            ng++;
        }
        gr[g].size += rl; gr[g].records++;
        at += RT_ENTRY_HDR + tl + rl;
    }
    if (at != bytes) { free(gr); free(stream); set_err("malformed re-tagged stream%s%s", NULL, NULL); return -1; }
    f->rt_bufs = calloc(ng ? ng : 1, sizeof(void *));
    fill = calloc(ng ? ng : 1, sizeof(size_t));
    if (!f->rt_bufs || !fill) { free(fill); free(f->rt_bufs); f->rt_bufs = NULL; free(gr); free(stream); set_err("out of memory%s%s", NULL, NULL); return -1; }
    f->rt_groups = gr; f->rt_n = ng; f->rt_stream = stream;
    for (g = 0; g < ng; g++) {
        f->rt_bufs[g] = malloc(gr[g].size ? gr[g].size : 1);
        if (!f->rt_bufs[g]) { free(fill); rtag_release(f); set_err("out of memory%s%s", NULL, NULL); return -1; }
        gr[g].data = f->rt_bufs[g];
    }
    /* pass 2: the records, in order, behind one another per group */
    for (at = 0; at < bytes; ) {
        uint32_t tl, rl;
        memcpy(&tl, stream + at, 4); memcpy(&rl, stream + at + 4, 4);
        for (g = 0; g < ng; g++) if (gr[g].tag_len == tl && !memcmp(gr[g].tag, stream + at + RT_ENTRY_HDR, tl)) break;
        memcpy((uint8_t *) f->rt_bufs[g] + fill[g], stream + at + RT_ENTRY_HDR + tl, rl);
        fill[g] += rl;
        at += RT_ENTRY_HDR + tl + rl;
    }
    free(fill);
    return 0;
}

/* What a call leaves behind once no other form will redo it: its metrics folded into the filter's table and, with a
 * routed rewrite_tag filter, the re-tagged stream of its n_rec records.  Those go to the emitter whatever the filter's own
 * verdict is (a chunk that does not decode to its end makes it NOTOUCH after the fact, rewrite_tag.c:500-546). */
static int call_commit(flbgpu_chain *c, struct bk_chain_args *a, const uint8_t *d_in, size_t bytes, uint32_t n_rec, const uint32_t *flags)
{
    const int again = l2m_want_observations(c);
    if (again) return again;                         /* 1: evaluate the call again (its result is not committed), -1 */
    if (l2m_merge(c, n_rec)) return -1;
    if (c->rtag_index < 0 || !((c->active >> c->rtag_index) & 1)) return 0;
    fill_args(c, a, d_in, bytes, n_rec);
    return rtag_collect(c, a, n_rec, (flags[c->rtag_index] & CHF_CAUSE) != 0);
}

/* the host buffer a result of `need` bytes goes to: the caller's (flbgpu_chain_set_result_buffer) while it fits, else a
 * malloc() of `size` bytes; res_drop() releases it on failure */
static void *res_take(flbgpu_chain *c, size_t need, size_t size)
{
    return (c->res_buf && c->res_cap >= need) ? (void *) c->res_buf : malloc(size);
}
static void res_drop(flbgpu_chain *c, void *p)
{
    if ((uint8_t *) p != c->res_buf) free(p);
}

static void hugepage_hint(void *p, size_t n)
{
#ifdef MADV_HUGEPAGE
    const char *e = getenv("FLBGPU_HUGEPAGE");
    if (e && e[0] == '0') return;
    if (n >= ((size_t) 8 << 20)) {                    /* fewer, larger page faults while the result is filled in */
        uintptr_t lo = ((uintptr_t) p + ((size_t) 2 << 20) - 1) & ~(((uintptr_t) 2 << 20) - 1);
        uintptr_t hi = ((uintptr_t) p + n) & ~(((uintptr_t) 2 << 20) - 1);
        if (hi > lo) madvise((void *) lo, hi - lo, MADV_HUGEPAGE);
    }
#else
    (void) p; (void) n;
#endif
}

static float ms_since(const struct timespec *t0)
{
    struct timespec t1;
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (float) ((t1.tv_sec - t0->tv_sec) * 1e3 + (t1.tv_nsec - t0->tv_nsec) / 1e6);
}

static int chain_run(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in_ext, size_t bytes,
                     uint8_t *ext_out, size_t ext_cap, void **host_out, size_t *out_size)
{
    struct bk_chain_args a;
    const uint8_t *d_in;
    uint32_t n_rec = 0, h_flags[FLBGPU_MAX_FILTERS + 1], nb;
    size_t off = 0, S = slice_bytes();
    uint64_t total;
    int clean, pass, r;
    struct timespec t0;

    if (call_start(c, bytes, out_size, &t0) || !(d_in = place_input(c, h_in, d_in_ext, bytes)) ||
        call_args(c, &a, bytes, initial_assume(c))) return -1;

    /* ---- index + evaluate, slice by slice, while the upload is still running ---- */
    while (off < bytes) {
        size_t len = bytes - off < S ? bytes - off : S;
        uint32_t n_valid;
        uint64_t end_off;
        if (index_slice(c, d_in, off, len, n_rec, &n_valid, &end_off)) return -1;
        if (n_valid == 0) {
            if (off + len < bytes) { S *= 2; continue; }       /* a record longer than the slice: widen it */
            break;                                             /* nothing decodable from here to the end */
        }
        fill_args(c, &a, d_in, bytes, n_rec + n_valid);
        bk_hint_streaming(c->q, a.d_in + off, (size_t) end_off - off);
        if (bk_chain_eval(c->q, &a, n_rec, n_rec + n_valid)) return -1;
        n_rec += n_valid;
        off = (size_t) end_off;
    }
    clean = ends_cleanly(c->q, h_in, d_in, off, bytes);
    if (refuse_wide_arrays(c, h_in, d_in, off, bytes)) return -1;
    c->st.records_in = n_rec;
    c->st.passes = 1;
    fill_args(c, &a, d_in, bytes, n_rec);

    /* ---- chunk-level verdicts; revise assumptions front to back until they hold ---- */
    for (pass = 0; pass <= c->nf; pass++) {
        if (bk_flags_fetch(c->q, c->d_flags, h_flags)) return -1;
        if (refused(c, h_flags[FLBGPU_MAX_FILTERS])) return -1;
        if (settle(c, a.assume, h_flags, clean, &a.assume) < 0) break;
        /* later filters saw the wrong input: re-evaluate */
        if (bk_flags_clear(c->q, c->d_flags) || l2m_clear(c) || report_clear(c) || bk_chain_eval(c->q, &a, 0, n_rec)) return -1;
        c->st.passes++;
    }
    c->st.kernel_launches = bk_launch_count();
    c->st.phase_ms[0] = ms_since(&t0);
    while ((r = call_commit(c, &a, d_in, bytes, n_rec, h_flags)) == 1) {      /* again, writing the metric observations */
        fill_args(c, &a, d_in, bytes, n_rec);
        if (bk_flags_clear(c->q, c->d_flags) || l2m_clear(c) || report_clear(c) || bk_chain_eval(c->q, &a, 0, n_rec)) return -1;
        c->st.passes++;
    }
    if (r) return -1;
    if (a.assume == 0) return FLBGPU_FILTER_NOTOUCH;

    /* ---- output offsets ---- */
    if (sizes_to_offsets(c, c->d_size, n_rec, NULL, NULL, "result larger than 4 GiB", &total)) return -1;
    a.d_bsum = c->d_bsum;
    nb = (n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    c->st.bytes_out = total;
    *out_size = (size_t) total;
    c->st.phase_ms[1] = ms_since(&t0) - c->st.phase_ms[0];
    if (total == 0) return FLBGPU_FILTER_MODIFIED;

    /* ---- emit (+ download) ---- */
    if (!host_out) {
        if (!ext_out && c->keep_result) {
            if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0)) return -1;
            ext_out = c->d_out; ext_cap = c->cap_out;
        }
        if (ext_cap < total) { set_err("device output buffer too small%s%s", NULL, NULL); return -1; }
        if (bk_chain_emit(c->q, &a, ext_out, 0, nb)) return -1;
    }
    else {
        const uint32_t step = 2048;                   /* blocks per emission launch (512 K records) */
        uint32_t b0;
        void *out = res_take(c, total, total);
        if (!out) return -1;
        if ((uint8_t *) out != c->res_buf) hugepage_hint(out, total);
        if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_download_begin(c->q, out, c->d_out)) { res_drop(c, out); return -1; }
        for (b0 = 0; b0 < nb; b0 += step) {
            uint32_t b1 = b0 + step < nb ? b0 + step : nb;
            if (bk_chain_emit(c->q, &a, c->d_out, b0, b1) || bk_download_push(c->q, (size_t) c->h_bsum[b0], (size_t) c->h_bsum[b1])) {
                bk_download_end(c->q);
                res_drop(c, out);
                return -1;
            }
        }
        if (bk_download_end(c->q)) { res_drop(c, out); return -1; }
        *host_out = out;
    }
    c->st.kernel_launches = bk_launch_count();
    if (host_out) bk_records_out(c->q, &c->st.records_out);     /* (the device-output form leaves the stream running) */
    c->st.phase_ms[3] = ms_since(&t0);
    c->st.phase_ms[2] = c->st.phase_ms[3] - c->st.phase_ms[1] - c->st.phase_ms[0];
    return FLBGPU_FILTER_MODIFIED;
}

/* Copy-out of result pieces from the pinned staging ring into the caller's malloc()ed chunk.  The
 * destination is written once and not read again by this library, so on x86-64 with AVX2 the body
 * goes out with non-temporal stores: no read-for-ownership of the destination lines and no cache
 * pollution -- with several GPUs per host the copy-out traffic is what saturates host memory. */
#if defined(__x86_64__) && defined(__GNUC__)
#include <immintrin.h>
__attribute__((target("avx2")))
static void stream_copy_avx2(uint8_t *d, const uint8_t *s, size_t n)
{
    size_t head = ((uintptr_t) d & 31) ? 32 - ((uintptr_t) d & 31) : 0, i;
    if (head > n) head = n;
    memcpy(d, s, head);
    d += head; s += head; n -= head;
    for (i = 0; i + 128 <= n; i += 128) {
        __m256i a = _mm256_loadu_si256((const __m256i *) (s + i)), b = _mm256_loadu_si256((const __m256i *) (s + i + 32));
        __m256i c = _mm256_loadu_si256((const __m256i *) (s + i + 64)), e = _mm256_loadu_si256((const __m256i *) (s + i + 96));
        _mm256_stream_si256((__m256i *) (d + i), a); _mm256_stream_si256((__m256i *) (d + i + 32), b);
        _mm256_stream_si256((__m256i *) (d + i + 64), c); _mm256_stream_si256((__m256i *) (d + i + 96), e);
    }
    _mm_sfence();
    memcpy(d + i, s + i, n - i);
}
#endif

void flbgpu_stream_copy(void *dst, const void *src, size_t n)
{
#if defined(__x86_64__) && defined(__GNUC__)
    static int have = -1;
    if (have < 0) { const char *e = getenv("FLBGPU_NT_COPY"); have = __builtin_cpu_supports("avx2") && !(e && e[0] == '0'); }
    if (have && n >= 4096) { stream_copy_avx2(dst, src, n); return; }
#endif
    memcpy(dst, src, n);
}

/* The streaming form's result so far: the host buffer and its capacity, the bytes placed in it, the record blocks emitted,
 * and whether a download into it is open. */
struct stream_out { uint8_t *out; size_t cap_out_h; uint64_t placed; uint32_t b_done; int dl_open; };

/* Emit the record blocks [so->b_done, upto) of the n_rec records evaluated so far (input bytes [0, off)) behind what has
 * been placed, and send them to the host buffer, which grows with the result. */
static int stream_flush(flbgpu_chain *c, struct bk_chain_args *a, struct stream_out *so, uint32_t upto, uint32_t n_rec, size_t off, size_t bytes)
{
    uint64_t end;
    if (upto <= so->b_done) return 0;
    fill_args(c, a, c->d_in, bytes, n_rec);
    if (bk_sizes_scan_range(c->q, c->d_size, n_rec, so->b_done, upto, c->d_bsum, c->h_bsum, so->placed)) return -1;
    end = c->h_bsum[upto];
    if (end >= 0xfff00000ull) { set_err("result larger than 4 GiB%s%s", NULL, NULL); return -1; }
    if (end > so->placed) {
        if (end > so->cap_out_h) {
            /* first estimate from the output/input ratio so far; grown (rarely) when it was too low */
            double ratio = (double) end / (double) (off ? off : 1);
            size_t want = (size_t) (ratio * 1.15 * (double) bytes) + ((size_t) 8 << 20);
            uint8_t *no;
            if (want < end) want = (size_t) end + ((size_t) 8 << 20);
            if (so->dl_open) { so->dl_open = 0; if (bk_download_end(c->q)) return -1; }
            if (!so->out) no = res_take(c, (size_t) end, want);
            else if (so->out == c->res_buf) { no = malloc(want); if (no) memcpy(no, so->out, (size_t) so->placed); }     /* outgrown: what has arrived moves */
            else no = realloc(so->out, want);
            if (!no) return -1;
            if (no == c->res_buf) want = c->res_cap;
            so->out = no; so->cap_out_h = want;
            if (so->out != c->res_buf) hugepage_hint(so->out, want);
            /* the device output buffer grows with the host one; bytes already emitted stay where they are */
            if (dev_grow(c, (void **) &c->d_out, &c->cap_out, want, 1, (size_t) so->placed)) return -1;
        }
        if (!so->dl_open) { if (bk_download_begin(c->q, so->out, c->d_out)) return -1; so->dl_open = 1; }
        if (bk_chain_emit(c->q, a, c->d_out, so->b_done, upto) || bk_download_push(c->q, (size_t) so->placed, (size_t) end)) return -1;
    }
    so->placed = end;
    so->b_done = upto;
    return 0;
}

/* the streaming form gives its result up: the download closes, the buffer is released (the caller's stays the caller's) */
static void stream_drop(flbgpu_chain *c, struct stream_out *so)
{
    if (so->dl_open) bk_download_end(c->q);
    res_drop(c, so->out);
}

/* Streaming form of chain_run for host buffers.  The chunk-level verdicts are only known when the
 * whole chunk has been evaluated, but they almost never differ from the previous call's (and from
 * "every filter modifies" on the first call), so each slice is emitted and sent back as soon as it
 * has been evaluated, speculating on that vector: upload of slice k+1, evaluation of slice k and
 * emission + download of slice k-1 overlap.  If the settled verdicts differ from the speculation the
 * speculative result is thrown away and the classic path runs (returns 1 = "use chain_run"). */
static int chain_run_stream(flbgpu_chain *c, const uint8_t *h_in, size_t bytes, void **host_out, size_t *out_size, int *ret)
{
    struct bk_chain_args a;
    struct stream_out so = { NULL, 0, 0, 0, 0 };
    uint32_t n_rec = 0, h_flags[FLBGPU_MAX_FILTERS + 1], assume = speculated_assume(c), nb_max;
    size_t off = 0, S = slice_bytes(), force = 0;
    const int taper = !(getenv("FLBGPU_TAPER") && getenv("FLBGPU_TAPER")[0] == '0');
    int clean;
    struct timespec t0;

    if (assume == 0) return 1;                       /* nothing would be emitted: the classic path decides */
    if (call_start(c, bytes, out_size, &t0) || !place_input(c, h_in, NULL, bytes)) return -1;
    nb_max = (uint32_t) (bytes / (3 * BK_REC_BLOCK)) + 4;       /* an event is at least 3 bytes */
    if (dev_grow(c, (void **) &c->d_bsum, &c->cap_bsum, nb_max, sizeof(uint64_t), 0) ||
        host_grow((void **) &c->h_bsum, &c->cap_hbsum, nb_max, sizeof(uint64_t)) || call_args(c, &a, bytes, assume)) return -1;

    while (off < bytes) {
        /* slices shrink towards the end of the chunk: what is left to do after the last upload piece
         * arrives (index, evaluate, emit, download of the last slice) is proportional to its size */
        size_t rem = bytes - off, want = S, len;
        uint32_t n_valid;
        uint64_t end_off;
        if (taper && rem < 3 * S) { want = rem / 3; if (want < ((size_t) 16 << 20)) want = (size_t) 16 << 20; if (want > S) want = S; }
        if (want < force) want = force;
        len = rem < want ? rem : want;
        if (index_slice(c, c->d_in, off, len, n_rec, &n_valid, &end_off)) goto fail;
        if (n_valid == 0) {
            if (off + len < bytes) { force = 2 * len; continue; }   /* a record longer than the slice: widen it */
            break;
        }
        force = 0;
        /* the previous slice has been evaluated by now (or is about to finish): place and send it */
        if (stream_flush(c, &a, &so, n_rec / BK_REC_BLOCK, n_rec, off, bytes)) goto fail;
        fill_args(c, &a, c->d_in, bytes, n_rec + n_valid);
        bk_hint_streaming(c->q, a.d_in + off, (size_t) end_off - off);
        if (bk_chain_eval(c->q, &a, n_rec, n_rec + n_valid)) goto fail;
        n_rec += n_valid;
        off = (size_t) end_off;
    }
    clean = ends_cleanly(c->q, h_in, c->d_in, off, bytes);
    if (refuse_wide_arrays(c, h_in, c->d_in, off, bytes)) goto fail;
    c->st.records_in = n_rec;
    c->st.passes = 1;
    if (stream_flush(c, &a, &so, (n_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK, n_rec, off, bytes)) goto fail;

    /* ---- the verdicts must be the ones speculated on ---- */
    if (bk_flags_fetch(c->q, c->d_flags, h_flags)) goto fail;
    if (refused(c, h_flags[FLBGPU_MAX_FILTERS])) goto fail;
    if (settle(c, assume, h_flags, clean, &assume) >= 0) {
        /* evidence of the later filters was gathered under a wrong assumption: redo classically (the next call
         * speculates on the verdict as found) */
        stream_drop(c, &so);
        return 1;
    }
    c->st.kernel_launches = bk_launch_count();
    if (so.dl_open) { so.dl_open = 0; if (bk_download_end(c->q)) goto fail; }
    switch (call_commit(c, &a, c->d_in, bytes, n_rec, h_flags)) {          /* every record of the call is still indexed */
    case 0: break;
    case 1: stream_drop(c, &so); return 1;          /* the metric observations are wanted: the classic path writes them */
    default: goto fail;
    }
    bk_records_out(c->q, &c->st.records_out);
    c->st.bytes_out = so.placed;
    *out_size = (size_t) so.placed;
    if (so.placed == 0) { res_drop(c, so.out); so.out = NULL; }
    else if (so.out != c->res_buf && so.cap_out_h > so.placed + so.placed / 2) {     /* badly over-estimated: give the excess back */
        uint8_t *sh = realloc(so.out, (size_t) so.placed);
        if (sh) so.out = sh;
    }
    *host_out = so.out;
    c->st.phase_ms[3] = ms_since(&t0);
    *ret = FLBGPU_FILTER_MODIFIED;
    return 0;
fail:
    stream_drop(c, &so);
    return -1;
}

/* the largest append the small-chunk form takes */
static size_t small_bytes(void)
{
    const char *e = getenv("FLBGPU_SMALL_MB");
    long mb = e ? atol(e) : 8;
    size_t v, s = slice_bytes();
    if (mb < 0) mb = 0;
    if (mb > 256) mb = 256;
    v = (size_t) mb << 20;
    return v < s ? v : s;                            /* the small form is a single slice */
}

/* One append as flb_filter_do() hands it over (tens of KB to a few MB): the whole call is one stream of work
 * without a host synchronisation in between (bk_small_run), under the verdict vector the previous call settled
 * on.  Returns 0 (done, *ret set), 1 (not for this form or the speculation did not hold: use the general
 * paths), -1 error. */
static int chain_run_small(flbgpu_chain *c, const uint8_t *h_in, size_t bytes, void **host_out, size_t *out_size, int *ret)
{
    struct bk_chain_args a;
    struct bk_small_res res;
    uint32_t assume = speculated_assume(c), n_tiles, cap_rec, nb_cap;
    size_t off, cap_out;
    int clean;
    struct timespec t0;

    if (assume == 0) return 1;                       /* nothing would be emitted: the classic path decides */
    if (call_start(c, bytes, out_size, &t0)) return -1;
    /* records of the shapes this path serves are tens of bytes at least; a chunk of tinier events overflows
     * the arrays, which the device reports (res.overflow) and the general path then handles */
    cap_rec = (uint32_t) (bytes / 24) + 1024;
    if (c->small_cap_rec > cap_rec) cap_rec = c->small_cap_rec;
    nb_cap = (cap_rec + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    n_tiles = (uint32_t) ((bytes + BK_INDEX_TILE - 1) / BK_INDEX_TILE);
    cap_out = bytes + bytes / 2 + 4096;
    if (c->small_cap_out > cap_out) cap_out = c->small_cap_out;
    /* (bk_small_run uploads the chunk itself, through the queue's own pinned buffer) */
    if (dev_grow(c, (void **) &c->d_in, &c->cap_in, bytes + 64, 1, 0) ||
        dev_grow(c, (void **) &c->d_tile, &c->cap_tile, n_tiles + 1, sizeof(uint32_t), 0) ||
        dev_grow(c, (void **) &c->d_bsum, &c->cap_bsum, nb_cap + 2, sizeof(uint64_t), 0) ||
        ensure_rec_cap(c, cap_rec, 0) ||
        dev_grow(c, (void **) &c->d_out, &c->cap_out, cap_out, 1, 0) ||
        call_args(c, &a, bytes, assume)) return -1;
    cap_out = c->cap_out;
    fill_args(c, &a, c->d_in, bytes, 0);
    if (bk_small_run(c->q, &a, h_in, c->d_in, bytes, cap_rec, c->d_tile, n_tiles, c->d_out, cap_out, &res)) return -1;
    c->st.kernel_launches = bk_launch_count();
    if (res.overflow) {                              /* denser events than assumed, or a slice-sized tangle of broken links */
        if (res.overflow == 1 && res.n_cand < 0x7fffffffu) c->small_cap_rec = res.n_cand + res.n_cand / 4 + 1024;
        return 1;
    }
    off = (size_t) res.end_off;
    clean = ends_cleanly(c->q, h_in, c->d_in, off, bytes);
    if (refuse_wide_arrays(c, h_in, c->d_in, off, bytes)) return -1;
    c->st.records_in = res.n_valid;
    c->st.passes = 1;
    if (refused(c, res.flags[FLBGPU_MAX_FILTERS])) return -1;
    if (settle(c, assume, res.flags, clean, &assume) >= 0) return 1;
    if (res.total >= 0xfff00000ull) { set_err("result larger than 4 GiB%s%s", NULL, NULL); return -1; }
    if (!res.emitted) {                              /* the result outgrew the output buffer: remember, let the general path do this call */
        c->small_cap_out = (size_t) res.total + (size_t) res.total / 4 + 4096;
        return 1;
    }
    switch (call_commit(c, &a, c->d_in, bytes, res.n_valid, res.flags)) {
    case 0: break;
    case 1: return 1;                                /* the metric observations are wanted: the general paths write them */
    default: return -1;
    }
    c->st.records_out = res.n_out;
    c->st.bytes_out = res.total;
    *out_size = (size_t) res.total;
    *host_out = NULL;
    if (res.total) {
        void *out = res_take(c, (size_t) res.total, (size_t) res.total);
        if (!out) { set_err("out of memory%s%s", NULL, NULL); return -1; }
        if (bk_small_fetch(c->q, out, c->d_out, (size_t) res.total)) { res_drop(c, out); return -1; }
        *host_out = out;
    }
    c->st.phase_ms[3] = ms_since(&t0);
    *ret = FLBGPU_FILTER_MODIFIED;
    return 0;
}

int flbgpu_chain_do_device(flbgpu_chain *c, const void *d_data, size_t bytes, void *d_out, size_t out_cap, size_t *out_size)
{
    int r;
    if (!c || !c->inited) return -1;
    g_rt_err[0] = 0;
    pthread_mutex_lock(&c->lock);
    c->ctx->last_q = c->q;
    {   /* no tag here: every filter that is not switched off */
        int k;
        c->active = 0;
        for (k = 0; k < c->nf; k++) if (!c->f[k]->inactive) c->active |= 1u << k;
    }
    if (c->ml_post) r = ml_then_rest(c, NULL, d_data, bytes, d_out, out_cap, NULL, out_size);
    else if (c->ml_index >= 0 && c->nf > 1) { set_err("a multiline filter inside a longer chain runs filter by filter: host buffers only%s%s", NULL, NULL); r = -1; }
    else if (c->ml_index >= 0) r = ml_run(c, NULL, d_data, bytes, d_out, out_cap, NULL, out_size);
    else r = chain_run(c, NULL, d_data, bytes, d_out, out_cap, NULL, out_size);
    if (r >= 0 && bk_sync(c->q)) r = -1;
    pthread_mutex_unlock(&c->lock);
    return r;
}

/* flb_filter_do() as the reference runs it (src/flb_filter.c:119-323): one filter after the other on the device, each
 * on the chunk the previous one returned.  The fused form hands fields from filter to filter by reference and cannot
 * parse a value an earlier filter of the same chain made (a decoded JSON string, a `Set` constant); it refuses with
 * FLBGPU_E_FIELDS and the chain is run this way instead -- same result, one round trip per filter. */
static int chain_do_one_by_one(flbgpu_chain *c, const void *data, size_t bytes, const char *tag, int tag_len, void **out_buf, size_t *out_size)
{
    const void *cur = data;
    size_t cur_n = bytes;
    void *owned = NULL;
    int k;
    for (k = 0; k < c->nf; k++) {
        void *o = NULL;
        size_t on = 0;
        int r = flbgpu_filter_cb(c->f[k], cur, cur_n, tag, tag_len, &o, &on);
        if (r < 0) { free(owned); return -1; }
        if (r != FLBGPU_FILTER_MODIFIED) { free(o); continue; }
        free(owned);
        owned = o;
        if (on == 0) { free(owned); *out_buf = NULL; *out_size = 0; return FLBGPU_FILTER_MODIFIED; }   /* nothing left: the chain ends */
        cur = o; cur_n = on;
    }
    if (!owned) return FLBGPU_FILTER_NOTOUCH;
    *out_buf = owned; *out_size = cur_n;
    return FLBGPU_FILTER_MODIFIED;
}
/* A fused call failed.  When all it refused were values an earlier filter of the chain made (FLBGPU_E_FIELDS, FLBGPU_E_DEEP),
 * the filter-by-filter form redoes the call from an empty result; any other failure stands. */
static int one_by_one_if_refused(flbgpu_chain *c, const void *data, size_t bytes, const char *tag, int tag_len, void **out_buf, size_t *out_size)
{
    if (!(c->nf > 1 && c->st.error_bits && !(c->st.error_bits & ~(FLBGPU_E_FIELDS | FLBGPU_E_DEEP)))) return -1;
    *out_buf = NULL; *out_size = 0;
    return chain_do_one_by_one(c, data, bytes, tag, tag_len, out_buf, out_size);
}

static int chain_do_locked(flbgpu_chain *c, const void *data, size_t bytes, const char *tag, int tag_len, void **out_buf, size_t *out_size)
{
    const char *sv;
    int r;
    if (c->rtag_index == -2) return chain_do_one_by_one(c, data, bytes, tag, tag_len, out_buf, out_size);     /* one re-tagged stream per chain */
    if (c->ml_index >= 0) {
        /* a multiline filter makes new records out of runs of records: it runs on its own, the filters around it on what it made */
        if (c->ml_post) {
            r = ml_then_rest(c, data, NULL, bytes, NULL, 0, out_buf, out_size);
            return r < 0 ? one_by_one_if_refused(c, data, bytes, tag, tag_len, out_buf, out_size) : r;
        }
        if (c->nf > 1) return chain_do_one_by_one(c, data, bytes, tag, tag_len, out_buf, out_size);
        r = ml_run(c, data, NULL, bytes, NULL, 0, out_buf, out_size);
        bk_upload_end(c->q);
        return r;
    }
    if (c->rtag_index >= 0) {                        /* the templates of a rewrite_tag filter may name the tag of the call */
        c->tag_len = (uint32_t) (tag && tag_len > 0 ? tag_len : 0);
        if (bk_tag_upload(c->q, tag, c->tag_len, &c->d_tag)) { set_err("%s%s", bk_last_error(), NULL); return -1; }
    }
    sv = getenv("FLBGPU_STREAM");
    if (!(sv && sv[0] == '0')) {                     /* FLBGPU_STREAM=0: the two-pass form only */
        int ret = 0;
        r = bytes <= small_bytes() ? chain_run_small(c, data, bytes, out_buf, out_size, &ret) : chain_run_stream(c, data, bytes, out_buf, out_size, &ret);
        bk_upload_end(c->q);                         /* `data` is not read after this call returns */
        if (r == 0) return ret;
        if (r < 0) return one_by_one_if_refused(c, data, bytes, tag, tag_len, out_buf, out_size);
        *out_buf = NULL; *out_size = 0;              /* not for this form, or its speculation did not hold: the two-pass form */
    }
    r = chain_run(c, data, NULL, bytes, NULL, 0, out_buf, out_size);
    bk_upload_end(c->q);
    return r < 0 ? one_by_one_if_refused(c, data, bytes, tag, tag_len, out_buf, out_size) : r;
}

int flbgpu_chain_do(flbgpu_chain *c, const void *data, size_t bytes, const char *tag, int tag_len,
                    void **out_buf, size_t *out_size)
{
    int r;
    if (!c || !c->inited || !out_buf || !out_size) return -1;
    g_rt_err[0] = 0;
    *out_buf = NULL; *out_size = 0;
    if (bytes == 0) return FLBGPU_FILTER_NOTOUCH;
    pthread_mutex_lock(&c->lock);
    c->ctx->last_q = c->q;
    c->active = chain_active_mask(c, tag, tag_len);
    if (c->active == 0) r = FLBGPU_FILTER_NOTOUCH;    /* no filter of the chain is routed this tag */
    else r = chain_do_locked(c, data, bytes, tag, tag_len, out_buf, out_size);
    pthread_mutex_unlock(&c->lock);
    return r;
}


#include "runtime_pool.h"

/* ---- rewrite_tag: what the last call re-tagged ---------------------------------- */
int flbgpu_filter_emitted(flbgpu_filter *f, const struct flbgpu_emit_group **groups, size_t *n_groups)
{
    if (!f || f->kind != FLBGPU_F_REWRITE_TAG || !groups || !n_groups) return -1;
    *groups = f->rt_groups; *n_groups = f->rt_n;
    return 0;
}

/* ---- log_to_metrics state ------------------------------------------------------ */
int flbgpu_l2m_info(flbgpu_filter *f, int *mode, int *n_labels, int *n_buckets, int *n_sets)
{
    if (!f || !f->l2m) return -1;
    *mode = f->l2m->mode; *n_labels = f->l2m->n_labels; *n_buckets = f->l2m->n_buckets; *n_sets = f->l2m->n_sets;
    return 0;
}

int flbgpu_l2m_get(flbgpu_filter *f, int i, uint64_t *hash, uint64_t *count, double *sum, uint64_t *buckets, char *labels)
{
    struct l2m_state *st = f ? f->l2m : NULL;
    if (!st || i < 0 || i >= st->n_sets) return -1;
    *hash = st->sets[i].hash; *count = st->sets[i].count; *sum = st->sets[i].sum;
    if (buckets) memcpy(buckets, st->sets[i].buckets, sizeof(uint64_t) * (st->n_buckets + 1));
    if (labels) memcpy(labels, st->sets[i].labels, (size_t) (st->n_labels ? st->n_labels : 1) * L2M_LABEL_BYTES);
    return 0;
}

int flbgpu_l2m_reset(flbgpu_filter *f)
{
    struct l2m_state *st = f ? f->l2m : NULL;
    int i;
    if (!st) return -1;
    for (i = 0; i < st->n_sets; i++) { free(st->sets[i].labels); free(st->sets[i].buckets); }
    st->n_sets = 0;
    return 0;
}

int flbgpu_l2m_put(flbgpu_filter *f, uint64_t hash, uint64_t count, double sum, const uint64_t *buckets, const char *labels)
{
    struct l2m_state *st = f ? f->l2m : NULL;
    struct l2m_set *set;
    size_t lb;
    if (!st) return -1;
    lb = (size_t) (st->n_labels ? st->n_labels : 1) * L2M_LABEL_BYTES;
    if (st->n_sets == st->cap_sets) {
        struct l2m_set *ns_ = realloc(st->sets, sizeof(*st->sets) * (size_t) (st->cap_sets ? st->cap_sets * 2 : 64));
        if (!ns_) return -1;
        st->sets = ns_;
        st->cap_sets = st->cap_sets ? st->cap_sets * 2 : 64;
    }
    set = &st->sets[st->n_sets++];
    memset(set, 0, sizeof(*set));
    set->hash = hash; set->count = count; set->sum = sum; set->bound = l2m_sum_bound(sum);
    set->labels = malloc(lb); memcpy(set->labels, labels, lb);
    set->buckets = calloc(st->n_buckets + 1, sizeof(uint64_t));
    if (buckets) memcpy(set->buckets, buckets, sizeof(uint64_t) * (st->n_buckets + 1));
    return 0;
}

/* Text of the metric in the format of cmt_encode_text_create() (lib/cmetrics/src/cmt_encode_text.c:
 * 273-336, 468-600) without the leading timestamp, label sets in first-seen order; malloc()ed */
char *flbgpu_l2m_text(flbgpu_filter *f)
{
    struct l2m_state *st = f ? f->l2m : NULL;
    size_t cap = 4096, len = 0;
    char *out;
    int i, j, k;
    if (!st) return NULL;
    out = malloc(cap);
    out[0] = 0;
#define L2M_APPEND(...) do { for (;;) { int w_ = snprintf(out + len, cap - len, __VA_ARGS__); \
        if ((size_t) w_ < cap - len) { len += (size_t) w_; break; } cap *= 2; out = realloc(out, cap); } } while (0)
    /* a metric without label keys is cmetrics' static metric: it exists, at 0, before anything was counted
     * (cmt_map.c: metric_static; a histogram in that state has no buckets yet and is not printable) */
    /* cmt_opts_init(): the fully qualified name joins namespace, subsystem and name, leaving out what is empty */
#define L2M_FQNAME() do { if (*st->ns) L2M_APPEND("%s_", st->ns); if (*st->subsystem) L2M_APPEND("%s_", st->subsystem); L2M_APPEND("%s", st->name); } while (0)
    if (st->n_sets == 0 && st->n_labels == 0 && st->mode != L2M_HISTOGRAM) { L2M_FQNAME(); L2M_APPEND(" = 0\n"); }
    for (i = 0; i < st->n_sets; i++) {
        struct l2m_set *s = &st->sets[i];
        L2M_FQNAME();
        for (j = 0; j < st->n_labels; j++) {
            const unsigned char *v = (const unsigned char *) s->labels + (size_t) j * L2M_LABEL_BYTES;
            L2M_APPEND("%s%s=\"%.*s\"", j ? "," : "{", st->label_keys[j], (int) v[0], (const char *) v + 1);
        }
        if (st->n_labels) L2M_APPEND("}");
        if (st->mode == L2M_COUNTER) L2M_APPEND(" = %.17g\n", (double) s->count);
        else if (st->mode == L2M_GAUGE) L2M_APPEND(" = %.17g\n", s->sum);
        else {
            L2M_APPEND(" = { buckets = { ");
            for (k = 0; k < st->n_buckets; k++) L2M_APPEND("%g=%llu, ", st->bounds[k], (unsigned long long) s->buckets[k]);
            L2M_APPEND("+Inf=%llu }, sum=%g, count=%llu }\n", (unsigned long long) s->buckets[st->n_buckets], s->sum,
                       (unsigned long long) s->count);
        }
    }
    return out;
}

int flbgpu_filter_cb(flbgpu_filter *f, const void *data, size_t bytes, const char *tag, int tag_len,
                     void **out_buf, size_t *out_size)
{
    if (!f || !f->inited) return -1;
    if (!f->solo) {
        flbgpu_chain *c = flbgpu_chain_new(f->ctx);
        if (flbgpu_chain_add(c, f) || flbgpu_chain_init(c)) { flbgpu_chain_destroy(c); return -1; }
        f->solo = c;
    }
    return flbgpu_chain_do(f->solo, data, bytes, tag, tag_len, out_buf, out_size);
}

/* end of the msgpack object at p (host side, for unwrapping results), or NULL */
static const uint8_t *host_mp_skip(const uint8_t *p, const uint8_t *end, int depth)
{
    uint32_t n = 0, c, i;
    int is_map = 0;
    if (p >= end || depth > 64) return NULL;
    c = *p;
    if (c <= 0x7f || c >= 0xe0 || c == 0xc0 || c == 0xc2 || c == 0xc3) return p + 1;
    if (c >= 0xa0 && c <= 0xbf) return (size_t) (end - p) >= 1 + (c & 31) ? p + 1 + (c & 31) : NULL;
    if (c >= 0x90 && c <= 0x9f) { n = c & 15; p += 1; goto cont; }
    if (c >= 0x80 && c <= 0x8f) { n = c & 15; is_map = 1; p += 1; goto cont; }
#define HM_NEED(k) do { if ((size_t) (end - p) < (size_t) (k)) return NULL; } while (0)
#define HM_BE16(q) (((uint32_t) (q)[0] << 8) | (q)[1])
#define HM_BE32(q) (((uint32_t) (q)[0] << 24) | ((uint32_t) (q)[1] << 16) | ((uint32_t) (q)[2] << 8) | (q)[3])
    switch (c) {
    case 0xcc: case 0xd0: HM_NEED(2); return p + 2;
    case 0xcd: case 0xd1: HM_NEED(3); return p + 3;
    case 0xce: case 0xd2: case 0xca: HM_NEED(5); return p + 5;
    case 0xcf: case 0xd3: case 0xcb: HM_NEED(9); return p + 9;
    case 0xd9: case 0xc4: HM_NEED(2); n = p[1]; HM_NEED(2 + n); return p + 2 + n;
    case 0xda: case 0xc5: HM_NEED(3); n = HM_BE16(p + 1); HM_NEED(3 + (size_t) n); return p + 3 + n;
    case 0xdb: case 0xc6: HM_NEED(5); n = HM_BE32(p + 1); HM_NEED(5 + (size_t) n); return p + 5 + n;
    case 0xd4: HM_NEED(3); return p + 3;
    case 0xd5: HM_NEED(4); return p + 4;
    case 0xd6: HM_NEED(6); return p + 6;
    case 0xd7: HM_NEED(10); return p + 10;
    case 0xd8: HM_NEED(18); return p + 18;
    case 0xc7: HM_NEED(3); n = p[1]; HM_NEED(3 + (size_t) n); return p + 3 + n;
    case 0xc8: HM_NEED(4); n = HM_BE16(p + 1); HM_NEED(4 + (size_t) n); return p + 4 + n;
    case 0xc9: HM_NEED(6); n = HM_BE32(p + 1); HM_NEED(6 + (size_t) n); return p + 6 + n;
    case 0xdc: HM_NEED(3); n = HM_BE16(p + 1); p += 3; break;
    case 0xdd: HM_NEED(5); n = HM_BE32(p + 1); p += 5; break;
    case 0xde: HM_NEED(3); n = HM_BE16(p + 1); p += 3; is_map = 1; break;
    case 0xdf: HM_NEED(5); n = HM_BE32(p + 1); p += 5; is_map = 1; break;
    default: return NULL;
    }
cont:
    for (i = 0; i < n * (is_map ? 2u : 1u); i++) {
        p = host_mp_skip(p, end, depth + 1);
        if (!p) return NULL;
    }
    return p;
}

static int parser_solo(flbgpu_parser *p)
{
    if (!p->solo) {
        flbgpu_filter *f = flbgpu_filter_new(p->ctx, "parser");
        flbgpu_chain *c;
        if (!f) return -1;
        flbgpu_filter_set_property(f, "key_name", "_");
        flbgpu_filter_set_property(f, "parser", p->name);
        if (flbgpu_filter_init(f)) { flbgpu_filter_destroy(f); return -1; }
        c = flbgpu_chain_new(p->ctx);
        if (!c) { flbgpu_filter_destroy(f); return -1; }
        c->want_report = 1;
        if (flbgpu_chain_add(c, f) || flbgpu_chain_init(c)) { flbgpu_chain_destroy(c); flbgpu_filter_destroy(f); return -1; }
        p->solo = c; p->solo_filter = f;
    }
    return 0;
}

static size_t put_line_event(uint8_t *rec, const char *buf, size_t length)
{
    size_t n = 0, i;
    rec[n++] = 0x92; rec[n++] = 0x92; rec[n++] = 0xd7; rec[n++] = 0x00;
    for (i = 0; i < 8; i++) rec[n++] = 0;
    rec[n++] = 0x80; rec[n++] = 0x81; rec[n++] = 0xa1; rec[n++] = '_';
    if (length < 32) rec[n++] = 0xa0 | (uint8_t) length;
    else if (length < 256) { rec[n++] = 0xd9; rec[n++] = (uint8_t) length; }
    else if (length < 65536) { rec[n++] = 0xda; rec[n++] = (uint8_t) (length >> 8); rec[n++] = (uint8_t) length; }
    else { rec[n++] = 0xdb; rec[n++] = (uint8_t) (length >> 24); rec[n++] = (uint8_t) (length >> 16); rec[n++] = (uint8_t) (length >> 8); rec[n++] = (uint8_t) length; }
    memcpy(rec + n, buf, length);
    return n + length;
}

/* the parser's own report of the call just made on its solo chain: 6 ints per line (dev_chain.cuh: ch_env.prep) */
static const int32_t *parser_report(flbgpu_chain *c, uint32_t n)
{
    if (c->st.records_in != n) { set_err("parser call: the lines did not come back one to one%s%s", NULL, NULL); return NULL; }
    if (host_grow((void **) &c->h_prep, &c->cap_hprep, (size_t) n * 6, sizeof(int32_t))) return NULL;
    if (bk_d2h(c->q, c->h_prep, c->d_prep, (size_t) n * 6 * sizeof(int32_t)) || bk_sync(c->q)) return NULL;
    return c->h_prep;
}

/* flb_parser_do() over n lines in ONE device pass (the entry a batched caller such as a GPU
 * filter_parser or an input plugin uses): line i = base[off[i] .. off[i]+len[i]).  Results: the
 * msgpack maps of the parsed lines back to back in *out_buf (malloc), map i at
 * [out_off[i], out_off[i+1]) (empty when ret[i] < 0), its time in out_time[i], ret[i] as
 * flb_parser_do would return it: the position the parser consumed the line up to (end of the last named capture,
 * src/flb_regex.c:50-54; end of the JSON document plus the white space behind it, src/flb_pack.c:427-499; where the
 * LTSV / logfmt scan stopped), or -1. */
int flbgpu_parser_do_batch(flbgpu_parser *p, const char *base, const uint32_t *off, const uint32_t *len, uint32_t n,
                           void **out_buf, size_t *out_size, uint64_t *out_off, struct flbgpu_time *out_time, int *ret)
{
    uint8_t *chunk, *o = NULL, *maps;
    const uint8_t *q, *end;
    const int32_t *rep;
    size_t total = 0, at = 0, osz = 0, mo = 0;
    uint32_t i;
    int r;
    if (!p || !base || !off || !len || !out_buf || !out_size || !out_off || !ret) return -1;
    *out_buf = NULL; *out_size = 0;
    if (parser_solo(p)) return -1;
    if (n == 0) { out_off[0] = 0; return 0; }
    for (i = 0; i < n; i++) total += (size_t) len[i] + 22;
    chunk = malloc(total + 1);
    if (!chunk) { set_err("out of memory%s%s", NULL, NULL); return -1; }
    for (i = 0; i < n; i++) at += put_line_event(chunk + at, base + off[i], len[i]);
    pthread_mutex_lock(&p->solo->lock);              /* the report belongs to this call: keep the instance until it is read */
    p->ctx->last_q = p->solo->q;
    p->solo->active = 1;
    r = chain_do_locked(p->solo, chunk, at, "", 0, (void **) &o, &osz);
    rep = r == FLBGPU_FILTER_MODIFIED ? parser_report(p->solo, n) : NULL;
    if (!rep) { pthread_mutex_unlock(&p->solo->lock); free(chunk); free(o); return -1; }
    maps = malloc(osz ? osz : 1);
    if (!maps) { pthread_mutex_unlock(&p->solo->lock); free(chunk); free(o); set_err("out of memory%s%s", NULL, NULL); return -1; }
    q = o; end = o + osz;
    for (i = 0; i < n; i++) {
        /* filter_parser emits exactly one record per input record, in order */
        const uint8_t *body, *nx;
        const int32_t *ri = rep + (size_t) 6 * i;
        out_off[i] = mo;
        if ((size_t) (end - q) < 13 || !(nx = host_mp_skip(q + 13, end, 0))) {
            pthread_mutex_unlock(&p->solo->lock);
            free(chunk); free(o); free(maps); set_err("malformed parser result%s%s", NULL, NULL); return -1;
        }
        body = q + 13;
        if (!ri[0]) {                                    /* no parser took the line */
            ret[i] = -1;
            if (out_time) { out_time[i].tv_sec = 0; out_time[i].tv_nsec = 0; }
        }
        else {
            ret[i] = ri[1];
            if (out_time) {
                out_time[i].tv_sec = (int64_t) (((uint64_t) (uint32_t) ri[3] << 32) | (uint32_t) ri[2]);
                out_time[i].tv_nsec = (int64_t) ri[4];
            }
            memcpy(maps + mo, body, (size_t) (nx - body));
            mo += (size_t) (nx - body);
        }
        q = nx;
    }
    pthread_mutex_unlock(&p->solo->lock);
    out_off[n] = mo;
    free(chunk); free(o);
    *out_buf = maps; *out_size = mo;
    return 0;
}

/* flb_parser_do() for one line: wrap it as one event {"_": line}, run filter_parser
 * with Key_Name "_" and unwrap the body map. */
int flbgpu_parser_do(flbgpu_parser *p, const char *buf, size_t length, void **out_buf, size_t *out_size,
                     struct flbgpu_time *out_time)
{
    uint32_t off = 0, len = (uint32_t) length;
    uint64_t ooff[2];
    struct flbgpu_time t;
    int ret = -1;
    if (!p || !buf || !out_buf || !out_size || length >= 0x7fffffffu) return -1;
    *out_buf = NULL; *out_size = 0;
    if (out_time) { out_time->tv_sec = 0; out_time->tv_nsec = 0; }
    if (flbgpu_parser_do_batch(p, buf, &off, &len, 1, out_buf, out_size, ooff, &t, &ret) != 0) return -1;
    if (ret < 0) { free(*out_buf); *out_buf = NULL; *out_size = 0; return -1; }
    if (out_time) *out_time = t;
    return ret;
}

/* ---- flb_pack_json_state(): the streaming JSON packer of the inputs (src/flb_pack.c:758-829) -----------------
 * One device lane per stream buffer (dev_jsmn.cuh); a single call is a batch of one. */
int flbgpu_pack_state_init(struct flbgpu_pack_state *s)
{
    if (!s) return -1;
    memset(s, 0, sizeof(*s));
    return 0;
}
void flbgpu_pack_state_reset(struct flbgpu_pack_state *s) { if (s) memset(s, 0, sizeof(*s)); }

int flbgpu_pack_json_state_batch(flbgpu_ctx *ctx, int n, const char *const *js, const size_t *len,
                                 char **buffers, int *sizes, struct flbgpu_pack_state *states, int *rets)
{
    bk_q *q;
    struct bk_jsmn_args a;
    uint32_t *h_off = NULL, *h_len = NULL, *h_tok_off = NULL, *h_tok_cap = NULL, *h_out_off = NULL;
    struct jm_result *h_res = NULL;
    uint8_t *h_js = NULL, *h_out = NULL, *d_js = NULL, *d_tmp = NULL, *d_out = NULL;
    uint32_t *d_meta = NULL;
    struct jm_tok *d_tok = NULL;
    struct jm_result *d_res = NULL;
    size_t total = 0, tok_total = 0, out_total = 0;
    int i, rc = -1, pass;

    if (!ctx || n < 0 || (n && (!js || !len || !buffers || !sizes || !states || !rets))) return -1;
    g_rt_err[0] = 0;
    if (n == 0) return 0;
    q = ctx->q0;
    for (i = 0; i < n; i++) {
        buffers[i] = NULL; sizes[i] = 0; rets[i] = -1;
        if (len[i] >= 0x7fffffffu) { set_err("stream buffer larger than 2 GiB%s%s", NULL, NULL); return -1; }
        total += (len[i] + 15) & ~(size_t) 15;
    }
    if (total >= 0xfff00000ull) { set_err("batch larger than 4 GiB: split it%s%s", NULL, NULL); return -1; }
    h_off = malloc(sizeof(uint32_t) * 5 * (size_t) n);
    h_res = malloc(sizeof(*h_res) * (size_t) n);
    h_js = malloc(total + 16);
    if (!h_off || !h_res || !h_js) { set_err("out of memory%s%s", NULL, NULL); goto done; }
    h_len = h_off + n; h_tok_off = h_len + n; h_tok_cap = h_tok_off + n; h_out_off = h_tok_cap + n;
    {
        size_t at = 0;
        for (i = 0; i < n; i++) {
            h_off[i] = (uint32_t) at; h_len[i] = (uint32_t) len[i];
            if (len[i]) memcpy(h_js + at, js[i], len[i]);
            at += (len[i] + 15) & ~(size_t) 15;
            /* a token takes at least one byte of text; most documents need far fewer: start at half, retry at the bound */
            h_tok_cap[i] = (uint32_t) (len[i] / 2 + 64);
        }
    }
    d_js = bk_alloc(q, total + 64);
    d_tmp = bk_alloc(q, total + (size_t) n + 64);
    d_meta = bk_alloc(q, sizeof(uint32_t) * 5 * (size_t) n);
    d_res = bk_alloc(q, sizeof(*d_res) * (size_t) n);
    if (!d_js || !d_tmp || !d_meta || !d_res) goto done;
    if (bk_h2d(q, d_js, h_js, total)) goto done;
    for (pass = 0; pass < 2; pass++) {
        int again = 0;
        tok_total = 0;
        for (i = 0; i < n; i++) { h_tok_off[i] = (uint32_t) tok_total; tok_total += h_tok_cap[i]; }
        if (tok_total >= 0x7fffffffu / sizeof(struct jm_tok) * 4) { set_err("token scratch too large: split the batch%s%s", NULL, NULL); goto done; }
        bk_free(q, d_tok);
        d_tok = bk_alloc(q, sizeof(struct jm_tok) * tok_total);
        if (!d_tok) goto done;
        if (bk_h2d(q, d_meta, h_off, sizeof(uint32_t) * 5 * (size_t) n)) goto done;
        memset(&a, 0, sizeof(a));
        a.d_js = d_js; a.d_off = d_meta; a.d_len = d_meta + n; a.n = (uint32_t) n;
        a.d_tok = d_tok; a.d_tok_off = d_meta + 2 * (size_t) n; a.d_tok_cap = d_meta + 3 * (size_t) n;
        a.d_tmp = d_tmp; a.d_res = d_res; a.d_out_off = d_meta + 4 * (size_t) n;
        if (bk_jsmn_scan(q, &a) || bk_d2h(q, h_res, d_res, sizeof(*h_res) * (size_t) n) || bk_sync(q)) goto done;
        for (i = 0; i < n; i++) if (h_res[i].status == JM_NOMEM) { h_tok_cap[i] = (uint32_t) len[i] + 1; again = 1; }
        if (!again) break;
    }
    for (i = 0; i < n; i++) {
        if (h_res[i].status == JM_NOMEM) { set_err("token scratch exhausted%s%s", NULL, NULL); goto done; }
        if (h_res[i].status == JM_REFUSED) {
            set_err("a number text needs a strtod() form that is not restated on the device (hex float, nan(payload))%s%s", NULL, NULL);
            goto done;
        }
        h_out_off[i] = (uint32_t) out_total;
        if (h_res[i].status == JM_OK) out_total += h_res[i].out_size;
    }
    if (out_total) {
        d_out = bk_alloc(q, out_total + 64);
        h_out = malloc(out_total);
        if (!d_out || !h_out) { set_err("out of memory%s%s", NULL, NULL); goto done; }
        if (bk_h2d(q, d_meta + 4 * (size_t) n, h_out_off, sizeof(uint32_t) * (size_t) n)) goto done;
        a.d_out = d_out;
        if (bk_jsmn_emit(q, &a) || bk_d2h(q, h_out, d_out, out_total) || bk_sync(q)) goto done;
    }
    for (i = 0; i < n; i++) {
        const struct jm_result *r = &h_res[i];
        states[i].multiple = 1;                          /* flb_pack_json_state() sets it (src/flb_pack.c:773) */
        rets[i] = r->status;
        if (r->status == JM_OK) {
            states[i].tokens_count = r->tokens_count;
            states[i].last_byte = r->last_byte;
            sizes[i] = (int) r->out_size;
            buffers[i] = malloc(r->out_size ? r->out_size : 1);
            if (!buffers[i]) { set_err("out of memory%s%s", NULL, NULL); goto done; }
            if (r->out_size) memcpy(buffers[i], h_out + h_out_off[i], r->out_size);
        }
        else if (r->status == JM_INVAL && r->tret == JM_OK) states[i].last_byte = 0;      /* "tokens_count == 0": last_byte = last (0) */
        else if (r->status == JM_FAIL) states[i].tokens_count = r->tokens_count;
    }
    rc = 0;
done:
    if (rc != 0) for (i = 0; i < n; i++) { free(buffers[i]); buffers[i] = NULL; }
    bk_free(q, d_js); bk_free(q, d_tmp); bk_free(q, d_meta); bk_free(q, d_res); bk_free(q, d_tok); bk_free(q, d_out);
    free(h_off); free(h_res); free(h_js); free(h_out);
    return rc;
}

int flbgpu_pack_json_state(flbgpu_ctx *ctx, const char *js, size_t len, char **buffer, int *size, struct flbgpu_pack_state *state)
{
    int ret = -1;
    if (!ctx || !js || !buffer || !size || !state) return -1;
    if (flbgpu_pack_json_state_batch(ctx, 1, &js, &len, buffer, size, state, &ret) != 0) return -1;
    return ret;
}

/* ---- the exchange step of the path: filter_log_to_metrics tables of N shards -> one table (SURVEY 8e) ------------
 * Every rank holds the table of its record range.  The merged table is what the reference's single cmetrics context
 * would hold for the whole chunk: label sets in first-seen order -- rank-major, since the ranges are consecutive --
 * counts and cumulative buckets summed (uint64, exact), histogram sums added in double (exact for integer-valued
 * observations; the order of a floating-point reduction is not the record order), gauges last-writer-wins = the
 * value of the highest rank that saw the set.  Three collectives over NVLink: an all-gather of the per-rank set
 * counts, an all-gather of the label keys, ONE all-reduce of the value matrix (two for histograms: uint64 + double). */
int flbgpu_comm_unique_id(uint8_t id[128]) { g_rt_err[0] = 0; return id ? bk_comm_unique_id(id) : -1; }

int flbgpu_comm_init(flbgpu_ctx *ctx, int nranks, int rank, const uint8_t id[128])
{
    g_rt_err[0] = 0;
    if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return -1;
    return bk_comm_init(ctx->q0, nranks, rank, id);
}

int flbgpu_l2m_allreduce(flbgpu_filter *f)
{
    struct l2m_state *st = f ? f->l2m : NULL;
    bk_q *q;
    int nranks = 0, rank = 0, r, i, rc = -1;
    size_t lb, K, maxn = 0, nu = 0, cols, j;
    uint64_t *h_cnt = NULL, *h_mat = NULL, *d_cnt = NULL, *d_mat = NULL;
    uint8_t *h_keys = NULL, *h_all = NULL, *d_keys = NULL, *d_all = NULL;
    double *h_sum = NULL, *d_sum = NULL;
    struct l2m_set *merged = NULL;
    size_t *map = NULL;                                   /* local set -> row of the union */

    if (!st) { set_err("not a log_to_metrics filter%s%s", NULL, NULL); return -1; }
    g_rt_err[0] = 0;
    q = f->ctx->q0;
    if (bk_comm_info(q, &nranks, &rank) != 0) { set_err("no communicator: call flbgpu_comm_init first%s%s", NULL, NULL); return -1; }
    lb = (size_t) (st->n_labels ? st->n_labels : 1) * L2M_LABEL_BYTES;
    K = 8 + lb;
    /* 1: how many label sets every rank holds */
    h_cnt = calloc((size_t) nranks + 1, 8);
    d_cnt = bk_alloc(q, ((size_t) nranks + 1) * 8);
    if (!h_cnt || !d_cnt) goto done;
    h_cnt[nranks] = (uint64_t) st->n_sets;
    if (bk_h2d(q, d_cnt + nranks, h_cnt + nranks, 8) || bk_sync(q) || bk_comm_allgather(q, d_cnt + nranks, d_cnt, 8) ||
        bk_d2h(q, h_cnt, d_cnt, (size_t) nranks * 8) || bk_sync(q)) goto done;
    for (r = 0; r < nranks; r++) if (h_cnt[r] > maxn) maxn = (size_t) h_cnt[r];
    if (maxn == 0) { rc = 0; goto done; }
    /* 2: the label keys of every rank, in its first-seen order */
    h_keys = calloc(maxn, K);
    h_all = malloc((size_t) nranks * maxn * K);
    d_keys = bk_alloc(q, maxn * K);
    d_all = bk_alloc(q, (size_t) nranks * maxn * K);
    if (!h_keys || !h_all || !d_keys || !d_all) goto done;
    for (i = 0; i < st->n_sets; i++) { memcpy(h_keys + (size_t) i * K, &st->sets[i].hash, 8); memcpy(h_keys + (size_t) i * K + 8, st->sets[i].labels, lb); }
    if (bk_h2d(q, d_keys, h_keys, maxn * K) || bk_sync(q) || bk_comm_allgather(q, d_keys, d_all, maxn * K) ||
        bk_d2h(q, h_all, d_all, (size_t) nranks * maxn * K) || bk_sync(q)) goto done;
    /* 3: the union, rank-major */
    merged = calloc((size_t) nranks * maxn, sizeof(*merged));
    map = calloc((size_t) st->n_sets + 1, sizeof(*map));
    if (!merged || !map) goto done;
    for (r = 0; r < nranks; r++) {
        for (j = 0; j < (size_t) h_cnt[r]; j++) {
            const uint8_t *k = h_all + ((size_t) r * maxn + j) * K;
            uint64_t h;
            size_t u;
            memcpy(&h, k, 8);
            for (u = 0; u < nu; u++) if (merged[u].hash == h) break;
            if (u == nu) {
                merged[nu].hash = h;
                merged[nu].labels = malloc(lb);
                merged[nu].buckets = calloc((size_t) st->n_buckets + 1, sizeof(uint64_t));
                if (!merged[nu].labels || !merged[nu].buckets) goto done;
                memcpy(merged[nu].labels, k + 8, lb);
                nu++;
            }
            if (r == rank) map[j] = u;
        }
    }
    /* 4: the values */
    cols = st->mode == L2M_GAUGE ? 1 + 2 * (size_t) nranks : 1 + (size_t) st->n_buckets + 1;
    h_mat = calloc(nu * cols, 8);
    d_mat = bk_alloc(q, nu * cols * 8);
    if (!h_mat || !d_mat) goto done;
    for (i = 0; i < st->n_sets; i++) {
        uint64_t *row = h_mat + map[i] * cols;
        row[0] = st->sets[i].count;
        if (st->mode == L2M_GAUGE) { row[1 + 2 * (size_t) rank] = 1; memcpy(&row[2 + 2 * (size_t) rank], &st->sets[i].sum, 8); }
        else memcpy(row + 1, st->sets[i].buckets, ((size_t) st->n_buckets + 1) * 8);
    }
    if (bk_h2d(q, d_mat, h_mat, nu * cols * 8) || bk_sync(q) || bk_comm_allreduce_u64(q, d_mat, nu * cols) ||
        bk_d2h(q, h_mat, d_mat, nu * cols * 8) || bk_sync(q)) goto done;
    if (st->mode != L2M_GAUGE) {
        h_sum = calloc(nu, 8);
        d_sum = bk_alloc(q, nu * 8);
        if (!h_sum || !d_sum) goto done;
        for (i = 0; i < st->n_sets; i++) h_sum[map[i]] = st->sets[i].sum;
        if (bk_h2d(q, d_sum, h_sum, nu * 8) || bk_sync(q) || bk_comm_allreduce_f64(q, d_sum, nu) ||
            bk_d2h(q, h_sum, d_sum, nu * 8) || bk_sync(q)) goto done;
    }
    /* 5: this rank's table becomes the merged one */
    for (j = 0; j < nu; j++) {
        const uint64_t *row = h_mat + j * cols;
        merged[j].count = row[0];
        if (st->mode == L2M_GAUGE) {
            for (r = nranks - 1; r >= 0; r--) if (row[1 + 2 * (size_t) r]) { memcpy(&merged[j].sum, &row[2 + 2 * (size_t) r], 8); break; }
        }
        else {
            memcpy(merged[j].buckets, row + 1, ((size_t) st->n_buckets + 1) * 8);
            merged[j].sum = h_sum[j];
            merged[j].bound = l2m_sum_bound(merged[j].sum);
        }
    }
    for (i = 0; i < st->n_sets; i++) { free(st->sets[i].labels); free(st->sets[i].buckets); }
    free(st->sets);
    st->sets = merged; st->n_sets = (int) nu; st->cap_sets = (int) ((size_t) nranks * maxn);
    merged = NULL;
    rc = 0;
done:
    if (merged) { for (j = 0; j < nu + 1 && j < (size_t) nranks * maxn; j++) { free(merged[j].labels); free(merged[j].buckets); } free(merged); }
    if (rc != 0 && !g_rt_err[0]) set_err("metric-table exchange failed: %s%s", bk_last_error(), NULL);
    bk_free(q, d_cnt); bk_free(q, d_mat); bk_free(q, d_keys); bk_free(q, d_all); bk_free(q, d_sum);
    free(h_cnt); free(h_mat); free(h_keys); free(h_all); free(h_sum); free(map);
    return rc;
}
