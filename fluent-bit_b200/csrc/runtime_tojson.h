/* runtime_tojson.h -- host side of the chunk -> JSON text conversion (part of runtime.c, included there).
 * flb_pack_msgpack_to_json_format(), src/flb_pack.c:1320-1602. */

#define TJ_MARKS_CAP 65536u      /* group markers per chunk */

static flbgpu_chain *tj_chain(flbgpu_ctx *ctx)
{
    flbgpu_chain *c = ctx->util;
    if (c) return c;
    c = flbgpu_chain_new(ctx);                         /* a queue and the growable buffers of a chain, no filters */
    if (!c) return NULL;
    c->d_flags = bk_alloc(c->q, sizeof(uint32_t) * (FLBGPU_MAX_FILTERS + 1));
    if (!c->d_flags) { flbgpu_chain_destroy(c); return NULL; }
    c->l2m_index = c->rtag_index = c->ml_index = -1;
    c->inited = 1;
    ctx->util = c;
    return c;
}

static int tj_run(flbgpu_chain *c, const uint8_t *h_in, size_t bytes, int json_format, int date_format, const char *date_key,
                  int escape_unicode, char **out, size_t *out_size, size_t *undefined_strings)
{
    struct tj_env e;
    const uint8_t *d_in;
    uint32_t n_rec, h_flags[FLBGPU_MAX_FILTERS + 1];
    size_t off, at, need;
    unsigned long long undef = 0, cnt[2] = { 0, 0 };
    uint32_t *d_groups = NULL;
    uint64_t total;
    char *res;
    int pass;

    if (call_start(c, bytes, out_size, NULL)) return -1;
    memset(&e, 0, sizeof(e));
    e.key_len = 0xffffffffu;
    if (date_key) {
        size_t kl = strlen(date_key);
        if (kl > sizeof(e.key)) { set_err("date key longer than %s bytes%s", "128", NULL); return -1; }
        memcpy(e.key, date_key, kl);
        e.key_len = (uint32_t) kl;
    }
    e.json_format = (uint32_t) json_format; e.date_format = (uint32_t) date_format; e.escape_unicode = escape_unicode ? 1u : 0u;
    if (bytes) {
        if (dev_grow(c, (void **) &c->d_in, &c->cap_in, bytes + 64, 1, 0)) return -1;
        if (bk_upload_start(c->q, c->d_in, h_in, bytes)) return -1;
    }
    d_in = c->d_in;
    if (bk_flags_clear(c->q, c->d_flags) || index_chunk(c, d_in, bytes, &n_rec, &off)) return -1;
    if (refuse_wide_arrays(c, h_in, d_in, off, bytes)) return -1;
    c->st.records_in = n_rec;
    total = 0;
    if (n_rec) {
        e.in = d_in; e.off = c->d_off; e.len = c->d_len; e.kind = c->d_kind; e.n_rec = n_rec;
        e.err = c->d_flags + FLBGPU_MAX_FILTERS;
        e.scr_pad = TJ_SCR_PAD(e.key_len == 0xffffffffu ? 0u : e.key_len);
        e.size = c->d_size;
        /* work memory: the counters (undefined strings, group markers), the marker lists, the packed lengths, the scratch slices */
        e.marks_cap = TJ_MARKS_CAP;
        need = 16 + 3 * sizeof(uint32_t) * (size_t) TJ_MARKS_CAP + sizeof(uint32_t) * (size_t) n_rec + 64;
        if (dev_grow(c, (void **) &c->d_mlw, &c->cap_mlw, need, 1, 0)) return -1;
        at = 0;
        e.undefined = (unsigned long long *) (c->d_mlw + at); e.n_marks = e.undefined + 1; at += 16;
        e.marks = (uint32_t *) (c->d_mlw + at); at += 2 * sizeof(uint32_t) * (size_t) TJ_MARKS_CAP;
        d_groups = (uint32_t *) (c->d_mlw + at); at += sizeof(uint32_t) * (size_t) TJ_MARKS_CAP;
        e.plen = (uint32_t *) (c->d_mlw + at);
        /* sized once, and once more when the chunk holds group markers: the events behind a start carry its body as
         * group_attributes */
        for (pass = 0; ; pass++) {
            if (dev_grow(c, (void **) &c->d_scr, &c->cap_scr, bytes + (size_t) n_rec * e.scr_pad + 64, 1, 0)) return -1;
            e.scr = c->d_scr;
            if (bk_zero(c->q, e.undefined, pass ? 8 : 16) || bk_tj_sizes(c->q, &e) || bk_flags_fetch(c->q, c->d_flags, h_flags)) return -1;
            if (h_flags[FLBGPU_MAX_FILTERS] & FLBGPU_E_JSONDATE) return 1;          /* the reference returns NULL for such a chunk */
            if (refused(c, h_flags[FLBGPU_MAX_FILTERS])) return -1;
            if (sizes_to_offsets(c, c->d_size, n_rec, NULL, NULL, "result larger than 4 GiB", &total)) return -1;
            if (bk_d2h(c->q, cnt, e.undefined, sizeof(cnt)) || bk_sync(c->q)) return -1;
            if (pass || !cnt[1]) break;
            {
                /* the markers' list in record order */
                uint32_t *h = malloc(2 * sizeof(uint32_t) * (size_t) cnt[1]), maxlen = 0;
                size_t a, b2;
                if (!h) return -1;
                if (bk_d2h(c->q, h, e.marks, 2 * sizeof(uint32_t) * (size_t) cnt[1]) || bk_sync(c->q)) { free(h); return -1; }
                for (a = 0; a < (size_t) cnt[1]; a++) { if (h[2 * a + 1] > maxlen) maxlen = h[2 * a + 1]; h[a] = h[2 * a]; }
                for (a = 1; a < (size_t) cnt[1]; a++) {      /* a handful: insertion sort */
                    const uint32_t v = h[a];
                    for (b2 = a; b2 > 0 && h[b2 - 1] > v; b2--) h[b2] = h[b2 - 1];
                    h[b2] = v;
                }
                if (bk_h2d(c->q, d_groups, h, sizeof(uint32_t) * (size_t) cnt[1]) || bk_sync(c->q)) { free(h); return -1; }
                free(h);
                e.groups = d_groups; e.n_groups = (uint32_t) cnt[1];
                e.scr_pad += maxlen + 32;                   /* an event's packed map now holds a marker's body too */
            }
        }
        undef = cnt[0];
    }
    bk_upload_end(c->q);
    c->st.kernel_launches = bk_launch_count();
    if (undefined_strings) *undefined_strings = (size_t) undef;
    /* json: "[" records joined by "," "]" -- also for no record at all; lines / stream: nothing converted -> NULL */
    if (json_format == (int) TJ_FORMAT_JSON) {
        res = malloc((size_t) total + 3);
        if (!res) return -1;
        if (total) {
            if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_tj_emit(c->q, &e, c->d_bsum, c->d_out) || bk_d2h(c->q, res, c->d_out, (size_t) total) || bk_sync(c->q)) { free(res); return -1; }
            res[0] = '[';
            res[total] = ']'; res[total + 1] = 0;
            *out_size = (size_t) total + 1;
        }
        else { res[0] = '['; res[1] = ']'; res[2] = 0; *out_size = 2; }
        *out = res;
        return 0;
    }
    if (total == 0) return 1;
    res = malloc((size_t) total + 1);
    if (!res) return -1;
    if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_tj_emit(c->q, &e, c->d_bsum, c->d_out) || bk_d2h(c->q, res, c->d_out, (size_t) total) || bk_sync(c->q)) { free(res); return -1; }
    res[total] = 0;
    *out = res; *out_size = (size_t) total;
    c->st.bytes_out = total;
    return 0;
}

/* 0: *out is the malloc()ed, NUL-terminated text; 1: the reference returns NULL for this input (nothing to convert);
 * -1: the call failed (flbgpu_last_error) */
int flbgpu_msgpack_to_json_format(flbgpu_ctx *ctx, const void *data, size_t bytes, int json_format, int date_format,
                                  const char *date_key, int escape_unicode, char **out, size_t *out_size, size_t *undefined_strings)
{
    flbgpu_chain *c;
    int r;
    g_rt_err[0] = 0;
    if (!ctx || !out || !out_size || (!data && bytes)) return -1;
    *out = NULL; *out_size = 0;
    if (undefined_strings) *undefined_strings = 0;
    if (json_format < 1 || json_format > 3) { set_err("json_format must be 1 (json), 2 (stream) or 3 (lines)%s%s", NULL, NULL); return -1; }
    if (date_format < 0 || date_format > 4) { set_err("unknown date format%s%s", NULL, NULL); return -1; }
    c = tj_chain(ctx);
    if (!c) return -1;

    pthread_mutex_lock(&c->lock);
    ctx->last_q = c->q;
    r = tj_run(c, data, bytes, json_format, date_format, date_key, escape_unicode, out, out_size, undefined_strings);
    if (r < 0) bk_upload_end(c->q);
    pthread_mutex_unlock(&c->lock);
    return r;
}

/* ---- chunk -> GELF messages: flb_msgpack_to_gelf() (src/flb_pack_gelf.c) on every event, as out_gelf and out_http flush a
 * chunk ---- */

static int gf_copy_key(uint8_t *dst, uint32_t *len, const char *key, const char *what)
{
    const size_t kl = strlen(key);
    if (kl > GF_KEY_MAX) { set_err("%s longer than 128 bytes%s", what, NULL); return -1; }
    memcpy(dst, key, kl);
    *len = (uint32_t) kl;
    return 0;
}

/* the call's arguments as the kernels take them (e->in and the buffers are set by gelf_run) */
static int gf_args(struct gf_env *e, const struct flbgpu_gelf_fields *fields, const char *tag_key, const char *tag, size_t tag_len,
                   int separator)
{
    static const char *const names[5] = { "host", "short_message", "timestamp", "level", "full_message" };   /* GF_HOST ... */
    const char *keys[5] = { NULL, NULL, NULL, NULL, NULL };
    int k;
    memset(e, 0, sizeof(*e));
    if (separator != 0 && separator != '\n') { set_err("separator must be 0 (out_gelf over TCP / TLS) or '\\n' (out_http)%s%s", NULL, NULL); return -1; }
    e->sep = (uint32_t) separator;
    if (fields) {
        keys[GF_HOST] = fields->host_key; keys[GF_SHORT] = fields->short_message_key; keys[GF_TIMESTAMP] = fields->timestamp_key;
        keys[GF_LEVEL] = fields->level_key; keys[GF_FULL] = fields->full_message_key;
    }
    for (k = 0; k < 5; k++)
        if (gf_copy_key(e->fkey[k], &e->fkey_len[k], keys[k] ? keys[k] : names[k], "a GELF field key")) return -1;
    e->tag_key_len = GF_NONE;
    if (tag_key) {
        if (!tag) { set_err("tag_key is set but the tag is NULL%s%s", NULL, NULL); return -1; }
        if (gf_copy_key(e->tag_key, &e->tag_key_len, tag_key, "tag_key")) return -1;
        if (tag_len > GF_TAG_MAX) { set_err("tag longer than 256 bytes%s%s", NULL, NULL); return -1; }
        memcpy(e->tag, tag, tag_len);
        e->tag_len = (uint32_t) tag_len;
    }
    return 0;
}

static int gelf_run(flbgpu_chain *c, const uint8_t *h_in, size_t bytes, struct gf_env *e, char **out, size_t *out_size,
                    size_t *failed, size_t *undefined_strings)
{
    const uint8_t *d_in = c->d_in;
    uint32_t n_rec, h_flags[FLBGPU_MAX_FILTERS + 1];
    size_t off;
    unsigned long long cnt[2] = { 0, 0 };
    uint64_t total = 0;
    char *res;

    if (call_start(c, bytes, out_size, NULL)) return -1;
    if (bytes && !(d_in = place_input(c, h_in, NULL, bytes))) return -1;
    if (bk_flags_clear(c->q, c->d_flags) || index_chunk(c, d_in, bytes, &n_rec, &off)) return -1;
    if (refuse_wide_arrays(c, h_in, d_in, off, bytes)) return -1;
    c->st.records_in = n_rec;
    if (n_rec) {
        e->in = d_in; e->in_len = bytes; e->off = c->d_off; e->len = c->d_len; e->kind = c->d_kind; e->n_rec = n_rec;
        e->err = c->d_flags + FLBGPU_MAX_FILTERS;
        e->size = c->d_size;
        /* work memory: the two counters (undefined strings, failed events), then the re-packed lengths */
        if (dev_grow(c, (void **) &c->d_mlw, &c->cap_mlw, 16 + sizeof(uint32_t) * (size_t) n_rec + 64, 1, 0)) return -1;
        e->undefined = (unsigned long long *) c->d_mlw; e->failed = e->undefined + 1;
        e->plen = (uint32_t *) (c->d_mlw + 16);
        if (e->tag_key_len != GF_NONE) {
            /* a re-packed event is its body (canonical encodings are never longer), a map header up to 4 bytes longer and
             * the two strings with their headers */
            e->scr_pad = 4 + 5 + e->tag_key_len + 5 + e->tag_len + 64;
            if (dev_grow(c, (void **) &c->d_scr, &c->cap_scr, bytes + (size_t) n_rec * e->scr_pad + 64, 1, 0)) return -1;
            e->scr = c->d_scr;
        }
        if (bk_zero(c->q, e->undefined, 16) || bk_gf_sizes(c->q, e) || bk_flags_fetch(c->q, c->d_flags, h_flags)) return -1;
        if (refused(c, h_flags[FLBGPU_MAX_FILTERS])) return -1;
        if (sizes_to_offsets(c, c->d_size, n_rec, NULL, NULL, "result larger than 4 GiB", &total)) return -1;
        if (bk_d2h(c->q, cnt, e->undefined, sizeof(cnt)) || bk_sync(c->q)) return -1;
    }
    bk_upload_end(c->q);
    c->st.kernel_launches = bk_launch_count();
    if (failed) *failed = (size_t) cnt[1];
    if (undefined_strings) *undefined_strings = (size_t) cnt[0];
    if (total == 0) return 1;
    res = malloc((size_t) total + 1);
    if (!res) { set_err("out of memory%s%s", NULL, NULL); return -1; }
    if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_gf_emit(c->q, e, c->d_bsum, c->d_out) ||
        bk_d2h(c->q, res, c->d_out, (size_t) total) || bk_sync(c->q)) { free(res); return -1; }
    res[total] = 0;
    *out = res; *out_size = (size_t) total;
    c->st.bytes_out = total;
    return 0;
}

/* 0: *out is the malloc()ed, NUL-terminated text; 1: no event was converted; -1: the call failed (flbgpu_last_error) */
int flbgpu_msgpack_to_gelf(flbgpu_ctx *ctx, const void *data, size_t bytes, const struct flbgpu_gelf_fields *fields,
                           const char *tag_key, const char *tag, size_t tag_len, int separator,
                           char **out, size_t *out_size, size_t *failed, size_t *undefined_strings)
{
    struct gf_env e;
    flbgpu_chain *c;
    int r;
    g_rt_err[0] = 0;
    if (!ctx || !out || !out_size || (!data && bytes)) return -1;
    *out = NULL; *out_size = 0;
    if (failed) *failed = 0;
    if (undefined_strings) *undefined_strings = 0;
    if (gf_args(&e, fields, tag_key, tag, tag_len, separator)) return -1;
    c = tj_chain(ctx);
    if (!c) return -1;

    pthread_mutex_lock(&c->lock);
    ctx->last_q = c->q;
    r = gelf_run(c, data, bytes, &e, out, out_size, failed, undefined_strings);
    if (r < 0) bk_upload_end(c->q);
    pthread_mutex_unlock(&c->lock);
    return r;
}
