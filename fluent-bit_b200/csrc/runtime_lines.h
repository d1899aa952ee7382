/* runtime_lines.h -- host side of the raw text -> log events conversion (part of runtime.c, included there).
 * The line loop of in_tail: plugins/in_tail/tail_file.c:629-700, :338-391. */

/* the arguments both line calls take: checked, the outputs cleared, the call's constants and strings in *e, the strings packed
 * into strs (*n_strs bytes, 1 KB at most).  1: nothing to do (no text); -1: refused */
static int ln_args(struct ln_env *e, uint8_t *strs, size_t *n_strs, const char *text, size_t bytes, const char *key, int skip_empty_lines,
                   int64_t sec, int64_t nsec, const char *path_key, const char *path, const char *offset_key, uint64_t stream_offset,
                   void **out_buf, size_t *out_size, size_t *consumed, size_t *lines)
{
    size_t at = 0;
    if (!out_buf || !out_size || !key || (!text && bytes)) return -1;
    *out_buf = NULL; *out_size = 0;
    if (consumed) *consumed = 0;
    if (lines) *lines = 0;
    if (bytes == 0) return 1;
    if (bytes >= 0xfff00000ull) { set_err("more than 4 GiB of text in one call%s%s", NULL, NULL); return -1; }
    if ((path_key && !path) || strlen(key) + (path_key ? strlen(path_key) + strlen(path) : 0) + (offset_key ? strlen(offset_key) : 0) > 1024) {
        set_err("key / path_key / path / offset_key: missing or longer than 1 KB together%s%s", NULL, NULL);
        return -1;
    }
    e->bytes = bytes; e->sec = sec; e->nsec = nsec; e->skip_empty_lines = skip_empty_lines ? 1u : 0u; e->stream_offset = stream_offset;
#define LN_STR(s, off_field, len_field) do { if (s) { e->off_field = (uint32_t) at; e->len_field = (uint32_t) strlen(s); memcpy(strs + at, s, e->len_field); at += e->len_field; } \
        else e->len_field = 0xffffffffu; } while (0)
    LN_STR(key, key_off, key_len);
    LN_STR(path_key, path_key_off, path_key_len);
    if (path_key) LN_STR(path, path_off, path_len); else e->path_len = 0xffffffffu;
    LN_STR(offset_key, offset_key_off, offset_key_len);
#undef LN_STR
    e->n_tiles = (uint32_t) ((bytes + LN_TILE - 1) / LN_TILE);
    *n_strs = at;
    return 0;
}

/* the text and the strings to e->text / e->strs, then the line feeds counted per tile and placed: e->n_lines, the tile offsets
 * in d_tiles / h_bsum (NULL: the chain's own).  All on the compute stream, where the line kernels run: the staged upload
 * (bk_upload_start) orders only the index stream, so the counting pass could read text that has not arrived and the filling
 * pass write more line feeds than were counted. */
static int ln_count_lines(flbgpu_chain *c, struct ln_env *e, const char *text, const uint8_t *strs, size_t n_strs,
                          uint64_t *d_tiles, uint64_t *h_bsum)
{
    uint64_t n;
    if (bk_h2d(c->q, (void *) e->text, text, e->bytes) || bk_h2d(c->q, (void *) e->strs, strs, n_strs ? n_strs : 1) ||
        bk_zero(c->q, e->n_events, 16) || bk_ln_count(c->q, e) ||
        sizes_to_offsets(c, e->cnt, e->n_tiles, d_tiles, h_bsum, "too many lines in one call", &n)) return -1;
    e->n_lines = (uint32_t) n;
    return 0;
}

int flbgpu_lines_to_events(flbgpu_ctx *ctx, const char *text, size_t bytes, const char *key, int skip_empty_lines,
                           int64_t sec, int64_t nsec, const char *path_key, const char *path, const char *offset_key,
                           uint64_t stream_offset, void **out_buf, size_t *out_size, size_t *consumed, size_t *lines)
{
    flbgpu_chain *c;
    struct ln_env e;
    uint8_t strs[1024];
    uint32_t last_nl = 0;
    unsigned long long n_events = 0;
    size_t n_strs = 0;
    uint64_t total;
    int r;
    g_rt_err[0] = 0;
    if (!ctx) return -1;
    memset(&e, 0, sizeof(e));
    r = ln_args(&e, strs, &n_strs, text, bytes, key, skip_empty_lines, sec, nsec, path_key, path, offset_key, stream_offset,
                out_buf, out_size, consumed, lines);
    if (r) return r < 0 ? -1 : 0;
    c = tj_chain(ctx);
    if (!c) return -1;
    pthread_mutex_lock(&c->lock);
    ctx->last_q = c->q;
#define LN_FAIL() do { bk_upload_end(c->q); pthread_mutex_unlock(&c->lock); return -1; } while (0)
    /* the text; work memory: the strings, the counts per tile; the line arrays once the number of lines is known */
    if (dev_grow(c, (void **) &c->d_in, &c->cap_in, bytes + 64, 1, 0) ||
        dev_grow(c, (void **) &c->d_mlw, &c->cap_mlw, 1024 + 16 + sizeof(uint32_t) * (size_t) e.n_tiles + 64, 1, 0)) LN_FAIL();
    e.text = c->d_in;
    e.strs = c->d_mlw;
    e.n_events = (unsigned long long *) (c->d_mlw + 1024);
    e.cnt = (uint32_t *) (c->d_mlw + 1024 + 16);
    if (ln_count_lines(c, &e, text, strs, n_strs, NULL, NULL)) LN_FAIL();
    bk_upload_end(c->q);
    c->st.records_in = e.n_lines;
    if (e.n_lines == 0) { pthread_mutex_unlock(&c->lock); return 0; }               /* no complete line yet */
    if (ensure_rec_cap(c, e.n_lines, 0)) LN_FAIL();
    e.nl = c->d_off; e.size = c->d_size;                                            /* (the record arrays of the chain, by another name) */
    if (bk_ln_fill(c->q, &e, c->d_bsum) || bk_ln_sizes(c->q, &e) ||
        sizes_to_offsets(c, e.size, e.n_lines, NULL, NULL, "result larger than 4 GiB", &total)) LN_FAIL();
    if (bk_d2h(c->q, &last_nl, e.nl + (e.n_lines - 1), sizeof(last_nl)) || bk_d2h(c->q, &n_events, e.n_events, sizeof(n_events)) || bk_sync(c->q)) LN_FAIL();
    if (consumed) *consumed = (size_t) last_nl + 1;
    if (lines) *lines = (size_t) n_events;                                          /* (`lines` of the reference counts what reached go_next) */
    if (total) {
        void *out = malloc((size_t) total);
        if (!out) LN_FAIL();
        if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_ln_emit(c->q, &e, c->d_bsum, c->d_out) ||
            bk_d2h(c->q, out, c->d_out, (size_t) total) || bk_sync(c->q)) { free(out); LN_FAIL(); }
        *out_buf = out; *out_size = (size_t) total;
    }
    c->st.bytes_in = bytes; c->st.bytes_out = total; c->st.kernel_launches = bk_launch_count();
    pthread_mutex_unlock(&c->lock);
    return 0;
#undef LN_FAIL
}

/* ---- with a parser: in_tail's `Parser` branch, plugins/in_tail/tail_file.c:721-746 ----
 * On the parser's solo chain (the one behind flbgpu_parser_do()), under its lock for the whole call, all on its queue's stream:
 *   line feeds (ln_count, ln_fill) -> the parser's input {"_": line} per kept line (tl_mid_*) -> the chain, device-resident,
 *   with the parser's report -> per line: its record, the bytes of its event (tl_sizes) -> the events (tl_emit).
 * The host waits for the counts the sizes need; the parser's input and its result stay on the device. */
static int parser_solo(flbgpu_parser *p);
static int chain_run(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in_ext, size_t bytes,
                     uint8_t *ext_out, size_t ext_cap, void **host_out, size_t *out_size);

/* a line the device would not parse: the call fails, naming the FLBGPU_E_* bits */
static void tl_refused(uint32_t bits)
{
    static const struct { uint32_t bit; const char *name; } nm[] = {
        { FLBGPU_E_FIELDS, "FIELDS" }, { FLBGPU_E_RXSTACK, "RXSTACK" }, { FLBGPU_E_RXBUDGET, "RXBUDGET" }, { FLBGPU_E_FLOAT, "FLOAT" },
        { FLBGPU_E_INDEX, "INDEX" }, { FLBGPU_E_ESCAPE, "ESCAPE" }, { FLBGPU_E_L2M, "L2M" }, { FLBGPU_E_RXUNICODE, "RXUNICODE" },
        { FLBGPU_E_DEEP, "DEEP" }, { FLBGPU_E_TAGVALUE, "TAGVALUE" }, { FLBGPU_E_MLLIMIT, "MLLIMIT" }, { FLBGPU_E_MLMETA, "MLMETA" },
        { FLBGPU_E_JSONDATE, "JSONDATE" }, { FLBGPU_E_JSONGROUP, "JSONGROUP" } };
    char names[256];
    size_t i, at = 0;
    names[0] = 0;
    for (i = 0; i < sizeof(nm) / sizeof(nm[0]); i++)
        if ((bits & nm[i].bit) && at < sizeof(names)) at += (size_t) snprintf(names + at, sizeof(names) - at, "%sFLBGPU_E_%s", at ? " " : "", nm[i].name);
    snprintf(g_rt_err, sizeof(g_rt_err), "the device refused to parse some lines (error bits 0x%x: %s); the reference parses them, "
             "so they are not passed on unparsed", bits, names);
}

int flbgpu_lines_to_events_parsed(flbgpu_parser *p, const char *text, size_t bytes, const char *key, int skip_empty_lines,
                                  int64_t sec, int64_t nsec, const char *path_key, const char *path, const char *offset_key,
                                  uint64_t stream_offset, void **out_buf, size_t *out_size, size_t *consumed, size_t *lines)
{
    flbgpu_chain *c;
    struct tl_env t;
    struct ln_env *e = &t.ln;
    uint8_t strs[1024];
    uint32_t nbt, nbl_max, last_nl = 0, bad = 0, h_flags[FLBGPU_MAX_FILTERS + 1];
    unsigned long long n_events = 0;
    size_t n_strs = 0, text_room, osz = 0;
    uint64_t *d_tiles, *d_fbsum, mid_total, total;
    int r;
    g_rt_err[0] = 0;
    if (!p) return -1;
    memset(&t, 0, sizeof(t));
    r = ln_args(e, strs, &n_strs, text, bytes, key, skip_empty_lines, sec, nsec, path_key, path, offset_key, stream_offset,
                out_buf, out_size, consumed, lines);
    if (r) return r < 0 ? -1 : 0;
    if (parser_solo(p)) return -1;
    c = p->solo;
    pthread_mutex_lock(&c->lock);
    p->ctx->last_q = c->q;
    c->active = 1;
    nbt = (e->n_tiles + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    nbl_max = (uint32_t) ((bytes + BK_REC_BLOCK - 1) / BK_REC_BLOCK);          /* (a line takes one byte at least: its '\n') */
#define TL_FAIL() do { c->keep_result = 0; pthread_mutex_unlock(&c->lock); return -1; } while (0)
    /* the text, then the strings, the counters (events, lines without a record) and the line feeds per tile */
    text_room = (bytes + 64 + 15) & ~(size_t) 15;
    if (dev_grow(c, (void **) &c->d_tl_text, &c->cap_tl_text, text_room + 1024 + 16 + sizeof(uint32_t) * (size_t) e->n_tiles, 1, 0)) TL_FAIL();
    e->text = c->d_tl_text;
    e->strs = c->d_tl_text + text_room;
    e->n_events = (unsigned long long *) (c->d_tl_text + text_room + 1024);
    t.bad = (uint32_t *) (c->d_tl_text + text_room + 1024 + 8);
    e->cnt = (uint32_t *) (c->d_tl_text + text_room + 1024 + 16);
    /* block offsets: of the tiles, of the parser's input per line, of the events per line */
    if (dev_grow(c, (void **) &c->d_tl_bsum, &c->cap_tl_bsum, (size_t) nbt + 2 + 2 * ((size_t) nbl_max + 2), sizeof(uint64_t), 0) ||
        host_grow((void **) &c->h_tl_bsum, &c->cap_tl_hbsum, (size_t) (nbt > nbl_max ? nbt : nbl_max) + 2, sizeof(uint64_t))) TL_FAIL();
    d_tiles = c->d_tl_bsum;
    t.mbsum = c->d_tl_bsum + nbt + 2;
    d_fbsum = c->d_tl_bsum + nbt + 2 + nbl_max + 2;
    if (ln_count_lines(c, e, text, strs, n_strs, d_tiles, c->h_tl_bsum)) TL_FAIL();
    if (e->n_lines == 0) { pthread_mutex_unlock(&c->lock); return 0; }             /* no complete line yet */
    /* per line: line feed, bytes in the parser's input, record, bytes of the event */
    if (dev_grow(c, (void **) &c->d_tl_line, &c->cap_tl_line, 4 * (size_t) e->n_lines, sizeof(uint32_t), 0)) TL_FAIL();
    e->nl = c->d_tl_line;
    t.msize = c->d_tl_line + e->n_lines;
    t.rec = c->d_tl_line + 2 * (size_t) e->n_lines;
    t.size = c->d_tl_line + 3 * (size_t) e->n_lines;
    if (bk_ln_fill(c->q, e, d_tiles) || bk_tl_mid_size(c->q, &t) ||
        sizes_to_offsets(c, t.msize, e->n_lines, (uint64_t *) t.mbsum, c->h_tl_bsum, "parser input larger than 4 GiB", &mid_total)) TL_FAIL();
    if (mid_total) {
        if (dev_grow(c, (void **) &c->d_tl_mid, &c->cap_tl_mid, mid_total + 64, 1, 0)) TL_FAIL();
        t.mid = c->d_tl_mid;
        /* the chain's index kernels run on a stream of their own: the parser's input is complete before they start */
        if (bk_tl_mid_emit(c->q, &t) || bk_sync(c->q)) TL_FAIL();
        c->keep_result = 1;                                                     /* (its result stays in the chain's d_out) */
        r = chain_run(c, NULL, c->d_tl_mid, (size_t) mid_total, NULL, 0, NULL, &osz);
        c->keep_result = 0;
        if (r < 0) { if (c->st.error_bits & ~FLBGPU_E_INDEX) tl_refused(c->st.error_bits); TL_FAIL(); }
        if (r != FLBGPU_FILTER_MODIFIED || osz == 0) { set_err("parser call: no result for the lines%s%s", NULL, NULL); TL_FAIL(); }
        /* (a value nested to msgpack-c's unpack limit: the repacking of flb_tail_pack_line_map() unpacks the parser's map) */
        if (bk_flags_fetch(c->q, c->d_flags, h_flags)) TL_FAIL();
        if (h_flags[FLBGPU_MAX_FILTERS] & FLBGPU_E_DEEP) { c->st.error_bits = h_flags[FLBGPU_MAX_FILTERS]; tl_refused(h_flags[FLBGPU_MAX_FILTERS]); TL_FAIL(); }
        t.n_rec = (uint32_t) c->st.records_in;
        t.r_off = c->d_off; t.r_len = c->d_len; t.r_kind = c->d_kind; t.r_size = c->d_size; t.r_bsum = c->d_bsum;
        t.res = c->d_out; t.prep = c->d_prep;
        if (dev_grow(c, (void **) &c->d_tl_rec, &c->cap_tl_rec, (size_t) t.n_rec + 1, sizeof(uint32_t), 0)) TL_FAIL();
        t.r_out = c->d_tl_rec;
        if (bk_tl_sizes(c->q, &t)) TL_FAIL();
    }
    if (bk_d2h(c->q, &last_nl, e->nl + (e->n_lines - 1), sizeof(last_nl)) || bk_d2h(c->q, &n_events, e->n_events, sizeof(n_events)) ||
        bk_d2h(c->q, &bad, t.bad, sizeof(bad)) ||
        sizes_to_offsets(c, t.size, mid_total ? e->n_lines : 0, d_fbsum, c->h_tl_bsum, "result larger than 4 GiB", &total)) TL_FAIL();
    if (bad) { set_err("parser call: the lines did not come back one to one%s%s", NULL, NULL); TL_FAIL(); }
    if (consumed) *consumed = (size_t) last_nl + 1;
    if (lines) *lines = (size_t) n_events;
    if (total) {
        void *out;
        if (dev_grow(c, (void **) &c->d_tl_out, &c->cap_tl_out, total, 1, 0)) TL_FAIL();
        out = malloc((size_t) total);
        if (!out) { set_err("out of memory%s%s", NULL, NULL); TL_FAIL(); }
        if (bk_tl_emit(c->q, &t, d_fbsum, c->d_tl_out) || bk_d2h(c->q, out, c->d_tl_out, (size_t) total) || bk_sync(c->q)) { free(out); TL_FAIL(); }
        *out_buf = out; *out_size = (size_t) total;
    }
    c->st.bytes_in = bytes; c->st.bytes_out = total; c->st.kernel_launches = bk_launch_count();
    pthread_mutex_unlock(&c->lock);
    return 0;
#undef TL_FAIL
}
