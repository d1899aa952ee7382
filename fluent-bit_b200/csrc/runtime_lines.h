/* runtime_lines.h -- host side of the raw text -> log events conversion (part of runtime.c, included there).
 * The line loop of in_tail: plugins/in_tail/tail_file.c:629-700, :338-391. */

int flbgpu_lines_to_events(flbgpu_ctx *ctx, const char *text, size_t bytes, const char *key, int skip_empty_lines,
                           int64_t sec, int64_t nsec, const char *path_key, const char *path, const char *offset_key,
                           uint64_t stream_offset, void **out_buf, size_t *out_size, size_t *consumed, size_t *lines)
{
    flbgpu_chain *c;
    struct ln_env e;
    uint8_t strs[1024];
    uint32_t nbt, nbl, last_nl = 0;
    unsigned long long n_events = 0;
    size_t at = 0, need;
    uint64_t total;
    int r = -1;
    g_rt_err[0] = 0;
    if (!ctx || !out_buf || !out_size || !key || (!text && bytes)) return -1;
    *out_buf = NULL; *out_size = 0;
    if (consumed) *consumed = 0;
    if (lines) *lines = 0;
    if (bytes == 0) return 0;
    if (bytes >= 0xfff00000ull) { set_err("more than 4 GiB of text in one call%s%s", NULL, NULL); return -1; }
    if ((path_key && !path) || strlen(key) + (path_key ? strlen(path_key) + strlen(path) : 0) + (offset_key ? strlen(offset_key) : 0) > sizeof(strs)) {
        set_err("key / path_key / path / offset_key: missing or longer than 1 KB together%s%s", NULL, NULL);
        return -1;
    }
    c = tj_chain(ctx);
    if (!c) return -1;
    pthread_mutex_lock(&c->lock);
    ctx->last_q = c->q;
    memset(&e, 0, sizeof(e));
    e.bytes = bytes; e.sec = sec; e.nsec = nsec; e.skip_empty_lines = skip_empty_lines ? 1u : 0u; e.stream_offset = stream_offset;
#define LN_STR(s, off_field, len_field) do { if (s) { e.off_field = (uint32_t) at; e.len_field = (uint32_t) strlen(s); memcpy(strs + at, s, e.len_field); at += e.len_field; } \
        else e.len_field = 0xffffffffu; } while (0)
    LN_STR(key, key_off, key_len);
    LN_STR(path_key, path_key_off, path_key_len);
    if (path_key) LN_STR(path, path_off, path_len); else e.path_len = 0xffffffffu;
    LN_STR(offset_key, offset_key_off, offset_key_len);
#undef LN_STR
    e.n_tiles = (uint32_t) ((bytes + LN_TILE - 1) / LN_TILE);
    nbt = (e.n_tiles + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
#define LN_FAIL() do { bk_upload_end(c->q); pthread_mutex_unlock(&c->lock); return -1; } while (0)
#define LN_GROW(ptr, cap, n_, type) do { if ((cap) < (size_t) (n_)) { size_t nc_ = (size_t) (n_) + (size_t) (n_) / 4 + 64; \
        bk_free(c->q, ptr); (ptr) = (type *) bk_alloc(c->q, nc_ * sizeof(type)); if (!(ptr)) { (cap) = 0; LN_FAIL(); } (cap) = nc_; } } while (0)
    LN_GROW(c->d_in, c->cap_in, bytes + 64, uint8_t);
    /* on the compute stream, where the line kernels run: the staged upload (bk_upload_start) orders only the index stream, so
     * the counting pass could read text that has not arrived and the filling pass write more line feeds than were counted */
    if (bk_h2d(c->q, c->d_in, text, bytes)) LN_FAIL();
    e.text = c->d_in;
    /* work memory: the strings, the counts per tile; the line arrays once the number of lines is known */
    need = 1024 + 16 + sizeof(uint32_t) * (size_t) e.n_tiles + 64;
    LN_GROW(c->d_mlw, c->cap_mlw, need, uint8_t);
    e.strs = c->d_mlw;
    e.n_events = (unsigned long long *) (c->d_mlw + 1024);
    e.cnt = (uint32_t *) (c->d_mlw + 1024 + 16);
    if (bk_zero(c->q, e.n_events, 16)) LN_FAIL();
    LN_GROW(c->d_bsum, c->cap_bsum, nbt + 2, uint64_t);
    if (c->cap_hbsum < (size_t) nbt + 2) {
        free(c->h_bsum);
        c->cap_hbsum = (size_t) nbt + nbt / 4 + 64;
        c->h_bsum = malloc(c->cap_hbsum * sizeof(uint64_t));
        if (!c->h_bsum) { c->cap_hbsum = 0; LN_FAIL(); }
    }
    if (bk_h2d(c->q, c->d_mlw, strs, at ? at : 1) || bk_ln_count(c->q, &e) || bk_sizes_scan(c->q, e.cnt, e.n_tiles, c->d_bsum, c->h_bsum)) LN_FAIL();
    if (c->h_bsum[nbt] >= 0xfff00000ull) { set_err("too many lines in one call%s%s", NULL, NULL); LN_FAIL(); }
    e.n_lines = (uint32_t) c->h_bsum[nbt];
    bk_upload_end(c->q);
    c->st.records_in = e.n_lines;
    if (e.n_lines == 0) { pthread_mutex_unlock(&c->lock); return 0; }               /* no complete line yet */
    if (ensure_rec_cap(c, e.n_lines, 0)) LN_FAIL();
    e.nl = c->d_off; e.size = c->d_size;                                            /* (the record arrays of the chain, by another name) */
    if (bk_ln_fill(c->q, &e, c->d_bsum)) LN_FAIL();
    nbl = (e.n_lines + BK_REC_BLOCK - 1) / BK_REC_BLOCK;
    LN_GROW(c->d_bsum, c->cap_bsum, nbl + 2, uint64_t);                             /* (ln_fill has run: the tile offsets are not needed again... */
    if (c->cap_hbsum < (size_t) nbl + 2) {
        free(c->h_bsum);
        c->cap_hbsum = (size_t) nbl + nbl / 4 + 64;
        c->h_bsum = malloc(c->cap_hbsum * sizeof(uint64_t));
        if (!c->h_bsum) { c->cap_hbsum = 0; LN_FAIL(); }
    }
    if (bk_sync(c->q)) LN_FAIL();                                                    /* ... once it has really run) */
    if (bk_ln_sizes(c->q, &e) || bk_sizes_scan(c->q, e.size, e.n_lines, c->d_bsum, c->h_bsum)) LN_FAIL();
    total = c->h_bsum[nbl];
    if (total >= 0xfff00000ull) { set_err("result larger than 4 GiB%s%s", NULL, NULL); LN_FAIL(); }
    if (bk_d2h(c->q, &last_nl, e.nl + (e.n_lines - 1), sizeof(last_nl)) || bk_d2h(c->q, &n_events, e.n_events, sizeof(n_events)) || bk_sync(c->q)) LN_FAIL();
    if (consumed) *consumed = (size_t) last_nl + 1;
    if (lines) *lines = (size_t) n_events;                                          /* (`lines` of the reference counts what reached go_next) */
    r = 0;
    if (total) {
        void *out = malloc((size_t) total);
        if (!out) LN_FAIL();
        LN_GROW(c->d_out, c->cap_out, total, uint8_t);
        if (bk_ln_emit(c->q, &e, c->d_bsum, c->d_out) || bk_d2h(c->q, out, c->d_out, (size_t) total) || bk_sync(c->q)) { free(out); LN_FAIL(); }
        *out_buf = out; *out_size = (size_t) total;
    }
    c->st.bytes_in = bytes; c->st.bytes_out = total; c->st.kernel_launches = bk_launch_count();
    pthread_mutex_unlock(&c->lock);
    return r;
#undef LN_GROW
#undef LN_FAIL
}
