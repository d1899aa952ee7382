/* dev_lines.cuh -- the ingest side of the path: raw text to log events (row f4, input side).
 *
 * Reference: the line loop of in_tail, plugins/in_tail/tail_file.c process_content() :629-700 (cut at '\n'; with
 * skip_empty_lines an empty line and a lone "\r" are stepped over; a line of two bytes or more loses its trailing '\r') and
 * go_next :776-785 (processed_bytes), and flb_tail_file_pack_line() :338-391: one event per line --
 *     92 92 d7 00 <sec> <nsec> df 00000000 df <n> [path_key: path] [offset_key: stream_offset + processed_bytes] key: line
 * (the encoder's forced map32 headers for metadata and body, flb_mp.c:591-640).  Docker mode and the tail's own multiline modes
 * are other code paths of that function and not built here.
 *
 *   ln_count .... one lane per tile of LN_TILE bytes: line feeds in the tile
 *   ln_fill ..... the positions of the line feeds, at the tile's offset in the list
 *   ln_size ..... one lane per line: where it starts, what it keeps, the bytes of its event (0: stepped over)
 *   ln_emit ..... one lane per line: the event
 * With a parser (flbgpu_lines_to_events_parsed): tl_mid_* write each kept line as an event of the parser's input, the parser's chain
 * runs on that, and tl_event makes the line's event from the chain's result and the parser's report.
 * Functions of a "thread index" like the rest, so that the CPU emulation of the tests runs the same code.
 */
#ifndef FLBGPU_DEV_LINES_CUH
#define FLBGPU_DEV_LINES_CUH
#include "dev_msgpack.cuh"

/* 0x80 in every byte of x that is a line feed (exact: no borrow between bytes) */
FLB_HD uint64_t ln_nl_mask(uint64_t x)
{
    const uint64_t m = x ^ 0x0a0a0a0a0a0a0a0aull, k = 0x7f7f7f7f7f7f7f7full;
    return ~(((m & k) + k) | m | k);
}
FLB_HD int ln_popc64(uint64_t v)
{
#ifdef __CUDA_ARCH__
    return __popcll(v);
#else
    return __builtin_popcountll(v);
#endif
}
FLB_HD int ln_ctz64(uint64_t v)
{
#ifdef __CUDA_ARCH__
    return __ffsll((long long) v) - 1;
#else
    return __builtin_ctzll(v);
#endif
}
/* a whole tile is read as 64-bit words (the text starts at an allocation, tiles at multiples of LN_TILE); the last one by bytes */
FLB_HD uint32_t ln_count(const struct ln_env *e, uint32_t t)
{
    const size_t lo = (size_t) t * LN_TILE, hi = lo + LN_TILE < e->bytes ? lo + LN_TILE : e->bytes;
    uint32_t n = 0;
    size_t i;
    if (hi - lo == LN_TILE && (((uintptr_t) (e->text + lo)) & 7u) == 0) {
        const uint64_t *w = (const uint64_t *) (e->text + lo);
        for (i = 0; i < LN_TILE / 8; i++) n += (uint32_t) ln_popc64(ln_nl_mask(w[i]));
        return n;
    }
    for (i = lo; i < hi; i++) n += e->text[i] == '\n';
    return n;
}
FLB_HD void ln_fill(const struct ln_env *e, uint32_t t, uint64_t at)
{
    const size_t lo = (size_t) t * LN_TILE, hi = lo + LN_TILE < e->bytes ? lo + LN_TILE : e->bytes;
    size_t i;
    if (hi - lo == LN_TILE && (((uintptr_t) (e->text + lo)) & 7u) == 0) {
        const uint64_t *w = (const uint64_t *) (e->text + lo);
        for (i = 0; i < LN_TILE / 8; i++) {
            uint64_t m = ln_nl_mask(w[i]);                /* little-endian: byte j of the word is bits 8j .. 8j + 7 */
            while (m) { e->nl[at++] = (uint32_t) (lo + 8 * i + (size_t) (ln_ctz64(m) >> 3)); m &= m - 1; }
        }
        return;
    }
    for (i = lo; i < hi; i++) if (e->text[i] == '\n') e->nl[at++] = (uint32_t) i;
}
FLB_HD uint32_t ln_put(uint8_t *o, const uint8_t *s, uint32_t n) { uint32_t i; for (i = 0; i < n; i++) o[i] = s[i]; return n; }
/* the 22 bytes in front of an event's body members: [[time, {}], {<entries>... (the encoder's forced map32 headers) */
FLB_HD void ln_head(uint8_t *o, int64_t sec, int64_t nsec, uint32_t entries)
{
    o[0] = 0x92; o[1] = 0x92; o[2] = 0xd7; o[3] = 0x00;
    mp_put_be32(o + 4, (uint32_t) sec); mp_put_be32(o + 8, (uint32_t) nsec);        /* (the encoder's (uint32_t) casts) */
    o[12] = 0xdf; o[13] = o[14] = o[15] = o[16] = 0;
    o[17] = 0xdf; mp_put_be32(o + 18, entries);
}
/* [path_key: path] [offset_key: stream_offset + start], counted in *entries; o == NULL: only their size */
FLB_HD uint32_t ln_path_offset(const struct ln_env *e, uint32_t start, uint8_t *o, uint32_t *entries)
{
    uint32_t n = 0;
    if (e->path_key_len != 0xffffffffu) {
        n += o ? mp_put_str_hdr(o + n, e->path_key_len) : mp_str_hdr_size(e->path_key_len);
        if (o) ln_put(o + n, e->strs + e->path_key_off, e->path_key_len);
        n += e->path_key_len;
        n += o ? mp_put_str_hdr(o + n, e->path_len) : mp_str_hdr_size(e->path_len);
        if (o) ln_put(o + n, e->strs + e->path_off, e->path_len);
        n += e->path_len;
        (*entries)++;
    }
    if (e->offset_key_len != 0xffffffffu) {
        n += o ? mp_put_str_hdr(o + n, e->offset_key_len) : mp_str_hdr_size(e->offset_key_len);
        if (o) ln_put(o + n, e->strs + e->offset_key_off, e->offset_key_len);
        n += e->offset_key_len;
        n += o ? mp_put_uint(o + n, e->stream_offset + start) : mp_uint_size(e->stream_offset + start);
        (*entries)++;
    }
    return n;
}
/* bytes of the event ln_plain() writes */
FLB_HD uint32_t ln_plain_size(const struct ln_env *e, uint32_t start, uint32_t keep)
{
    uint32_t entries = 0;
    return 22 + ln_path_offset(e, start, 0, &entries) + mp_str_hdr_size(e->key_len) + e->key_len + mp_str_hdr_size(keep) + keep;
}
/* line k: [start, start + keep) is what the event carries; returns the event's size, 0 when the line is stepped over */
FLB_HD uint32_t ln_line(const struct ln_env *e, uint32_t k, uint32_t *start, uint32_t *keep)
{
    const uint32_t s = k ? e->nl[k - 1] + 1u : 0u, len = e->nl[k] - s;
    uint32_t crlf = 0;
    *start = s;
    if (e->skip_empty_lines && (len == 0 || (len == 1 && e->text[s] == '\r'))) return 0;
    if (len >= 2) crlf = e->text[s + len - 1] == '\r';
    *keep = len - crlf;
    return ln_plain_size(e, s, *keep);
}
/* the event of the line at `start`, `keep` bytes of it under `key`, stamped with the call's time */
FLB_HD void ln_plain(const struct ln_env *e, uint32_t start, uint32_t keep, uint8_t *o)
{
    uint32_t entries = 1, n = 22;
    n += ln_path_offset(e, start, o + n, &entries);
    n += mp_put_str_hdr(o + n, e->key_len); n += ln_put(o + n, e->strs + e->key_off, e->key_len);
    n += mp_put_str_hdr(o + n, keep);
    mp_copy(o + n, e->text + start, keep);               /* (the text buffer is padded like every device buffer) */
    ln_head(o, e->sec, e->nsec, entries);
}
FLB_HD void ln_emit(const struct ln_env *e, uint32_t k, uint8_t *o)
{
    uint32_t start, keep = 0;
    if (ln_line(e, k, &start, &keep)) ln_plain(e, start, keep, o);
}


/* ---- with a parser: in_tail's `Parser` branch, plugins/in_tail/tail_file.c:721-746 ----
 * line k in the parser's input: [[0, {}], {"_": line[0, keep)}], the event flbgpu_parser_do() hands its chain (Key_Name _);
 * the parser sees the line without its trailing '\r' (:724) */
FLB_HD uint32_t tl_mid_size(const struct tl_env *t, uint32_t k)
{
    uint32_t start, keep = 0;
    if (!ln_line(&t->ln, k, &start, &keep)) return 0;
    return 16 + mp_str_hdr_size(keep) + keep;
}
FLB_HD void tl_mid_emit(const struct tl_env *t, uint32_t k, uint8_t *o)
{
    uint32_t start, keep = 0, i;
    if (!ln_line(&t->ln, k, &start, &keep)) return;
    o[0] = 0x92; o[1] = 0x92; o[2] = 0xd7; o[3] = 0x00;
    for (i = 4; i < 12; i++) o[i] = 0;
    o[12] = 0x80; o[13] = 0x81; o[14] = 0xa1; o[15] = '_';
    mp_copy(o + 16 + mp_put_str_hdr(o + 16, keep), t->ln.text + start, keep);
}
/* the chain's record that starts at `off` and is `len` bytes long, or TL_NONE.  The index lists candidates in offset order; a
 * piece of a line that happens to frame as an event is a candidate of kind 2 at an offset inside the line's event, never at its start */
FLB_HD uint32_t tl_find(const struct tl_env *t, uint32_t off, uint32_t len)
{
    uint32_t lo = 0, hi = t->n_rec;
    while (lo < hi) {
        const uint32_t m = lo + (hi - lo) / 2;
        if (t->r_off[m] < off) lo = m + 1; else hi = m;
    }
    if (lo < t->n_rec && t->r_off[lo] == off && t->r_len[lo] == len && t->r_kind[lo] == 0) return lo;
    return TL_NONE;
}
/* line k's event from record r of the chain; o == NULL: only its size (0: the record is not a map event).
 * Parsed (report flag set): flb_tail_pack_line_map() :281-336 -- the parsed time, or the call's when flb_time_to_nanosec() of it
 * is 0 (:727-729); the members of the parser's map, each re-encoded as msgpack_pack_object() writes it (flb_tail_repack_map()
 * :228-279); then path_key and offset_key.  Not parsed: flb_tail_file_pack_line() of the line as read, '\r' and all (:744). */
FLB_HD uint32_t tl_event(const struct tl_env *t, uint32_t k, uint32_t r, uint8_t *o)
{
    const struct ln_env *e = &t->ln;
    const int32_t *pr = t->prep + (size_t) 6 * r;
    const uint32_t start = k ? e->nl[k - 1] + 1u : 0u, len = e->nl[k] - start;
    const uint8_t *p = t->res + t->r_out[r] + 13, *end = t->res + t->r_out[r] + t->r_size[r];   /* (13: [[time, {}] of the result) */
    struct mp_tok mt;
    int64_t sec, nsec;
    uint32_t n = 22, i, used, entries;
    if (!pr[0]) {
        if (o) ln_plain(e, start, len, o);
        return ln_plain_size(e, start, len);
    }
    if (p >= end || mp_token(p, end, &mt) != 0 || mt.type != MPT_MAP) return 0;
    entries = mt.len;
    p += mt.hdr;
    for (i = 0; i < 2 * mt.len; i++) {
        n += mp_canon(p, end, o ? o + n : 0, &used);
        p += used;
    }
    n += ln_path_offset(e, start, o ? o + n : 0, &entries);
    if (o) {
        sec = (int64_t) (((uint64_t) (uint32_t) pr[3] << 32) | (uint32_t) pr[2]); nsec = pr[4];
        if ((uint64_t) sec * 1000000000ull + (uint64_t) nsec == 0) { sec = e->sec; nsec = e->nsec; }
        ln_head(o, sec, nsec, entries);
    }
    return n;
}

#endif
