/* dev_gelf.cuh -- a chunk of log events as GELF messages: what out_gelf (Graylog) and out_http (`format gelf`) send.
 *
 * Reference: flb_msgpack_to_gelf() src/flb_pack_gelf.c:407-785 with flb_msgpack_gelf_flatten() :191-405,
 * flb_msgpack_gelf_key() :23-110, flb_msgpack_gelf_value() :112-147 and flb_msgpack_gelf_value_ext() :149-189; the flush
 * loops plugins/out_gelf/gelf.c:265-392 (inject_tag() :233-262) and plugins/out_http/http.c:378-440.
 *
 * One lane per event, two passes (size, bytes), like dev_tojson.cuh, whose escaped string writer, integer writer and event
 * time it uses.  Without tag_key the reference converts the body where the decoder found it, in the chunk, so the bytes its
 * string writer reads past a string are the chunk's own: they are read here too, up to the chunk's end.  With tag_key it
 * converts the map inject_tag() re-encoded, which a lane first rebuilds in its scratch slice.  The flattening's recursion is
 * an explicit stack of containers; msgpack-c's unpack depth bounds it.
 */
#ifndef FLBGPU_DEV_GELF_CUH
#define FLBGPU_DEV_GELF_CUH
#include "dev_tojson.cuh"

#define GF_MAXDEPTH 40

/* valid_char[] of flb_msgpack_gelf_key(): every other byte of a key becomes '_' */
FLB_HD int gf_valid(uint8_t c)
{
    return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '.' || c == '_' || c == '-';
}

/* a key as flb_msgpack_gelf_key() writes it.  cut: the key went through strncpy() into a zeroed buffer (the top-level
 * prefix, :619-627), so a NUL byte zero-fills the rest, and each of those zeroes becomes '_' */
FLB_HD uint32_t gf_put_key(const uint8_t *k, uint32_t len, int cut, uint8_t *o)
{
    uint32_t i;
    int z = 0;
    if (o) for (i = 0; i < len; i++) { const uint8_t c = k[i]; if (c == 0 && cut) z = 1; o[i] = (z || !gf_valid(c)) ? '_' : c; }
    return len;
}

FLB_HD uint32_t gf_put_raw(const uint8_t *s, uint32_t len, uint8_t *o)
{
    uint32_t i;
    if (o) for (i = 0; i < len; i++) o[i] = s[i];
    return len;
}

/* "%f" of a MSGPACK_OBJECT_FLOAT32 / _FLOAT64 (via.f64), at most cap bytes of it */
FLB_HD uint32_t gf_real(const struct mp_tok *t, uint8_t *buf, uint32_t cap)
{
    union { uint64_t u; double d; } cv;
    if (t->type == MPT_F32) { union { uint32_t u; float f; } a; a.u = (uint32_t) t->u; cv.d = (double) a.f; }
    else cv.u = t->u;
    return dj_fmt_f6(cv.u, buf, cap);
}

/* the syslog keyword of a level string, matched case-insensitively (:573-586): its index, or -1 */
FLB_HD int gf_level_name(const uint8_t *s, uint32_t len)
{
    const char *w = "emerg\0alert\0crit\0err\0warning\0notice\0info\0debug";
    int idx;
    for (idx = 0; idx < 8; idx++) {
        uint32_t wl = 0, k;
        while (w[wl]) wl++;
        if (wl == len) {
            for (k = 0; k < len; k++) { uint8_t c = s[k]; if (c >= 'A' && c <= 'Z') c += 32; if (c != (uint8_t) w[k]) break; }
            if (k == len) return idx;
        }
        w += wl + 1;
    }
    return -1;
}

/* the name a field key is written under */
FLB_HD const uint8_t *gf_field_name(int f, uint32_t *len)
{
    switch (f) {
    case GF_HOST: *len = 4; return (const uint8_t *) "host";
    case GF_SHORT: *len = 13; return (const uint8_t *) "short_message";
    case GF_TIMESTAMP: *len = 9; return (const uint8_t *) "timestamp";
    case GF_LEVEL: *len = 5; return (const uint8_t *) "level";
    }
    *len = 12; return (const uint8_t *) "full_message";
}

/* flb_msgpack_gelf_flatten() of a value that is not a container.  q: quoted (outside an array); inside an array strings are a
 * plain flb_sds_cat(), neither quoted nor escaped */
FLB_HDN uint32_t gf_scalar(const struct mp_tok *t, const uint8_t *p, const uint8_t *lim, int q, uint8_t *o, uint32_t *undef)
{
    uint32_t n = 0, x;
    switch (t->type) {
    case MPT_NIL: TJ_PUT('n'); TJ_PUT('u'); TJ_PUT('l'); TJ_PUT('l'); break;
    case MPT_BOOL:
        if (q) TJ_PUT('"');
        if (t->u) { TJ_PUT('t'); TJ_PUT('r'); TJ_PUT('u'); TJ_PUT('e'); } else { TJ_PUT('f'); TJ_PUT('a'); TJ_PUT('l'); TJ_PUT('s'); TJ_PUT('e'); }
        if (q) TJ_PUT('"');
        break;
    case MPT_UINT: n += tj_put_u64(t->u, o); break;
    case MPT_INT: {                                      /* (msgpack-c: a non-negative int is POSITIVE_INTEGER) */
        const int64_t v = (int64_t) t->u;
        if (v < 0) { TJ_PUT('-'); n += tj_put_u64((uint64_t) 0 - (uint64_t) v, o ? o + n : 0); }
        else n += tj_put_u64((uint64_t) v, o);
        break;
    }
    case MPT_F32: case MPT_F64: {                        /* flb_sds_printf("%f"): never cut */
        uint8_t f[320];
        n += gf_put_raw(f, gf_real(t, f, sizeof(f)), o);
        break;
    }
    case MPT_STR: case MPT_BIN:
        if (!q) { n += gf_put_raw(p + t->hdr, t->len, o); break; }
        TJ_PUT('"');
        if (t->len) n += tj_write_str(p + t->hdr, t->len, lim, 1, o ? o + n : 0, undef);     /* flb_sds_cat_utf8() */
        TJ_PUT('"');
        break;
    case MPT_EXT:                                        /* each byte as \xNN, lower-case hex of the unsigned byte */
        if (q) TJ_PUT('"');
        for (x = 0; x < t->len; x++) {
            const uint8_t c = p[t->hdr + x];
            TJ_PUT('\\'); TJ_PUT('x'); TJ_PUT("0123456789abcdef"[c >> 4]); TJ_PUT("0123456789abcdef"[c & 15]);
        }
        if (q) TJ_PUT('"');
        break;
    }
    return n;
}

/* The prefix of the map at stack level s: the keys of the maps from level pb (the first map behind the last array) up to s,
 * each behind a '_' once the prefix holds something (:331-352).  The top-level map's own part is '_' + its key (:619-627).
 * A map straight inside an array has no key (GF_NONE). */
FLB_HD uint32_t gf_put_prefix(const uint8_t *const *ck, const uint32_t *cl, uint32_t pb, uint32_t s, int top, uint8_t *o)
{
    uint32_t n = 0, L = 0, j;
    for (j = pb; j <= s; j++) {
        if (cl[j] == GF_NONE) continue;
        if (j == 0 && top) { TJ_PUT('_'); n += gf_put_key(ck[0], cl[0], 1, o ? o + n : 0); L = 1 + cl[0]; continue; }
        if (L) { TJ_PUT('_'); L++; }
        n += gf_put_key(ck[j], cl[j], 0, o ? o + n : 0);
        L += cl[j];
    }
    return n;
}

/* msgpack-c hands out a zero-length fixstr as a NULL pointer until the unpack call has read a token with bytes behind its
 * first one (unpack_template.h: `n` starts NULL, and each trail read sets it), and flb_msgpack_to_gelf() leaves a top-level
 * scalar member whose key or value pointer is NULL out (`if (!val || !key) continue`).  Returns where the first such token lies
 * in the buffer an unpack call starts at p. */
FLB_HD const uint8_t *gf_null_end(const uint8_t *p, const uint8_t *lim)
{
    while (p < lim) {
        const uint8_t c = *p;
        if (c <= 0x7f || c >= 0xe0 || (c >= 0x80 && c <= 0x9f) || c == 0xa0 || c == 0xc0 || c == 0xc2 || c == 0xc3) p++;
        else break;
    }
    return p;
}

/* flb_msgpack_to_gelf() of the map at p, in a buffer that ends at lim; sec / nsec: the event's time; nul_end: gf_null_end() of
 * the unpack call.  Returns the text's length, 0 where the reference returns NULL (or the event nests deeper than the stack:
 * e->err gets FLBGPU_E_FIELDS). */
FLB_HDN uint32_t gf_convert(const struct gf_env *e, const uint8_t *p, const uint8_t *lim, const uint8_t *nul_end, int64_t sec,
                            int64_t nsec, uint8_t *o, uint32_t *undef)
{
    const uint8_t *ck[GF_MAXDEPTH];
    uint32_t cl[GF_MAXDEPTH], rem[GF_MAXDEPTH], idx[GF_MAXDEPTH], plen[GF_MAXDEPTH], pb[GF_MAXDEPTH];
    uint8_t isarr[GF_MAXDEPTH], flag[GF_MAXDEPTH];     /* flag: a map's members are written as inside an array; an array closes with '"' */
    uint32_t n = 0, top_rem, found = 0;
    int sp = 0, topmap = 0;
    struct mp_tok t, tv;
    const uint8_t *vp;
    mp_token(p, lim, &t);
    top_rem = t.len;
    p += t.hdr;
    TJ_PUT('{'); TJ_PUT('"'); TJ_PUT('v'); TJ_PUT('e'); TJ_PUT('r'); TJ_PUT('s'); TJ_PUT('i'); TJ_PUT('o'); TJ_PUT('n');
    TJ_PUT('"'); TJ_PUT(':'); TJ_PUT('"'); TJ_PUT('1'); TJ_PUT('.'); TJ_PUT('1'); TJ_PUT('"');
    for (;;) {
        if (sp == 0) {
            /* ---- a member of the record (:497-753) */
            const uint8_t *key, *nx;
            uint32_t klen;
            int which = -1, custom = 0, lvl = -1, f, key_null, val_null;
            uint8_t fb[49];
            uint32_t fm = 0;
            if (!top_rem) break;
            top_rem--;
            key_null = *p == 0xa0 && p < nul_end;
            mp_token(p, lim, &t);
            vp = mp_skip(p, lim);
            nx = mp_skip(vp, lim);
            if (t.type != MPT_STR && t.type != MPT_BIN) { p = nx; continue; }
            key = p + t.hdr; klen = t.len;
            mp_token(vp, lim, &tv);
            val_null = *vp == 0xa0 && vp < nul_end;
            for (f = 0; f < 5 && which < 0; f++) if (klen == e->fkey_len[f] && bytes_eq(key, e->fkey[f], klen)) which = f;
            if (which >= 0) {
                if ((found >> which) & 1) { p = nx; continue; }          /* the first occurrence wins */
                found |= 1u << which;
                key = gf_field_name(which, &klen);
                if (which == GF_LEVEL) {
                    if (tv.type == MPT_UINT || (tv.type == MPT_INT && (int64_t) tv.u >= 0)) { }
                    else if (tv.type == MPT_STR) {
                        if (tv.len == 1 && vp[tv.hdr] >= '0' && vp[tv.hdr] <= '7') lvl = vp[tv.hdr] - '0';
                        else lvl = gf_level_name(vp + tv.hdr, tv.len);           /* -1: stays a string */
                    }
                    else return 0;
                }
            }
            else if (klen == 2 && key[0] == 'i' && key[1] == 'd') { p = nx; continue; }
            else custom = 1;
            if (tv.type == MPT_MAP) {
                p = vp + tv.hdr;
                if (tv.len) {
                    isarr[0] = 0; flag[0] = 0; rem[0] = tv.len; idx[0] = 0; ck[0] = key; cl[0] = klen; plen[0] = 1 + klen; pb[0] = 0;
                    sp = 1; topmap = 1;
                }
                continue;
            }
            /* nil is left out; so is a float32, which is not MSGPACK_OBJECT_FLOAT (= FLOAT64) and matches no branch (:659-727).
             * A float64 is measured first: snprintf(temp, 47, "%f") into char temp[48] = {0}, then val_len bytes of temp -- a
             * 47- or 48-character result keeps 46 characters and brings NUL bytes along, a longer one fails the event even when
             * the member would then be left out.  Then a scalar with a NULL key or value pointer goes (a field key's name
             * replaces a NULL key). */
            if (tv.type == MPT_NIL || tv.type == MPT_F32) { p = nx; continue; }
            if (tv.type == MPT_F64 && (fm = gf_real(&tv, fb, 49)) > 48) return 0;
            if ((val_null || (custom && key_null)) && tv.type != MPT_ARRAY) { p = nx; continue; }
            TJ_PUT(','); TJ_PUT(' '); TJ_PUT('"');
            if (custom) TJ_PUT('_');
            n += gf_put_key(key, klen, 0, o ? o + n : 0);
            TJ_PUT('"'); TJ_PUT(':');
            if (tv.type == MPT_ARRAY) {
                TJ_PUT('"');
                isarr[0] = 1; flag[0] = 1; rem[0] = tv.len; idx[0] = 0; cl[0] = GF_NONE;
                sp = 1; topmap = 0;
                p = vp + tv.hdr;
                continue;
            }
            if (lvl >= 0) n += tj_put_u64((uint64_t) lvl, o ? o + n : 0);
            else if (tv.type == MPT_F64) { uint32_t x; for (x = 0; x < fm; x++) TJ_PUT(x < 46 ? fb[x] : 0); }
            else n += gf_scalar(&tv, vp, lim, 1, o ? o + n : 0, undef);
            p = nx;
            continue;
        }
        {
            const int s = sp - 1;
            if (!rem[s]) {
                if (isarr[s] && flag[s]) TJ_PUT('"');
                sp--;
                continue;
            }
            rem[s]--;
            mp_token(p, lim, &t);
            if (isarr[s]) {
                /* ---- an array element: ", " between elements, everything as inside an array (:276-313) */
                if (idx[s]++) { TJ_PUT(','); TJ_PUT(' '); }
                if (t.type == MPT_MAP || t.type == MPT_ARRAY) {
                    if (sp >= GF_MAXDEPTH) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
                    isarr[sp] = t.type == MPT_ARRAY; flag[sp] = t.type == MPT_MAP; rem[sp] = t.len; idx[sp] = 0;
                    cl[sp] = GF_NONE; plen[sp] = 0; pb[sp] = (uint32_t) sp;
                    sp++;
                    p += t.hdr;
                }
                else { n += gf_scalar(&t, p, lim, 0, o ? o + n : 0, undef); p = mp_skip(p, lim); }
                continue;
            }
            /* ---- a member of a nested map (:315-398): keys that are not strings are skipped */
            {
                const uint32_t i = idx[s]++;
                const int in_array = flag[s];
                vp = mp_skip(p, lim);
                if (t.type != MPT_STR) { p = mp_skip(vp, lim); continue; }
                mp_token(vp, lim, &tv);
                if (tv.type == MPT_MAP) {
                    if (sp >= GF_MAXDEPTH) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
                    isarr[sp] = 0; flag[sp] = (uint8_t) in_array; rem[sp] = tv.len; idx[sp] = 0; ck[sp] = p + t.hdr; cl[sp] = t.len;
                    plen[sp] = plen[s] ? plen[s] + 1 + t.len : t.len; pb[sp] = pb[s];
                    sp++;
                    p = vp + tv.hdr;
                    continue;
                }
                if (in_array && i > 0) TJ_PUT(' ');
                if (!in_array) { TJ_PUT(','); TJ_PUT(' '); TJ_PUT('"'); }
                if (!in_array || plen[s]) { n += gf_put_prefix(ck, cl, pb[s], (uint32_t) s, topmap, o ? o + n : 0); TJ_PUT('_'); }
                n += gf_put_key(p + t.hdr, t.len, 0, o ? o + n : 0);
                if (in_array) TJ_PUT('='); else { TJ_PUT('"'); TJ_PUT(':'); }
                if (tv.type == MPT_ARRAY) {
                    if (!in_array) TJ_PUT('"');
                    if (sp >= GF_MAXDEPTH) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
                    isarr[sp] = 1; flag[sp] = (uint8_t) !in_array; rem[sp] = tv.len; idx[sp] = 0; cl[sp] = GF_NONE;
                    sp++;
                    p = vp + tv.hdr;
                    continue;
                }
                n += gf_scalar(&tv, vp, lim, !in_array, o ? o + n : 0, undef);
                p = mp_skip(vp, lim);
            }
        }
    }
    if (!((found >> GF_TIMESTAMP) & 1)) {
        /* "%li.%03lu" of tv_sec and tv_nsec / 1000000 (a long divided, printed unsigned) */
        const uint64_t ms = (uint64_t) (nsec / 1000000);
        TJ_PUT(','); TJ_PUT(' '); TJ_PUT('"');
        n += gf_put_raw((const uint8_t *) "timestamp", 9, o ? o + n : 0);
        TJ_PUT('"'); TJ_PUT(':');
        if (sec < 0) { TJ_PUT('-'); n += tj_put_u64((uint64_t) 0 - (uint64_t) sec, o ? o + n : 0); }
        else n += tj_put_u64((uint64_t) sec, o ? o + n : 0);
        TJ_PUT('.');
        if (ms < 100) TJ_PUT('0');
        if (ms < 10) TJ_PUT('0');
        n += tj_put_u64(ms, o ? o + n : 0);
    }
    if (!((found >> GF_SHORT) & 1)) return 0;
    TJ_PUT('}');
    return n;
}

/* inject_tag(): the body's members through msgpack_pack_object() into a map one larger, then tag_key: tag */
FLB_HDN uint32_t gf_pack_tag(const struct gf_env *e, const uint8_t *q, const uint8_t *end, uint8_t *b)
{
    struct mp_tok t;
    uint32_t n, k;
    mp_token(q, end, &t);
    n = mp_put_map_hdr(b, t.len + 1);
    q += t.hdr;
    for (k = 0; k < 2 * t.len; k++) {
        const uint8_t *nx = mp_skip(q, end);
        n += mp_canon(q, nx, b + n, 0);
        q = nx;
    }
    n += mp_put_str_hdr(b + n, e->tag_key_len); n += gf_put_raw(e->tag_key, e->tag_key_len, b + n);
    n += mp_put_str_hdr(b + n, e->tag_len); n += gf_put_raw(e->tag, e->tag_len, b + n);
    return n;
}

/* Event i's message and separator (o == NULL: sized only; the sizing pass re-packs the event when tag_key is set and counts
 * what fails).  Events the decoder steps over (kind != 0) and events that fail give 0 bytes. */
FLB_HDN uint32_t gf_event(const struct gf_env *e, uint32_t i, uint8_t *o)
{
    const uint8_t *p, *end, *q, *lim, *nul_end;
    int64_t sec, nsec;
    uint32_t n, undef = 0;
    if (e->kind[i] != 0) return 0;
    p = e->in + e->off[i]; end = p + e->len[i]; q = p + 1;
    if (*q == 0x92) q = mp_skip(tj_event_time(q + 1, end, &sec, &nsec), end);     /* [[ts, meta], body] */
    else q = tj_event_time(q, end, &sec, &nsec);
    if (e->tag_key_len != GF_NONE) {
        uint8_t *b = e->scr + e->off[i] + (size_t) i * e->scr_pad;
        if (!o) e->plen[i] = gf_pack_tag(e, q, end, b);
        q = b; lim = b + e->plen[i];
        nul_end = gf_null_end(b, lim);                   /* flb_msgpack_raw_to_gelf() unpacks the re-packed map */
    }
    else {
        lim = e->in + e->in_len;
        nul_end = gf_null_end(p, end);                   /* the decoder unpacks the whole event */
    }
    n = gf_convert(e, q, lim, nul_end, sec, nsec, o, &undef);
    if (!n) { if (!o) CH_ATOMIC_ADD(e->failed, 1); return 0; }
    if (o) o[n] = (uint8_t) e->sep;
    n++;
    if (undef && !o) CH_ATOMIC_ADD(e->undefined, 1);
    return n;
}

#endif
