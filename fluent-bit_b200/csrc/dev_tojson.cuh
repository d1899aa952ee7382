/* dev_tojson.cuh -- the output side of the path: a chunk of log events as JSON text (row f4).
 *
 * Reference: flb_pack_msgpack_to_json_format() src/flb_pack.c:1320-1602 (what out_stdout, out_http, out_file, out_kafka ...
 * call on a chunk: json / json_stream / json_lines, the date key in five formats), msgpack2json() :984-1146 (numbers, the
 * "%.1f" / "%.16g" rule for reals, duplicate string keys dropped in favour of the last one, ext bodies as \xNN),
 * flb_utils_write_str() src/flb_utils.c:883-1372 (the escaped and the raw string writer), flb_utf8_decode() src/flb_utf8.c:42-102.
 *
 * One lane per event, two passes (size, bytes).  Like the reference, a lane first packs the event as ONE msgpack map --
 * date key, `__internal__` for non-empty metadata, the body's members re-encoded canonically (msgpack_pack_object) -- into its
 * slice of a scratch buffer, then converts that buffer.  The detour is not for show: the reference's string writers test
 * 16 bytes at a time and, after a multi-byte character has put them out of step, test (and copy!) up to 15 bytes past the end
 * of a string -- the bytes that follow it in that very buffer.  Where those bytes exist the behaviour is reproduced; where
 * they lie beyond the event's buffer (uninitialised or stale memory in the reference) the window is taken as "not plain" and
 * the string is counted (tj_env.undefined).
 */
#ifndef FLBGPU_DEV_TOJSON_CUH
#define FLBGPU_DEV_TOJSON_CUH
#include "dev_json.cuh"

/* ---- printf("%.16g") / ("%.1f") as msgpack2json uses them ---- */
FLB_HD void djb_sub(struct dj_big *a, const struct dj_big *b)          /* a -= b, a >= b */
{
    uint64_t borrow = 0;
    uint32_t i;
    for (i = 0; i < a->n; i++) {
        const uint64_t x = (uint64_t) a->v[i], y = (i < b->n ? (uint64_t) b->v[i] : 0) + borrow;
        a->v[i] = (uint32_t) (x - y);
        borrow = x < y ? 1 : 0;
    }
    while (a->n && a->v[a->n - 1] == 0) a->n--;
}

#define TJ_PUT(c) do { if (o) o[n] = (uint8_t) (c); n++; } while (0)

FLB_HD uint32_t tj_put_u64(uint64_t v, uint8_t *o)
{
    uint8_t t[20];
    uint32_t k = 0, n = 0;
    do { t[k++] = (uint8_t) ('0' + v % 10); v /= 10; } while (v);
    while (k) { const uint8_t c = t[--k]; TJ_PUT(c); }         /* (TJ_PUT evaluates its argument only when it writes) */
    return n;
}

/* a MSGPACK_OBJECT_FLOAT{32,64} value (as a double's bits) */
FLB_HDN uint32_t tj_fmt_real(uint64_t bits, uint8_t *o)
{
    const uint32_t ef = (uint32_t) ((bits >> 52) & 0x7ff);
    const int neg = (int) (bits >> 63);
    uint64_t M = bits & (((uint64_t) 1 << 52) - 1);
    uint32_t n = 0;
    int k;
    if (ef == 0x7ff) {                                   /* "%.16g": inf, -inf, nan, -nan */
        if (neg) TJ_PUT('-');
        if (M) { TJ_PUT('n'); TJ_PUT('a'); TJ_PUT('n'); } else { TJ_PUT('i'); TJ_PUT('n'); TJ_PUT('f'); }
        return n;
    }
    if (ef) { M |= (uint64_t) 1 << 52; k = (int) ef - 1075; } else k = -1074;
    /* f64 == (double)(long long) f64: an integer below 2^63 in magnitude (-2^63 included: what the x86 conversion returns for
     * everything out of range) -> "%.1f" */
    {
        int integral = 0;
        uint64_t mag = 0;
        if (M == 0) integral = 1;
        else if (k >= 0) { if (k <= 10) { integral = 1; mag = M << k; } else if (k == 11 && M == ((uint64_t) 1 << 52) && neg) { integral = 1; mag = (uint64_t) 1 << 63; } }
        else if (-k <= 52 && (M & (((uint64_t) 1 << -k) - 1)) == 0) { integral = 1; mag = M >> -k; }
        if (integral) {
            if (neg) TJ_PUT('-');
            n += tj_put_u64(mag, o ? o + n : 0);
            TJ_PUT('.'); TJ_PUT('0');
            return n;
        }
    }
    /* "%.16g": sixteen significant digits of the exact binary value, round-half-even; v = R / S * 10^e10, 1 <= R / S < 10 */
    {
        struct dj_big R, S, T;
        uint8_t d[17];
        int e10, i, nd, nb = 64 - dj_clz64(M) + k, up;
        e10 = (int) (((long long) (nb - 1) * 78913) >> 18);            /* floor((nb - 1) * log10(2)), give or take one */
        R.v[0] = (uint32_t) M; R.v[1] = (uint32_t) (M >> 32); R.n = R.v[1] ? 2 : 1;
        S.v[0] = 1; S.n = 1;
        if (k >= 0) djb_shl(&R, (uint32_t) k); else djb_shl(&S, (uint32_t) -k);
        if (e10 >= 0) { djb_mul_pow5(&S, (uint32_t) e10); djb_shl(&S, (uint32_t) e10); }
        else { djb_mul_pow5(&R, (uint32_t) -e10); djb_shl(&R, (uint32_t) -e10); }
        while (djb_cmp(&R, &S) < 0) { djb_mul_small(&R, 10u, 0); e10--; }
        for (;;) {
            T = S;
            djb_mul_small(&T, 10u, 0);
            if (djb_cmp(&R, &T) < 0) break;
            S = T; e10++;
        }
        for (i = 0; i < 16; i++) {
            int q = 0;
            while (djb_cmp(&R, &S) >= 0) { djb_sub(&R, &S); q++; }
            d[i] = (uint8_t) q;
            if (i < 15) djb_mul_small(&R, 10u, 0);
        }
        djb_mul_small(&R, 2u, 0);
        i = djb_cmp(&R, &S);
        up = i > 0 || (i == 0 && (d[15] & 1));
        if (up) {
            for (i = 15; i >= 0; i--) { if (d[i] < 9) { d[i]++; break; } d[i] = 0; }
            if (i < 0) { d[0] = 1; e10++; }
        }
        nd = 16;
        while (nd > 1 && d[nd - 1] == 0) nd--;
        if (neg) TJ_PUT('-');
        if (e10 < -4 || e10 >= 16) {
            int ex = e10 < 0 ? -e10 : e10;
            TJ_PUT('0' + d[0]);
            if (nd > 1) { TJ_PUT('.'); for (i = 1; i < nd; i++) TJ_PUT('0' + d[i]); }
            TJ_PUT('e'); TJ_PUT(e10 < 0 ? '-' : '+');
            if (ex >= 100) { TJ_PUT('0' + ex / 100); ex %= 100; }
            TJ_PUT('0' + ex / 10); TJ_PUT('0' + ex % 10);
        }
        else if (e10 >= 0) {
            for (i = 0; i <= e10; i++) TJ_PUT('0' + (i < nd ? d[i] : 0));
            if (nd > e10 + 1) { TJ_PUT('.'); for (i = e10 + 1; i < nd; i++) TJ_PUT('0' + d[i]); }
        }
        else {
            TJ_PUT('0'); TJ_PUT('.');
            for (i = 0; i < -e10 - 1; i++) TJ_PUT('0');
            for (i = 0; i < nd; i++) TJ_PUT('0' + d[i]);
        }
    }
    return n;
}

/* ---- flb_utils_write_str(): the two string writers ---- */
/* a 16-byte window none of whose bytes is <= 0x1f, '"', '\\' or >= 0x80 (flb_vector8_has_le / _has / _is_highbit_set) */
FLB_HD int tj_chunk_plain(const uint8_t *p)
{
    int i;
    for (i = 0; i < 16; i++) { const uint8_t c = p[i]; if (c <= 0x1f || c == '"' || c == '\\' || c >= 0x80) return 0; }
    return 1;
}

FLB_HD uint32_t tj_hex4(uint32_t cp, uint8_t *o)      /* "\\u%.4x" */
{
    uint32_t n = 0;
    int sh, started = 0;
    TJ_PUT('\\'); TJ_PUT('u');
    for (sh = 28; sh >= 0; sh -= 4) {
        const uint32_t h = (cp >> sh) & 15u;
        if (h || started || sh <= 12) { TJ_PUT("0123456789abcdef"[h]); started = 1; }
    }
    return n;
}

/* flb_utf8_decode(): 0 accept, 1 reject, 2 continue */
FLB_HD int tj_utf8_decode(uint32_t *state, uint32_t *cp, uint8_t byte)
{
    if (*state == 0) {
        if (byte <= 0x7f) { *cp = byte; return 0; }
        else if ((byte & 0xe0) == 0xc0) { *cp = byte & 0x1f; *state = 1; }
        else if ((byte & 0xf0) == 0xe0) { *cp = byte & 0x0f; *state = 2; }
        else if ((byte & 0xf8) == 0xf0) { *cp = byte & 0x07; *state = 3; }
        else { *state = 1; return 1; }
    }
    else {
        if ((byte & 0xc0) == 0x80) { *cp = (*cp << 6) | (byte & 0x3f); (*state)--; }
        else { *state = 1; return 1; }
    }
    if (*state == 0) {
        if ((*cp >= 0xd800 && *cp <= 0xdfff) || *cp > 0x10ffff) { *state = 1; return 1; }
        return 0;
    }
    return 2;
}

/* flb_utf8_validate_char() of the raw writer: length of the valid sequence at s (max_len bytes left), 0 = invalid */
FLB_HD int tj_utf8_validate(const uint8_t *s, int max_len)
{
    const uint8_t c = s[0];
    int len, i;
    if (c <= 0x7f) return 1;
    else if ((c & 0xe0) == 0xc0) { if (c < 0xc2) return 0; len = 2; }
    else if ((c & 0xf0) == 0xe0) {
        if (max_len > 1 && c == 0xe0 && s[1] < 0xa0) return 0;
        if (max_len > 1 && c == 0xed && s[1] >= 0xa0) return 0;
        len = 3;
    }
    else if ((c & 0xf8) == 0xf0) {
        if (max_len > 1 && c == 0xf0 && s[1] < 0x90) return 0;
        if (c > 0xf4) return 0;
        if (max_len > 1 && c == 0xf4 && s[1] > 0x8f) return 0;
        len = 4;
    }
    else return 0;
    if (max_len < len) return 0;
    for (i = 1; i < len; i++) if ((s[i] & 0xc0) != 0x80) return 0;
    return len;
}

/* str[0, len) inside a buffer that ends at lim; returns the bytes written (o == NULL: counted only); *undef is set when a
 * 16-byte test reaches past lim */
FLB_HDN uint32_t tj_write_str(const uint8_t *str, uint32_t len, const uint8_t *lim, int escape_unicode, uint8_t *o, uint32_t *undef)
{
    const uint32_t vlen = len & ~15u;
    uint32_t i = 0, copypos = 0, n = 0, b, x;
    for (;;) {
        for (; i < vlen; i += 16) {
            if (str + i + 16 > lim) { *undef = 1; break; }
            if (!tj_chunk_plain(str + i)) break;
        }
        if (copypos < i) {                               /* (i may have stepped past the string: the reference copies that too) */
            for (x = copypos; x < i; x++) TJ_PUT(str[x]);
            copypos = i;
        }
        for (b = 0; b < 16; b++) {
            uint32_t c;
            if (i >= len) return n;
            c = str[i];
            if (c < 128 && (c < 0x20 || c == '"' || c == '\\' || c == 0x7f)) {        /* json_escape_table */
                TJ_PUT('\\');
                if (c == '"' || c == '\\') TJ_PUT(c);
                else if (c == '\n') TJ_PUT('n');
                else if (c == '\r') TJ_PUT('r');
                else if (c == '\t') TJ_PUT('t');
                else if (c == '\b') TJ_PUT('b');
                else if (c == '\f') TJ_PUT('f');
                else { TJ_PUT('u'); TJ_PUT('0'); TJ_PUT('0'); TJ_PUT("0123456789abcdef"[c >> 4]); TJ_PUT("0123456789abcdef"[c & 15]); }
            }
            else if (c < 0x80) TJ_PUT(c);
            else if (!escape_unicode) {                  /* flb_utils_write_str_raw(): valid sequences verbatim, U+FFFD for the rest */
                const int ul = tj_utf8_validate(str + i, (int) (len - i));
                if (ul == 0 || i + (uint32_t) ul > len) { TJ_PUT(0xef); TJ_PUT(0xbf); TJ_PUT(0xbd); }
                else { for (x = 0; x < (uint32_t) ul; x++) TJ_PUT(str[i + x]); i += (uint32_t) ul - 1; }
            }
            else {
                /* flb_utils_write_str_escaped(), the branch every byte >= 0x80 takes (`c` is a sign-extended char there) */
                uint32_t ulen, state = 0, cp = 0, un;
                uint8_t tmp[8];
                int valid = 1;
                ulen = c < 0xc0 ? 1u : c < 0xe0 ? 2u : c < 0xf0 ? 3u : c < 0xf8 ? 4u : c < 0xfc ? 5u : 6u;    /* flb_utf8_len() */
                if (i + ulen > len) { i++; break; }      /* "skip truncated UTF-8": one byte is dropped without a trace */
                for (un = 0; un < ulen; un++) {
                    const int r = tj_utf8_decode(&state, &cp, str[i]);
                    if (r == 1) {
                        if (un == 0) { tmp[0] = str[i]; ulen = 1; i++; }
                        else ulen = un;
                        valid = 0;
                        break;
                    }
                    tmp[un] = str[i];
                    i++;
                }
                i--;
                if (valid) {
                    if (cp > 0xffff) {
                        n += tj_hex4(0xd800 + ((cp - 0x10000) >> 10), o ? o + n : 0);
                        n += tj_hex4(0xdc00 + ((cp - 0x10000) & 0x3ff), o ? o + n : 0);
                    }
                    else n += tj_hex4(cp, o ? o + n : 0);
                }
                else {
                    for (x = 0; x < ulen; x++) {         /* each fragment as U+E0xx, in UTF-8 */
                        TJ_PUT(0xe0 | (0xe0 >> 4));
                        TJ_PUT(0x80 | ((0xe0 << 2) & 0x3f) | ((tmp[x] >> 6) & 0x03));
                        TJ_PUT(0x80 | (tmp[x] & 0x3f));
                    }
                }
            }
            i++;
        }
        copypos = i;
    }
}

/* ---- one event ---- */

/* (mp_copy() reads whole aligned words around its source, which buffers from bk_alloc() are padded for -- a string literal is not) */
FLB_HD uint32_t tj_put_lit(uint8_t *o, const char *s, uint32_t n) { uint32_t i; for (i = 0; i < n; i++) o[i] = (uint8_t) s[i]; return n; }

FLB_HD uint32_t tj_put2(uint32_t v, uint8_t *o) { o[0] = (uint8_t) ('0' + v / 10 % 10); o[1] = (uint8_t) ('0' + v % 10); return 2; }

/* strftime("%Y-%m-%d?%H:%M:%S") of gmtime_r(sec) + ".%06lu" of the microseconds (+ 'Z'); returns the length (<= 37) */
FLB_HD uint32_t tj_datetime(int64_t sec, uint64_t usec, int iso, uint8_t *o)
{
    int64_t days = sec / 86400, rem = sec % 86400, y;
    uint32_t n = 0, k, m, dd;
    int64_t z, era, doe, yoe, doy, mp;
    uint8_t t[24];
    if (rem < 0) { rem += 86400; days--; }
    z = days + 719468;                                   /* civil_from_days */
    era = (z >= 0 ? z : z - 146096) / 146097;
    doe = z - era * 146097;
    yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    y = yoe + era * 400;
    doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    mp = (5 * doy + 2) / 153;
    dd = (uint32_t) (doy - (153 * mp + 2) / 5 + 1);
    m = (uint32_t) (mp < 10 ? mp + 3 : mp - 9);
    if (m <= 2) y++;
    k = 0;
    { int64_t yy = y < 0 ? -y : y; do { t[k++] = (uint8_t) ('0' + yy % 10); yy /= 10; } while (yy); }
    if (y < 0) o[n++] = '-';
    while (k) o[n++] = t[--k];
    o[n++] = '-'; n += tj_put2(m, o + n); o[n++] = '-'; n += tj_put2(dd, o + n);
    o[n++] = iso ? 'T' : ' ';
    n += tj_put2((uint32_t) (rem / 3600), o + n); o[n++] = ':';
    n += tj_put2((uint32_t) (rem % 3600 / 60), o + n); o[n++] = ':';
    n += tj_put2((uint32_t) (rem % 60), o + n);
    o[n++] = '.';
    {
        uint8_t u[24];
        uint32_t ku = 0;
        do { u[ku++] = (uint8_t) ('0' + usec % 10); usec /= 10; } while (usec);
        while (ku < 6) u[ku++] = '0';
        while (ku) o[n++] = u[--ku];
    }
    if (iso) o[n++] = 'Z';
    return n;
}


/* the timestamp at q of an event rec_frame() accepted, as flb_log_event_decoder_decode_timestamp() converts it; returns the
 * position behind it */
FLB_HD const uint8_t *tj_event_time(const uint8_t *q, const uint8_t *end, int64_t *sec, int64_t *nsec)
{
    struct mp_tok t;
    mp_token(q, end, &t);
    *nsec = 0;
    if (t.type == MPT_UINT || t.type == MPT_INT) *sec = (int64_t) t.u;
    else if (t.type == MPT_F64) {
        union { uint64_t u; double d; } cv;
        cv.u = t.u;
        *sec = mp_d2i64(cv.d);
        *nsec = mp_d2i64((cv.d - (double) *sec) * 1000000000.0);
    }
    else { *sec = (int64_t) (int32_t) mp_be32(q + t.hdr); *nsec = (int64_t) (int32_t) mp_be32(q + t.hdr + 4); }
    return q + t.hdr + (t.type == MPT_EXT ? t.len : 0);
}

/* the event as one msgpack map in its scratch slice (flb_pack.c:1380-1497); returns its length */
FLB_HDN uint32_t tj_pack_event(const struct tj_env *e, uint32_t i, uint8_t *b)
{
    const uint8_t *p = e->in + e->off[i], *end = p + e->len[i], *q = p + 1, *meta = 0, *meta_end = 0;
    struct mp_tok t;
    int64_t sec, nsec;
    uint32_t n = 5, entries = 0, k;
    const int v2 = (*q == 0x92);
    if (v2) q++;
    q = tj_event_time(q, end, &sec, &nsec);
    if (v2) { meta = q; q = mp_skip(q, end); meta_end = q; }
    if (e->key_len != 0xffffffffu) {
        n += mp_put_str_hdr(b + n, e->key_len);
        for (k = 0; k < e->key_len; k++) b[n + k] = e->key[k];
        n += e->key_len;
        switch (e->date_format) {
        case TJ_DATE_DOUBLE: {
            union { uint64_t u; double d; } cv;
            cv.d = (double) sec + ((double) nsec / 1000000000.0);         /* flb_time_to_double() */
            b[n] = 0xcb; mp_put_be64(b + n + 1, cv.u); n += 9;
            break;
        }
        case TJ_DATE_ISO8601: case TJ_DATE_JAVA_SQL: {
            uint8_t txt[48];
            const uint32_t tl = tj_datetime(sec, (uint64_t) nsec / 1000u, e->date_format == TJ_DATE_ISO8601, txt);
            if (tl >= 38u) CH_ATOMIC_OR(e->err, FLBGPU_E_JSONDATE);      /* the reference gives the whole chunk up (char time_formatted[38]) */
            n += mp_put_str_hdr(b + n, tl);
            mp_copy(b + n, txt, tl); n += tl;
            break;
        }
        case TJ_DATE_EPOCH: n += mp_put_uint(b + n, (uint64_t) sec); break;
        default: n += mp_put_uint(b + n, (uint64_t) sec * 1000u + (uint64_t) (nsec / 1000000)); break;     /* flb_time_to_millisec(): the nanoseconds divide as a signed long */
        }
        entries++;
    }
    {
        /* "__internal__": { "group_attributes": the governing group start's body, "log_metadata": metadata } when either holds
         * something (flb_pack.c:1432-1474; a legacy event's metadata is the decoder's empty map) */
        const uint8_t *ga = 0, *ga_end = 0;
        uint32_t meta_n = 0, ga_n = 0;
        if (meta) { mp_token(meta, meta_end, &t); meta_n = t.len; }
        if (e->n_groups) {
            uint32_t lo = 0, hi = e->n_groups;           /* the last marker in front of event i */
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((e->groups[mid] >> 1) < i) lo = mid + 1; else hi = mid; }
            if (lo && (e->groups[lo - 1] & 1u)) {
                const uint32_t g = e->groups[lo - 1] >> 1;
                const uint8_t *gp = e->in + e->off[g], *gend = gp + e->len[g], *gq = gp + 1;
                struct mp_tok tg;
                if (*gq == 0x92) { gq++; mp_token(gq, gend, &tg); gq += tg.hdr + (tg.type == MPT_EXT ? tg.len : 0); gq = mp_skip(gq, gend); }
                else { mp_token(gq, gend, &tg); gq += tg.hdr + (tg.type == MPT_EXT ? tg.len : 0); }
                ga = gq; ga_end = gend;
                mp_token(ga, ga_end, &tg);
                ga_n = tg.len;
            }
        }
        if (meta_n > 0 || ga_n > 0) {
            n += mp_put_str_hdr(b + n, 12); n += tj_put_lit(b + n, "__internal__", 12);
            b[n] = 0xdf; mp_put_be32(b + n + 1, ga ? 2u : 1u); n += 5;
            if (ga) {
                n += mp_put_str_hdr(b + n, 16); n += tj_put_lit(b + n, "group_attributes", 16);
                n += mp_canon(ga, ga_end, b + n, 0);
            }
            n += mp_put_str_hdr(b + n, 12); n += tj_put_lit(b + n, "log_metadata", 12);
            if (meta) n += mp_canon(meta, meta_end, b + n, 0); else b[n++] = 0x80;
            entries++;
        }
    }
    mp_token(q, end, &t);
    q += t.hdr;
    for (k = 0; k < 2 * t.len; k++) {
        const uint8_t *nx = mp_skip(q, end);
        n += mp_canon(q, nx, b + n, 0);
        q = nx;
    }
    entries += t.len;
    b[0] = 0xdf; mp_put_be32(b + 1, entries);
    return n;
}

/* msgpack2json() over the packed object at p (ends at lim); returns the text length */
#define TJ_MAXDEPTH 40
FLB_HDN uint32_t tj_convert(const struct tj_env *e, const uint8_t *p, const uint8_t *lim, uint8_t *o, uint32_t *undef)
{
    uint32_t n = 0, rem[TJ_MAXDEPTH], packed[TJ_MAXDEPTH];
    uint8_t kind[TJ_MAXDEPTH], phase[TJ_MAXDEPTH];       /* kind 0 array, 1 map; map phase 0 key next, 1 key written, 2 value written */
    int sp = 0;
    struct mp_tok t;
    for (;;) {
        int done_value = 0;
        if (sp && kind[sp - 1] == 1 && phase[sp - 1] == 0) {
            /* a map entry: dropped when a later entry has the same string key (key_exists_in_map) */
            int dup = 0;
            mp_token(p, lim, &t);
            if (t.type == MPT_STR) {
                const uint8_t *q = mp_skip(mp_skip(p, lim), lim);
                uint32_t j;
                for (j = 1; j < rem[sp - 1] && !dup; j++) {
                    struct mp_tok tq;
                    mp_token(q, lim, &tq);
                    if (tq.type == MPT_STR && tq.len == t.len && bytes_eq(q + tq.hdr, p + t.hdr, t.len)) dup = 1;
                    q = mp_skip(mp_skip(q, lim), lim);
                }
            }
            if (dup) {
                p = mp_skip(mp_skip(p, lim), lim);
                if (--rem[sp - 1] == 0) { TJ_PUT('}'); sp--; done_value = 1; }
                else continue;
            }
            else {
                if (packed[sp - 1]) TJ_PUT(',');
                packed[sp - 1]++;
                phase[sp - 1] = 1;
            }
        }
        if (!done_value) {
            mp_token(p, lim, &t);
            switch (t.type) {
            case MPT_NIL: TJ_PUT('n'); TJ_PUT('u'); TJ_PUT('l'); TJ_PUT('l'); p += t.hdr; done_value = 1; break;
            case MPT_BOOL:
                if (t.u) { TJ_PUT('t'); TJ_PUT('r'); TJ_PUT('u'); TJ_PUT('e'); } else { TJ_PUT('f'); TJ_PUT('a'); TJ_PUT('l'); TJ_PUT('s'); TJ_PUT('e'); }
                p += t.hdr; done_value = 1; break;
            case MPT_UINT: n += tj_put_u64(t.u, o ? o + n : 0); p += t.hdr; done_value = 1; break;
            case MPT_INT: {
                const int64_t v = (int64_t) t.u;
                if (v < 0) { TJ_PUT('-'); n += tj_put_u64((uint64_t) 0 - (uint64_t) v, o ? o + n : 0); }
                else n += tj_put_u64((uint64_t) v, o ? o + n : 0);          /* (msgpack-c: a non-negative int is POSITIVE_INTEGER) */
                p += t.hdr; done_value = 1; break;
            }
            case MPT_F32: {
                union { uint32_t u; float f; } a; union { uint64_t u; double d; } cv;
                a.u = (uint32_t) t.u; cv.d = (double) a.f;
                n += tj_fmt_real(cv.u, o ? o + n : 0); p += t.hdr; done_value = 1; break;
            }
            case MPT_F64: n += tj_fmt_real(t.u, o ? o + n : 0); p += t.hdr; done_value = 1; break;
            case MPT_STR: case MPT_BIN:
                TJ_PUT('"');
                if (t.len) n += tj_write_str(p + t.hdr, t.len, lim, (int) e->escape_unicode, o ? o + n : 0, undef);
                TJ_PUT('"');
                p += t.hdr + t.len; done_value = 1; break;
            case MPT_EXT: {
                uint32_t x;
                TJ_PUT('"');
                for (x = 0; x < t.len; x++) {            /* "\\x%02x" of a (char): bytes >= 0x80 print as ffffffXX */
                    const uint8_t c = p[t.hdr + x];
                    TJ_PUT('\\'); TJ_PUT('x');
                    if (c >= 0x80) { int z; for (z = 0; z < 6; z++) TJ_PUT('f'); }
                    TJ_PUT("0123456789abcdef"[c >> 4]); TJ_PUT("0123456789abcdef"[c & 15]);
                }
                TJ_PUT('"');
                p += t.hdr + t.len; done_value = 1; break;
            }
            case MPT_ARRAY:
                TJ_PUT('[');
                p += t.hdr;
                if (t.len == 0) { TJ_PUT(']'); done_value = 1; }
                else if (sp >= TJ_MAXDEPTH) return 0;
                else { kind[sp] = 0; rem[sp] = t.len; packed[sp] = 0; phase[sp] = 0; sp++; }
                break;
            case MPT_MAP:
                TJ_PUT('{');
                p += t.hdr;
                if (t.len == 0) { TJ_PUT('}'); done_value = 1; }
                else if (sp >= TJ_MAXDEPTH) return 0;
                else { kind[sp] = 1; rem[sp] = t.len; packed[sp] = 0; phase[sp] = 0; sp++; }
                break;
            default: return 0;
            }
        }
        while (done_value) {                             /* a value is complete: what does its container do next */
            if (!sp) return n;
            if (kind[sp - 1] == 0) {
                if (--rem[sp - 1] == 0) { TJ_PUT(']'); sp--; }
                else { TJ_PUT(','); done_value = 0; }
            }
            else if (phase[sp - 1] == 1) { TJ_PUT(':'); phase[sp - 1] = 2; done_value = 0; }
            else {
                if (--rem[sp - 1] == 0) { TJ_PUT('}'); sp--; }
                else { phase[sp - 1] = 0; done_value = 0; }
            }
        }
    }
}

/* sizing pass (o == NULL): packs the event, leaves plen[i]; emission pass: converts from the packed map.
 * Text of event i: json "," + map (the host turns the first ',' into '[' and appends ']'), stream: map, lines: map + "\n". */
FLB_HDN uint32_t tj_event(const struct tj_env *e, uint32_t i, uint8_t *o)
{
    uint8_t *b = e->scr + e->off[i] + (size_t) i * e->scr_pad;
    uint32_t n = 0, undef = 0, pl;
    if (e->kind[i] != 0) {
        /* an event the decoder steps over; group markers (seconds -1: start, -2: end) are listed for the host */
        if (!o && e->kind[i] == 1 && !e->groups) {
            const uint8_t *p = e->in + e->off[i], *q = p + 1;
            struct mp_tok t;
            long long sec = 0;
            if (*q == 0x92) q++;
            mp_token(q, p + e->len[i], &t);
            if (t.type == MPT_EXT) sec = (long long) (int32_t) mp_be32(q + t.hdr);
            else if (t.type == MPT_INT || t.type == MPT_UINT) sec = (long long) (int32_t) (uint32_t) t.u;
            else if (t.type == MPT_F64) { union { uint64_t u; double d; } cv; cv.u = t.u; sec = (long long) (int32_t) (uint32_t) mp_d2i64(cv.d); }
            if (sec == -1 || sec == -2) {
#ifdef __CUDA_ARCH__
                const unsigned long long at = atomicAdd(e->n_marks, 1ull);
#else
                const unsigned long long at = (*e->n_marks)++;
#endif
                if (at < e->marks_cap) { e->marks[2 * at] = i * 2u + (sec == -1 ? 1u : 0u); e->marks[2 * at + 1] = e->len[i]; }
                else CH_ATOMIC_OR(e->err, FLBGPU_E_JSONGROUP);
            }
        }
        return 0;
    }
    if (!o) { pl = tj_pack_event(e, i, b); e->plen[i] = pl; }
    else pl = e->plen[i];
    if (e->json_format == TJ_FORMAT_JSON) TJ_PUT(',');
    {
        const uint32_t m = tj_convert(e, b, b + pl, o ? o + n : 0, &undef);
        if (!m) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
        n += m;
    }
    if (e->json_format == TJ_FORMAT_LINES) TJ_PUT('\n');
    if (undef && !o) CH_ATOMIC_ADD(e->undefined, 1);
    return n;
}

#endif
