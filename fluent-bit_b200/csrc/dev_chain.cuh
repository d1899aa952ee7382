/* dev_chain.cuh -- one log record through the configured filter chain (one lane = one
 * record).  The record is held as a FIELD LIST of references into the input chunk /
 * the program's constant pool; every filter is an operation on that list and a single
 * encoder at the end writes msgpack.  The same function runs twice per record:
 * EMIT=false measures (output size, keep/drop, chunk-level evidence) and EMIT=true
 * writes at the offset the prefix sum assigned.
 *
 * Reference behaviour mirrored here (file:line in /root/reference):
 *   record framing ........ src/flb_log_event_decoder.c:180-297, :309-456
 *   record encoding ....... src/flb_log_event_encoder.c:172-218 (92 92 d7 00 sec nsec meta body)
 *   filter_parser ......... plugins/filter_parser/filter_parser.c:174-442
 *   regex parser .......... src/flb_parser_regex.c:44-227, src/flb_regex.c:28-58,294-316
 *   typecast .............. src/flb_parser.c:1280-1377
 *   filter_grep ........... plugins/filter_grep/grep.c:167-194,250-284,286-392
 *   record accessor ....... src/flb_ra_key.c:108-134,151-240,303-340,374-435
 *   filter_modify ......... plugins/filter_modify/modify.c:523-953 (conditions), :955-1339 (rules),
 *                           :1341-1457 (sequential application)
 *   filter_record_modifier  plugins/filter_record_modifier/filter_modifier.c:213-279,298-486
 */
#ifndef FLBGPU_DEV_CHAIN_CUH
#define FLBGPU_DEV_CHAIN_CUH

#include <stdint.h>
#include "flbgpu_prog.h"
#include "dev_msgpack.cuh"
#include "dev_regex.cuh"
#include "dev_time.cuh"
#include "dev_json.cuh"

#define CH_MAXF        64
#define CH_RX_STACK    192      /* 32-bit words of backtrack stack per lane */
#define CH_RX_BUDGET   4000000u /* VM steps per search: guards against catastrophic backtracking */

#ifdef __CUDA_ARCH__
/* evidence / error words: every record would hit the same word; once the bits are there (after the
 * first few warps) a plain cached read is all it takes */
#define CH_ATOMIC_OR(p, v)  do { if ((*(volatile const unsigned int *) (p) & (unsigned int) (v)) != (unsigned int) (v)) \
                                     atomicOr((unsigned int *) (p), (unsigned int) (v)); } while (0)
#define CH_ATOMIC_ADD(p, v) atomicAdd((unsigned long long *) (p), (unsigned long long) (v))
#else
#define CH_ATOMIC_OR(p, v)  (*(p) |= (v))
#define CH_ATOMIC_ADD(p, v) (*(p) += (v))
#endif

/* reference = kind:4 | len:28 | off:32 */
typedef uint64_t ref_t;
enum { RK_MP_IN = 1, RK_MP_CONST, RK_MP_SCR, RK_STR_IN, RK_INT_IN, RK_HEX_IN, RK_FLT_IN, RK_TRUE, RK_FALSE,
       RK_STR_SCR };
FLB_HD ref_t mkref(uint32_t kind, uint32_t off, uint32_t len) { return ((uint64_t) kind << 60) | ((uint64_t) (len & 0x0fffffffu) << 32) | off; }
FLB_HD uint32_t r_kind(ref_t r) { return (uint32_t) (r >> 60); }
FLB_HD uint32_t r_len(ref_t r) { return (uint32_t) (r >> 32) & 0x0fffffffu; }
FLB_HD uint32_t r_off(ref_t r) { return (uint32_t) r; }

enum { ST_CANON = 0, ST_MAP32 = 1, ST_PRESET = 2 };

struct ch_env {
    const uint8_t *in;
    uint32_t in_len;
    const uint8_t *blob;
    uint8_t *scr;
    uint32_t scr_mul;         /* scratch bytes per record byte (the record's region starts at scr + scr_mul * record offset) */
    int32_t *capcache;        /* capture cache, one COLUMN per word: word w of record r at capcache[w * cap_n + r], so that the
                                 lanes of a warp (adjacent records) touch adjacent words -- coalesced in both passes */
    uint32_t cap_stride;      /* words per record */
    uint32_t cap_n;           /* records per column */
    int64_t now;
    uint32_t assume;          /* bit k: filter k is chunk-level MODIFIED */
    uint32_t active;          /* bit k: filter k is routed this chunk (Match / Match_Regex), else skipped like flb_filter_do() does */
    uint32_t *fl_flags;       /* [n_filters] CHF_* evidence (evaluation pass only) */
    uint32_t *err;            /* FLBGPU_E_* */
    struct l2m_table l2m;     /* log_to_metrics delta table of this call (hash == NULL: none) */
    int32_t *prep;            /* parser report (flbgpu_parser_do): 6 ints per record -- parsed flag, position consumed,
                                 seconds lo / hi, nanoseconds, spare -- or NULL */
    uint32_t *esize;          /* chains with a rewrite_tag filter: bytes of the record's entry in the re-tagged stream (0 = none) */
    const uint8_t *tag;       /* the tag of this call (rewrite_tag templates: $TAG, $TAG[n]) */
    uint32_t tag_len;
};

/* What differs from lane to lane.  struct ch_env itself is the same for every record of a launch and is read where the
 * kernel parameters live (constant bank); only these few words sit in the lane's registers / local memory. */
struct ch_lane {
    uint8_t *scr;             /* this record's scratch region (ch_env.scr + scr_mul * record offset), or NULL */
    uint32_t dec_at;          /* where the field decoders write inside it (behind the parser's part) */
    const uint32_t *bm;       /* JSON stage-1 bitmap of the warp's byte range (shared memory), or NULL */
    uint32_t bm_base, bm_end; /* input offsets it covers */
    uint32_t defer_ok;        /* a record the stage-2 walker cannot take returns CH_DEFER instead of being scanned in place */
    /* log_to_metrics follow-up (k_l2m_fixup): probe != NULL: report whether this record assigns a metric value (probe[0] = 1,
     * the value's bits in probe[1]) and touch nothing; forced != NULL: the value to observe for a record whose text does not convert */
    unsigned long long *l2m_probe;
    const double *l2m_forced;
    uint32_t raw_lo;          /* chains with a rewrite_tag filter: where the bytes the reference's decoder consumed for this record begin
                                 (the end of the previous decoded record: events the decoder steps over in between belong to it) */
};

#define CW(p, x) (p)[(size_t) (x) * cs]          /* word x of a record's capture-cache row (cs = e->cap_n) */

struct ch_rec {
    int64_t ts_sec, ts_nsec;
    ref_t meta;
    int nf;
    ref_t k[CH_MAXF], v[CH_MAXF];
    uint32_t kh[CH_MAXF];        /* ch_khash() of each STR/BIN key (0 for other key types): key tests compare this first */
    int style;
    uint32_t preset_n;
    int reenc;
};

FLB_HD const uint8_t *ref_ptr(const struct ch_env *e, const struct ch_lane *ln, ref_t r)
{
    uint32_t k = r_kind(r);
    if (k == RK_MP_CONST) return e->blob + r_off(r);
    if (k == RK_MP_SCR || k == RK_STR_SCR) return ln->scr + r_off(r);
    return e->in + r_off(r);
}

/* string view of a key/value: 1 STR, 2 BIN, 3 true, 4 false, 0 anything else */
FLB_HD int ref_view(const struct ch_env *e, const struct ch_lane *ln, ref_t r, const uint8_t **p, uint32_t *n)
{
    uint32_t k = r_kind(r);
    const uint8_t *b = ref_ptr(e, ln, r);
    if (k == RK_STR_IN || k == RK_STR_SCR) { *p = b; *n = r_len(r); return 1; }
    if (k == RK_TRUE) return 3;
    if (k == RK_FALSE) return 4;
    if (k == RK_MP_IN || k == RK_MP_CONST || k == RK_MP_SCR) {
        struct mp_tok t;
        if (mp_token(b, b + r_len(r), &t) != 0) return 0;
        if (t.type == MPT_STR) { *p = b + t.hdr; *n = t.len; return 1; }
        if (t.type == MPT_BIN) { *p = b + t.hdr; *n = t.len; return 2; }
        if (t.type == MPT_BOOL) return t.u ? 3 : 4;
    }
    return 0;
}

/* O(1) fingerprint of a key (length, first, middle and last byte), never 0.  Only a pre-filter: a key
 * test compares the bytes when the fingerprints agree.  key_hash() in runtime.c is the same function. */
FLB_HD uint32_t ch_khash(const uint8_t *s, uint32_t n)
{
    uint32_t h = n * 2654435761u;
    if (n) h ^= (uint32_t) s[0] ^ ((uint32_t) s[n - 1] << 8) ^ ((uint32_t) s[n >> 1] << 16);
    return h | 1u;
}
FLB_HD uint32_t ref_khash(const struct ch_env *e, const struct ch_lane *ln, ref_t r)
{
    const uint8_t *p; uint32_t n;
    int t = ref_view(e, ln, r, &p, &n);
    return (t == 1 || t == 2) ? ch_khash(p, n) : 0u;
}

FLB_HD int bytes_eq(const uint8_t *a, const uint8_t *b, uint32_t n)
{
    /* Callers come here after the fingerprints agreed, so the strings are almost always equal: compare in groups of eight
     * without a branch per byte, so that the loads of a group are in flight together instead of one behind the other. */
    uint32_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint32_t d = (uint32_t) (a[i] ^ b[i]) | (uint32_t) (a[i + 1] ^ b[i + 1]) | (uint32_t) (a[i + 2] ^ b[i + 2]) | (uint32_t) (a[i + 3] ^ b[i + 3]) |
                     (uint32_t) (a[i + 4] ^ b[i + 4]) | (uint32_t) (a[i + 5] ^ b[i + 5]) | (uint32_t) (a[i + 6] ^ b[i + 6]) | (uint32_t) (a[i + 7] ^ b[i + 7]);
        if (d) return 0;
    }
    {
        uint32_t d = 0;
        for (; i < n; i++) d |= (uint32_t) (a[i] ^ b[i]);
        return d == 0;
    }
}

/* strtoll(s, NULL, 10) on a counted string (atoll in flb_parser_typecast) */
FLB_HD int64_t ch_atoll(const uint8_t *s, uint32_t n)
{
    uint32_t i = 0;
    int neg = 0;
    uint64_t v = 0, lim;
    while (i < n && dt_isspace(s[i])) i++;
    if (i < n && (s[i] == '+' || s[i] == '-')) { neg = s[i] == '-'; i++; }
    lim = neg ? 9223372036854775808ull : 9223372036854775807ull;
    if (n - i <= 18) {                            /* cannot reach the limit: no check per digit */
        for (; i < n && s[i] >= '0' && s[i] <= '9'; i++) v = v * 10 + (uint64_t) (s[i] - '0');
        return neg ? (int64_t) (0 - v) : (int64_t) v;
    }
    for (; i < n && s[i] >= '0' && s[i] <= '9'; i++) {
        uint64_t d = s[i] - '0';
        if (v > (lim - d) / 10) { v = lim; while (i < n && s[i] >= '0' && s[i] <= '9') i++; break; }
        v = v * 10 + d;
    }
    return neg ? (int64_t) (0 - v) : (int64_t) v;
}

/* strtoull(s, NULL, 16) */
FLB_HD uint64_t ch_strtoull16(const uint8_t *s, uint32_t n)
{
    uint32_t i = 0;
    int neg = 0, any = 0, ovf = 0;
    uint64_t v = 0;
    while (i < n && dt_isspace(s[i])) i++;
    if (i < n && (s[i] == '+' || s[i] == '-')) { neg = s[i] == '-'; i++; }
    if (i + 1 < n && s[i] == '0' && (s[i + 1] == 'x' || s[i + 1] == 'X')) {
        int h = (i + 2 < n) ? s[i + 2] : 0;
        if ((h >= '0' && h <= '9') || ((h | 0x20) >= 'a' && (h | 0x20) <= 'f')) i += 2;
    }
    for (; i < n; i++) {
        int c = s[i], d;
        if (c >= '0' && c <= '9') d = c - '0';
        else if ((c | 0x20) >= 'a' && (c | 0x20) <= 'f') d = (c | 0x20) - 'a' + 10;
        else break;
        any = 1;
        if (v >> 60) ovf = 1;
        v = (v << 4) | (uint64_t) d;
    }
    (void) any;
    if (ovf) return 0xffffffffffffffffull;
    return neg ? (uint64_t) (0 - v) : v;
}

/* ------------------------------------------------------------ emission */
/* size (o == NULL) or bytes of one field reference */
FLB_HD uint32_t ref_emit(const struct ch_env *e, const struct ch_lane *ln, ref_t r, uint8_t *o)
{
    uint32_t k = r_kind(r), n = r_len(r);
    const uint8_t *b = ref_ptr(e, ln, r);
    switch (k) {
    case RK_MP_IN:
        return mp_canon(b, b + n, o, 0);
    case RK_MP_CONST:
    case RK_MP_SCR:
        if (o) mp_copy(o, b, n);
        return n;
    case RK_STR_IN:
    case RK_STR_SCR:
        if (o) { uint32_t h = mp_put_str_hdr(o, n); mp_copy(o + h, b, n); }
        return mp_str_hdr_size(n) + n;
    case RK_INT_IN: {
        int64_t v = ch_atoll(b, n);
        if (o) mp_put_int(o, v);
        return mp_int_size(v);
    }
    case RK_HEX_IN: {
        uint64_t v = ch_strtoull16(b, n);
        if (o) mp_put_uint(o, v);
        return mp_uint_size(v);
    }
    case RK_FLT_IN: {
        int ok;                                    /* decided in the sizing pass too: that is where refusals are read */
        const uint64_t u = dj_strtod(b, (int) n, &ok);
        if (!ok) CH_ATOMIC_OR(e->err, FLBGPU_E_FLOAT);
        if (o) { o[0] = 0xcb; mp_put_be64(o + 1, u); }
        return 9;
    }
    case RK_TRUE: if (o) o[0] = 0xc3; return 1;
    case RK_FALSE: if (o) o[0] = 0xc2; return 1;
    }
    return 0;
}

FLB_HD uint32_t rec_emit(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, uint8_t *o)
{
    uint32_t n = 0;
    int i;
    if (o) {
        o[0] = 0x92; o[1] = 0x92; o[2] = 0xd7; o[3] = 0x00;
        mp_put_be32(o + 4, (uint32_t) rc->ts_sec);
        mp_put_be32(o + 8, (uint32_t) rc->ts_nsec);
    }
    n = 12;
    n += ref_emit(e, ln, rc->meta, o ? o + n : 0);
    if (rc->style == ST_MAP32) {
        if (o) { o[n] = 0xdf; mp_put_be32(o + n + 1, (uint32_t) rc->nf); }
        n += 5;
    }
    else if (rc->style == ST_PRESET) {
        /* header type chosen for preset_n (msgpack_pack_map(n)), count patched afterwards
         * (src/flb_parser_regex.c:182-199) */
        if (rc->preset_n < 16) { if (o) o[n] = 0x80 | (uint8_t) rc->nf; n += 1; }
        else if (rc->preset_n < 65536) { if (o) { o[n] = 0xde; mp_put_be16(o + n + 1, (uint32_t) rc->nf); } n += 3; }
        else { if (o) { o[n] = 0xdf; mp_put_be32(o + n + 1, (uint32_t) rc->nf); } n += 5; }
    }
    else {
        if (o) mp_put_map_hdr(o + n, (uint32_t) rc->nf);
        n += mp_cnt_hdr_size((uint32_t) rc->nf);
    }
    for (i = 0; i < rc->nf; i++) {
        n += ref_emit(e, ln, rc->k[i], o ? o + n : 0);
        n += ref_emit(e, ln, rc->v[i], o ? o + n : 0);
    }
    return n;
}

/* ------------------------------------------------------------- decoding */
/* Frame check of ONE record starting at p: returns its end or NULL.
 * kind: 0 normal, 1 skipped by the decoder (negative 32-bit seconds). */
FLB_HD const uint8_t *rec_frame(const uint8_t *p, const uint8_t *end, int *kind)
{
    struct mp_tok t;
    const uint8_t *q;
    int64_t sec = 0;
    if (end - p < 3 || p[0] != 0x92) return 0;
    q = p + 1;
    if (*q == 0x92) q++;                        /* [ [ts, meta], body ] */
    else if ((*q & 0xf0) == 0x90 || *q == 0xdc || *q == 0xdd) return 0;   /* header array of another size */
    if (q >= end || mp_token(q, end, &t) != 0) return 0;
    if (t.type == MPT_UINT) sec = (int64_t) t.u;
    else if (t.type == MPT_INT) { if ((int64_t) t.u < 0) return 0; sec = (int64_t) t.u; }
    else if (t.type == MPT_F64) { union { uint64_t u; double d; } cv; cv.u = t.u; sec = mp_d2i64(cv.d); }   /* whether the decoder steps over it: as x86-64 converts */
    else if (t.type == MPT_EXT) {
        if (t.ext_type != 0 || t.len != 8 || (size_t) (end - q) < t.hdr + 8u) return 0;
        sec = (int64_t) (int32_t) mp_be32(q + t.hdr);
    }
    else return 0;
    q += t.hdr + (t.type == MPT_EXT ? t.len : 0);
    if (p[1] == 0x92) {                          /* metadata must be a map */
        if (q >= end || mp_token(q, end, &t) != 0 || t.type != MPT_MAP) return 0;
        q = mp_skip_lim(q, end, 2);              /* open around it: the event array and the header array */
        if (!q) return 0;
    }
    if (q >= end || mp_token(q, end, &t) != 0 || t.type != MPT_MAP) return 0;
    q = mp_skip_lim(q, end, 1);
    if (!q) return 0;
    *kind = ((int32_t) (uint32_t) sec) < 0 ? 1 : 0;
    return q;
}

/* A candidate at p is the HEADER ARRAY of a v2 record, not a record, when the byte
 * before it starts a well-formed [[ts, meta], body] frame: "[ts, meta]" on its own has
 * the shape of a legacy [ts, body] event.  (If p-1 frames as v2, then p cannot also be
 * a record start: the outer body would have to be both a map and an array.) */
FLB_HD int rec_is_shadowed(const uint8_t *base, const uint8_t *p, const uint8_t *end)
{
    int kind;
    if (p == base || p[-1] != 0x92) return 0;
    return rec_frame(p - 1, end, &kind) != 0;
}

/* Split a framed record into timestamp, metadata and the top-level field list.
 * Returns 0, or -1 when it has more than CH_MAXF keys. */
FLB_HD int rec_decode(const struct ch_env *e, const struct ch_lane *ln, uint32_t off, uint32_t len, struct ch_rec *rc, uint32_t empty_map_off)
{
    const uint8_t *p = e->in + off, *end = p + len, *q = p + 1, *nx;
    struct mp_tok t;
    uint32_t i;
    int v2 = (*q == 0x92);
    if (v2) q++;
    mp_token(q, end, &t);
    rc->ts_nsec = 0;
    if (t.type == MPT_UINT || t.type == MPT_INT) rc->ts_sec = (int64_t) t.u;
    else if (t.type == MPT_F64) {
        union { uint64_t u; double d; } cv;
        cv.u = t.u;
        rc->ts_sec = (int64_t) cv.d;
        rc->ts_nsec = (int64_t) ((cv.d - (double) rc->ts_sec) * 1000000000.0);
    }
    else {
        rc->ts_sec = (int64_t) (int32_t) mp_be32(q + t.hdr);
        rc->ts_nsec = (int64_t) (int32_t) mp_be32(q + t.hdr + 4);
    }
    q += t.hdr + (t.type == MPT_EXT ? t.len : 0);
    if (v2) {
        nx = mp_skip(q, end);
        rc->meta = mkref(RK_MP_IN, (uint32_t) (q - e->in), (uint32_t) (nx - q));
        q = nx;
    }
    else rc->meta = mkref(RK_MP_CONST, empty_map_off, 1);
    mp_token(q, end, &t);
    q += t.hdr;
    rc->style = ST_CANON; rc->preset_n = 0; rc->reenc = 0;
    if (t.len > CH_MAXF) { rc->nf = 0; return -1; }
    rc->nf = (int) t.len;
    for (i = 0; i < t.len; i++) {
        nx = mp_skip(q, end);
        rc->k[i] = mkref(RK_MP_IN, (uint32_t) (q - e->in), (uint32_t) (nx - q));
        q = nx;
        nx = mp_skip(q, end);
        rc->v[i] = mkref(RK_MP_IN, (uint32_t) (q - e->in), (uint32_t) (nx - q));
        q = nx;
        rc->kh[i] = ref_khash(e, ln, rc->k[i]);
    }
    return 0;
}

/* -------------------------------------------------------- record accessor */
/* ra_key_val_id(): index of the LAST field whose key is a STR equal to name */
FLB_HD int ra_find(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, const uint8_t *name, uint32_t nlen)
{
    const uint32_t h = ch_khash(name, nlen);
    int i;
    for (i = rc->nf - 1; i >= 0; i--) {
        const uint8_t *kp; uint32_t kn;
        if (rc->kh[i] != h) continue;
        if (ref_view(e, ln, rc->k[i], &kp, &kn) != 1) continue;
        if (kn == nlen && bytes_eq(kp, name, nlen)) return i;
    }
    return -1;
}

/* subkey_to_object() over raw msgpack: on success *vp..*ve is the value object and
 * *key_is_null tells whether the last step was an array index */
FLB_HDN int ra_walk_sub(const struct ch_env *e, const struct ch_lane *ln, const struct cf_ra *ra, const uint8_t *p, const uint8_t *end,
                       const uint8_t **vp, const uint8_t **ve, int *key_is_null)
{
    const struct cf_ra_sub *sub = (const struct cf_ra_sub *) (e->blob + ra->sub_off);
    uint32_t levels = ra->n_sub, matched = 0, s;
    const uint8_t *cur = p, *cur_end = end;
    struct mp_tok t;
    if (levels == 0) return -1;
    for (s = 0; s < levels; s++) {
        if (mp_token(cur, cur_end, &t) != 0) return -1;
        if (sub[s].is_index) {
            const uint8_t *q;
            uint32_t i;
            if (t.type != MPT_ARRAY) return -1;
            if (sub[s].index == 0x7fffffffu || sub[s].index >= t.len) return -1;
            q = cur + t.hdr;
            for (i = 0; i < sub[s].index; i++) q = mp_skip(q, cur_end);
            cur = q; cur_end = mp_skip(q, cur_end);
            *key_is_null = 1;
            matched++;
            if (matched == levels) break;
            continue;
        }
        if (t.type != MPT_MAP) break;
        {
            /* last matching STR key wins */
            const uint8_t *q = cur + t.hdr, *found = 0, *found_end = 0;
            const uint8_t *want = e->blob + sub[s].str_off;
            uint32_t i;
            for (i = 0; i < t.len; i++) {
                struct mp_tok kt;
                const uint8_t *kq = q, *vq;
                mp_token(q, cur_end, &kt);
                vq = mp_skip(q, cur_end);
                q = mp_skip(vq, cur_end);
                if (kt.type == MPT_STR && kt.len == sub[s].str_len && bytes_eq(kq + kt.hdr, want, kt.len)) {
                    found = vq; found_end = q;
                }
            }
            if (!found) continue;               /* "try next entry" (src/flb_ra_key.c:214) */
            cur = found; cur_end = found_end;
            *key_is_null = 0;
            matched++;
            if (matched == levels) break;
        }
    }
    if (matched == 0 || levels != matched) return -1;
    *vp = cur; *ve = cur_end;
    return 0;
}

/* flb_ra_key_value_get(): 0 found (flags: *okey_null), -1 not found.
 * On success either *top >= 0 (the top-level field itself) or *vp and *ve (nested). */
FLB_HD int ra_get(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, const struct cf_ra *ra, int *top,
                  const uint8_t **vp, const uint8_t **ve, int *okey_null)
{
    int i = ra_find(e, ln, rc, e->blob + ra->key_off, ra->key_len);
    uint32_t k;
    *top = -1; *okey_null = 0;
    if (i < 0) return -1;
    k = r_kind(rc->v[i]);
    if (ra->n_sub > 0 && (k == RK_MP_IN || k == RK_MP_CONST || k == RK_MP_SCR)) {
        const uint8_t *b = ref_ptr(e, ln, rc->v[i]);
        struct mp_tok t;
        if (mp_token(b, b + r_len(rc->v[i]), &t) == 0 && (t.type == MPT_MAP || t.type == MPT_ARRAY)) {
            return ra_walk_sub(e, ln, ra, b, b + r_len(rc->v[i]), vp, ve, okey_null);
        }
    }
    *top = i;
    return 0;
}

/* view of a located value as STR/BIN/bool (same codes as ref_view) */
FLB_HD int loc_view(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, int top, const uint8_t *vp, const uint8_t *ve,
                    const uint8_t **p, uint32_t *n)
{
    struct mp_tok t;
    if (top >= 0) return ref_view(e, ln, rc->v[top], p, n);
    if (mp_token(vp, ve, &t) != 0) return 0;
    if (t.type == MPT_STR) { *p = vp + t.hdr; *n = t.len; return 1; }
    if (t.type == MPT_BIN) { *p = vp + t.hdr; *n = t.len; return 2; }
    if (t.type == MPT_BOOL) return t.u ? 3 : 4;
    return 0;
}

FLB_HDN int rx_run(const struct ch_env *e, const struct ch_lane *ln, uint32_t rx_off, const uint8_t *s, uint32_t n, int *caps, uint32_t *stk)
{
    uint32_t budget = CH_RX_BUDGET;
    int r = rx_search((const struct rx_prog *) (e->blob + rx_off), s, (int) n, caps, stk, CH_RX_STACK, &budget);
    if (r == RX_R_ESTACK) { CH_ATOMIC_OR(e->err, FLBGPU_E_RXSTACK); return 0; }
    if (r == RX_R_EBUDGET) { CH_ATOMIC_OR(e->err, FLBGPU_E_RXBUDGET); return 0; }
    if (r == RX_R_EUNICODE) { CH_ATOMIC_OR(e->err, FLBGPU_E_RXUNICODE); return 0; }
    return r == RX_R_MATCH;
}

/* flb_ra_regex_match() > 0 ? */
FLB_HD int ra_regex_match(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, uint32_t ra_off, uint32_t rx_off,
                          int *caps, uint32_t *stk)
{
    const struct cf_ra *ra = (const struct cf_ra *) (e->blob + ra_off);
    const uint8_t *vp = 0, *ve = 0, *s;
    uint32_t n;
    int top, kn;
    if (ra_get(e, ln, rc, ra, &top, &vp, &ve, &kn) != 0) return 0;
    if (loc_view(e, ln, rc, top, vp, ve, &s, &n) != 1) return 0;      /* value must be a STR */
    return rx_run(e, ln, rx_off, s, n, caps, stk);
}

/* ---------------------------------------------------------- filter_parser */
/* One regex parser over s[0,n): returns 1 parsed (fields appended to out_*), 0 not.
 * Timestamp result in *t_sec and *t_nsec (0/0 when no time was resolved). */
/* tslot (4 ints of the capture cache, or NULL): the evaluation pass stores the Time_Key lookup there
 * (state 1 ok / 2 failed, seconds lo/hi, nanoseconds) and the emission pass (use_cached) reads it
 * instead of running strptime again */
FLB_HD int pdef_regex(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, uint32_t val_off, const uint8_t *s,
                      uint32_t n, const int *caps, ref_t *ok_, ref_t *ov_, int *on, int64_t *t_sec,
                      int64_t *t_nsec, int32_t *tslot, int use_cached, uint32_t *th, int *pos)
{
    const struct cf_pname *nm = (const struct cf_pname *) (e->blob + pd->names_off);
    uint32_t i;
    int any_end = 0, cnt = 0, have_nsec = 0;
    const size_t cs = e->cap_n;
    int64_t lookup = 0, nsec_cached = 0;
    double frac = 0;
    if (pd->n_groups == 0) return 0;                 /* flb_parser_regex_do: n <= 0 -> -1 */
    /* decided before anything is written: the caller may hand in the record's own field arrays */
    for (i = 0; i < pd->n_names; i++) if (caps[2 * nm[i].group + 1] >= 0) { any_end = 1; *pos = caps[2 * nm[i].group + 1]; }   /* cb_onig_named: last_pos */
    if (!any_end) return 0;                          /* flb_regex_parse: last_pos == -1 */
    for (i = 0; i < pd->n_names; i++) {
        int b = caps[2 * nm[i].group], en = caps[2 * nm[i].group + 1];
        uint32_t vlen = (uint32_t) (en - b);
        const uint8_t *v = s + b;
        if (vlen == 0 && pd->skip_empty) continue;
        if (pd->has_time && nm[i].is_time && use_cached && tslot && CW(tslot, 0)) {
            if (CW(tslot, 0) == 2) continue;
            lookup = (int64_t) (((uint64_t) (uint32_t) CW(tslot, 2) << 32) | (uint32_t) CW(tslot, 1));
            nsec_cached = CW(tslot, 3); have_nsec = 1;
            if (!pd->time_keep) continue;
        }
        else if (pd->has_time && nm[i].is_time) {
            struct dt_tm tm;
            struct dt_parser tp;
            double ns;
            int r;
            tm.sec = tm.min = tm.hour = tm.mday = tm.mon = tm.year = tm.wday = tm.yday = tm.isdst = 0;
            tm.gmtoff = 0;
            tp.fmt = (const char *) (e->blob + pd->fmt_off);
            tp.frac_fmt = pd->has_frac ? (const char *) (e->blob + pd->frac_off) : 0;
            tp.with_year = (int) pd->time_with_year; tp.with_tz = (int) pd->time_with_tz;
            tp.strict = (int) pd->time_strict; tp.offset = pd->time_offset; tp.fast_apache = (pd->has_time & 2) != 0; tp.tfast = pd->tfast_off ? e->blob + pd->tfast_off : 0;
            r = dt_time_lookup(vlen ? v : s, vlen, e->now, &tp, &tm, &ns);
            if (r == -1) { if (tslot && !use_cached) CW(tslot, 0) = 2; continue; }
            frac = ns;
            lookup = dt_timegm(&tm) - tm.gmtoff;
            if (tslot && !use_cached) {
                CW(tslot, 0) = 1; CW(tslot, 1) = (int32_t) (uint32_t) lookup; CW(tslot, 2) = (int32_t) (uint32_t) ((uint64_t) lookup >> 32);
#ifdef __CUDA_ARCH__
                CW(tslot, 3) = (int32_t) (int64_t) __dmul_rn(frac, 1000000000.0);
#else
                CW(tslot, 3) = (int32_t) (int64_t) (frac * 1000000000.0);
#endif
            }
            if (!pd->time_keep) continue;
        }
        if (cnt >= CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
        ok_[cnt] = mkref(RK_MP_CONST, nm[i].kmp_off, nm[i].kmp_len);
        th[cnt] = nm[i].hash;
        {
            uint32_t kind = RK_STR_IN, voff = val_off + (uint32_t) (vlen ? b : 0);
            if (nm[i].cast == FLBGPU_TYPE_INT) kind = RK_INT_IN;
            else if (nm[i].cast == FLBGPU_TYPE_HEX) kind = RK_HEX_IN;
            else if (nm[i].cast == FLBGPU_TYPE_FLOAT) kind = RK_FLT_IN;
            else if (nm[i].cast == FLBGPU_TYPE_BOOL) {
                if (vlen >= 4 && dt_lower(v[0]) == 't' && dt_lower(v[1]) == 'r' && dt_lower(v[2]) == 'u' && dt_lower(v[3]) == 'e') kind = RK_TRUE;
                else if (vlen >= 5 && dt_lower(v[0]) == 'f' && dt_lower(v[1]) == 'a' && dt_lower(v[2]) == 'l' && dt_lower(v[3]) == 's' && dt_lower(v[4]) == 'e') kind = RK_FALSE;
            }
            ov_[cnt] = mkref(kind, voff, vlen);
        }
        cnt++;
    }
    *on = cnt;
    *t_sec = lookup;
    if (have_nsec) { *t_nsec = nsec_cached; return 1; }
#ifdef __CUDA_ARCH__
    *t_nsec = (int64_t) __dmul_rn(frac, 1000000000.0);
#else
    *t_nsec = (int64_t) (frac * 1000000000.0);
#endif
    return 1;
}

/* Types cast of a parsed (key, value) pair: flb_parser_typecast(), src/flb_parser.c:1280-1377 */
FLB_HD ref_t cast_value(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, const uint8_t *key, uint32_t klen,
                        const uint8_t *v, uint32_t voff, uint32_t vlen)
{
    const struct cf_ptype *ty = (const struct cf_ptype *) (e->blob + pd->types_off);
    uint32_t i;
    for (i = 0; i < pd->n_types; i++) {
        if (ty[i].key_len != klen || !bytes_eq(e->blob + ty[i].key_off, key, klen)) continue;
        if (ty[i].type == FLBGPU_TYPE_INT) return mkref(RK_INT_IN, voff, vlen);
        if (ty[i].type == FLBGPU_TYPE_HEX) return mkref(RK_HEX_IN, voff, vlen);
        if (ty[i].type == FLBGPU_TYPE_FLOAT) return mkref(RK_FLT_IN, voff, vlen);
        if (ty[i].type == FLBGPU_TYPE_BOOL) {
            if (vlen >= 4 && dt_lower(v[0]) == 't' && dt_lower(v[1]) == 'r' && dt_lower(v[2]) == 'u' && dt_lower(v[3]) == 'e') return mkref(RK_TRUE, 0, 0);
            if (vlen >= 5 && dt_lower(v[0]) == 'f' && dt_lower(v[1]) == 'a' && dt_lower(v[2]) == 'l' && dt_lower(v[3]) == 's' && dt_lower(v[4]) == 'e') return mkref(RK_FALSE, 0, 0);
        }
        break;
    }
    return mkref(RK_STR_IN, voff, vlen);
}

FLB_HDN int pdef_time(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, const uint8_t *v, uint32_t vlen,
                     int64_t *lookup, double *frac)
{
    struct dt_tm tm;
    struct dt_parser tp;
    double ns;
    tm.sec = tm.min = tm.hour = tm.mday = tm.mon = tm.year = tm.wday = tm.yday = tm.isdst = 0;
    tm.gmtoff = 0;
    tp.fmt = (const char *) (e->blob + pd->fmt_off);
    tp.frac_fmt = pd->has_frac ? (const char *) (e->blob + pd->frac_off) : 0;
    tp.with_year = (int) pd->time_with_year; tp.with_tz = (int) pd->time_with_tz;
    tp.strict = (int) pd->time_strict; tp.offset = pd->time_offset; tp.fast_apache = (pd->has_time & 2) != 0; tp.tfast = pd->tfast_off ? e->blob + pd->tfast_off : 0;
    if (dt_time_lookup(v, vlen, e->now, &tp, &tm, &ns) == -1) return -1;
    *frac = ns;
    *lookup = dt_timegm(&tm) - tm.gmtoff;
    return 0;
}

FLB_HD int64_t frac_to_nsec(double frac)
{
#ifdef __CUDA_ARCH__
    return (int64_t) __dmul_rn(frac, 1000000000.0);
#else
    return (int64_t) (frac * 1000000000.0);
#endif
}

/* ltsv_parser(), src/flb_parser_ltsv.c:82-197.  label bytes [0-9A-Za-z_.-] (:43-60),
 * field bytes = everything but NUL, TAB, LF, CR (:62-79). */
FLB_HD int ltsv_label(uint32_t c) { return (c >= '0' && c <= '9') || ((c | 0x20) >= 'a' && (c | 0x20) <= 'z') || c == '_' || c == '.' || c == '-'; }
FLB_HD int ltsv_field(uint32_t c) { return c != 0 && c != 9 && c != 10 && c != 13; }

FLB_HDN int pdef_ltsv(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, uint32_t val_off, const uint8_t *s, uint32_t n,
                     ref_t *ok_, ref_t *ov_, int *on, int64_t *t_sec, int64_t *t_nsec, int *pos)
{
    uint32_t c = 0;
    int cnt = 0;
    int64_t lookup = 0;
    double frac = 0;
    while (c < n) {
        uint32_t label = c, label_len, field, field_len;
        while (c < n && ltsv_label(s[c])) c++;
        label_len = c - label;
        if (c == n) break;
        if (s[c] != ':') break;
        c++;
        field = c;
        while (c < n && ltsv_field(s[c])) c++;
        field_len = c - field;
        if (label_len > 0) {
            int time_found = 0;
            if (pd->has_time && label_len == pd->time_key_len && field_len > 0 &&
                bytes_eq(s + label, e->blob + pd->time_key_off, label_len)) {
                if (pdef_time(e, ln, pd, s + field, field_len, &lookup, &frac) != 0) return 0;
                time_found = 1;
            }
            if (!time_found || pd->time_keep) {
                if (cnt >= CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
                ok_[cnt] = mkref(RK_STR_IN, val_off + label, label_len);
                ov_[cnt] = pd->n_types ? cast_value(e, ln, pd, s + label, label_len, s + field, val_off + field, field_len)
                                       : mkref(RK_STR_IN, val_off + field, field_len);
                cnt++;
            }
        }
        if (c == n) break;
        if (s[c] == '\t') c++;
        if (c == n) break;
        if (s[c] == '\r' || s[c] == '\n') {          /* the line end is consumed: CR, CR LF or LF (:180-193) */
            if (s[c] == '\r') { c++; if (c < n && s[c] == '\n') c++; } else c++;
            break;
        }
    }
    if (cnt == 0) return 0;
    *on = cnt; *t_sec = lookup; *t_nsec = frac_to_nsec(frac); *pos = (int) c;      /* last_byte: where the scan stopped */
    return 1;
}

/* flb_unescape_string_utf8() followed by strlen(), src/flb_unescape.c:40-271: what logfmt does to a
 * quoted value that contains a backslash (src/flb_parser_logfmt.c:195-214).  Decodes s[0,n) to o and
 * returns the length up to the first NUL the decoding produced. */
FLB_HD uint32_t lf_hexv(uint32_t c)
{
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return 0xffu;
}
FLB_HD uint32_t lf_sx(uint32_t b) { return (b & 0x80u) ? (b | 0xffffff00u) : b; }     /* (uint32_t)(signed char) */

/* the decoded bytes, NULs included: what flb_unescape_string_utf8() returns */
FLB_HD uint32_t lf_unescape_raw(const uint8_t *s, uint32_t n, uint8_t *o)
{
    uint32_t in = 0, out = 0;
    while (in < n && s[in]) {
        uint32_t ch, used = 1, len;
        if (s[in] == '\\' && in + 1 < n) {
            const uint8_t *q = s + in + 1;
            const uint32_t size = n - in - 1;
            uint32_t c = q[0];
            used = 2;
            switch (c) {
            case '"': case '\'': case '\\': case '/': ch = c; break;
            case 'n': ch = 10; break;
            case 'b': ch = 8; break;
            case 't': ch = 9; break;
            case 'f': ch = 12; break;
            case 'r': ch = 13; break;
            default: {
                /* u8_read_escape_sequence(): returns the characters it consumed after the backslash */
                uint32_t k = 1, dno = 0, v = 0;
                ch = lf_sx(c);
                if (c == 'v') ch = 11;
                else if (c == 'a') ch = 7;
                else if (c >= '0' && c <= '7') {
                    k = 0;
                    do { v = v * 8 + (q[k] - '0'); k++; dno++; } while (k < size && q[k] >= '0' && q[k] <= '7' && dno < 3);
                    ch = v;
                }
                else if (c == 'x') {
                    while (k < size && lf_hexv(q[k]) != 0xffu && dno < 2) { v = v * 16 + lf_hexv(q[k]); k++; dno++; }
                    if (dno > 0) ch = v;
                }
                else if (c == 'u') {
                    while (k < size && lf_hexv(q[k]) != 0xffu && dno < 4) { v = v * 16 + lf_hexv(q[k]); k++; dno++; }
                    if (dno != 4 && dno > 0) ch = 0xfffd;
                    else {
                        ch = v;                                        /* no digit at all: strtol("") = 0 */
                        if (ch >= 0xdc00 && ch <= 0xdfff) ch = 0xfffd;
                        else if (ch >= 0xd800 && ch <= 0xdbff) {
                            if (k + 2 < size && q[k] == '\\' && q[k + 1] == 'u') {
                                uint32_t low = 0;
                                dno = 0;
                                k += 2;
                                while (k < size && lf_hexv(q[k]) != 0xffu && dno < 4) { low = low * 16 + lf_hexv(q[k]); k++; dno++; }
                                if (dno != 4 && dno > 0) ch = 0xfffd;
                                else if (low >= 0xdc00 && low <= 0xdfff) ch = 0x10000 + (((ch - 0xd800) << 10) | (low - 0xdc00));
                                else ch = 0xfffd;
                            }
                            else ch = 0xfffd;
                        }
                    }
                }
                else if (c == 'U') {
                    while (k < size && lf_hexv(q[k]) != 0xffu && dno < 8) { v = v * 16 + lf_hexv(q[k]); k++; dno++; }
                    if (dno > 0) ch = v;
                }
                used = k + 1;
            }
            }
        }
        else ch = lf_sx(s[in]);
        in += used;
        len = ch < 0x80 ? 1 : ch < 0x800 ? 2 : ch < 0x10000 ? 3 : ch < 0x110000 ? 4 : 0;
        if (len > n - out) break;                                      /* "Crossing over string boundary" */
        if (len <= 1) o[out++] = (uint8_t) ch;
        else if (len == 2) { o[out++] = (uint8_t) ((ch >> 6) | 0xc0); o[out++] = (uint8_t) ((ch & 0x3f) | 0x80); }
        else if (len == 3) { o[out++] = (uint8_t) ((ch >> 12) | 0xe0); o[out++] = (uint8_t) (((ch >> 6) & 0x3f) | 0x80); o[out++] = (uint8_t) ((ch & 0x3f) | 0x80); }
        else { o[out++] = (uint8_t) ((ch >> 18) | 0xf0); o[out++] = (uint8_t) (((ch >> 12) & 0x3f) | 0x80); o[out++] = (uint8_t) (((ch >> 6) & 0x3f) | 0x80); o[out++] = (uint8_t) ((ch & 0x3f) | 0x80); }
    }
    return out;
}

FLB_HD uint32_t lf_unescape(const uint8_t *s, uint32_t n, uint8_t *o)
{
    const uint32_t out = lf_unescape_raw(s, n, o);
    uint32_t i;
    for (i = 0; i < out; i++) if (!o[i]) return i;                     /* the caller's strlen() */
    return out;
}

/* logfmt_parser(), src/flb_parser_logfmt.c:63-254.  ident bytes: > ' ' and not '=' '"' (:44-61) */
FLB_HD int logfmt_ident(uint32_t c) { return c > ' ' && c != '=' && c != '"'; }

FLB_HDN int pdef_logfmt(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, uint32_t val_off, const uint8_t *s, uint32_t n,
                       ref_t *ok_, ref_t *ov_, int *on, int64_t *t_sec, int64_t *t_nsec, int *pos)
{
    uint32_t c = 0, sk = 0;          /* sk: next free byte of the record's scratch (decoded escapes) */
    int cnt = 0;
    int64_t lookup = 0;
    double frac = 0;
    while (c < n) {
        uint32_t key, key_len, value = 0, value_len = 0;
        int value_set = 0, value_str = 0, value_escape = 0;
        while (c < n && !logfmt_ident(s[c])) c++;
        if (c == n) break;
        key = c;
        while (c < n && logfmt_ident(s[c])) c++;
        key_len = c - key;
        if (c < n && s[c] == '=') {
            value_set = 1;
            c++;
            if (c < n) {
                if (s[c] == '"') {
                    c++;
                    value = c;
                    value_str = 1;
                    while (c < n) {
                        if (s[c] != '\\' && s[c] != '"') c++;
                        else if (s[c] == '\\') { value_escape = 1; c++; if (c == n) break; c++; }
                        else break;
                    }
                    value_len = c - value;
                    if (c < n && s[c] == '"') c++;
                }
                else {
                    value = c;
                    while (c < n && logfmt_ident(s[c])) c++;
                    value_len = c - value;
                }
            }
        }
        if (key_len > 0) {
            int time_found = 0;
            if (pd->logfmt_no_bare_keys && value_len == 0 && !value_set) return 0;
            if (pd->has_time && key_len == pd->time_key_len && value_len > 0 &&
                bytes_eq(s + key, e->blob + pd->time_key_off, key_len)) {
                if (pdef_time(e, ln, pd, s + value, value_len, &lookup, &frac) != 0) return 0;
                time_found = 1;
            }
            if (!time_found || pd->time_keep) {
                if (cnt >= CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
                ok_[cnt] = mkref(RK_STR_IN, val_off + key, key_len);
                if (pd->n_types) ov_[cnt] = cast_value(e, ln, pd, s + key, key_len, s + value, val_off + value, value_len);
                else if (value_len == 0) ov_[cnt] = value_str ? mkref(RK_STR_IN, val_off + value, 0) : mkref(RK_TRUE, 0, 0);
                else if (value_escape) {
                    if (!ln->scr) { CH_ATOMIC_OR(e->err, FLBGPU_E_ESCAPE); ov_[cnt] = mkref(RK_STR_IN, val_off + value, value_len); }
                    else {
                        const uint32_t dl = lf_unescape(s + value, value_len, ln->scr + sk);
                        ov_[cnt] = mkref(RK_STR_SCR, sk, dl);
                        sk += value_len;                               /* the decoded text is never longer */
                    }
                }
                else ov_[cnt] = mkref(RK_STR_IN, val_off + value, value_len);
                cnt++;
            }
        }
        if (c == n) break;
        if (s[c] == '\r' || s[c] == '\n') {          /* src/flb_parser_logfmt.c:236-249 */
            if (s[c] == '\r') { c++; if (c < n && s[c] == '\n') c++; } else c++;
            break;
        }
    }
    if (cnt == 0) return 0;
    *on = cnt; *t_sec = lookup; *t_nsec = frac_to_nsec(frac); *pos = (int) c;
    return 1;
}

/* ---- JSON fast path ------------------------------------------------------------------
 * One flat token loop per lane, written so that a warp stays together: every iteration handles
 * one token, lanes agree on the grammar state they execute (the lowest one goes first, the rest
 * wait -- same trick as RX_ALIGN_PC), and strings are scanned eight bytes at a time.  Top-level
 * members become field references straight into the input text (plain strings, integers) so
 * nothing is copied in the common case; escapes, reals, null and nested containers are written to
 * the record's scratch.  It only ever answers "valid document, here are the fields" (1) or
 * "not an object" (0, src/flb_parser_json.c:70-85); anything unusual -- bytes >= 0x80 or < 0x20 in a
 * string, surrogates, long numbers, trailing text, depth -- returns -1 and the exact transcoder
 * (dj_parse_record, yyjson-identical) decides. */
/* Reconvergence points.  Lanes of a warp leave data-dependent loops at different times and the
 * hardware does not bring them back together by itself; CH_SYNC() is placed where every lane that
 * is still running a record is guaranteed to pass (uniform, configuration-driven loop heads), so
 * the next filter / rule / regex starts with the warp together again.  Lanes whose record was
 * dropped have returned to the kernel and exited, which __syncwarp() tolerates. */
#ifdef __CUDA_ARCH__
#define CH_STCS(p, v) __stcs((int *) (p), (int) (v))
#else
#define CH_STCS(p, v) (*(p) = (v))
#endif

#ifdef __CUDA_ARCH__
#define CH_SYNC() __syncwarp()
#else
#define CH_SYNC()
#endif

#ifdef __CUDA_ARCH__
#define DJF_ALIGN(st) { const unsigned m_ = __activemask(); \
        if ((unsigned) (st) != __reduce_min_sync(m_, (unsigned) (st))) continue; }
#else
#define DJF_ALIGN(st)
#endif
#define DJF_KEY   0
#define DJF_COLON 1
#define DJF_VAL   2
#define DJF_AFTER 3
#define DJF_DONE  4

/* first position in [p, n) holding '"', '\\', a control byte or a byte >= 0x80; n if none.
 * Reads whole aligned 8-byte words: the buffer behind s is padded (bk_alloc). */
FLB_HD int djf_scan_plain(const uint8_t *s, int p, int n)
{
    while (p < n) {
        const uintptr_t a = (uintptr_t) (s + p);
        const unsigned sh = (unsigned) (a & 7) * 8;
        uint64_t w = *(const uint64_t *) (a & ~(uintptr_t) 7), t, sp;
        w >>= sh;
        if (sh) w |= 0x6161616161616161ull << (64 - sh);
        t = w ^ 0x2222222222222222ull; sp = (t - 0x0101010101010101ull) & ~t;
        t = w ^ 0x5c5c5c5c5c5c5c5cull; sp |= (t - 0x0101010101010101ull) & ~t;
        sp |= (w - 0x2020202020202020ull) & ~w;
        sp |= w;
        sp &= 0x8080808080808080ull;
        if (sp) {
#ifdef __CUDA_ARCH__
            p += (__ffsll((long long) sp) - 1) >> 3;
#else
            p += __builtin_ctzll(sp) >> 3;
#endif
            return p < n ? p : n;
        }
        p += 8 - (int) (sh >> 3);
    }
    return n;
}

/* first position in [p, n) that is not an ASCII digit (n if none); same word-at-a-time walk */
FLB_HD int djf_scan_digits(const uint8_t *s, int p, int n)
{
    while (p < n) {
        const uintptr_t a = (uintptr_t) (s + p);
        const unsigned sh = (unsigned) (a & 7) * 8;
        uint64_t w = *(const uint64_t *) (a & ~(uintptr_t) 7), t, nd;
        w >>= sh;
        if (sh) w |= 0x3030303030303030ull << (64 - sh);
        t = w ^ 0x3030303030303030ull;                           /* digits become 0..9 */
        nd = ((t + 0x7676767676767676ull) | t) & 0x8080808080808080ull;   /* bit 7 set where t >= 10 */
        if (nd) {
#ifdef __CUDA_ARCH__
            p += (__ffsll((long long) nd) - 1) >> 3;
#else
            p += __builtin_ctzll(nd) >> 3;
#endif
            return p < n ? p : n;
        }
        p += 8 - (int) (sh >> 3);
    }
    return n;
}

/* string whose opening quote is at s[p].  Plain: *raw = 1, [*b, *b + *len) are input offsets.
 * With escapes: decoded to scr + at, *raw = 0, *len decoded bytes.  Returns the position after the
 * closing quote or -1. */
FLB_HD int djf_string(const uint8_t *s, int p, int n, uint8_t *scr, uint32_t at, int *raw, uint32_t *b, uint32_t *len)
{
    int q = djf_scan_plain(s, p + 1, n);
    uint32_t k = 0;
    if (q >= n) return -1;
    if (s[q] == '"') { *raw = 1; *b = (uint32_t) (p + 1); *len = (uint32_t) (q - p - 1); return q + 1; }
    if (s[q] != '\\') return -1;
    *raw = 0;
    {
        int i;
        for (i = p + 1; i < q; i++) scr[at + k++] = s[i];
    }
    for (;;) {
        uint32_t c;
        if (q >= n) return -1;
        c = s[q];
        if (c == '"') break;
        if (c < 0x20 || c >= 0x80) return -1;
        if (c != '\\') { scr[at + k++] = (uint8_t) c; q++; continue; }
        if (q + 1 >= n) return -1;
        c = s[q + 1];
        q += 2;
        switch (c) {
        case '"': case '\\': case '/': break;
        case 'b': c = 8; break;
        case 'f': c = 12; break;
        case 'n': c = 10; break;
        case 'r': c = 13; break;
        case 't': c = 9; break;
        case 'u': {
            int h0, h1, h2, h3;
            if (q + 4 > n) return -1;
            h0 = dj_hex(s[q]); h1 = dj_hex(s[q + 1]); h2 = dj_hex(s[q + 2]); h3 = dj_hex(s[q + 3]);
            if ((h0 | h1 | h2 | h3) < 0) return -1;
            c = (uint32_t) ((h0 << 12) | (h1 << 8) | (h2 << 4) | h3);
            if (c == 0 || (c >= 0xd800 && c <= 0xdfff)) return -1;
            q += 4;
            if (c >= 0x800) { scr[at + k++] = (uint8_t) (0xe0 | (c >> 12)); scr[at + k++] = (uint8_t) (0x80 | ((c >> 6) & 63)); c = 0x80 | (c & 63); }
            else if (c >= 0x80) { scr[at + k++] = (uint8_t) (0xc0 | (c >> 6)); c = 0x80 | (c & 63); }
            break;
        }
        default: return -1;
        }
        scr[at + k++] = (uint8_t) c;
    }
    *len = k;
    return q + 1;
}

FLB_HD int djf_record(const struct ch_env *e, const struct ch_lane *ln, const uint8_t *s, int n, uint32_t val_off, ref_t *ok_, ref_t *ov_, uint32_t *th,
                      int *on)
{
    uint8_t *scr = ln->scr;
    uint32_t hpos[DJ_MAX_DEPTH + 1], ccnt[DJ_MAX_DEPTH + 1];
    uint32_t k = 0, isobj = 2, top_start = 0;
    int p = 0, st = DJF_KEY, depth = 1, cnt = 0, first = 1;
    ref_t keyref = 0, valref = 0;
    uint32_t keyhash = 0;

    if (!scr) return -1;
    while (p < n && dj_ws(s[p])) p++;
    if (p >= n || s[p] != '{') return 0;
    p++;
    for (;;) {
        uint32_t c;
        int done = 0;                      /* 1: a value just completed, 2: a container closes */
        DJF_ALIGN(st)
        if (st == DJF_DONE) break;
        if (p >= n) return -1;
        c = s[p];
        if (c <= ' ') {                    /* whitespace between tokens is the exception in log lines */
            while (p < n && dj_ws(s[p])) p++;
            if (p >= n) return -1;
            c = s[p];
        }
        if (st == DJF_COLON) {
            if (c != ':') return -1;
            p++; st = DJF_VAL;
            continue;
        }
        if (st == DJF_AFTER) {
            if (c == ',') { p++; first = 0; st = ((isobj >> depth) & 1) ? DJF_KEY : DJF_VAL; continue; }
            if (c != (((isobj >> depth) & 1) ? '}' : ']')) return -1;
            done = 2;
        }
        else if (st == DJF_KEY) {
            if (c == '}' && first) done = 2;
            else {
                int raw; uint32_t b, len;
                if (c != '"') return -1;
                p = djf_string(s, p, n, scr, depth == 1 ? k : k + 5, &raw, &b, &len);
                if (p < 0) return -1;
                if (depth == 1) {
                    if (raw) { keyref = mkref(RK_STR_IN, val_off + b, len); keyhash = ch_khash(s + b, len); }
                    else { keyref = mkref(RK_STR_SCR, k, len); keyhash = ch_khash(scr + k, len); k += len; }
                }
                else {
                    uint32_t h = mp_put_str_hdr(scr + k, len), i;
                    if (raw) for (i = 0; i < len; i++) scr[k + h + i] = s[b + i];
                    else for (i = 0; i < len; i++) scr[k + h + i] = scr[k + 5 + i];
                    k += h + len;
                }
                /* the colon normally follows at once: take it here and save a round of the loop */
                if (p < n && s[p] == ':') { p++; st = DJF_VAL; }
                else st = DJF_COLON;
                continue;
            }
        }
        else {                             /* DJF_VAL */
            if (c == '"') {
                int raw; uint32_t b, len;
                p = djf_string(s, p, n, scr, depth == 1 ? k : k + 5, &raw, &b, &len);
                if (p < 0) return -1;
                if (depth == 1) {
                    if (raw) valref = mkref(RK_STR_IN, val_off + b, len);
                    else { valref = mkref(RK_STR_SCR, k, len); k += len; }
                }
                else {
                    uint32_t h = mp_put_str_hdr(scr + k, len), i;
                    if (raw) for (i = 0; i < len; i++) scr[k + h + i] = s[b + i];
                    else for (i = 0; i < len; i++) scr[k + h + i] = scr[k + 5 + i];
                    k += h + len;
                }
                done = 1;
            }
            else if (c == '{' || c == '[') {
                if (depth >= DJ_DEEP_HINT) return -1;         /* nesting near the unpacker's limit: the exact transcoder decides and reports it */
                if (depth == 1) top_start = k;
                depth++;
                hpos[depth] = k; ccnt[depth] = 0;
                scr[k++] = 0;
                if (c == '{') { isobj |= 1u << depth; st = DJF_KEY; } else { isobj &= ~(1u << depth); st = DJF_VAL; }
                first = 1;
                p++;
                continue;
            }
            else if (c == ']' && first && !((isobj >> depth) & 1)) done = 2;
            else if (c == '-' || (c >= '0' && c <= '9')) {
                int q = p, nd = 0, neg = 0, plain = 1;
                uint64_t v = 0;
                if (c == '-') { neg = 1; q++; }
                if (q >= n || s[q] < '0' || s[q] > '9') return -1;
                if (s[q] == '0') { q++; if (q < n && s[q] >= '0' && s[q] <= '9') return -1; }
                else {
                    const int q0 = q;
                    q = djf_scan_digits(s, q, n);
                    nd = q - q0;
                    if (nd > 18) plain = 0;
                    else if (depth != 1 || (q < n && s[q] == '.')) { int z; for (z = q0; z < q; z++) v = v * 10 + (s[z] - '0'); }
                }
                if (plain && q < n && s[q] == '.') {
                    /* short decimal without exponent: mantissa / 10^k with both exact in binary64
                     * (<= 15 digits) is correctly rounded -- Clinger's fast path, same result as
                     * dj_number / yyjson */
                    int r = q + 1, fd = 0;
                    uint64_t m = v;
                    while (r < n && s[r] >= '0' && s[r] <= '9' && nd + fd < 15) { m = m * 10 + (s[r] - '0'); r++; fd++; }
                    if (fd > 0 && !(r < n && ((s[r] >= '0' && s[r] <= '9') || s[r] == 'e' || s[r] == 'E'))) {
                        union { double d; uint64_t u; } cv;
                        cv.d = (double) m / dj_p10[fd];
                        if (neg) cv.u |= (uint64_t) 1 << 63;
                        scr[k] = 0xcb; mp_put_be64(scr + k + 1, cv.u);
                        if (depth == 1) valref = mkref(RK_MP_SCR, k, 9);
                        k += 9;
                        p = r;
                        done = 1;
                        plain = 2;
                    }
                    else plain = 0;
                }
                else if (plain && q < n && (s[q] == 'e' || s[q] == 'E')) plain = 0;
                if (plain == 2) { }
                else if (plain) {
                    if (depth == 1) valref = mkref(RK_INT_IN, val_off + (uint32_t) p, (uint32_t) (q - p));
                    else { int64_t iv = neg ? -(int64_t) v : (int64_t) v; mp_put_int(scr + k, iv); k += mp_int_size(iv); }
                    p = q;
                }
                else {
                    int kind = 0;
                    uint64_t u = 0;
                    uint32_t jerr = 0, sz;
                    q = dj_number(s, n, p, &kind, &u, &jerr);
                    if (q < 0) return -1;
                    if (jerr) CH_ATOMIC_OR(e->err, FLBGPU_E_FLOAT);
                    if (kind == 0) { mp_put_uint(scr + k, u); sz = mp_uint_size(u); }
                    else if (kind == 1) { mp_put_int(scr + k, (int64_t) u); sz = mp_int_size((int64_t) u); }
                    else { scr[k] = 0xcb; mp_put_be64(scr + k + 1, u); sz = 9; }
                    if (depth == 1) valref = mkref(RK_MP_SCR, k, sz);
                    k += sz;
                    p = q;
                }
                done = 1;
            }
            else if (c == 't' && p + 4 <= n && s[p + 1] == 'r' && s[p + 2] == 'u' && s[p + 3] == 'e') {
                if (depth == 1) valref = mkref(RK_TRUE, 0, 0); else scr[k++] = 0xc3;
                p += 4; done = 1;
            }
            else if (c == 'f' && p + 5 <= n && s[p + 1] == 'a' && s[p + 2] == 'l' && s[p + 3] == 's' && s[p + 4] == 'e') {
                if (depth == 1) valref = mkref(RK_FALSE, 0, 0); else scr[k++] = 0xc2;
                p += 5; done = 1;
            }
            else if (c == 'n' && p + 4 <= n && s[p + 1] == 'u' && s[p + 2] == 'l' && s[p + 3] == 'l') {
                if (depth == 1) valref = mkref(RK_MP_SCR, k, 1);
                scr[k++] = 0xc0;
                p += 4; done = 1;
            }
            else return -1;
        }

        if (done == 2) {                   /* the container at `depth` closes at s[p] */
            p++;
            if (depth == 1) { st = DJF_DONE; continue; }
            {
                uint32_t cn = ccnt[depth], hp = hpos[depth], ob = (isobj >> depth) & 1;
                if (cn < 16) scr[hp] = (uint8_t) ((ob ? 0x80 : 0x90) | cn);
                else {
                    uint32_t extra = cn < 65536 ? 2 : 4, i;
                    for (i = k - 1; i > hp; i--) scr[i + extra] = scr[i];
                    if (extra == 2) { scr[hp] = ob ? 0xde : 0xdc; mp_put_be16(scr + hp + 1, cn); }
                    else { scr[hp] = ob ? 0xdf : 0xdd; mp_put_be32(scr + hp + 1, cn); }
                    k += extra;
                }
            }
            depth--;
            if (depth == 1) valref = mkref(RK_MP_SCR, top_start, k - top_start);
        }
        /* a value completed inside the container at `depth` */
        if (depth == 1) {
            if (cnt >= CH_MAXF) return -1;
            ok_[cnt] = keyref; ov_[cnt] = valref; th[cnt] = keyhash; cnt++;
        }
        else ccnt[depth]++;
        first = 0;
        /* likewise the comma */
        if (p < n && s[p] == ',') { p++; st = ((isobj >> depth) & 1) ? DJF_KEY : DJF_VAL; }
        else st = DJF_AFTER;
    }
    while (p < n && dj_ws(s[p])) p++;
    if (p < n) return -1;                  /* trailing text: a second document would reject the line */
    *on = cnt;
    return 1;
}

/* ---- field decoders: flb_parser_decoder_do(), src/flb_parser_decoder.c:215-535 -------------------------------------
 * Applied to the map a parser produced (regex / LTSV / logfmt: after the map is complete; JSON: before the time key is
 * looked up, src/flb_parser_json.c:101-117).  Decoded texts and objects go to the decoders' half of the record's scratch. */
/* flb_unescape_string(), src/flb_unescape.c:279-334 */
FLB_HD uint32_t pdec_unescape(const uint8_t *b, uint32_t n, uint8_t *o)
{
    uint32_t i = 0, j = 0;
    while (i < n) {
        if (b[i] == 0x5c) {
            if (i + 1 < n) {
                const uint32_t c = b[i + 1];
                if (c == 'n') { o[j++] = 10; i++; }
                else if (c == 'a') { o[j++] = 7; i++; }
                else if (c == 'b') { o[j++] = 8; i++; }
                else if (c == 't') { o[j++] = 9; i++; }
                else if (c == 'v') { o[j++] = 11; i++; }
                else if (c == 'f') { o[j++] = 12; i++; }
                else if (c == 'r') { o[j++] = 13; i++; }
                else if (c == 0x5c) { o[j++] = 0x5c; i++; }
                i++;
                continue;
            }
            /* a backslash at the very end: the reference steps over it and then copies the byte behind the text -- the
             * terminator of its sds buffer -- so a NUL comes out */
            o[j++] = 0;
            break;
        }
        o[j++] = b[i++];
    }
    return j;
}

/* flb_mysql_unquote_string(), src/flb_unescape.c:338-391 */
FLB_HD uint32_t pdec_mysql_unquote(const uint8_t *b, uint32_t n, uint8_t *o)
{
    uint32_t i = 0, j = 0;
    while (i < n) {
        uint32_t c = b[i++];
        if (c != 0x5c) o[j++] = (uint8_t) c;
        else if (i >= n) o[j++] = (uint8_t) c;
        else {
            c = b[i++];
            switch (c) {
            case 'n': o[j++] = 10; break;
            case 'r': o[j++] = 13; break;
            case 't': o[j++] = 9; break;
            case 0x5c: o[j++] = 0x5c; break;
            case 0x27: o[j++] = 0x27; break;
            case '"': o[j++] = '"'; break;
            case '0': o[j++] = 0; break;
            case 'Z': o[j++] = 0x1a; break;
            default: o[j++] = 0x5c; o[j++] = (uint8_t) c; break;
            }
        }
    }
    return j;
}

#define PDEC_OUT_STRING 0
#define PDEC_OUT_OBJECT 1
/* one backend over text[0,n): result at scr + *at (advanced), *out_len bytes, *out_type; -1 = the decoder failed */
FLB_HDN int pdec_backend(const struct ch_env *e, const struct ch_lane *ln, uint32_t backend, const uint8_t *text, uint32_t n, uint32_t *at, uint32_t *out_off,
                         uint32_t *out_len, int *out_type)
{
    uint8_t *o = ln->scr + *at;
    *out_off = *at;
    if (backend == PDEC_JSON) {
        /* decode_json(): leading blanks skipped, a map or array must start there, exactly one document, and it must be a map */
        uint32_t p = 0, mplen = 0, jerr = 0;
        int consumed = 0;
        while (p < n && text[p] == ' ') p++;
        if (p >= n || (text[p] != '{' && text[p] != '[')) return -1;
        if (!dj_parse_record(text + p, (int) (n - p), o, &mplen, &jerr, &consumed)) return -1;
        if (jerr & DJ_E_FLOAT) CH_ATOMIC_OR(e->err, FLBGPU_E_FLOAT);
        if (jerr & DJ_E_DEEP) CH_ATOMIC_OR(e->err, FLBGPU_E_DEEP);
        *out_len = mplen; *out_type = PDEC_OUT_OBJECT;
    }
    else if (backend == PDEC_ESCAPED) { *out_len = pdec_unescape(text, n, o); *out_type = PDEC_OUT_STRING; }
    else if (backend == PDEC_ESCAPED_UTF8) { *out_len = lf_unescape_raw(text, n, o); *out_type = PDEC_OUT_STRING; }
    else {                                             /* decode_mysql_quoted() */
        if (n < 2) { uint32_t i; for (i = 0; i < n; i++) o[i] = text[i]; *out_len = n; }
        else if ((text[0] == 0x27 && text[n - 1] == 0x27) || (text[0] == '"' && text[n - 1] == '"')) *out_len = pdec_mysql_unquote(text + 1, n - 2, o);
        else { uint32_t i; for (i = 0; i < n; i++) o[i] = text[i]; *out_len = n; }
        *out_type = PDEC_OUT_STRING;
    }
    *at += *out_len + 1;
    return 0;
}

/* returns 1 when some key had a decoder (the reference then re-packs the map: canonical header), 0 when none, -1 when the
 * field list overflowed */
FLB_HDN int apply_decoders(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, ref_t *K, ref_t *V, uint32_t *TH, int *cnt_io)
{
    const struct cf_pdec *decs = (const struct cf_pdec *) (e->blob + pd->dec_off);
    int cnt = *cnt_io, i, matched = -1, extra_keys = 0, extra_has = 0;
    uint32_t at = ln->dec_at, extra_off = 0, extra_len = 0, d;
    if (!ln->scr || !pd->n_dec) return 0;
    /* the first STR key some decoder is registered for: nothing happens before it (and nothing at all without one) */
    for (i = 0; i < cnt && matched < 0; i++) {
        const uint8_t *kp; uint32_t kn;
        if (ref_view(e, ln, K[i], &kp, &kn) != 1) continue;
        for (d = 0; d < pd->n_dec; d++) if (decs[d].key_len == kn && bytes_eq(kp, e->blob + decs[d].key_off, kn)) { matched = i; break; }
    }
    if (matched < 0) return 0;
    for (i = matched; i < cnt; i++) {
        const uint8_t *kp, *vp, *data;
        uint32_t kn, vn, data_n, r;
        const struct cf_pdec *dec = 0;
        const struct cf_pdec_rule *rules;
        int is_decoded = 0, is_decoded_as = 0, in_type = PDEC_OUT_STRING, out_type = PDEC_OUT_STRING;
        uint32_t in_off = 0, in_len = 0, out_off = 0, out_len = 0;
        if (ref_view(e, ln, K[i], &kp, &kn) != 1 || ref_view(e, ln, V[i], &vp, &vn) != 1) continue;
        for (d = 0; d < pd->n_dec; d++) if (decs[d].key_len == kn && bytes_eq(kp, e->blob + decs[d].key_off, kn)) { dec = &decs[d]; break; }
        if (!dec) continue;
        data = vp; data_n = vn;
        if (dec->add_extra_keys) { extra_keys = 1; extra_has = 0; }      /* the extra-keys buffer starts over with every such key */
        rules = (const struct cf_pdec_rule *) (e->blob + dec->rules_off);
        for (r = 0; r < dec->n_rules; r++) {
            uint32_t o_off = 0, o_len = 0;
            int o_type = 0, ret;
            if (rules[r].type == PDEC_DEFAULT && rules[r].action == PDEC_ACT_DO_NEXT && is_decoded) continue;
            if (is_decoded_as && in_type != PDEC_OUT_STRING) continue;
            ret = pdec_backend(e, ln, rules[r].backend, data, data_n, &at, &o_off, &o_len, &o_type);
            if (ret == -1) {
                if (rules[r].action == PDEC_ACT_TRY_NEXT || rules[r].action == PDEC_ACT_DO_NEXT) continue;
                break;
            }
            if (rules[r].type == PDEC_AS) {
                in_off = o_off; in_len = o_len; in_type = o_type; is_decoded_as = 1;
                data = ln->scr + o_off; data_n = o_len;               /* the next rule decodes what this one made */
            }
            else { out_off = o_off; out_len = o_len; out_type = o_type; is_decoded = 1; }
            if (rules[r].action == PDEC_ACT_DO_NEXT) continue;
            break;
        }
        if (is_decoded_as) V[i] = mkref(in_type == PDEC_OUT_STRING ? RK_STR_SCR : RK_MP_SCR, in_off, in_len);
        if (is_decoded && out_type == PDEC_OUT_OBJECT) { extra_has = 1; extra_off = out_off; extra_len = out_len; }
    }
    /* merge_record_and_extra_keys(): the members of the (last) decoded object follow the record's own */
    if (extra_keys && extra_has) {
        const uint8_t *q = ln->scr + extra_off, *end = q + extra_len, *nx;
        struct mp_tok t;
        uint32_t m;
        if (mp_token(q, end, &t) == 0 && t.type == MPT_MAP) {
            q += t.hdr;
            for (m = 0; m < t.len; m++) {
                if (cnt >= CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return -1; }
                nx = mp_skip(q, end);
                K[cnt] = mkref(RK_MP_SCR, (uint32_t) (q - ln->scr), (uint32_t) (nx - q));
                q = nx;
                nx = mp_skip(q, end);
                V[cnt] = mkref(RK_MP_SCR, (uint32_t) (q - ln->scr), (uint32_t) (nx - q));
                q = nx;
                TH[cnt] = 0;
                cnt++;
            }
        }
    }
    *cnt_io = cnt;
    return 1;
}

/* first input offset >= p_abs inside the bitmap's range whose byte is '"', '\\', < 0x20 or >= 0x80; bm_end if none */
FLB_HD uint32_t djf_bm_next(const struct ch_env *e, const struct ch_lane *ln, uint32_t p_abs)
{
    uint32_t rel = p_abs - ln->bm_base, w = rel >> 5;
    const uint32_t nw = (ln->bm_end - ln->bm_base + 31u) >> 5;
    uint32_t m;
    if (p_abs >= ln->bm_end) return ln->bm_end;
    m = ln->bm[w] & (0xffffffffu << (rel & 31u));
    while (!m) { if (++w >= nw) return ln->bm_end; m = ln->bm[w]; }
#ifdef __CUDA_ARCH__
    rel = (w << 5) + (uint32_t) (__ffs((int) m) - 1);
#else
    rel = (w << 5) + (uint32_t) __builtin_ctz(m);
#endif
    return ln->bm_base + rel;
}

/* Stage 2 over the stage-1 bitmap: the flat object of a log line -- string keys, values that are plain strings, integers of
 * up to 18 digits, short decimals, true / false / null -- one O(1) step per token.  Same answers as djf_record() on what it
 * accepts (1 + fields, or 0 "not an object"); -2 = something else is in the line (escapes, non-ASCII, nesting, exponents, white
 * space in odd places ...): djf_record() decides.  val_off is the input offset of s[0]. */
FLB_HD int djf_record_bm(const struct ch_env *e, const struct ch_lane *ln, const uint8_t *s, int n, uint32_t val_off, ref_t *ok_, ref_t *ov_, uint32_t *th, int *on)
{
    uint8_t *scr = ln->scr;
    uint32_t k = 0;
    int p = 0, cnt = 0, state = 0;             /* 0 running, 1 finished, <0 verdict */
    if (!scr || val_off < ln->bm_base || val_off + (uint32_t) n > ln->bm_end) return -2;
    while (p < n && dj_ws(s[p])) p++;
    if (p >= n || s[p] != '{') return 0;
    p++;
    if (p < n && s[p] == '}') { p++; state = 1; }
#ifdef __CUDA_ARCH__
    const unsigned wm = __activemask();
#endif
    for (;;) {
#ifdef __CUDA_ARCH__
        if (!__any_sync(wm, state == 0)) break;    /* the lanes that came in together leave together: one member per round */
        if (state != 0) continue;
#else
        if (state != 0) break;
#endif
        {
            ref_t keyref, valref;
            uint32_t keyhash, c, q;
            /* key */
            if (p >= n || s[p] != '"') { state = -2; continue; }
            q = djf_bm_next(e, ln, val_off + (uint32_t) p + 1) - val_off;
            if (q >= (uint32_t) n || s[q] != '"') { state = -2; continue; }
            keyref = mkref(RK_STR_IN, val_off + (uint32_t) p + 1, q - (uint32_t) p - 1);
            keyhash = ch_khash(s + p + 1, q - (uint32_t) p - 1);
            p = (int) q + 1;
            if (p >= n || s[p] != ':') { state = -2; continue; }
            p++;
            if (p >= n) { state = -2; continue; }
            /* value */
            c = s[p];
            if (c == '"') {
                q = djf_bm_next(e, ln, val_off + (uint32_t) p + 1) - val_off;
                if (q >= (uint32_t) n) { state = -2; continue; }
                if (s[q] == '"') { valref = mkref(RK_STR_IN, val_off + (uint32_t) p + 1, q - (uint32_t) p - 1); p = (int) q + 1; }
                else if (s[q] == 0x5c) {
                    /* a string value with escapes: decoded into scratch exactly as djf_record() does */
                    int raw; uint32_t b, len;
                    const int np = djf_string(s, p, n, scr, k, &raw, &b, &len);
                    if (np < 0 || raw) { state = -2; continue; }
                    valref = mkref(RK_STR_SCR, k, len); k += len;
                    p = np;
                }
                else { state = -2; continue; }
            }
            else if (c == '-' || (c >= '0' && c <= '9')) {
                int z = p, nd = 0, neg = 0, z0;
                uint64_t v = 0;
                if (c == '-') { neg = 1; z++; }
                if (z >= n || s[z] < '0' || s[z] > '9') { state = -2; continue; }
                if (s[z] == '0') { z++; if (z < n && s[z] >= '0' && s[z] <= '9') { state = -2; continue; } }
                else {
                    z0 = z;
                    z = djf_scan_digits(s, z, n);
                    nd = z - z0;
                    if (nd > 18) { state = -2; continue; }
                    if (z < n && s[z] == '.') { int y; for (y = z0; y < z; y++) v = v * 10 + (s[y] - '0'); }
                }
                if (z < n && s[z] == '.') {
                    /* short decimal without exponent (Clinger's exact case), as in djf_record() */
                    int r = z + 1, fd = 0;
                    uint64_t m = v;
                    while (r < n && s[r] >= '0' && s[r] <= '9' && nd + fd < 15) { m = m * 10 + (s[r] - '0'); r++; fd++; }
                    if (fd > 0 && !(r < n && ((s[r] >= '0' && s[r] <= '9') || s[r] == 'e' || s[r] == 'E'))) {
                        union { double d; uint64_t u; } cv;
                        cv.d = (double) m / dj_p10[fd];
                        if (neg) cv.u |= (uint64_t) 1 << 63;
                        scr[k] = 0xcb; mp_put_be64(scr + k + 1, cv.u);
                        valref = mkref(RK_MP_SCR, k, 9);
                        k += 9;
                        p = r;
                    }
                    else { state = -2; continue; }
                }
                else if (z < n && (s[z] == 'e' || s[z] == 'E')) { state = -2; continue; }
                else { valref = mkref(RK_INT_IN, val_off + (uint32_t) p, (uint32_t) (z - p)); p = z; }
            }
            else if (c == 't' && p + 4 <= n && s[p + 1] == 'r' && s[p + 2] == 'u' && s[p + 3] == 'e') { valref = mkref(RK_TRUE, 0, 0); p += 4; }
            else if (c == 'f' && p + 5 <= n && s[p + 1] == 'a' && s[p + 2] == 'l' && s[p + 3] == 's' && s[p + 4] == 'e') { valref = mkref(RK_FALSE, 0, 0); p += 5; }
            else if (c == 'n' && p + 4 <= n && s[p + 1] == 'u' && s[p + 2] == 'l' && s[p + 3] == 'l') { valref = mkref(RK_MP_SCR, k, 1); scr[k++] = 0xc0; p += 4; }
            else { state = -2; continue; }
            if (cnt >= CH_MAXF) { state = -2; continue; }
            ok_[cnt] = keyref; ov_[cnt] = valref; th[cnt] = keyhash; cnt++;
            if (p < n && s[p] == ',') { p++; continue; }
            if (p < n && s[p] == '}') { p++; state = 1; continue; }
            state = -2;
        }
    }
    if (state != 1) return -2;
    while (p < n && dj_ws(s[p])) p++;
    if (p < n) return -2;
    *on = cnt;
    return 1;
}

/* flb_parser_json_do(), src/flb_parser_json.c:29-247.  The document is transcoded into
 * this record's scratch region by the evaluation pass (msgpack, canonical); both passes
 * then read the top-level map back as the field list.  Time key: first member whose key
 * equals Time_Key; its value must be a STR; a failed lookup keeps the member and leaves
 * the timestamp at 0 (:198-209). */
template <bool EMIT>
FLB_HD int pdef_json(const struct ch_env *e, const struct ch_lane *ln, const struct cf_pdef *pd, uint32_t val_off, const uint8_t *s, uint32_t n,
                     ref_t *ok_, ref_t *ov_, uint32_t *th, int *on, int64_t *t_sec, int64_t *t_nsec, uint32_t ridx,
                     uint32_t *cache_pos, int *pos)
{
    int32_t *slot = 0;
    const size_t cs = e->cap_n;
    uint32_t mplen = 0, i;
    int ok, cnt = 0, skip = -1;
    struct mp_tok t;
    const uint8_t *q, *end, *nx;
    int64_t lookup = 0;
    double frac = 0;

    if (!ln->scr) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
    if (e->capcache && e->cap_stride >= RC_CACHE_INTS && *cache_pos + 2 <= e->cap_stride - RC_CACHE_INTS)
        slot = e->capcache + (size_t) *cache_pos * cs + ridx;
    *cache_pos += 2;
    /* slot[0]: 0/1 = result of the exact transcoder (msgpack of slot[1] bytes in scratch),
     * 2 = the fast path produced the fields (it is re-run by the emission pass, nothing cached) */
    if (!(EMIT && slot && CW(slot, 0) != 2)) {
        ok = ln->bm ? djf_record_bm(e, ln, s, (int) n, val_off, ok_, ov_, th, &cnt) : -2;
        if (ok == -2) {
            if (!EMIT && ln->bm && ln->defer_ok) return -2;         /* put off to the follow-up launch (CH_DEFER) */
            cnt = 0; ok = djf_record(e, ln, s, (int) n, val_off, ok_, ov_, th, &cnt);
        }
        if (ok == 0) { if (!EMIT && slot) { CW(slot, 0) = 0; CW(slot, 1) = 0; } return 0; }
        if (ok == 1) { if (!EMIT && slot) { CW(slot, 0) = 2; CW(slot, 1) = 0; } *pos = (int) n; goto have_fields; }   /* nothing but white space behind the document */
    }
    cnt = 0;
    if (EMIT && slot) { ok = CW(slot, 0); mplen = (uint32_t) CW(slot, 1); }
    else {
        uint32_t jerr = 0;
        ok = dj_parse_record(s, (int) n, ln->scr, &mplen, &jerr, pos);
        if (jerr & DJ_E_FLOAT) CH_ATOMIC_OR(e->err, FLBGPU_E_FLOAT);
        if (ok && (jerr & DJ_E_DEEP)) CH_ATOMIC_OR(e->err, FLBGPU_E_DEEP);
        if (!EMIT && slot) { CW(slot, 0) = ok; CW(slot, 1) = (int32_t) mplen; }
    }
    if (!ok) return 0;
    q = ln->scr; end = q + mplen;
    mp_token(q, end, &t);
    q += t.hdr;
    if (t.len > CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
    for (i = 0; i < t.len; i++) {
        nx = mp_skip(q, end);
        ok_[cnt] = mkref(RK_MP_SCR, (uint32_t) (q - ln->scr), (uint32_t) (nx - q));
        q = nx;
        nx = mp_skip(q, end);
        ov_[cnt] = mkref(RK_MP_SCR, (uint32_t) (q - ln->scr), (uint32_t) (nx - q));
        q = nx;
        th[cnt] = 0;                 /* fingerprint computed when the list is merged */
        cnt++;
    }
have_fields:
    if (pd->n_dec) apply_decoders(e, ln, pd, ok_, ov_, th, &cnt);
    if (pd->has_time) {
        /* the first field whose fingerprint is the key's, or unknown: found without a branch per field, so that the loads of the
         * fingerprints are in flight together (most records do not carry the key at all) */
        uint32_t first = (uint32_t) cnt;
        for (i = (uint32_t) cnt; i-- > 0; ) { const uint32_t h_ = th[i]; if (h_ == 0 || h_ == pd->time_key_hash) first = i; }
        for (i = first; i < (uint32_t) cnt; i++) {
            const uint8_t *kp; uint32_t kn;
            if (th[i] && th[i] != pd->time_key_hash) continue;      /* a known fingerprint that differs: not the key */
            if (ref_view(e, ln, ok_[i], &kp, &kn) != 1) continue;
            if (kn != pd->time_key_len || !bytes_eq(kp, e->blob + pd->time_key_off, kn)) continue;
            {
                const uint8_t *vp; uint32_t vn;
                if (ref_view(e, ln, ov_[i], &vp, &vn) != 1) break;            /* value is not a STR: no time */
                if (pdef_time(e, ln, pd, vp, vn, &lookup, &frac) != 0) { lookup = 0; frac = 0; break; }
                if (!pd->time_keep) skip = (int) i;
            }
            break;
        }
    }
    if (skip >= 0) {
        for (i = (uint32_t) skip; i + 1 < (uint32_t) cnt; i++) { ok_[i] = ok_[i + 1]; ov_[i] = ov_[i + 1]; th[i] = th[i + 1]; }
        cnt--;
    }
    *on = cnt; *t_sec = lookup; *t_nsec = frac_to_nsec(frac);
    return 1;
}

struct ch_scratch {              /* per-lane working memory */
    int caps[2 * (RX_MAX_GROUPS + 1)];
    uint32_t stk[CH_RX_STACK];
    ref_t tk[CH_MAXF], tv[CH_MAXF];
    uint32_t th[CH_MAXF];         /* ch_khash of tk[] where the producer knows it cheaply, else 0 */
    int defer;                    /* set by f_parser: this record goes to the follow-up launch */
};
#define CH_DEFER 0xffffffffu

template <bool EMIT>
FLB_HD void f_parser(const struct ch_env *e, const struct ch_lane *ln, const struct cf_parser *cf, struct ch_rec *rc, struct ch_scratch *w,
                     uint32_t ridx, uint32_t *cache_pos, int pristine, uint32_t rec_off, uint32_t rec_len, uint32_t empty_map_off)
{
    uint64_t keep;                /* bit i: original field i is appended after the parsed ones */
    int i, parse_ok = 0, np = 0, preserved = -1, have_arr, pi, in_place = 0;
    int64_t ps = 0, pns = 0;
    uint32_t preset = 0;
    int style = ST_CANON;
    const size_t cs = e->cap_n;

    const uint32_t key_hash = cf->ra_off ? 0u : ch_khash(e->blob + cf->key_off, cf->key_len);
    have_arr = cf->reserve_data || cf->preserve_key;
    keep = cf->reserve_data ? ~0ull : 0ull;

    for (i = (cf->ra_off ? -1 : 0); i < (cf->ra_off ? 0 : rc->nf); i++) {
        const uint8_t *vp = 0; uint32_t vn = 0;
        uint32_t val_off;
        if (cf->ra_off) {
            const struct cf_ra *ra = (const struct cf_ra *) (e->blob + cf->ra_off);
            const uint8_t *np_ = 0, *ne_ = 0;
            int top, kn, vt;
            if (ra_get(e, ln, rc, ra, &top, &np_, &ne_, &kn) != 0) break;
            vt = loc_view(e, ln, rc, top, np_, ne_, &vp, &vn);
            if (vt != 1 && vt != 2) break;
        }
        else {
            const uint8_t *kp; uint32_t kn; int kt, vt;
            if (rc->kh[i] != key_hash) continue;
            kt = ref_view(e, ln, rc->k[i], &kp, &kn);
            if (kt != 1 && kt != 2) continue;
            if (kn != cf->key_len || !bytes_eq(kp, e->blob + cf->key_off, kn)) continue;
            vt = ref_view(e, ln, rc->v[i], &vp, &vn);
            if (vt != 1 && vt != 2) continue;
        }
        if (vp < e->in || vp + vn > e->in + e->in_len) {     /* (an empty value may sit at the very end of the chunk) */
            /* the value was produced by an earlier filter (scratch / constant pool): parsed fields
             * could not reference it by input offset -- refused loudly rather than mis-parsed */
            CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS);
            break;
        }
        val_off = (uint32_t) (vp - e->in);
        parse_ok = 0;
        for (pi = 0; pi < (int) cf->n_parsers; pi++) {
            const struct cf_pdef *pd = (const struct cf_pdef *) (e->blob + cf->pdef_off[pi]);
            int64_t ts = 0, tns = 0;
            int got = 0, cnt = 0, pos = 0;
            if (pd->type == FLBGPU_PARSER_REGEX) {
                uint32_t need = 1 + 2 * (pd->n_groups + 1), c;      /* + 4 ints of parsed time behind them */
                int32_t *slot = 0;
                int matched;
                const uint32_t lim = e->cap_stride >= RC_CACHE_INTS ? e->cap_stride - RC_CACHE_INTS : 0;
                /* the last-field case: nothing of the old list is looked at again, so the parsed fields
                 * go straight into the record's arrays instead of through the staging lists */
                const int direct = !have_arr && !cf->ra_off && i == rc->nf - 1;
                if (e->capcache && *cache_pos + need + 4 <= lim)
                    slot = e->capcache + (size_t) *cache_pos * cs + ridx;
                *cache_pos += need + 4;
                if (EMIT && slot) {
                    matched = CW(slot, 0);
                    for (c = 0; c + 1 < need; c++) w->caps[c] = CW(slot, 1 + c);
                }
                else {
                    matched = rx_run(e, ln, pd->rx_off, vp, vn, w->caps, w->stk);
                    if (!EMIT && slot) {
                        CW(slot, 0) = matched;
                        for (c = 0; c + 1 < need; c++) CW(slot, 1 + c) = w->caps[c];
                        CW(slot, need) = 0;
                    }
                }
                if (matched) got = pdef_regex(e, ln, pd, val_off, vp, vn, w->caps, direct ? rc->k : w->tk, direct ? rc->v : w->tv, &cnt,
                                              &ts, &tns, slot ? slot + (size_t) need * cs : 0, EMIT ? 1 : 0, direct ? rc->kh : w->th, &pos);
                if (got) { preset = pd->n_groups; style = ST_PRESET; in_place = direct; }
            }
            else if (pd->type == FLBGPU_PARSER_JSON) {
                /* same in-place case as for the regex parser, possible while the record is still exactly
                 * what rec_decode() produced: a document that turns out not to parse after some fields
                 * were written is undone by decoding the record again */
                const int direct = pristine && !have_arr && !cf->ra_off && i == rc->nf - 1;
                got = pdef_json<EMIT>(e, ln, pd, val_off, vp, vn, direct ? rc->k : w->tk, direct ? rc->v : w->tv, direct ? rc->kh : w->th,
                                      &cnt, &ts, &tns, ridx, cache_pos, &pos);
                if (got == -2) { w->defer = 1; return; }
                if (got) { style = ST_CANON; in_place = direct; }
                else if (direct) {
                    /* (the time an earlier key of the same name parsed stays: filter_parser.c:296-300 keeps the last non-zero one) */
                    const int64_t s0 = rc->ts_sec, n0 = rc->ts_nsec;
                    rec_decode(e, ln, rec_off, rec_len, rc, empty_map_off);
                    rc->ts_sec = s0; rc->ts_nsec = n0;
                }
            }
            else if (pd->type == FLBGPU_PARSER_LTSV) {
                got = pdef_ltsv(e, ln, pd, val_off, vp, vn, w->tk, w->tv, &cnt, &ts, &tns, &pos);
                if (got) style = ST_CANON;
            }
            else if (pd->type == FLBGPU_PARSER_LOGFMT) {
                got = pdef_logfmt(e, ln, pd, val_off, vp, vn, w->tk, w->tv, &cnt, &ts, &tns, &pos);
                if (got) style = ST_CANON;
            }
            if (got) {
                if (pd->type == FLBGPU_PARSER_LTSV || pd->type == FLBGPU_PARSER_LOGFMT) { int z; for (z = 0; z < cnt; z++) w->th[z] = 0; }
                if (pd->n_dec && pd->type != FLBGPU_PARSER_JSON) {
                    /* (the JSON parser decodes before it looks for the time key: pdef_json) */
                    const int r = apply_decoders(e, ln, pd, in_place ? rc->k : w->tk, in_place ? rc->v : w->tv, in_place ? rc->kh : w->th, &cnt);
                    if (r > 0) style = ST_CANON;                   /* flb_parser_decoder_do() packs a map of its own */
                }
                if (in_place && pd->type == FLBGPU_PARSER_JSON) {
                    /* the walkers leave the fingerprints, the exact transcoder leaves zeroes: look first (loads in flight together), fill only then */
                    int z; uint32_t missing = 0;
                    for (z = 0; z < cnt; z++) missing |= (rc->kh[z] == 0);
                    if (missing) for (z = 0; z < cnt; z++) if (!rc->kh[z]) rc->kh[z] = ref_khash(e, ln, rc->k[z]);
                }
                parse_ok = 1;
                np = cnt;
                if (!EMIT && e->prep) {             /* what flb_parser_do() hands back beside the map: position, time as parsed */
                    int32_t *pr = e->prep + (size_t) 6 * ridx;
                    pr[0] = 1; pr[1] = pos; pr[2] = (int32_t) (uint32_t) ts; pr[3] = (int32_t) (uint32_t) ((uint64_t) ts >> 32); pr[4] = (int32_t) tns;
                }
                if ((uint64_t) ts * 1000000000ull + (uint64_t) tns != 0) { ps = ts; pns = tns; }
                if ((uint64_t) ts * 1000000000ull + (uint64_t) tns != 0) { rc->ts_sec = ts; rc->ts_nsec = tns; }
                if (have_arr && !cf->ra_off) {
                    if (!cf->preserve_key) keep &= ~(1ull << i);
                    else if (!cf->reserve_data) preserved = i;
                }
                break;
            }
        }
    }
    (void) ps; (void) pns;
    rc->reenc = 1;
    if (!parse_ok) { rc->style = ST_CANON; return; }
    if (in_place) { rc->nf = np; rc->style = style; rc->preset_n = preset; return; }
    {
        /* parsed keys first, then the reserved originals (src/flb_pack.c:1716-1723) */
        int extra = 0, j = np;
        if (cf->reserve_data) { for (i = 0; i < rc->nf; i++) if ((keep >> i) & 1) extra++; }
        else if (preserved >= 0) extra = 1;
        if (np + extra > CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return; }
        if (cf->reserve_data) {
            for (i = 0; i < rc->nf; i++) if ((keep >> i) & 1) { w->tk[j] = rc->k[i]; w->tv[j] = rc->v[i]; w->th[j] = rc->kh[i]; j++; }
        }
        else if (preserved >= 0) { w->tk[j] = rc->k[preserved]; w->tv[j] = rc->v[preserved]; w->th[j] = rc->kh[preserved]; j++; }
        for (i = 0; i < j; i++) { rc->k[i] = w->tk[i]; rc->v[i] = w->tv[i]; rc->kh[i] = w->th[i] ? w->th[i] : ref_khash(e, ln, w->tk[i]); }
        rc->nf = j;
        if (extra > 0) rc->style = ST_CANON;
        else { rc->style = style; rc->preset_n = preset; }
    }
}

/* ------------------------------------------------------------ filter_grep */
/* returns 1 keep, 0 exclude */
FLB_HD int f_grep(const struct ch_env *e, const struct ch_lane *ln, const struct cf_grep *cf, const struct ch_rec *rc, struct ch_scratch *w)
{
    const struct cf_grep_rule *r = (const struct cf_grep_rule *) (e->blob + cf->rules_off);
    uint32_t i;
    int found = 0;
    if (cf->op == GREP_OP_LEGACY) {
        int verdict = -1;                 /* decided lanes idle through the remaining rules (CH_SYNC) */
        for (i = 0; i < cf->n_rules; i++) {
            CH_SYNC();
            if (verdict < 0) {
                int m = ra_regex_match(e, ln, rc, r[i].ra_off, r[i].rx_off, w->caps, w->stk);
                if (!m) { if (r[i].type == GREP_REGEX) verdict = 0; }
                else verdict = r[i].type == GREP_EXCLUDE ? 0 : 1;
            }
        }
        return verdict < 0 ? 1 : verdict;
    }
    if (cf->n_rules == 0) return 1;
    {
        uint32_t stop = cf->n_rules;
        for (i = 0; i < cf->n_rules; i++) {
            CH_SYNC();
            if (stop == cf->n_rules) {
                found = ra_regex_match(e, ln, rc, r[i].ra_off, r[i].rx_off, w->caps, w->stk);
                if ((cf->op == GREP_OP_OR && found) || (cf->op == GREP_OP_AND && !found)) stop = i;
            }
        }
        i = stop;
    }
    if (i == cf->n_rules) i = cf->n_rules - 1;
    if (r[i].type == GREP_REGEX) return found ? 1 : 0;
    return found ? 0 : 1;
}

/* ---------------------------------------------------------- filter_modify */
FLB_HD int key_eq(const struct ch_env *e, const struct ch_lane *ln, ref_t k, const uint8_t *s, uint32_t n)
{
    const uint8_t *kp; uint32_t kn;
    int t = ref_view(e, ln, k, &kp, &kn);
    return (t == 1 || t == 2) && kn == n && bytes_eq(kp, s, n);
}
/* helper_msgpack_object_matches_wildcard(): prefix test (defined as length-guarded) */
FLB_HD int key_prefix(const struct ch_env *e, const struct ch_lane *ln, ref_t k, const uint8_t *s, uint32_t n)
{
    const uint8_t *kp; uint32_t kn;
    int t = ref_view(e, ln, k, &kp, &kn);
    return (t == 1 || t == 2) && kn >= n && bytes_eq(kp, s, n);
}
/* helper_msgpack_object_matches_regex(): STR, or BOOLEAN as "true"/"false" */
FLB_HD int obj_rx(const struct ch_env *e, const struct ch_lane *ln, int vt, const uint8_t *p, uint32_t n, uint32_t rx_off, struct ch_scratch *w)
{
    if (vt == 1) return rx_run(e, ln, rx_off, p, n, w->caps, w->stk);
    if (vt == 3) return rx_run(e, ln, rx_off, (const uint8_t *) "true", 4, w->caps, w->stk);
    if (vt == 4) return rx_run(e, ln, rx_off, (const uint8_t *) "false", 5, w->caps, w->stk);
    return 0;
}
FLB_HD int ref_rx(const struct ch_env *e, const struct ch_lane *ln, ref_t r, uint32_t rx_off, struct ch_scratch *w)
{
    const uint8_t *p = 0; uint32_t n = 0;
    int vt = ref_view(e, ln, r, &p, &n);
    return obj_rx(e, ln, vt, p, n, rx_off, w);
}

FLB_HD int mod_conditions(const struct ch_env *e, const struct ch_lane *ln, const struct cf_modify *cf, const struct ch_rec *rc,
                          struct ch_scratch *w)
{
    const struct cf_mod_cond *c = (const struct cf_mod_cond *) (e->blob + cf->conds_off);
    uint32_t ci;
    int ok = 1, i;
    for (ci = 0; ci < cf->n_conds; ci++) {
        CH_SYNC();
        const struct cf_ra *ra = c[ci].ra_off ? (const struct cf_ra *) (e->blob + c[ci].ra_off) : 0;
        const uint8_t *vp = 0, *ve = 0, *sp = 0;
        uint32_t sn = 0;
        int top = -1, kn = 0, exists = 0, vt = 0, r = 0, cnt = 0;
        if (ra) {
            exists = (ra_get(e, ln, rc, ra, &top, &vp, &ve, &kn) == 0) && !kn;
            if (exists) vt = loc_view(e, ln, rc, top, vp, ve, &sp, &sn);
        }
        switch (c[ci].type) {
        case MODC_KEY_EXISTS: r = exists; break;
        case MODC_KEY_DOES_NOT_EXIST: r = !exists; break;
        case MODC_A_KEY_MATCHES:
        case MODC_NO_KEY_MATCHES:
            for (i = 0; i < rc->nf; i++) if (ref_rx(e, ln, rc->k[i], c[ci].a_rx, w)) cnt++;
            r = (c[ci].type == MODC_A_KEY_MATCHES) ? cnt > 0 : cnt == 0;
            break;
        case MODC_KEY_VALUE_EQUALS:
            r = exists && (vt == 1 || vt == 2) && sn == c[ci].b_len && bytes_eq(sp, e->blob + c[ci].b_off, sn);
            break;
        case MODC_KEY_VALUE_DOES_NOT_EQUAL:
            r = exists && !((vt == 1 || vt == 2) && sn == c[ci].b_len && bytes_eq(sp, e->blob + c[ci].b_off, sn));
            break;
        case MODC_KEY_VALUE_MATCHES:
            r = exists && obj_rx(e, ln, vt, sp, sn, c[ci].b_rx, w);
            break;
        case MODC_KEY_VALUE_DOES_NOT_MATCH:
            r = exists && !obj_rx(e, ln, vt, sp, sn, c[ci].b_rx, w);
            break;
        case MODC_MATCHING_KEYS_HAVE_MATCHING_VALUES:
        case MODC_MATCHING_KEYS_DO_NOT_HAVE_MATCHING_VALUES:
            r = 1;
            for (i = 0; i < rc->nf; i++) {
                if (ref_rx(e, ln, rc->k[i], c[ci].a_rx, w) && !ref_rx(e, ln, rc->v[i], c[ci].b_rx, w)) { r = 0; break; }
            }
            if (c[ci].type == MODC_MATCHING_KEYS_DO_NOT_HAVE_MATCHING_VALUES) r = !r;
            break;
        default: r = 0;
        }
        if (!r) ok = 0;
    }
    return ok;
}

/* key i of the record equals (s, n) whose ch_khash is h */
FLB_HD int key_is(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, int i, uint32_t h, const uint8_t *s, uint32_t n)
{
    return rc->kh[i] == h && key_eq(e, ln, rc->k[i], s, n);
}
FLB_HD int count_keys(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, uint32_t h, const uint8_t *s, uint32_t n)
{
    int i, c = 0;
    for (i = 0; i < rc->nf; i++) if (key_is(e, ln, rc, i, h, s, n)) c++;
    return c;
}

/* remove the fields whose bit is set in del: everything before the first deleted field stays put */
FLB_HD void compact(struct ch_rec *rc, uint64_t del)
{
    int i, j;
    if (!del) return;
#ifdef __CUDA_ARCH__
    j = __ffsll((long long) del) - 1;
#else
    j = __builtin_ctzll(del);
#endif
    for (i = j + 1; i < rc->nf; i++) if (!((del >> i) & 1)) { rc->k[j] = rc->k[i]; rc->v[j] = rc->v[i]; rc->kh[j] = rc->kh[i]; j++; }
    rc->nf = j;
}

/* returns 1 when the rule modified the map */
FLB_HD int mod_rule(const struct ch_env *e, const struct ch_lane *ln, const struct cf_mod_rule *r, struct ch_rec *rc, struct ch_scratch *w)
{
    const uint8_t *key = e->blob + r->key_off, *val = e->blob + r->val_off;
    ref_t kmp = mkref(RK_MP_CONST, r->kmp_off, r->kmp_len), vmp = mkref(RK_MP_CONST, r->vmp_off, r->vmp_len);
    uint64_t del = 0;                 /* bit i: field i goes away (CH_MAXF <= 64) */
    const uint32_t kh = r->key_hash, vh = r->val_hash;
    int i, j, match, conflict;

    switch (r->type) {
    case MOD_RENAME:
    case MOD_HARD_RENAME:
        match = count_keys(e, ln, rc, kh, key, r->key_len);
        conflict = count_keys(e, ln, rc, vh, val, r->val_len);
        if (match == 0) return 0;
        if (r->type == MOD_RENAME && conflict > 0) return 0;
        if (conflict > 0) for (i = 0; i < rc->nf; i++) if (key_is(e, ln, rc, i, vh, val, r->val_len)) del |= 1ull << i;
        for (i = 0; i < rc->nf; i++) if (!((del >> i) & 1) && key_is(e, ln, rc, i, kh, key, r->key_len)) { rc->k[i] = vmp; rc->kh[i] = vh; }
        compact(rc, del);
        return 1;
    case MOD_COPY:
    case MOD_HARD_COPY:
        match = count_keys(e, ln, rc, kh, key, r->key_len);
        conflict = count_keys(e, ln, rc, vh, val, r->val_len);
        if (match != 1) return 0;
        if (r->type == MOD_COPY && conflict > 0) return 0;
        if (r->type == MOD_HARD_COPY && conflict > 1) return 0;
        if (conflict == 1) {
            for (i = 0; i < rc->nf; i++) if (key_is(e, ln, rc, i, vh, val, r->val_len)) del |= 1ull << i;
            compact(rc, del);
        }
        if (rc->nf + 1 > CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
        for (i = 0; i < rc->nf; i++) if (key_is(e, ln, rc, i, kh, key, r->key_len)) break;
        if (i == rc->nf) return 1;       /* source vanished with the conflict key (same name): map repacked */
        for (j = rc->nf; j > i + 1; j--) { rc->k[j] = rc->k[j - 1]; rc->v[j] = rc->v[j - 1]; rc->kh[j] = rc->kh[j - 1]; }
        rc->k[i + 1] = vmp; rc->v[i + 1] = rc->v[i]; rc->kh[i + 1] = vh;
        rc->nf++;
        return 1;
    case MOD_ADD:
        if (count_keys(e, ln, rc, kh, key, r->key_len) != 0) return 0;
        if (rc->nf + 1 > CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 0; }
        rc->k[rc->nf] = kmp; rc->v[rc->nf] = vmp; rc->kh[rc->nf] = kh; rc->nf++;
        return 1;
    case MOD_SET:
        for (i = 0; i < rc->nf; i++) if (key_is(e, ln, rc, i, kh, key, r->key_len)) del |= 1ull << i;
        compact(rc, del);
        if (rc->nf + 1 > CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return 1; }
        rc->k[rc->nf] = kmp; rc->v[rc->nf] = vmp; rc->kh[rc->nf] = kh; rc->nf++;
        return 1;
    case MOD_REMOVE:
    case MOD_REMOVE_WILDCARD:
    case MOD_REMOVE_REGEX:
        match = 0;
        for (i = 0; i < rc->nf; i++) {
            int d;
            if (r->type == MOD_REMOVE) d = key_is(e, ln, rc, i, kh, key, r->key_len) ? 1 : 0;
            else if (r->type == MOD_REMOVE_WILDCARD) d = key_prefix(e, ln, rc->k[i], key, r->key_len) ? 1 : 0;
            else d = ref_rx(e, ln, rc->k[i], r->key_rx, w) ? 1 : 0;
            if (d) del |= 1ull << i;
            match += d;
        }
        if (match == 0) return 0;
        compact(rc, del);
        return 1;
    case MOD_MOVE_TO_START:
    case MOD_MOVE_TO_END:
        match = 0;
        for (i = 0; i < rc->nf; i++) if (key_prefix(e, ln, rc->k[i], key, r->key_len)) { del |= 1ull << i; match++; }
        if (match == 0) return 0;
        j = 0;
        for (i = 0; i < rc->nf; i++) if ((int) ((del >> i) & 1) == (r->type == MOD_MOVE_TO_START)) { w->tk[j] = rc->k[i]; w->tv[j] = rc->v[i]; j++; }
        for (i = 0; i < rc->nf; i++) if ((int) ((del >> i) & 1) != (r->type == MOD_MOVE_TO_START)) { w->tk[j] = rc->k[i]; w->tv[j] = rc->v[i]; j++; }
        for (i = 0; i < rc->nf; i++) { rc->k[i] = w->tk[i]; rc->v[i] = w->tv[i]; rc->kh[i] = ref_khash(e, ln, w->tk[i]); }
        return 1;
    }
    return 0;
}

/* returns 1 when the record was modified (and is re-encoded canonically) */
FLB_HD int f_modify(const struct ch_env *e, const struct ch_lane *ln, const struct cf_modify *cf, struct ch_rec *rc, struct ch_scratch *w)
{
    const struct cf_mod_rule *r = (const struct cf_mod_rule *) (e->blob + cf->rules_off);
    uint32_t i;
    int mod = 0;
    const int cond = mod_conditions(e, ln, cf, rc, w);
    for (i = 0; i < cf->n_rules; i++) {
        CH_SYNC();
        if (cond && mod_rule(e, ln, &r[i], rc, w)) mod = 1;
    }
    if (mod) { rc->reenc = 1; rc->style = ST_CANON; }
    return mod;
}

/* ------------------------------------------------- filter_record_modifier */
FLB_HD int ci_eq(const uint8_t *a, const uint8_t *b, uint32_t n)
{
    uint32_t i;
    for (i = 0; i < n; i++) {
        if (dt_lower(a[i]) != dt_lower(b[i])) return 0;
        if (a[i] == 0) break;                 /* strncasecmp stops at NUL */
    }
    return 1;
}

/* returns: 0 passes untouched evidence-wise, sets *cause; *drop when no field is left */
FLB_HDN void f_recmod(const struct ch_env *e, const struct ch_lane *ln, const struct cf_recmod *cf, struct ch_rec *rc, int *cause, int *drop)
{
    const struct cf_rm_key *keys = 0;
    const struct cf_rm_rec *recs = (const struct cf_rm_rec *) (e->blob + cf->records_off);
    uint64_t del = 0;
    uint32_t nk = 0, q;
    int is_delete = 0, i, remaining = rc->nf, total;

    if (cf->n_remove > 0) { keys = (const struct cf_rm_key *) (e->blob + cf->remove_off); nk = cf->n_remove; is_delete = 1; }
    else if (cf->n_allow > 0) { keys = (const struct cf_rm_key *) (e->blob + cf->allow_off); nk = cf->n_allow; is_delete = 0; }
    if (keys) {
        for (i = 0; i < rc->nf; i++) {
            const uint8_t *kp = 0; uint32_t kn = 0;
            int kt = ref_view(e, ln, rc->k[i], &kp, &kn), result = 0;
            for (q = 0; q < nk && (kt == 1 || kt == 2); q++) {
                if (!keys[q].dynamic && kn != keys[q].len) continue;
                if (keys[q].dynamic && kn < keys[q].len) continue;
                if (ci_eq(kp, e->blob + keys[q].off, keys[q].len)) { result = 1; break; }
            }
            if (result == is_delete) { del |= 1ull << i; remaining--; }
        }
    }
    *cause = (remaining != rc->nf) || cf->n_records > 0;
    total = remaining + (int) cf->n_records;
    *drop = total <= 0;
    if (*drop) return;
    compact(rc, del);
    if (rc->nf + (int) cf->n_records > CH_MAXF) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return; }
    for (q = 0; q < cf->n_records; q++) {
        rc->k[rc->nf] = mkref(RK_MP_CONST, recs[q].kmp_off, recs[q].kmp_len);
        rc->v[rc->nf] = mkref(RK_MP_CONST, recs[q].vmp_off, recs[q].vmp_len);
        rc->kh[rc->nf] = ref_khash(e, ln, rc->k[rc->nf]);
        rc->nf++;
    }
    rc->reenc = 1;
    rc->style = ST_MAP32;
}

/* ------------------------------------------------ filter_log_to_metrics */
#ifdef __CUDA_ARCH__
#define CH_CAS64(p, c, v)   atomicCAS((unsigned long long *) (p), (unsigned long long) (c), (unsigned long long) (v))
#define CH_MAX32(p, v)      atomicMax((unsigned int *) (p), (unsigned int) (v))
#define CH_ADDF64(p, v)     atomicAdd((double *) (p), (double) (v))
#define CH_ADD64(p, v)      atomicAdd((unsigned long long *) (p), (unsigned long long) (v))
#define CH_MAX64(p, v)      atomicMax((unsigned long long *) (p), (unsigned long long) (v))
/* gauge: the pair (record index + 1, value bits) of the LAST record of a label set wins, whatever order the
 * lanes arrive in -- cmt_gauge_set() overwrites in record order.  One 16-byte compare-and-swap (sm_90+). */
struct __align__(16) ch_pair16 { unsigned long long a, b; };
static __device__ __forceinline__ void ch_gauge_set(unsigned long long *p, unsigned long long a, unsigned long long b)
{
    struct ch_pair16 cur, want;
    cur.a = ((volatile unsigned long long *) p)[0]; cur.b = ((volatile unsigned long long *) p)[1];
    want.a = a; want.b = b;
    while (cur.a < a) {
        const struct ch_pair16 old = atomicCAS((struct ch_pair16 *) p, cur, want);
        if (old.a == cur.a && old.b == cur.b) break;
        cur = old;
    }
}
#else
static inline void ch_gauge_set(unsigned long long *p, unsigned long long a, unsigned long long b) { if (p[0] < a) { p[0] = a; p[1] = b; } }
static inline unsigned long long ch_cas64_host(unsigned long long *p, unsigned long long c, unsigned long long v) { unsigned long long o = *p; if (o == c) *p = v; return o; }
#define CH_CAS64(p, c, v)   ch_cas64_host((unsigned long long *) (p), (c), (v))
#define CH_MAX32(p, v)      do { if (*(p) < (v)) *(p) = (v); } while (0)
#define CH_ADDF64(p, v)     (*(p) += (v))
#define CH_MAX64(p, v)      do { if (*(p) < (v)) *(p) = (v); } while (0)
static inline unsigned long long ch_add64_host(unsigned long long *p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
#define CH_ADD64(p, v)      ch_add64_host((unsigned long long *) (p), (v))
#endif

/* flb_ra_get_value_object() as the label/value code uses it: the located msgpack token.
 * Returns 1 and the token, 0 when the accessor finds nothing. */
FLB_HD int l2m_lookup(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, uint32_t ra_off, struct mp_tok *t,
                      const uint8_t **payload, int *is_raw_str, uint32_t *raw_len)
{
    const struct cf_ra *ra = (const struct cf_ra *) (e->blob + ra_off);
    const uint8_t *vp = 0, *ve = 0;
    int top, kn, i;
    *is_raw_str = 0;
    i = ra_find(e, ln, rc, e->blob + ra->key_off, ra->key_len);
    if (i < 0) return 0;
    top = i;
    {
        uint32_t k = r_kind(rc->v[i]);
        if (k == RK_STR_IN || k == RK_STR_SCR) { *is_raw_str = 1; *payload = ref_ptr(e, ln, rc->v[i]); *raw_len = r_len(rc->v[i]); return 1; }
        if (k == RK_TRUE || k == RK_FALSE) { t->type = MPT_BOOL; return 1; }
        if (k == RK_INT_IN) { t->type = MPT_INT; t->u = (uint64_t) ch_atoll(ref_ptr(e, ln, rc->v[i]), r_len(rc->v[i])); return 1; }
        if (k == RK_HEX_IN) { t->type = MPT_UINT; t->u = ch_strtoull16(ref_ptr(e, ln, rc->v[i]), r_len(rc->v[i])); return 1; }
        if (k == RK_FLT_IN) {
            int okf;
            t->u = dj_strtod(ref_ptr(e, ln, rc->v[i]), (int) r_len(rc->v[i]), &okf);
            if (!okf) CH_ATOMIC_OR(e->err, FLBGPU_E_FLOAT);
            t->type = MPT_F64; return 1;
        }
        if (k != RK_MP_IN && k != RK_MP_CONST && k != RK_MP_SCR) { t->type = MPT_NIL; CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return 1; }
        vp = ref_ptr(e, ln, rc->v[i]); ve = vp + r_len(rc->v[i]);
        if (mp_token(vp, ve, t) != 0) return 0;
        if (ra->n_sub > 0 && (t->type == MPT_MAP || t->type == MPT_ARRAY)) {
            if (ra_walk_sub(e, ln, ra, vp, ve, &vp, &ve, &kn) != 0) return 0;
            if (mp_token(vp, ve, t) != 0) return 0;
        }
    }
    (void) top;
    *payload = vp + t->hdr;
    return 1;
}

FLB_HDN void f_l2m(const struct ch_env *e, const struct ch_lane *ln, const struct cf_l2m *cf, const struct ch_rec *rc, struct ch_scratch *w,
                  uint32_t ridx)
{
    const struct l2m_table *tb = &e->l2m;
    uint8_t *lab = (uint8_t *) w->stk;                     /* label strings: reuse the regex stack area */
    uint32_t li, lpos = 0;
    unsigned long long h = 1469598103934665603ull, hc = 1469598103934665603ull;
    uint32_t idx, probes = 0;
    double val = 0;

    if (!tb->hash) return;
    if (cf->grep_off && !f_grep(e, ln, (const struct cf_grep *) (e->blob + cf->grep_off), rc, w)) return;

    /* label values -> strings (log_to_metrics.c:1010-1043): STR "%s" (<= 251 bytes, stops at NUL),
     * integers "%ld", anything else "" */
    for (li = 0; li < cf->n_labels; li++) {
        struct mp_tok t;
        const uint8_t *pl = 0;
        int raw = 0;
        uint32_t rl = 0, n = 0, k;
        uint8_t *dst = lab + lpos + 1;
        if (lpos + 1 + 252 > sizeof(w->stk)) { CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return; }
        t.type = MPT_NIL; t.len = 0; t.u = 0; t.hdr = 0;
        if (l2m_lookup(e, ln, rc, cf->label_ra_off[li], &t, &pl, &raw, &rl)) {
            if (raw || t.type == MPT_STR) {
                uint32_t sl = raw ? rl : t.len;
                for (k = 0; k < sl && k < 251 && pl[k]; k++) dst[n++] = pl[k];
            }
            else if (t.type == MPT_UINT || t.type == MPT_INT) {
                int64_t v = (int64_t) t.u;
                uint64_t a = v < 0 ? (uint64_t) (0 - (uint64_t) v) : (uint64_t) v;
                uint8_t tmp[24];
                int m = 0;
                do { tmp[m++] = (uint8_t) ('0' + a % 10); a /= 10; } while (a);
                if (v < 0) dst[n++] = '-';
                while (m) dst[n++] = tmp[--m];
            }
            else if (t.type == MPT_F32 || t.type == MPT_F64) {                                       /* "%f" */
                uint64_t fb = t.u;
                if (t.type == MPT_F32) { union { uint32_t u; float f; } c4; union { double d; uint64_t u; } c8; c4.u = (uint32_t) t.u; c8.d = (double) c4.f; fb = c8.u; }
                n = dj_fmt_f6(fb, dst, 251);
            }
        }
        lab[lpos] = (uint8_t) n;
        for (k = 0; k <= n; k++) { h ^= lab[lpos + k]; h *= 1099511628211ull; }
        for (k = 1; k <= n; k++) { hc ^= lab[lpos + k]; hc *= 1099511628211ull; }
        lpos += 1 + n;
    }
    h |= 1ull;

    if (cf->mode != L2M_COUNTER) {                 /* gauge and histogram read the value the same way (:1052-1110) */
        struct mp_tok t;
        const uint8_t *pl = 0;
        int raw = 0, ok = 1;
        uint32_t rl = 0;
        t.type = MPT_NIL; t.len = 0; t.u = 0; t.hdr = 0;
        if (!l2m_lookup(e, ln, rc, cf->value_ra_off, &t, &pl, &raw, &rl)) return;    /* "value field is empty or not existent" */
        if (raw || t.type == MPT_STR) {
            /* sscanf("%lf"): a text that converts nothing leaves the PREVIOUS record's value in
             * place (log_to_metrics.c:984,1105) -- order dependent, refused; so are inf/nan/hex */
            uint32_t sl = raw ? rl : t.len, q = 0;
            while (q < sl && dt_isspace(pl[q])) q++;
            if (q < sl && (pl[q] == '+' || pl[q] == '-')) q++;
            if (q < sl && pl[q] == '.') q++;
            if (q < sl && pl[q] == '0' && q + 1 < sl && (pl[q + 1] | 0x20) == 'x') { CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return; }   /* hex float: not restated */
            if (q >= sl || pl[q] < '0' || pl[q] > '9') {
                /* "inf" / "nan" would convert: refused.  Anything else converts nothing: the value of the previous converting record */
                const uint32_t c0 = q < sl ? (uint32_t) (pl[q] | 0x20) : 0u;
                if (c0 == 'i' || c0 == 'n') { CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return; }
                if (ln->l2m_forced) val = *ln->l2m_forced;
                else if (ln->l2m_probe) return;                                     /* assigns nothing */
                else {
                    const unsigned long long at = tb->pending ? CH_ADD64(&tb->pending_n[0], 1ull) : (unsigned long long) L2M_PENDING_CAP;
                    if (at < tb->pending_cap) tb->pending[at] = ridx; else CH_ATOMIC_OR(e->err, FLBGPU_E_L2M);
                    return;
                }
            }
            else {
                union { uint64_t u; double d; } cv; cv.u = dj_strtod(pl, (int) sl, &ok); val = cv.d;
                if (!ok) { CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return; }
            }
        }
        else if (t.type == MPT_UINT || t.type == MPT_INT) val = (double) (int64_t) t.u;
        else if (t.type == MPT_F64) { union { uint64_t u; double d; } cv; cv.u = t.u; val = cv.d; }
        else if (t.type == MPT_F32) { union { uint32_t u; float f; } cv; cv.u = (uint32_t) t.u; val = (double) cv.f; }
        else return;                                                              /* "cannot convert given value to metric" */
        if (ln->l2m_probe) { union { uint64_t u; double d; } cv; cv.d = val; ln->l2m_probe[0] = 1ull; ln->l2m_probe[1] = cv.u; return; }
    }
    else if (ln->l2m_probe) return;

    /* find or claim the slot of this label set */
    idx = (uint32_t) (h >> 20) & tb->mask;
    for (;;) {
        unsigned long long cur = CH_CAS64(&tb->hash[idx], 0ull, h);
        if (cur == 0ull) {
            uint8_t *d = tb->str + (size_t) idx * cf->n_labels * L2M_LABEL_BYTES;
            uint32_t p = 0, k;
            for (li = 0; li < cf->n_labels; li++) {
                uint32_t n = lab[p];
                for (k = 0; k <= n; k++) d[(size_t) li * L2M_LABEL_BYTES + k] = lab[p + k];
                p += 1 + n;
            }
            break;
        }
        if (cur == h) break;
        idx = (idx + 1) & tb->mask;
        if (++probes > tb->mask) { CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return; }
    }
    tb->chash[idx] = hc | 1ull;                     /* every lane of this tuple stores the same value */
    CH_MAX32(&tb->first[idx], 0xffffffffu - ridx);
    CH_ATOMIC_ADD(&tb->cnt[idx], 1ull);
    if (cf->mode == L2M_HISTOGRAM) {
        const double *ub = (const double *) (e->blob + cf->buckets_off);
        int i;
        for (i = (int) cf->n_buckets - 1; i >= 0; i--) {
            if (val > ub[i]) break;
            CH_ATOMIC_ADD(&tb->bkt[(size_t) idx * (cf->n_buckets + 1) + i], 1ull);
        }
        CH_ATOMIC_ADD(&tb->bkt[(size_t) idx * (cf->n_buckets + 1) + cf->n_buckets], 1ull);
        CH_ADDF64(&tb->sum[idx], val);
        if (tb->amax) {
            union { double d; unsigned long long u; } cv;
            const double av = val < 0 ? -val : val;
            unsigned long long ai = av <= (double) L2M_EXACT_MAX ? (unsigned long long) av : L2M_NOT_EXACT;   /* NaN: not <= */
            cv.d = val;
            if ((double) ai != av || cv.u == 0x8000000000000000ull) ai = L2M_NOT_EXACT;
            if (ai > tb->amax[idx]) CH_MAX64(&tb->amax[idx], ai);      /* (a plain read first: the hot sets' maximum is soon reached) */
            if (tb->obs_slot) { tb->obs_slot[ridx] = idx + 1; tb->obs_val[ridx] = val; }
        }
    }
    else if (cf->mode == L2M_GAUGE) {              /* bkt is [slot][2] here: last record index + 1, value bits */
        union { double d; unsigned long long u; } cv;
        cv.d = val;
        ch_gauge_set(&tb->bkt[(size_t) idx * 2], (unsigned long long) ridx + 1, cv.u);
    }
}

/* Events the decoder steps over (group markers, negative timestamps: kind 1 in the record index) are still
 * objects of the chunk for log_to_metrics, which walks it with msgpack_unpack_next() and takes element 1 of
 * every root array as the map (log_to_metrics.c:993-1003).  It sees them when no earlier filter of the chain
 * rewrote the chunk -- a rewritten chunk holds decoded events only. */
FLB_HDN void chain_skipped_record(const struct ch_env *e, uint32_t ridx, uint32_t off, uint32_t len)
{
    const struct chain_hdr *h = (const struct chain_hdr *) e->blob;
    const struct chain_filter *f = (const struct chain_filter *) (e->blob + h->filters_off);
    struct ch_lane lane, *ln = &lane;
    uint32_t k;
    for (k = 0; k < h->n_filters; k++) {
        if (!((e->active >> k) & 1)) continue;
        if (f[k].kind == FLBGPU_F_LOG_TO_METRICS) break;
        if ((e->assume >> k) & 1) return;
    }
    if (k == h->n_filters) return;
    {
        struct ch_rec rc;
        struct ch_scratch w;
        lane.scr = e->scr ? e->scr + (size_t) e->scr_mul * off : 0; lane.dec_at = 4u * len;
        lane.bm = 0; lane.bm_base = lane.bm_end = 0; lane.defer_ok = 0; lane.l2m_probe = 0; lane.l2m_forced = 0;
        if (rec_decode(e, ln, off, len, &rc, h->empty_map_off) != 0) { CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS); return; }
        f_l2m(e, ln, (const struct cf_l2m *) (e->blob + f[k].cfg_off), &rc, &w, ridx);
    }
}

/* ------------------------------------------------------ filter_rewrite_tag */
/* plugins/filter_rewrite_tag/rewrite_tag.c:356-426 (process_record) + src/flb_record_accessor.c:483-690 (flb_ra_translate):
 * the first rule whose key holds a string its regex matches decides; the new tag is the rule's template with $TAG, $TAG[n],
 * $0..$9 and $key['sub'] filled in.  o == NULL: only the length. */
FLB_HD uint32_t rt_put(uint8_t *o, uint32_t k, const uint8_t *b, uint32_t n)
{
    if (o) { uint32_t i; for (i = 0; i < n; i++) o[k + i] = b[i]; }
    return n;
}
FLB_HD uint32_t rt_put_i64(uint8_t *o, uint32_t k, int64_t v)        /* snprintf("%" PRId64) */
{
    uint8_t tmp[20];
    int n = 0;
    uint32_t w = 0;
    uint64_t u = v < 0 ? 0 - (uint64_t) v : (uint64_t) v;
    do { tmp[n++] = (uint8_t) ('0' + (int) (u % 10)); u /= 10; } while (u);
    if (v < 0) { if (o) o[k] = '-'; w++; }
    while (n) { n--; if (o) o[k + w] = tmp[n]; w++; }
    return w;
}
/* one msgpack value as ra_translate_keymap() prints it; anything it prints nothing for returns 0 */
FLB_HD uint32_t rt_put_mp(const struct ch_env *e, const uint8_t *b, const uint8_t *end, uint8_t *o, uint32_t k)
{
    struct mp_tok t;
    if (mp_token(b, end, &t) != 0) return 0;
    switch (t.type) {
    case MPT_STR: return rt_put(o, k, b + t.hdr, t.len);
    case MPT_BIN: {                                  /* "%02x" per byte */
        uint32_t i;
        if (o) for (i = 0; i < t.len; i++) { const uint8_t c = b[t.hdr + i]; o[k + 2 * i] = "0123456789abcdef"[c >> 4]; o[k + 2 * i + 1] = "0123456789abcdef"[c & 15]; }
        return 2 * t.len;
    }
    case MPT_UINT: case MPT_INT: return rt_put_i64(o, k, (int64_t) t.u);
    case MPT_BOOL: return t.u ? rt_put(o, k, (const uint8_t *) "true", 4) : rt_put(o, k, (const uint8_t *) "false", 5);
    case MPT_NIL: return rt_put(o, k, (const uint8_t *) "null", 4);
    case MPT_F32: case MPT_F64: case MPT_MAP:        /* snprintf("%f") / flb_msgpack_to_json_str(): not restated -- refused, loudly */
        CH_ATOMIC_OR(e->err, FLBGPU_E_TAGVALUE);
        return 0;
    default: return 0;                               /* arrays, ext: flb_ra_key_to_value_ext() has no value for them */
    }
}
FLB_HD uint32_t rt_translate(const struct ch_env *e, const struct ch_lane *ln, const struct ch_rec *rc, const struct cf_rt_rule *rule,
                             const uint8_t *subj, const int *caps, uint8_t *o)
{
    const struct cf_rt_part *pt = (const struct cf_rt_part *) (e->blob + rule->parts_off);
    const struct rx_prog *pg = (const struct rx_prog *) (e->blob + rule->rx_off);
    uint32_t k = 0, i;
    for (i = 0; i < rule->n_parts; i++) {
        switch (pt[i].type) {
        case RT_STRING: k += rt_put(o, k, e->blob + pt[i].a, pt[i].b); break;
        case RT_TAG: k += rt_put(o, k, e->tag, e->tag_len); break;
        case RT_TAG_PART: {                          /* ra_translate_tag_part() */
            uint32_t at = 0;
            int id = -1, done = 0;
            while (at < e->tag_len) {
                uint32_t end = 0;
                int dot = 0;
                while (at + end < e->tag_len) { if (e->tag[at + end] == '.') { dot = 1; break; } end++; }
                if (!dot) { if (at == 0) break; end = e->tag_len - at; }
                id++;
                if ((int) pt[i].a == id) { k += rt_put(o, k, e->tag + at, end); done = 1; break; }
                at += end + 1;
            }
            if (!done && pt[i].a == 0 && id == -1 && at < e->tag_len) k += rt_put(o, k, e->tag, e->tag_len);      /* no dots in the tag */
            break;
        }
        case RT_REGEX_ID:                            /* flb_regex_do() keeps no region for a pattern without groups: not even $0 */
            if (pg->n_groups > 0 && pt[i].a <= pg->n_groups && caps[2 * pt[i].a] >= 0)
                k += rt_put(o, k, subj + caps[2 * pt[i].a], (uint32_t) (caps[2 * pt[i].a + 1] - caps[2 * pt[i].a]));
            break;
        case RT_KEYMAP: {
            const struct cf_ra *ra = (const struct cf_ra *) (e->blob + pt[i].a);
            const uint8_t *vp = 0, *ve = 0;
            int top, kn;
            if (ra_get(e, ln, rc, ra, &top, &vp, &ve, &kn) != 0) break;
            if (top < 0) { k += rt_put_mp(e, vp, ve, o, k); break; }
            {
                const ref_t r = rc->v[top];
                const uint32_t rk = r_kind(r);
                const uint8_t *b = ref_ptr(e, ln, r);
                if (rk == RK_STR_IN || rk == RK_STR_SCR) k += rt_put(o, k, b, r_len(r));
                else if (rk == RK_INT_IN) k += rt_put_i64(o, k, ch_atoll(b, r_len(r)));
                else if (rk == RK_HEX_IN) k += rt_put_i64(o, k, (int64_t) ch_strtoull16(b, r_len(r)));
                else if (rk == RK_TRUE) k += rt_put(o, k, (const uint8_t *) "true", 4);
                else if (rk == RK_FALSE) k += rt_put(o, k, (const uint8_t *) "false", 5);
                else if (rk == RK_FLT_IN) CH_ATOMIC_OR(e->err, FLBGPU_E_TAGVALUE);
                else k += rt_put_mp(e, b, b + r_len(r), o, k);
            }
            break;
        }
        default: break;
        }
    }
    return k;
}
/* the rule that takes the record: its index, or -1.  *subj / caps: what its regex matched on. */
FLB_HD int f_rtag_rule(const struct ch_env *e, const struct ch_lane *ln, const struct cf_rtag *cf, const struct ch_rec *rc, struct ch_scratch *w,
                       const uint8_t **subj)
{
    const struct cf_rt_rule *r = (const struct cf_rt_rule *) (e->blob + cf->rules_off);
    uint32_t i;
    int hit = -1;
    for (i = 0; i < cf->n_rules; i++) {
        CH_SYNC();
        if (hit < 0) {
            const struct cf_ra *ra = (const struct cf_ra *) (e->blob + r[i].ra_off);
            const uint8_t *vp = 0, *ve = 0, *s;
            uint32_t n;
            int top, kn;
            if (ra_get(e, ln, rc, ra, &top, &vp, &ve, &kn) != 0) continue;
            if (loc_view(e, ln, rc, top, vp, ve, &s, &n) != 1) continue;        /* the value must be a STR (flb_ra_key_regex_match) */
            if (rx_run(e, ln, r[i].rx_off, s, n, w->caps, w->stk)) { hit = (int) i; *subj = s; }
        }
    }
    return hit;
}

/* ------------------------------------------------------------- the chain */
/* Runs record `ridx` (framed at off/len, kind 0) through the chain.
 * EMIT=false: returns the output size (0 = dropped) and records evidence.
 * EMIT=true : writes the record at `out` (the caller only calls it for size>0).
 * PH (evaluation pass only) splits the chain into two launches whose code each fits the instruction cache better than
 * the whole interpreter does: CH_PH_HEAD = decode the record and run filter 0 (the parser), then leave the field list in the
 * record's capture-cache row and return 1 (alive) / 0 (dropped) / CH_DEFER (more fields than the row holds: the whole chain
 * is run for this record by the follow-up launch); CH_PH_TAIL = pick the field list up again and run filters 1..n-1. */
#define CH_PH_ALL  0
#define CH_PH_HEAD 1
#define CH_PH_TAIL 2
#define CH_PH_RTAG 3                        /* EMIT only: stop at the rewrite_tag filter and write the record's entry of the re-tagged stream */
#define RC_STATE_KH RC_CACHE_MAXF            /* split mode: the key fingerprints, in columns behind the row (cap_stride ..) */
template <bool EMIT, int PH = CH_PH_ALL>
FLB_HD uint32_t chain_record(const struct ch_env *e, struct ch_lane *ln, uint32_t ridx, uint32_t off, uint32_t len, uint8_t *out)
{
    const struct chain_hdr *h = (const struct chain_hdr *) e->blob;
    const struct chain_filter *f = (const struct chain_filter *) (e->blob + h->filters_off);
    struct ch_rec rc;
    struct ch_scratch w;
    uint32_t k, cache_pos = 0;
    w.defer = 0;
    if (!EMIT && PH != CH_PH_TAIL && e->esize) e->esize[ridx] = 0;
    /* this record's private scratch region: scr_mul bytes per record byte, the decoders' part behind the parser's */
    ln->scr = e->scr ? e->scr + (size_t) e->scr_mul * off : 0;
    ln->dec_at = 4u * len;
    /* The evaluation pass leaves the final field list of every surviving record (<= RC_CACHE_MAXF
     * fields) in the last RC_CACHE_INTS ints of its capture-cache row; the emission pass then only
     * encodes -- no decoding, no filters.  Longer records are re-run through the chain. */
    if (EMIT && PH != CH_PH_RTAG && e->capcache && e->cap_stride >= RC_CACHE_INTS) {
        const size_t cs = e->cap_n;
        const int32_t *c = e->capcache + (size_t) (e->cap_stride - RC_CACHE_INTS) * cs + ridx;
        const int32_t st = CW(c, 0);
        if (st == RC_CACHE_RAW) { mp_copy(out, e->in + off, len); return len; }
        if (st >= 0) {
            int i;
            rc.nf = st & 0xff; rc.style = (st >> 8) & 0xff; rc.reenc = 1;
            rc.preset_n = (uint32_t) CW(c, 1);
            rc.ts_sec = (int64_t) (uint32_t) CW(c, 2); rc.ts_nsec = (int64_t) (uint32_t) CW(c, 3);
            rc.meta = ((ref_t) (uint32_t) CW(c, 5) << 32) | (uint32_t) CW(c, 4);
            for (i = 0; i < rc.nf; i++) {
                rc.k[i] = ((ref_t) (uint32_t) CW(c, 8 + 4 * i + 1) << 32) | (uint32_t) CW(c, 8 + 4 * i);
                rc.v[i] = ((ref_t) (uint32_t) CW(c, 8 + 4 * i + 3) << 32) | (uint32_t) CW(c, 8 + 4 * i + 2);
            }
            return rec_emit(e, ln, &rc, out);
        }
    }
    if (PH == CH_PH_TAIL) {
        /* the head launch left the state here: field list, key fingerprints, style, time */
        const size_t cs = e->cap_n;
        const int32_t *c = e->capcache + (size_t) (e->cap_stride - RC_CACHE_INTS) * cs + ridx;
        const int32_t *kh = e->capcache + (size_t) e->cap_stride * cs + ridx;
        const int32_t st = CW(c, 0);
        int i;
        rc.nf = st & 0xff; rc.style = (st >> 8) & 0xff; rc.reenc = (st >> 16) & 1;
        rc.preset_n = (uint32_t) CW(c, 1);
        rc.ts_sec = (int64_t) (((uint64_t) (uint32_t) CW(c, 6) << 32) | (uint32_t) CW(c, 2)); rc.ts_nsec = (int64_t) (uint32_t) CW(c, 3);
        rc.meta = ((ref_t) (uint32_t) CW(c, 5) << 32) | (uint32_t) CW(c, 4);
        for (i = 0; i < rc.nf; i++) {
            rc.k[i] = ((ref_t) (uint32_t) CW(c, 8 + 4 * i + 1) << 32) | (uint32_t) CW(c, 8 + 4 * i);
            rc.v[i] = ((ref_t) (uint32_t) CW(c, 8 + 4 * i + 3) << 32) | (uint32_t) CW(c, 8 + 4 * i + 2);
            rc.kh[i] = (uint32_t) CW(kh, i);
        }
    }
    else if (rec_decode(e, ln, off, len, &rc, h->empty_map_off) != 0) {
        CH_ATOMIC_OR(e->err, FLBGPU_E_FIELDS);
        return 0;
    }
    for (k = (PH == CH_PH_TAIL ? h->split_at : 0u); k < (PH == CH_PH_HEAD ? h->split_at : h->n_filters); k++) {
        const uint8_t *cfg = e->blob + f[k].cfg_off;
        int assumed = (e->assume >> k) & 1;
        if (!((e->active >> k) & 1)) continue;
        CH_SYNC();
        switch (f[k].kind) {
        case FLBGPU_F_PARSER:
            if (!assumed) break;
            f_parser<EMIT>(e, ln, (const struct cf_parser *) cfg, &rc, &w, ridx, &cache_pos, k == 0, off, len, h->empty_map_off);
            if (!EMIT && w.defer) return CH_DEFER;
            if (PH == CH_PH_HEAD && rc.nf > RC_CACHE_MAXF) return CH_DEFER;      /* more fields than the hand-over row holds: before any filter behind it leaves evidence */
            if (!EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED);
            break;
        case FLBGPU_F_GREP:
            if (!f_grep(e, ln, (const struct cf_grep *) cfg, &rc, &w)) {
                if (!EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_CAUSE);
                if (assumed) return 0;
            }
            else if (!EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED);
            break;
        case FLBGPU_F_MODIFY: {
            /* evaluate on a copy when the filter is assumed NOTOUCH so the record passes unchanged */
            if (assumed) {
                if (f_modify(e, ln, (const struct cf_modify *) cfg, &rc, &w) && !EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_CAUSE);
            }
            else if (!EMIT) {
                struct ch_rec tmp = rc;
                if (f_modify(e, ln, (const struct cf_modify *) cfg, &tmp, &w)) CH_ATOMIC_OR(&e->fl_flags[k], CHF_CAUSE);
            }
            if (!EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED);
            break;
        }
        case FLBGPU_F_RECORD_MODIFIER: {
            int cause = 0, drop = 0;
            if (assumed) {
                f_recmod(e, ln, (const struct cf_recmod *) cfg, &rc, &cause, &drop);
                if (!EMIT) { if (cause) CH_ATOMIC_OR(&e->fl_flags[k], CHF_CAUSE); if (!drop) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED); }
                if (drop) return 0;
            }
            else if (!EMIT) {
                struct ch_rec tmp = rc;
                f_recmod(e, ln, (const struct cf_recmod *) cfg, &tmp, &cause, &drop);
                if (cause) CH_ATOMIC_OR(&e->fl_flags[k], CHF_CAUSE);
                if (!drop) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED);
            }
            break;
        }
        case FLBGPU_F_REWRITE_TAG: {
            /* rewrite_tag.c:468-497: a matched record goes to the emitter under its new tag -- as this filter sees it --
             * and stays in the chunk only when the rule says keep */
            const struct cf_rtag *cf = (const struct cf_rtag *) cfg;
            const uint8_t *subj = 0;
            const int hit = f_rtag_rule(e, ln, cf, &rc, &w, &subj);
            if (hit >= 0) {
                const struct cf_rt_rule *rule = (const struct cf_rt_rule *) (e->blob + cf->rules_off) + hit;
                /* untouched so far: the bytes are the decoder's `data + pre .. off`, events it stepped over included */
                const uint32_t lo = (!rc.reenc && (e->assume & e->active & ((1u << k) - 1u)) == 0) ? ln->raw_lo : off;
                if (PH == CH_PH_RTAG) {
                    const uint32_t tl = rt_translate(e, ln, &rc, rule, subj, w.caps, out + RT_ENTRY_HDR);
                    uint32_t rl;
                    if (!rc.reenc) { rl = off + len - lo; mp_copy(out + RT_ENTRY_HDR + tl, e->in + lo, rl); }
                    else rl = rec_emit(e, ln, &rc, out + RT_ENTRY_HDR + tl);
                    out[0] = (uint8_t) tl; out[1] = (uint8_t) (tl >> 8); out[2] = (uint8_t) (tl >> 16); out[3] = (uint8_t) (tl >> 24);
                    out[4] = (uint8_t) rl; out[5] = (uint8_t) (rl >> 8); out[6] = (uint8_t) (rl >> 16); out[7] = (uint8_t) (rl >> 24);
                    return RT_ENTRY_HDR + tl + rl;
                }
                if (!EMIT) {
                    CH_ATOMIC_OR(&e->fl_flags[k], CHF_CAUSE);
                    if (e->esize) e->esize[ridx] = RT_ENTRY_HDR + rt_translate(e, ln, &rc, rule, subj, w.caps, 0) + (rc.reenc ? rec_emit(e, ln, &rc, 0) : off + len - lo);
                }
                if (!rule->keep) { if (assumed) return 0; }
                else if (!EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED);
            }
            else {
                if (PH == CH_PH_RTAG) return 0;
                if (!EMIT) CH_ATOMIC_OR(&e->fl_flags[k], CHF_EMITTED);
            }
            break;
        }
        case FLBGPU_F_LOG_TO_METRICS:
            /* metrics are accumulated once per call, by the evaluation pass; logs pass
             * through unless discard_logs (log_to_metrics.c:1136-1141) */
            if (!EMIT) f_l2m(e, ln, (const struct cf_l2m *) cfg, &rc, &w, ridx);
            if (assumed) return 0;
            break;
        default:
            break;
        }
    }
    if (PH == CH_PH_RTAG) return 0;          /* (not reached for a record the evaluation pass sized an entry for) */
    if (PH == CH_PH_HEAD) {
        /* hand the record over to the tail launch */
        const size_t cs = e->cap_n;
        int32_t *c = e->capcache + (size_t) (e->cap_stride - RC_CACHE_INTS) * cs + ridx;
        int32_t *kh = e->capcache + (size_t) e->cap_stride * cs + ridx;
        int i;
        if (rc.nf > RC_CACHE_MAXF) return CH_DEFER;
        CH_STCS(&CW(c, 6), (int32_t) (uint32_t) ((uint64_t) rc.ts_sec >> 32));
        CH_STCS(c, (int32_t) ((uint32_t) rc.nf | ((uint32_t) rc.style << 8) | ((uint32_t) (rc.reenc ? 1 : 0) << 16)));
        CH_STCS(&CW(c, 1), (int32_t) rc.preset_n);
        CH_STCS(&CW(c, 2), (int32_t) (uint32_t) rc.ts_sec); CH_STCS(&CW(c, 3), (int32_t) (uint32_t) rc.ts_nsec);
        CH_STCS(&CW(c, 4), (int32_t) (uint32_t) rc.meta); CH_STCS(&CW(c, 5), (int32_t) (uint32_t) (rc.meta >> 32));
        for (i = 0; i < rc.nf; i++) {
            CH_STCS(&CW(c, 8 + 4 * i), (int32_t) (uint32_t) rc.k[i]); CH_STCS(&CW(c, 8 + 4 * i + 1), (int32_t) (uint32_t) (rc.k[i] >> 32));
            CH_STCS(&CW(c, 8 + 4 * i + 2), (int32_t) (uint32_t) rc.v[i]); CH_STCS(&CW(c, 8 + 4 * i + 3), (int32_t) (uint32_t) (rc.v[i] >> 32));
            CH_STCS(&CW(kh, i), (int32_t) rc.kh[i]);
        }
        return 1;
    }
    if (!EMIT && e->capcache && e->cap_stride >= RC_CACHE_INTS) {
        /* streaming stores: written once, read once by the emission pass -- they should not push the
         * lanes' local-memory lines out of L2 */
        const size_t cs = e->cap_n;
        int32_t *c = e->capcache + (size_t) (e->cap_stride - RC_CACHE_INTS) * cs + ridx;
        if (!rc.reenc) CH_STCS(c, RC_CACHE_RAW);
        else if (rc.nf > RC_CACHE_MAXF) CH_STCS(c, RC_CACHE_NONE);
        else {
            int i;
            CH_STCS(c, (int32_t) ((uint32_t) rc.nf | ((uint32_t) rc.style << 8)));
            CH_STCS(&CW(c, 1), (int32_t) rc.preset_n);
            CH_STCS(&CW(c, 2), (int32_t) (uint32_t) rc.ts_sec); CH_STCS(&CW(c, 3), (int32_t) (uint32_t) rc.ts_nsec);
            CH_STCS(&CW(c, 4), (int32_t) (uint32_t) rc.meta); CH_STCS(&CW(c, 5), (int32_t) (uint32_t) (rc.meta >> 32));
            for (i = 0; i < rc.nf; i++) {
                CH_STCS(&CW(c, 8 + 4 * i), (int32_t) (uint32_t) rc.k[i]); CH_STCS(&CW(c, 8 + 4 * i + 1), (int32_t) (uint32_t) (rc.k[i] >> 32));
                CH_STCS(&CW(c, 8 + 4 * i + 2), (int32_t) (uint32_t) rc.v[i]); CH_STCS(&CW(c, 8 + 4 * i + 3), (int32_t) (uint32_t) (rc.v[i] >> 32));
            }
        }
    }
    if (!rc.reenc) {
        if (EMIT) mp_copy(out, e->in + off, len);
        return len;
    }
    return rec_emit(e, ln, &rc, EMIT ? out : 0);
}

/* log_to_metrics: observe pending record `ridx` (its value text converts nothing) with the value the nearest earlier record of
 * the call assigned -- 0.0 when there is none (the reference's local starts at 0 in every cb_filter call).  Looking a record up
 * means running it through the chain in front of the filter again, without side effects (ln.l2m_probe). */
#define L2M_LOOKBACK_MAX 100000u
FLB_HD void l2m_fixup_record(const struct ch_env *e, uint32_t ridx, const uint32_t *off, const uint32_t *len, const uint8_t *kind)
{
    struct ch_lane ln;
    unsigned long long pr[2];
    double val = 0.0;
    uint32_t j = ridx, steps = 0;
    ln.bm = 0; ln.bm_base = ln.bm_end = 0; ln.defer_ok = 0; ln.l2m_forced = 0; ln.scr = 0; ln.dec_at = 0;
    while (j > 0) {
        j--;
        if (kind[j] != 0) continue;
        if (++steps > L2M_LOOKBACK_MAX) { CH_ATOMIC_OR(e->err, FLBGPU_E_L2M); return; }
        pr[0] = 0; pr[1] = 0;
        ln.l2m_probe = pr; ln.raw_lo = off[j];
        (void) chain_record<false>(e, &ln, j, off[j], len[j], 0);
        if (pr[0]) { union { uint64_t u; double d; } cv; cv.u = pr[1]; val = cv.d; break; }
    }
    ln.l2m_probe = 0; ln.l2m_forced = &val; ln.raw_lo = off[ridx];
    (void) chain_record<false>(e, &ln, ridx, off[ridx], len[ridx], 0);
}

#include "dev_jsmn.cuh"

#endif
