/* dev_msgpack.cuh -- msgpack walking / canonical re-encoding on the device.
 *
 * Byte rules follow msgpack-c 3.3.0 as vendored by the reference:
 *   integers .... lib/msgpack-c/include/msgpack/pack_template.h:221-277 (minimal width;
 *                 non-negative values use the unsigned family)
 *   str/bin ..... pack_template.h:762-830 (fixstr<32, str8<256, str16, str32; bin8/16/32)
 *   array/map ... pack_template.h:709-760 (fix<16, 16, 32)
 *   ext ......... pack_template.h:840-905 (fixext 1,2,4,8,16 else ext8/16/32)
 * "canonical copy" == what msgpack_pack_object() (lib/msgpack-c/src/objectc.c) writes
 * for an object that msgpack_unpack_next() read: every header re-emitted minimal,
 * payload bytes untouched; float32 stays float32.
 */
#ifndef FLBGPU_DEV_MSGPACK_CUH
#define FLBGPU_DEV_MSGPACK_CUH

#include <stdint.h>

#ifndef FLB_HD
#ifdef __CUDACC__
#define FLB_HD __host__ __device__ __forceinline__
#ifdef FLB_INLINE_ALL
#define FLB_HDN __host__ __device__ __forceinline__
#else
#define FLB_HDN __host__ __device__ __noinline__
#endif
#else
#define FLB_HD static inline
#define FLB_HDN static
#endif
#endif

FLB_HD uint32_t mp_be16(const uint8_t *p) { return ((uint32_t) p[0] << 8) | p[1]; }
FLB_HD uint32_t mp_be32(const uint8_t *p)
{
    return ((uint32_t) p[0] << 24) | ((uint32_t) p[1] << 16) | ((uint32_t) p[2] << 8) | p[3];
}
FLB_HD uint64_t mp_be64(const uint8_t *p) { return ((uint64_t) mp_be32(p) << 32) | mp_be32(p + 4); }

/* (int64_t) of a double as the reference's x86-64 build converts it (cvttsd2si): out of range and NaN give INT64_MIN, where
 * the device's conversion would saturate / give 0 */
FLB_HD int64_t mp_d2i64(double d)
{
    if (!(d >= -9223372036854775808.0 && d < 9223372036854775808.0)) return (int64_t) 0x8000000000000000ull;
    return (int64_t) d;
}

/* token classes */
enum { MPT_NIL = 0, MPT_BOOL, MPT_UINT, MPT_INT, MPT_F32, MPT_F64, MPT_STR, MPT_BIN, MPT_ARRAY, MPT_MAP,
       MPT_EXT, MPT_INVALID };

struct mp_tok {
    int      type;
    uint32_t hdr;      /* header bytes (including fixed payload for scalars) */
    uint32_t len;      /* str/bin/ext payload bytes; array/map element count */
    uint64_t u;        /* integer value (two's complement for MPT_INT), bool */
    int      ext_type;
};

/* Decode the token at p (p < end).  Returns 0, or -1 when truncated/invalid. */
FLB_HD int mp_token(const uint8_t *p, const uint8_t *end, struct mp_tok *t)
{
    uint32_t b = p[0];
    size_t rem = (size_t) (end - p);
    t->ext_type = 0; t->len = 0; t->u = 0;
    if (b < 0x80) { t->type = MPT_UINT; t->hdr = 1; t->u = b; return 0; }
    if (b >= 0xe0) { t->type = MPT_INT; t->hdr = 1; t->u = (uint64_t) (int64_t) (int8_t) b; return 0; }
    if (b <= 0x8f) { t->type = MPT_MAP; t->hdr = 1; t->len = b & 0x0f; return 0; }
    if (b <= 0x9f) { t->type = MPT_ARRAY; t->hdr = 1; t->len = b & 0x0f; return 0; }
    if (b <= 0xbf) { t->type = MPT_STR; t->hdr = 1; t->len = b & 0x1f; return 0; }
    switch (b) {
    case 0xc0: t->type = MPT_NIL; t->hdr = 1; return 0;
    case 0xc2: t->type = MPT_BOOL; t->hdr = 1; t->u = 0; return 0;
    case 0xc3: t->type = MPT_BOOL; t->hdr = 1; t->u = 1; return 0;
    case 0xc4: if (rem < 2) return -1; t->type = MPT_BIN; t->hdr = 2; t->len = p[1]; return 0;
    case 0xc5: if (rem < 3) return -1; t->type = MPT_BIN; t->hdr = 3; t->len = mp_be16(p + 1); return 0;
    case 0xc6: if (rem < 5) return -1; t->type = MPT_BIN; t->hdr = 5; t->len = mp_be32(p + 1); return 0;
    case 0xc7: if (rem < 3) return -1; t->type = MPT_EXT; t->hdr = 3; t->len = p[1]; t->ext_type = (int8_t) p[2]; return 0;
    case 0xc8: if (rem < 4) return -1; t->type = MPT_EXT; t->hdr = 4; t->len = mp_be16(p + 1); t->ext_type = (int8_t) p[3]; return 0;
    case 0xc9: if (rem < 6) return -1; t->type = MPT_EXT; t->hdr = 6; t->len = mp_be32(p + 1); t->ext_type = (int8_t) p[5]; return 0;
    case 0xca: if (rem < 5) return -1; t->type = MPT_F32; t->hdr = 5; t->u = mp_be32(p + 1); return 0;
    case 0xcb: if (rem < 9) return -1; t->type = MPT_F64; t->hdr = 9; t->u = mp_be64(p + 1); return 0;
    case 0xcc: if (rem < 2) return -1; t->type = MPT_UINT; t->hdr = 2; t->u = p[1]; return 0;
    case 0xcd: if (rem < 3) return -1; t->type = MPT_UINT; t->hdr = 3; t->u = mp_be16(p + 1); return 0;
    case 0xce: if (rem < 5) return -1; t->type = MPT_UINT; t->hdr = 5; t->u = mp_be32(p + 1); return 0;
    case 0xcf: if (rem < 9) return -1; t->type = MPT_UINT; t->hdr = 9; t->u = mp_be64(p + 1); return 0;
    case 0xd0: if (rem < 2) return -1; t->type = MPT_INT; t->hdr = 2; t->u = (uint64_t) (int64_t) (int8_t) p[1]; return 0;
    case 0xd1: if (rem < 3) return -1; t->type = MPT_INT; t->hdr = 3; t->u = (uint64_t) (int64_t) (int16_t) mp_be16(p + 1); return 0;
    case 0xd2: if (rem < 5) return -1; t->type = MPT_INT; t->hdr = 5; t->u = (uint64_t) (int64_t) (int32_t) mp_be32(p + 1); return 0;
    case 0xd3: if (rem < 9) return -1; t->type = MPT_INT; t->hdr = 9; t->u = mp_be64(p + 1); return 0;
    case 0xd4: if (rem < 2) return -1; t->type = MPT_EXT; t->hdr = 2; t->len = 1; t->ext_type = (int8_t) p[1]; return 0;
    case 0xd5: if (rem < 2) return -1; t->type = MPT_EXT; t->hdr = 2; t->len = 2; t->ext_type = (int8_t) p[1]; return 0;
    case 0xd6: if (rem < 2) return -1; t->type = MPT_EXT; t->hdr = 2; t->len = 4; t->ext_type = (int8_t) p[1]; return 0;
    case 0xd7: if (rem < 2) return -1; t->type = MPT_EXT; t->hdr = 2; t->len = 8; t->ext_type = (int8_t) p[1]; return 0;
    case 0xd8: if (rem < 2) return -1; t->type = MPT_EXT; t->hdr = 2; t->len = 16; t->ext_type = (int8_t) p[1]; return 0;
    case 0xd9: if (rem < 2) return -1; t->type = MPT_STR; t->hdr = 2; t->len = p[1]; return 0;
    case 0xda: if (rem < 3) return -1; t->type = MPT_STR; t->hdr = 3; t->len = mp_be16(p + 1); return 0;
    case 0xdb: if (rem < 5) return -1; t->type = MPT_STR; t->hdr = 5; t->len = mp_be32(p + 1); return 0;
    case 0xdc: if (rem < 3) return -1; t->type = MPT_ARRAY; t->hdr = 3; t->len = mp_be16(p + 1); return 0;
    case 0xdd: if (rem < 5) return -1; t->type = MPT_ARRAY; t->hdr = 5; t->len = mp_be32(p + 1); return 0;
    case 0xde: if (rem < 3) return -1; t->type = MPT_MAP; t->hdr = 3; t->len = mp_be16(p + 1); return 0;
    case 0xdf: if (rem < 5) return -1; t->type = MPT_MAP; t->hdr = 5; t->len = mp_be32(p + 1); return 0;
    default: t->type = MPT_INVALID; return -1;     /* 0xc1 */
    }
}

/* Skip one complete object starting at p.  Returns the first byte after it, or
 * NULL when the object is truncated or malformed.  Nesting needs no stack: a
 * single "objects still owed" counter is enough to find the end. */
FLB_HD const uint8_t *mp_skip(const uint8_t *p, const uint8_t *end)
{
    uint64_t owed = 1;
    struct mp_tok t;
    while (owed) {
        if (p >= end) return 0;
        if (mp_token(p, end, &t) != 0) return 0;
        owed--;
        p += t.hdr;
        if (t.type == MPT_STR || t.type == MPT_BIN || t.type == MPT_EXT) {
            if ((size_t) (end - p) < t.len) return 0;
            p += t.len;
        }
        else if (t.type == MPT_ARRAY) owed += t.len;
        else if (t.type == MPT_MAP) owed += 2 * (uint64_t) t.len;
    }
    return p;
}

/* msgpack-c's unpacker keeps its open containers on a stack of MSGPACK_EMBED_STACK_SIZE (32) entries and fails with
 * MSGPACK_UNPACK_NOMEM_ERROR when a container header -- empty or not -- arrives while `top` is already 32
 * (lib/msgpack-c/include/msgpack/unpack_template.h:140-144, start_container): to flb_log_event_decoder_next() such an event
 * is a deserialization failure like any malformed byte.  mp_skip_lim() is mp_skip() with that rule: `top0` containers are open
 * around the object at p.  The exact walk needs the count owed to every open container, so it runs only for objects that hold
 * enough container headers to reach the limit at all. */
#define MP_UNPACK_STACK 32
FLB_HD
#ifdef __CUDACC__
__noinline__
#endif
const uint8_t *mp_skip_exact(const uint8_t *p, const uint8_t *end, uint32_t top0)
{
    uint32_t owed[MP_UNPACK_STACK];
    uint32_t d = 0;                        /* containers of this object that are open */
    struct mp_tok t;
    for (;;) {
        uint32_t items = 0;
        int container = 0;
        if (p >= end) return 0;
        if (mp_token(p, end, &t) != 0) return 0;
        p += t.hdr;
        if (t.type == MPT_STR || t.type == MPT_BIN || t.type == MPT_EXT) {
            if ((size_t) (end - p) < t.len) return 0;
            p += t.len;
        }
        else if (t.type == MPT_ARRAY) { container = 1; items = t.len; }
        else if (t.type == MPT_MAP) { container = 1; if (t.len > 0x7fffffffu) return 0; items = 2 * t.len; }
        if (container) {
            if (top0 + d >= MP_UNPACK_STACK) return 0;
            if (items) { owed[d++] = items; continue; }
        }
        for (;;) {                         /* one object done: pay it to the containers it closes */
            if (d == 0) return p;
            if (--owed[d - 1]) break;
            d--;
        }
    }
}
FLB_HD const uint8_t *mp_skip_lim(const uint8_t *p, const uint8_t *end, uint32_t top0)
{
    const uint8_t *p0 = p;
    uint64_t owed = 1;
    uint32_t containers = 0;
    struct mp_tok t;
    while (owed) {
        if (p >= end) return 0;
        if (mp_token(p, end, &t) != 0) return 0;
        owed--;
        p += t.hdr;
        if (t.type == MPT_STR || t.type == MPT_BIN || t.type == MPT_EXT) {
            if ((size_t) (end - p) < t.len) return 0;
            p += t.len;
        }
        else if (t.type == MPT_ARRAY) { owed += t.len; containers++; }
        else if (t.type == MPT_MAP) { owed += 2 * (uint64_t) t.len; containers++; }
    }
    if (top0 + containers <= MP_UNPACK_STACK) return p;          /* even nested one inside the other they fit */
    return mp_skip_exact(p0, end, top0);
}

/* ---- sizes of canonical headers ---- */
FLB_HD uint32_t mp_str_hdr_size(uint32_t n) { return n < 32 ? 1 : n < 256 ? 2 : n < 65536 ? 3 : 5; }
FLB_HD uint32_t mp_bin_hdr_size(uint32_t n) { return n < 256 ? 2 : n < 65536 ? 3 : 5; }
FLB_HD uint32_t mp_cnt_hdr_size(uint32_t n) { return n < 16 ? 1 : n < 65536 ? 3 : 5; }
FLB_HD uint32_t mp_ext_hdr_size(uint32_t n)
{
    if (n == 1 || n == 2 || n == 4 || n == 8 || n == 16) return 2;
    return n < 256 ? 3 : n < 65536 ? 4 : 6;
}
FLB_HD uint32_t mp_uint_size(uint64_t v) { return v < 128 ? 1 : v < 256 ? 2 : v < 65536 ? 3 : v < 4294967296ull ? 5 : 9; }
FLB_HD uint32_t mp_int_size(int64_t v)
{
    if (v >= 0) return mp_uint_size((uint64_t) v);
    if (v >= -32) return 1;
    if (v >= -128) return 2;
    if (v >= -32768) return 3;
    if (v >= -2147483648ll) return 5;
    return 9;
}

/* ---- writers: return bytes written ---- */
FLB_HD uint32_t mp_put_be16(uint8_t *o, uint32_t v) { o[0] = (uint8_t) (v >> 8); o[1] = (uint8_t) v; return 2; }
FLB_HD uint32_t mp_put_be32(uint8_t *o, uint32_t v)
{
    o[0] = (uint8_t) (v >> 24); o[1] = (uint8_t) (v >> 16); o[2] = (uint8_t) (v >> 8); o[3] = (uint8_t) v;
    return 4;
}
FLB_HD uint32_t mp_put_be64(uint8_t *o, uint64_t v)
{
    mp_put_be32(o, (uint32_t) (v >> 32)); mp_put_be32(o + 4, (uint32_t) v);
    return 8;
}
FLB_HD uint32_t mp_put_str_hdr(uint8_t *o, uint32_t n)
{
    if (n < 32) { o[0] = 0xa0 | n; return 1; }
    if (n < 256) { o[0] = 0xd9; o[1] = (uint8_t) n; return 2; }
    if (n < 65536) { o[0] = 0xda; mp_put_be16(o + 1, n); return 3; }
    o[0] = 0xdb; mp_put_be32(o + 1, n); return 5;
}
FLB_HD uint32_t mp_put_bin_hdr(uint8_t *o, uint32_t n)
{
    if (n < 256) { o[0] = 0xc4; o[1] = (uint8_t) n; return 2; }
    if (n < 65536) { o[0] = 0xc5; mp_put_be16(o + 1, n); return 3; }
    o[0] = 0xc6; mp_put_be32(o + 1, n); return 5;
}
FLB_HD uint32_t mp_put_map_hdr(uint8_t *o, uint32_t n)
{
    if (n < 16) { o[0] = 0x80 | n; return 1; }
    if (n < 65536) { o[0] = 0xde; mp_put_be16(o + 1, n); return 3; }
    o[0] = 0xdf; mp_put_be32(o + 1, n); return 5;
}
FLB_HD uint32_t mp_put_array_hdr(uint8_t *o, uint32_t n)
{
    if (n < 16) { o[0] = 0x90 | n; return 1; }
    if (n < 65536) { o[0] = 0xdc; mp_put_be16(o + 1, n); return 3; }
    o[0] = 0xdd; mp_put_be32(o + 1, n); return 5;
}
FLB_HD uint32_t mp_put_ext_hdr(uint8_t *o, uint32_t n, int type)
{
    if (n == 1) { o[0] = 0xd4; o[1] = (uint8_t) type; return 2; }
    if (n == 2) { o[0] = 0xd5; o[1] = (uint8_t) type; return 2; }
    if (n == 4) { o[0] = 0xd6; o[1] = (uint8_t) type; return 2; }
    if (n == 8) { o[0] = 0xd7; o[1] = (uint8_t) type; return 2; }
    if (n == 16) { o[0] = 0xd8; o[1] = (uint8_t) type; return 2; }
    if (n < 256) { o[0] = 0xc7; o[1] = (uint8_t) n; o[2] = (uint8_t) type; return 3; }
    if (n < 65536) { o[0] = 0xc8; mp_put_be16(o + 1, n); o[3] = (uint8_t) type; return 4; }
    o[0] = 0xc9; mp_put_be32(o + 1, n); o[5] = (uint8_t) type; return 6;
}
FLB_HD uint32_t mp_put_uint(uint8_t *o, uint64_t v)
{
    if (v < 128) { o[0] = (uint8_t) v; return 1; }
    if (v < 256) { o[0] = 0xcc; o[1] = (uint8_t) v; return 2; }
    if (v < 65536) { o[0] = 0xcd; mp_put_be16(o + 1, (uint32_t) v); return 3; }
    if (v < 4294967296ull) { o[0] = 0xce; mp_put_be32(o + 1, (uint32_t) v); return 5; }
    o[0] = 0xcf; mp_put_be64(o + 1, v); return 9;
}
FLB_HD uint32_t mp_put_int(uint8_t *o, int64_t v)
{
    if (v >= 0) return mp_put_uint(o, (uint64_t) v);
    if (v >= -32) { o[0] = (uint8_t) v; return 1; }
    if (v >= -128) { o[0] = 0xd0; o[1] = (uint8_t) v; return 2; }
    if (v >= -32768) { o[0] = 0xd1; mp_put_be16(o + 1, (uint32_t) (uint16_t) v); return 3; }
    if (v >= -2147483648ll) { o[0] = 0xd2; mp_put_be32(o + 1, (uint32_t) v); return 5; }
    o[0] = 0xd3; mp_put_be64(o + 1, (uint64_t) v); return 9;
}

/* copy of n bytes between arbitrary alignments.  On the device: bytes until the destination is
 * 4-aligned, then one aligned 32-bit store per word, the source word assembled from two aligned
 * loads with a funnel shift (source buffers are padded, see bk_alloc); the emission pass is mostly
 * this loop. */
FLB_HD void mp_copy(uint8_t *o, const uint8_t *s, uint32_t n)
{
    uint32_t i = 0;
#ifdef __CUDA_ARCH__
    if (n >= 8) {
        while (((uintptr_t) (o + i)) & 3) { o[i] = s[i]; i++; }
        {
            const uintptr_t sa = (uintptr_t) (s + i);
            const uint32_t *sw = (const uint32_t *) (sa & ~(uintptr_t) 3);
            const uint32_t sh = (uint32_t) (sa & 3) * 8;
            uint32_t *ow = (uint32_t *) (o + i);
            uint32_t lo = *sw++;
            for (; i + 4 <= n; i += 4) {
                uint32_t hi = sh ? *sw++ : 0, v;
                if (sh) { v = __funnelshift_r(lo, hi, sh); lo = hi; }
                else { v = lo; lo = *sw++; }
                *ow++ = v;
            }
        }
    }
#endif
    for (; i < n; i++) o[i] = s[i];
}

/* Canonical re-encoding of the complete object at p (already validated by
 * mp_skip).  When o is NULL only the size is computed.  Returns the output size;
 * *consumed gets the input size. */
FLB_HDN uint32_t mp_canon(const uint8_t *p, const uint8_t *end, uint8_t *o, uint32_t *consumed)
{
    const uint8_t *p0 = p;
    uint64_t owed = 1;
    uint32_t out = 0;
    struct mp_tok t;
    while (owed) {
        if (p >= end || mp_token(p, end, &t) != 0) break;
        owed--;
        switch (t.type) {
        case MPT_UINT:
            if (o) mp_put_uint(o + out, t.u);
            out += mp_uint_size(t.u);
            break;
        case MPT_INT:
            if (o) mp_put_int(o + out, (int64_t) t.u);
            out += mp_int_size((int64_t) t.u);
            break;
        case MPT_STR:
            if (o) { mp_put_str_hdr(o + out, t.len); mp_copy(o + out + mp_str_hdr_size(t.len), p + t.hdr, t.len); }
            out += mp_str_hdr_size(t.len) + t.len;
            break;
        case MPT_BIN:
            if (o) { mp_put_bin_hdr(o + out, t.len); mp_copy(o + out + mp_bin_hdr_size(t.len), p + t.hdr, t.len); }
            out += mp_bin_hdr_size(t.len) + t.len;
            break;
        case MPT_EXT:
            if (o) { mp_put_ext_hdr(o + out, t.len, t.ext_type); mp_copy(o + out + mp_ext_hdr_size(t.len), p + t.hdr, t.len); }
            out += mp_ext_hdr_size(t.len) + t.len;
            break;
        case MPT_ARRAY:
            if (o) mp_put_array_hdr(o + out, t.len);
            out += mp_cnt_hdr_size(t.len);
            owed += t.len;
            break;
        case MPT_MAP:
            if (o) mp_put_map_hdr(o + out, t.len);
            out += mp_cnt_hdr_size(t.len);
            owed += 2 * (uint64_t) t.len;
            break;
        default:                      /* nil, bool, f32, f64: byte-identical */
            if (o) mp_copy(o + out, p, t.hdr);
            out += t.hdr;
            break;
        }
        p += t.hdr;
        if (t.type == MPT_STR || t.type == MPT_BIN || t.type == MPT_EXT) p += t.len;
    }
    if (consumed) *consumed = (uint32_t) (p - p0);
    return out;
}

#endif
