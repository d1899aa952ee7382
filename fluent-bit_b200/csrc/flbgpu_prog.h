/* flbgpu_prog.h -- plain-old-data layouts shared by the host-side compilers (C)
 * and the device interpreters (CUDA).  Everything a kernel needs at run time
 * (regex programs, strptime programs, the filter-chain program, the constant
 * pool) lives in ONE relocatable byte blob; every cross reference is a byte
 * offset from the blob base, so the blob is uploaded to HBM with one memcpy.
 */
#ifndef FLBGPU_PROG_H
#define FLBGPU_PROG_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ regex */
/* Instruction word: low 8 bits opcode, high 24 bits argument.  Semantics are
 * those of Onigmo's backtracking matcher (lib/onigmo/regexec.c:1431 match_at):
 * leftmost start, alternatives tried in priority order, captures restored on
 * backtrack. */
enum {
    RX_MATCH = 0,      /* success */
    RX_FAIL,           /* force backtrack */
    RX_BYTE,           /* arg = byte value */
    RX_STR,            /* arg = n bytes; bytes packed in following ceil(n/4) words */
    RX_CLASS,          /* arg = class index; consumes one character */
    RX_ANY,            /* any character except '\n' (OP_ANYCHAR) */
    RX_ANY_NL,         /* any character (OP_ANYCHAR_ML) */
    RX_JMP,            /* arg = absolute pc */
    RX_SPLIT,          /* continue at pc+1, alternative = arg (absolute pc) */
    RX_SPLIT_LAZY,     /* continue at arg, alternative = pc+1 */
    RX_SAVE,           /* arg = capture slot (2*g or 2*g+1) */
    RX_CSTAR_POSS,     /* arg = class: cls* with no alternatives left behind */
    RX_CSTAR_BT,       /* arg = class: greedy cls*, one back-off frame */
    RX_CSTAR_LAZY,     /* arg = class: lazy cls*? */
    RX_BOL,            /* ^  (ANCHOR_BEGIN_LINE) */
    RX_EOL,            /* $  (ANCHOR_END_LINE) */
    RX_BEGIN_BUF,      /* \A */
    RX_END_BUF,        /* \z */
    RX_SEMI_END_BUF,   /* \Z */
    RX_WORD_B,         /* \b */
    RX_NOT_WORD_B,     /* \B */
    RX_NULL_START,     /* arg = loop id: remember position (OP_NULL_CHECK_START) */
    RX_NULL_END,       /* arg = loop id: if iteration was empty skip next insn */
    RX_MARK,           /* arg = kind: push a cut mark (look-ahead / atomic) */
    RX_CUT_POS,        /* positive look-ahead end: cut to mark, restore position */
    RX_CUT_ATOMIC,     /* atomic group end: cut to mark, keep position */
    RX_CUT_NEG,        /* negative look-ahead body matched: cut to mark, drop the
                          alternative below it, fail */
    RX_BACKREF,        /* arg = group number */
    RX_OPCOUNT
};

#define RX_OP(w)   ((w) & 0xffu)
#define RX_ARG(w)  ((w) >> 8)
#define RX_MK(op, arg) (((uint32_t)(arg) << 8) | (uint32_t)(op))

/* class.mb_mode */
enum { RX_MB_NONE = 0, RX_MB_ALL = 1, RX_MB_RANGES = 2, RX_MB_NOT_RANGES = 3 };

struct rx_class {
    uint32_t bits[8];      /* membership of single-byte characters (incl. invalid high bytes) */
    uint32_t mb_mode;      /* how valid multi-byte characters are decided */
    uint32_t n_ranges;     /* code point ranges [lo,hi] for RX_MB_RANGES / RX_MB_NOT_RANGES */
    uint32_t ranges_off;   /* byte offset from the rx_prog header to uint32 pairs */
    uint32_t pad;
};

#define RX_MAX_GROUPS 47   /* named/numbered groups, group 0 excluded */
#define RX_F_ANCHOR_BOL   1u   /* every match starts at a line start   */
#define RX_F_ANCHOR_BUF   2u   /* every match starts at offset 0       */
#define RX_F_HAS_FIRSTSET 4u   /* first[] is a sound first-byte filter */
#define RX_F_NULLABLE     8u   /* the pattern can match the empty string */
#define RX_F_HAS_SECONDSET 32u /* second[] is a sound filter on the byte behind an ASCII first byte */
#define RX_F_ASCII_ONLY  16u   /* the pattern uses a construct whose non-ASCII behaviour is not restated (POSIX bracket, \b \B,
                                  case-insensitive matching: Onigmo consults its Unicode tables there): a subject with a byte >= 0x80
                                  is refused loudly (RX_R_EUNICODE), never matched approximately */

struct rx_prog {
    uint32_t total_bytes;  /* size of this program incl. header, code, classes, ranges */
    uint32_t n_code;       /* 32-bit words of code */
    uint32_t code_off;     /* byte offset of code[] from this header */
    uint32_t n_classes;
    uint32_t class_off;    /* byte offset of struct rx_class[] */
    uint32_t n_groups;     /* capture groups (group 0 excluded) */
    uint32_t flags;
    uint32_t n_null;       /* number of null-check loop ids */
    uint32_t first[8];     /* first-byte filter (valid when RX_F_HAS_FIRSTSET) */
    uint32_t second[8];    /* RX_F_HAS_SECONDSET: the pattern begins with exactly one character and cannot end right behind it --
                              the bytes that can follow that character.  A start whose first byte is ASCII (one byte wide) and whose
                              next byte is not in the set cannot match: `(.)(?:Exception|Error)` tries 3 starts per line, not 100 */
};

/* run-time status of one match attempt */
#define RX_R_NOMATCH   0
#define RX_R_MATCH     1
#define RX_R_ESTACK   -2   /* backtrack stack exhausted: rerun with a bigger stack */
#define RX_R_EBUDGET  -3   /* step budget exhausted (catastrophic backtracking guard) */
#define RX_R_EUNICODE -4   /* RX_F_ASCII_ONLY pattern met a non-ASCII subject */


/* ------------------------------------------------------- chain program */
/* All *_off fields are byte offsets from the blob base; 0 means "absent". */

enum { FLBGPU_F_PARSER = 1, FLBGPU_F_GREP, FLBGPU_F_MODIFY, FLBGPU_F_RECORD_MODIFIER, FLBGPU_F_LOG_TO_METRICS, FLBGPU_F_REWRITE_TAG,
       FLBGPU_F_MULTILINE };

/* parser types: include/fluent-bit/flb_parser.h:30-33 */
enum { FLBGPU_PARSER_REGEX = 1, FLBGPU_PARSER_JSON, FLBGPU_PARSER_LTSV, FLBGPU_PARSER_LOGFMT };
/* Types casts: include/fluent-bit/flb_parser.h:70-76 */
enum { FLBGPU_TYPE_INT = 1, FLBGPU_TYPE_FLOAT, FLBGPU_TYPE_BOOL, FLBGPU_TYPE_STRING, FLBGPU_TYPE_HEX };

struct cf_ra_sub { uint32_t is_index, index, str_off, str_len; };
/* final field list of a surviving record, left by the evaluation pass for the emission pass in the
 * last RC_CACHE_INTS ints of the record's capture-cache row: 8 header ints + 4 per field */
#define RC_CACHE_MAXF 16
#define RC_CACHE_INTS (8 + 4 * RC_CACHE_MAXF)
#define RC_CACHE_NONE (-1)
#define RC_CACHE_RAW  (-2)

struct cf_ra { uint32_t key_off, key_len, n_sub, sub_off; };

struct cf_pname {              /* one (name, group) pair in onig_foreach_name order */
    uint32_t kmp_off, kmp_len; /* the name as a msgpack str, in the constant pool */
    uint32_t raw_off, raw_len; /* the name's bytes */
    uint32_t group;
    uint32_t is_time;          /* this is the Time_Key */
    uint32_t cast;             /* FLBGPU_TYPE_* or 0 */
    uint32_t hash;             /* ch_khash() of the name */
};

struct cf_ptype { uint32_t key_off, key_len, type, pad; };

struct cf_pdef {               /* device view of struct flb_parser (flb_parser.h:41-68) */
    uint32_t type;
    uint32_t rx_off;
    uint32_t n_names, names_off;
    uint32_t skip_empty, time_keep, time_strict, has_time;
    uint32_t time_with_year, time_with_tz;
    int32_t  time_offset;
    uint32_t fmt_off, frac_off, has_frac;
    uint32_t time_key_off, time_key_len;
    uint32_t n_types, types_off;
    uint32_t logfmt_no_bare_keys;
    uint32_t n_groups;
    uint32_t tfast_off;        /* compiled fixed-shape time program (TF_* ops), 0 = none */
    uint32_t n_dec;            /* field decoders (Decode_Field / Decode_Field_As): struct cf_pdec[n_dec] at dec_off */
    uint32_t dec_off;
    uint32_t time_key_hash;    /* ch_khash() of the Time_Key */
};

/* struct flb_parser_dec / flb_parser_dec_rule, include/fluent-bit/flb_parser_decoder.h:27-59 */
enum { PDEC_DEFAULT = 0, PDEC_AS = 1 };                                        /* rule type */
enum { PDEC_JSON = 0, PDEC_ESCAPED = 1, PDEC_ESCAPED_UTF8 = 2, PDEC_MYSQL_QUOTED = 3 };   /* backend */
enum { PDEC_ACT_NONE = 0, PDEC_ACT_TRY_NEXT = 1, PDEC_ACT_DO_NEXT = 2 };
struct cf_pdec_rule { uint32_t type, backend, action, pad; };
struct cf_pdec { uint32_t key_off, key_len, add_extra_keys, n_rules, rules_off, pad0, pad1, pad2; };

/* Fixed-shape time program: what flb_strptime() does for the format when every numeric field has its
 * full width, spaces are single, month names are the 3-letter forms and the zone is Z or +hh[:]mm.
 * Any other value makes the program give up and the general interpreter decides. */
enum { TF_END = 0, TF_D2, TF_Y4, TF_LIT, TF_SPACE, TF_MON3, TF_TZ, TF_FRAC };
enum { TFF_MDAY = 0, TFF_MON, TFF_HOUR, TFF_MIN, TFF_SEC };

struct cf_parser {             /* filter_parser */
    uint32_t key_off, key_len;
    uint32_t ra_off;
    uint32_t reserve_data, preserve_key;
    uint32_t n_parsers;
    uint32_t pdef_off[8];
};

enum { GREP_REGEX = 1, GREP_EXCLUDE = 2 };
enum { GREP_OP_LEGACY = 0, GREP_OP_OR, GREP_OP_AND };
struct cf_grep_rule { uint32_t type, ra_off, rx_off, pad; };
struct cf_grep { uint32_t op, n_rules, rules_off, pad; };

/* plugins/filter_rewrite_tag/rewrite_tag.h: struct rewrite_rule, and the parts of its tag template as
 * ra_parse_buffer() (src/flb_record_accessor.c:75-214) cuts them */
enum { RT_STRING = 1, RT_KEYMAP, RT_REGEX_ID, RT_TAG, RT_TAG_PART };
struct cf_rt_part { uint32_t type, a, b, pad; };     /* STRING: a = offset, b = length; KEYMAP: a = struct cf_ra; REGEX_ID / TAG_PART: a = id */
struct cf_rt_rule { uint32_t ra_off, rx_off, keep, n_parts, parts_off, pad0, pad1, pad2; };
struct cf_rtag { uint32_t n_rules, rules_off, pad0, pad1; };
/* one entry of the re-tagged stream a rewrite_tag filter leaves beside its result: u32 tag length, u32 record bytes,
 * the tag, the record as the filter saw it (what the reference hands to in_emitter_add_record()) */
#define RT_ENTRY_HDR 8u

/* plugins/filter_modify/modify.h rule / condition kinds */
enum { MOD_RENAME = 1, MOD_HARD_RENAME, MOD_ADD, MOD_SET, MOD_REMOVE, MOD_REMOVE_WILDCARD, MOD_REMOVE_REGEX,
       MOD_COPY, MOD_HARD_COPY, MOD_MOVE_TO_START, MOD_MOVE_TO_END };
enum { MODC_KEY_EXISTS = 1, MODC_KEY_DOES_NOT_EXIST, MODC_A_KEY_MATCHES, MODC_NO_KEY_MATCHES,
       MODC_KEY_VALUE_EQUALS, MODC_KEY_VALUE_DOES_NOT_EQUAL, MODC_KEY_VALUE_MATCHES,
       MODC_KEY_VALUE_DOES_NOT_MATCH, MODC_MATCHING_KEYS_HAVE_MATCHING_VALUES,
       MODC_MATCHING_KEYS_DO_NOT_HAVE_MATCHING_VALUES };
struct cf_mod_cond { uint32_t type, ra_off, b_off, b_len, a_rx, b_rx, pad0, pad1; };
struct cf_mod_rule {
    uint32_t type;
    uint32_t key_off, key_len;     /* raw bytes */
    uint32_t kmp_off, kmp_len;     /* msgpack str */
    uint32_t val_off, val_len;
    uint32_t vmp_off, vmp_len;
    uint32_t key_rx;
    uint32_t key_hash, val_hash;   /* ch_khash() of key / val (dev_chain.cuh) */
};
struct cf_modify { uint32_t n_conds, conds_off, n_rules, rules_off; };

struct cf_rm_key { uint32_t off, len, dynamic, pad; };
struct cf_rm_rec { uint32_t kmp_off, kmp_len, vmp_off, vmp_len; };
struct cf_recmod { uint32_t n_records, records_off, n_remove, remove_off, n_allow, allow_off, pad0, pad1; };

/* filter_log_to_metrics (plugins/filter_log_to_metrics/log_to_metrics.c) */
enum { L2M_COUNTER = 0, L2M_GAUGE = 1, L2M_HISTOGRAM = 2 };
#define L2M_MAX_LABELS 16
#define L2M_LABEL_BYTES 256          /* MAX_LABEL_LENGTH 253 rounded up */
#define L2M_SLOTS_LOG2 16
struct cf_l2m {
    uint32_t grep_off;               /* struct cf_grep (legacy semantics) for Regex / Exclude */
    uint32_t mode;
    uint32_t n_labels;
    uint32_t label_ra_off[L2M_MAX_LABELS];
    uint32_t value_ra_off;
    uint32_t n_buckets;
    uint32_t buckets_off;            /* double[n_buckets], ascending */
    uint32_t discard;
};

/* per-call device table of label sets (open addressing on a 64-bit hash of the label values) */
struct l2m_table {
    unsigned long long *hash;        /* 0 = empty; over the label values WITH their lengths: one slot per exact label tuple */
    unsigned long long *chash;       /* over the label values run together, as cmetrics hashes them (cmt_map.c:208-222): tuples that
                                        concatenate to the same text are ONE metric there; the host folds such slots together */
    uint32_t *first;                 /* 0xffffffff - (smallest record index of the set) */
    unsigned long long *cnt;         /* counter value / histogram count */
    double *sum;                     /* histogram sum */
    unsigned long long *bkt;         /* [slot][n_buckets + 1] cumulative buckets, last = +Inf; gauge: [slot][2] = last record + 1, value bits */
    uint8_t *str;                    /* [slot][n_labels][L2M_LABEL_BYTES]: length byte + bytes */
    uint32_t mask;
    uint32_t pending_cap;
    /* gauge / histogram: records whose value text sscanf("%lf") cannot convert -- the reference then observes the value the
     * previous converting record of the call left in its local variable (log_to_metrics.c:983-984,1060,1090).  They are listed
     * here by the evaluation launch and observed by a follow-up launch that looks that value up (k_l2m_fixup).
     * pending_n[0] = listed, [1] = done. */
    uint32_t *pending;
    unsigned long long *pending_n;
    /* histogram: the reference adds every observation to the set's sum in record order (cmt_metric_hist_sum_add()), which
     * the atomic sum above matches only when every addition is exact.  amax[slot] = the largest |value| of the call's
     * observations when all of them are integers of at most 2^53 (and none is -0.0), else L2M_NOT_EXACT; the host keeps the
     * atomic sum where that proves it exact, and otherwise adds obs_val up in record order.  obs_slot[record] = slot + 1 of
     * the record's observation (0: none), indexed by the call's record index. */
    unsigned long long *amax;
    uint32_t *obs_slot;
    double *obs_val;
};
#define L2M_PENDING_CAP 65536u
#define L2M_NOT_EXACT 0xffffffffffffffffull
#define L2M_EXACT_MAX 9007199254740992ull      /* 2^53: every integer up to here is a double */

struct chain_filter { uint32_t kind, cfg_off; };

#define FLBGPU_MAX_FILTERS 16
struct chain_hdr {
    uint32_t total_bytes;
    uint32_t n_filters;
    uint32_t filters_off;      /* struct chain_filter[] */
    uint32_t cap_stride;       /* ints of capture cache per record (0 = none) */
    uint32_t empty_map_off;    /* one byte 0x80 */
    uint32_t needs_scratch;
    uint32_t split_at;         /* split evaluation: the head launch runs filters [0, split_at) -- the parser and the grep filters right
                                  behind it, which only look --, the tail launch the rest, over the records that are still there */
    uint32_t pad1;
};

/* per-filter chunk-level evidence accumulated by the evaluation pass */
#define CHF_CAUSE   1u   /* some record made this filter "modify" the chunk */
#define CHF_EMITTED 2u   /* some record left this filter */

/* record-level problems (bit set in the per-call error word; the call fails loudly) */
#define FLBGPU_E_FIELDS    1u   /* more top-level keys than the interpreter holds */
#define FLBGPU_E_RXSTACK   2u   /* regex backtrack stack exhausted */
#define FLBGPU_E_RXBUDGET  4u   /* regex step budget exhausted */
#define FLBGPU_E_FLOAT     8u   /* strtod() text that is not restated: hex float, nan(payload) */
#define FLBGPU_E_INDEX    16u   /* record index fast path failed */
#define FLBGPU_E_ESCAPE   32u   /* logfmt escapes met without a scratch region (cannot happen through the C ABI) */
#define FLBGPU_E_L2M      64u   /* log_to_metrics: label table full / float label / unparsable value */
#define FLBGPU_E_DEEP    256u   /* a parser made a value nested near msgpack-c's unpack limit: the filters behind it must see it as the
                                   reference's decoder does -- the call is run filter by filter */
#define FLBGPU_E_TAGVALUE 512u   /* rewrite_tag: a tag template names a float or a map (snprintf("%f") / JSON text are not restated) */
#define FLBGPU_E_RXUNICODE 128u /* a pattern with POSIX brackets / \b / case-insensitivity met a non-ASCII subject */

#define FLBGPU_E_MLLIMIT 1024u  /* multiline: a concatenated message reached the buffer limit (the reference truncates it and marks the record) */
#define FLBGPU_E_MLMETA  2048u  /* multiline: more metadata members in one message than the merge holds (ML_MD_MAX) */

/* ---------------------------------------------------- filter_multiline (dev_ml.cuh) */
/* One multiline parser instance as the filter runs it in `buffer off` mode (plugins/filter_multiline/ml.c:792-892,
 * src/multiline/flb_ml.c, flb_ml_rule.c).  The per-line work (find key_content, which rules' regexes match) is one lane per
 * record; what is sequential in the reference -- the rule state, "is the buffer empty", "is there a first-line context" -- is a
 * finite automaton over the records, composed over blocks of records and scanned (dev_ml.cuh). */
#define ML_MAX_RULES 15
enum { ML_T_REGEX = 0, ML_T_ENDSWITH = 1, ML_T_EQ = 2 };
struct cf_ml_rule {
    uint32_t rx_off;           /* regex program */
    uint32_t start;            /* from_states names start_state */
    uint32_t next_start;       /* some rule of to_state_map is a start state: the buffer is flushed right after this rule matched */
    uint32_t n_to;             /* to_state_map without its start-state rules, in list order */
    uint8_t to[16];
};
struct cf_ml {
    uint32_t type, negate, n_rules, rules_off;
    uint32_t key_off, key_len;        /* key_content; key_len 0xffffffff: none (every record passes through on its own) */
    uint32_t match_off, match_len;    /* ENDSWITH / EQ */
    uint32_t limit;                   /* multiline buffer limit in bytes, 0 = none */
    uint32_t pad[3];
};
/* per record, after the parallel pass */
#define MLF_MASK   0x7fffu     /* bit j: rule j matches the content (ENDSWITH / EQ: bit 0 = the match, negate applied) */
#define MLF_HAS    0x10000u    /* key_content found with a string value */
#define MLF_LENOK  0x20000u    /* ENDSWITH: the content is at least as long as the match string */
#define MLF_LIVE   0x40000u    /* an event the decoder yields */
struct ml_feat { uint32_t coff, clen, bits; };
/* per record, after the automaton ran over it */
#define MLA_FB      1u   /* the pending message is flushed (and comes out) before this record is looked at */
#define MLA_APP     2u   /* the record appends to the buffer */
#define MLA_NL      4u   /* ... a line feed only (a continuation line whose content is empty) */
#define MLA_SEP     8u   /* ... behind a line feed when the buffer does not end in one */
#define MLA_CTXMAP  16u  /* its map becomes the first-line context */
#define MLA_CTXTIME 32u  /* its timestamp becomes the message's */
#define MLA_FA      64u  /* the message is flushed (and comes out) right after this record */
#define MLA_ALONE   128u /* nothing took the line: what was pending went out, the record goes out on its own */
#define ML_MD_MAX 48u    /* metadata members of the lines of one message (before the duplicates go) */
#define ML_F1 64u        /* records per automaton block, blocks per super-block */
#define ML_F2 128u
#define ML_MAX_STATES ((ML_MAX_RULES + 1) * 4)
/* everything one call of the multiline filter works on (device pointers; dev_ml.cuh) */
struct ml_env {
    const uint8_t *in;
    const uint8_t *blob;
    uint32_t cfg_off;                 /* struct cf_ml */
    const uint32_t *off, *len; const uint8_t *kind;
    uint32_t n_rec;
    uint32_t *err;                    /* FLBGPU_E_* */
    /* per record */
    struct ml_feat *feat;
    uint8_t *act;
    uint32_t *tl;                     /* 1 + index of the last record at or before this one that registered its time, 0 = none yet */
    /* automaton tree */
    uint8_t *T1, *T2, *in1, *in2;     /* [nt1][S], [nt2][S], [nt1], [nt2] */
    uint32_t *cnt1, *lt1, *cnt2, *lt2, *base1, *tl1, *base2, *tl2;
    uint32_t nt1, nt2, S;
    uint32_t state_in;                /* the automaton's state when the call begins (rule carried over from the previous chunk) */
    int64_t time_in[2];               /* the group's mp_time when the call begins */
    int64_t now[2];                   /* what stands in for flb_time_get() when a message has no time */
    /* results of the plan: [0] events, [1] final state, [2] seconds, [3] nanoseconds of the group's mp_time afterwards */
    unsigned long long *res;
    /* per event (flush) */
    uint32_t *ev_slot, *ev_size, *ev_buflen, *ev_ctx;
};

#define FLBGPU_E_JSONGROUP 8192u /* to-JSON: more group markers in one chunk than the list holds */
#define FLBGPU_E_JSONDATE 4096u /* to-JSON: a date that does not fit the reference's 38-byte buffer (it returns NULL for the chunk) */

/* ---------------------------------------------------- chunk -> JSON text (dev_tojson.cuh) */
struct tj_env {
    const uint8_t *in;
    const uint32_t *off, *len; const uint8_t *kind;
    uint32_t n_rec;
    uint8_t *scr;                     /* event i packs its map at scr + off[i] + i * scr_pad */
    uint32_t scr_pad;
    uint32_t *plen;                   /* bytes of that map */
    uint32_t *size;                   /* bytes of text per event (separator included) */
    uint32_t json_format, date_format, escape_unicode;
    uint32_t key_len;                 /* 0xffffffff: no date key */
    uint8_t key[128];
    uint32_t *err;
    unsigned long long *undefined;    /* strings whose text depends, in the reference, on memory behind the event's buffer */
    /* group markers (events with seconds -1 / -2, flb_log_event_decoder.c:393-447): the sizing pass lists them in marks[]
     * (two words each: record index * 2 + is_start, record length; any order, n_marks[0] of them); when there are any, the host sorts the list and the passes
     * run again with it as groups[0, n_groups): an event's group_attributes are the body of the last marker in front of it,
     * if that is a start */
    uint32_t *marks; unsigned long long *n_marks; uint32_t marks_cap;
    const uint32_t *groups; uint32_t n_groups;
};
#define TJ_FORMAT_JSON 1u
#define TJ_FORMAT_STREAM 2u
#define TJ_FORMAT_LINES 3u
#define TJ_DATE_DOUBLE 0u
#define TJ_DATE_ISO8601 1u
#define TJ_DATE_EPOCH 2u
#define TJ_DATE_JAVA_SQL 3u
#define TJ_DATE_EPOCH_MS 4u
#define TJ_SCR_PAD(key_len) ((key_len) + 128u)

/* ---------------------------------------------------- chunk -> GELF messages (dev_gelf.cuh) */
#define GF_KEY_MAX 128u               /* bytes of a field key or of the tag key */
#define GF_TAG_MAX 256u               /* bytes of the tag */
#define GF_NONE 0xffffffffu
/* the five field keys in the order flb_msgpack_to_gelf() tests them (src/flb_pack_gelf.c:522-606) */
#define GF_HOST 0
#define GF_SHORT 1
#define GF_TIMESTAMP 2
#define GF_LEVEL 3
#define GF_FULL 4
struct gf_env {
    const uint8_t *in;
    uint64_t in_len;                  /* the chunk's end: what the string writer may read up to without tag_key */
    const uint32_t *off, *len; const uint8_t *kind;
    uint32_t n_rec;
    uint8_t *scr;                     /* tag_key: event i re-packed with the tag at scr + off[i] + i * scr_pad */
    uint32_t scr_pad;
    uint32_t *plen;                   /* bytes of that map */
    uint32_t *size;                   /* bytes of text per event (separator included), 0: left out */
    uint32_t *err;
    unsigned long long *undefined;    /* events with a string whose text depends, in the reference, on memory behind its buffer */
    unsigned long long *failed;       /* events flb_msgpack_to_gelf() returns NULL for */
    uint32_t sep;                     /* the byte behind each message */
    uint32_t fkey_len[5];             /* GF_HOST ...: the names the record's keys are matched against */
    uint8_t fkey[5][GF_KEY_MAX];
    uint32_t tag_key_len;             /* GF_NONE: no tag_key */
    uint8_t tag_key[GF_KEY_MAX];
    uint32_t tag_len;
    uint8_t tag[GF_TAG_MAX];
};

/* ---------------------------------------------------- raw text -> log events (dev_lines.cuh) */
#define LN_TILE 256u
struct ln_env {
    const uint8_t *text; size_t bytes;
    uint32_t n_tiles, n_lines;
    uint32_t *cnt;                    /* line feeds per tile */
    uint32_t *nl;                     /* position of line feed k */
    uint32_t *size;                   /* bytes of the event of line k */
    unsigned long long *n_events;     /* lines that became events */
    int64_t sec, nsec;                /* the timestamp of the call (the reference stamps every line with "now") */
    uint32_t skip_empty_lines;
    uint64_t stream_offset;
    const uint8_t *strs;              /* key, path_key, path, offset_key, back to back */
    uint32_t key_off, key_len, path_key_off, path_key_len, path_off, path_len, offset_key_off, offset_key_len;   /* _len 0xffffffff: absent */
};
/* ... with a parser (in_tail's `Parser`): every kept line goes through the parser's chain as the event {"_": line}; the events are
 * then made from the chain's result and the parser's report */
#define TL_NONE 0xffffffffu
struct tl_env {
    struct ln_env ln;                 /* the text, its line feeds, the call's strings and time (ln.size: unused) */
    uint32_t *msize;                  /* bytes of line k's event in the parser's input (0: stepped over) */
    const uint64_t *mbsum;            /* ... their offsets per BK_REC_BLOCK lines */
    uint8_t *mid;                     /* the parser's input: one event per kept line, back to back */
    const uint32_t *r_off, *r_len;    /* the chain's record index over `mid` (kind 2: an event-shaped piece inside a line) */
    const uint8_t *r_kind;
    uint32_t n_rec;
    const uint32_t *r_size;           /* bytes of record r in the chain's result, */
    const uint64_t *r_bsum;           /* ... their offsets per BK_REC_BLOCK records */
    uint32_t *r_out;                  /* record r's offset in the result */
    const uint8_t *res;               /* the chain's result */
    const int32_t *prep;              /* the parser's report: 6 ints per record (parsed, position, seconds lo / hi, nanoseconds, -) */
    uint32_t *rec;                    /* the record of line k (TL_NONE: stepped over) */
    uint32_t *size;                   /* bytes of line k's event */
    uint32_t *bad;                    /* lines whose event is not where the chain's index has a record */
};

/* ---------------------------------------------------- streaming JSON packer (dev_jsmn.cuh) */
enum { JM_UNDEFINED = 0, JM_OBJECT = 1, JM_ARRAY = 2, JM_STRING = 4, JM_PRIMITIVE = 8 };     /* jsmntype_t, lib/jsmn/jsmn.h */
struct jm_tok { int32_t type, start, end, size, parent; };

#define JM_OK        0
#define JM_INVAL   (-501)     /* FLB_ERR_JSON_INVAL, include/fluent-bit/flb_error.h:46 */
#define JM_PART    (-502)     /* FLB_ERR_JSON_PART, :47 */
#define JM_NOMEM   (-2)       /* token array too small (internal: the host retries with a larger one) */
#define JM_FAIL    (-1)       /* tokens_to_msgpack() returned NULL */
#define JM_REFUSED (-3)       /* a number text the device strtod does not restate (hex float, nan(payload)): loud, never wrong */

struct jm_result {
    int32_t status;           /* what flb_pack_json_state() returns */
    int32_t last_byte;        /* state->last_byte */
    int32_t tokens_count;     /* state->tokens_count */
    int32_t records;          /* top-level values packed */
    uint32_t out_size;        /* msgpack bytes */
    uint32_t toknext;         /* tokens the tokeniser allocated */
    int32_t tret;             /* the tokeniser's own verdict */
    int32_t pad;
};

#ifdef __cplusplus
}
#endif
#endif
