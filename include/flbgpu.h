/* flbgpu.h -- C ABI of libflbgpu.so: Fluent Bit's parse->filter hot path on H100.
 *
 * Plain C, plain pointers and sizes.  Each entry point names the reference
 * interface it stands in for (paths relative to the fluent-bit source tree, v5.0.2).
 * INTEGRATION.md shows the few lines of glue a Fluent Bit maintainer adds on the
 * reference side (a `struct flb_filter_plugin` whose callbacks forward here).
 *
 * There is no CPU implementation behind this ABI: flbgpu_init() fails when no CUDA
 * device is usable and every other call then returns an error.
 */
#ifndef FLBGPU_H
#define FLBGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* include/fluent-bit/flb_filter.h:42-43 */
#define FLBGPU_FILTER_MODIFIED 1
#define FLBGPU_FILTER_NOTOUCH  2

/* include/fluent-bit/flb_parser.h:70-76 (enum FLB_PARSER_TYPE_*) */
#define FLBGPU_PARSER_TYPE_INT    1
#define FLBGPU_PARSER_TYPE_FLOAT  2
#define FLBGPU_PARSER_TYPE_BOOL   3
#define FLBGPU_PARSER_TYPE_STRING 4
#define FLBGPU_PARSER_TYPE_HEX    5

typedef struct flbgpu_ctx    flbgpu_ctx;     /* one device context (per GPU)            */
typedef struct flbgpu_parser flbgpu_parser;  /* struct flb_parser, flb_parser.h:41-68   */
typedef struct flbgpu_filter flbgpu_filter;  /* struct flb_filter_instance + plugin ctx */
typedef struct flbgpu_chain  flbgpu_chain;   /* config->filters as one fused program    */

/* struct flb_parser_types, include/fluent-bit/flb_parser.h:35-39 */
struct flbgpu_parser_types {
    char *key;
    int   key_len;
    int   type;
};

/* The field decoders of a parser definition (`Decode_Field json log`, `Decode_Field_As escaped_utf8 log do_next`, ...):
 * the properties as the [PARSER] section spells them, in order, ended by an entry whose property is NULL.  This is what
 * flb_parser_decoder_list_create() (src/flb_parser_decoder.c:594) reads from the section; flbgpu_parser_create() takes
 * the array where flb_parser_create() takes the struct mk_list that function built. */
struct flbgpu_parser_decoder {
    const char *property;      /* "decode_field" | "decode_field_as" (any case) */
    const char *value;         /* "<json|escaped|escaped_utf8|mysql_quoted> <field> [try_next|do_next]" */
};

/* struct flb_time { struct timespec tm; }, include/fluent-bit/flb_time.h */
struct flbgpu_time {
    int64_t tv_sec;
    int64_t tv_nsec;
};

/* ---- context ---------------------------------------------------------- */
/* Stands in for the process-wide state flb_config_init() sets up for this path
 * (config->parsers, config->filters).  device = CUDA ordinal.  NULL on failure;
 * flbgpu_last_error() says why (e.g. "no CUDA device available"). */
flbgpu_ctx *flbgpu_init(int device);
void        flbgpu_shutdown(flbgpu_ctx *ctx);
const char *flbgpu_last_error(void);
const char *flbgpu_backend_name(void);
int         flbgpu_device_count(void);

/* ---- parsers ---------------------------------------------------------- */
/* flb_parser_create(), src/flb_parser.c:148-348 -- same arguments, same meaning; `decoders` is NULL or an array of
 * struct flbgpu_parser_decoder (above).  The parser is registered under `name` in the context, like config->parsers.
 * NULL on error. */
flbgpu_parser *flbgpu_parser_create(flbgpu_ctx *ctx, const char *name, const char *format,
                                    const char *p_regex, int skip_empty,
                                    const char *time_fmt, const char *time_key,
                                    const char *time_offset, int time_keep, int time_strict,
                                    int time_system_timezone, int logfmt_no_bare_keys,
                                    struct flbgpu_parser_types *types, int types_len,
                                    void *decoders /* struct flbgpu_parser_decoder[] or NULL */);
/* flb_parser_get(), src/flb_parser.c:1022 */
flbgpu_parser *flbgpu_parser_get(flbgpu_ctx *ctx, const char *name);
/* flb_parser_do(), src/flb_parser.c:1044-1066: one line in, one msgpack map out.
 * Returns what the reference returns: -1 when no record comes out, else the position inside the line the parser
 * consumed it up to -- end of the last named capture for regex (src/flb_regex.c:50-54), end of the JSON document plus
 * the white space behind it (src/flb_pack.c:427-499), where the LTSV / logfmt scan stopped (line end consumed).
 * *out_buf is malloc()ed, caller frees; *out_time is the parsed time with 64-bit seconds (0/0 when the parser has no
 * time key or the record none).  The device reports position, "parsed" and time per line itself; nothing is inferred
 * from the output bytes. */
int flbgpu_parser_do(flbgpu_parser *parser, const char *buf, size_t length,
                     void **out_buf, size_t *out_size, struct flbgpu_time *out_time);

/* The batched form (SURVEY 8b): n lines in one device pass.  line i = base[off[i], off[i]+len[i]).
 * *out_buf (malloc) holds the msgpack maps of the parsed lines back to back, map i at
 * [out_off[i], out_off[i+1]) (out_off has n+1 entries; empty range when ret[i] < 0); out_time[i]
 * and ret[i] are what flbgpu_parser_do() returns per line (position or -1).  Returns 0, or -1 when the call failed. */
int flbgpu_parser_do_batch(flbgpu_parser *p, const char *base, const uint32_t *off, const uint32_t *len, uint32_t n,
                           void **out_buf, size_t *out_size, uint64_t *out_off, struct flbgpu_time *out_time, int *ret);
void flbgpu_parser_destroy(flbgpu_parser *parser);

/* ---- streaming JSON packer ------------------------------------------------------------------------------------
 * flb_pack_json_state(), src/flb_pack.c:758-829: what in_tcp / in_lib / in_stdin / in_mqtt call on the bytes a stream
 * has received so far -- the jsmn tokeniser (strict mode, parent links) and tokens_to_msgpack() (:512-592): every
 * whole top-level JSON value comes out as msgpack, state->last_byte says how much of the buffer that was, and an
 * unfinished tail is reported as FLB_ERR_JSON_PART when nothing before it is whole.  Same return values
 * (0, FLB_ERR_JSON_INVAL -501, FLB_ERR_JSON_PART -502, -1), same malloc()ed *buffer.
 * struct flbgpu_pack_state mirrors the fields of struct flb_pack_state (include/fluent-bit/flb_pack.h:64-74) a caller
 * reads; the tokeniser's own state is not kept between calls: a buffer that grew is tokenised again from its start,
 * which is what resuming amounts to (the callers reset the state after every successful pack).
 * The batch form packs n independent stream buffers (one connection each) in one device pass. */
struct flbgpu_pack_state {
    int multiple;
    int tokens_count;
    int last_byte;
};
int  flbgpu_pack_state_init(struct flbgpu_pack_state *s);
void flbgpu_pack_state_reset(struct flbgpu_pack_state *s);
int  flbgpu_pack_json_state(flbgpu_ctx *ctx, const char *js, size_t len, char **buffer, int *size, struct flbgpu_pack_state *state);
int  flbgpu_pack_json_state_batch(flbgpu_ctx *ctx, int n, const char *const *js, const size_t *len,
                                  char **buffers, int *sizes, struct flbgpu_pack_state *states, int *rets);

/* ---- output side: a chunk as JSON text -----------------------------------------------------------------------------
 * flb_pack_msgpack_to_json_format(), src/flb_pack.c:1320-1602 -- what out_stdout, out_http, out_file, out_kafka ... call on
 * the chunk they flush.  json_format: 1 FLB_PACK_JSON_FORMAT_JSON (one array), 2 _STREAM (maps back to back), 3 _LINES (one
 * map per line); date_format: 0 double, 1 iso8601, 2 epoch, 3 java_sql_timestamp, 4 epoch_ms (FLB_PACK_JSON_DATE_*,
 * include/fluent-bit/flb_pack.h:38-42); date_key NULL: no date member; escape_unicode: config->json_escape_unicode.
 * Returns 0 with *out = malloc()ed NUL-terminated text of *out_size bytes (the reference returns an flb_sds_t), 1 when the
 * reference returns NULL for this input (nothing to convert; a date that overflows its 38-byte buffer), -1 on failure.
 * *undefined_strings (may be NULL) counts strings whose text in the reference depends on memory behind the event: its string
 * writers test 16 bytes at a time and, out of step after a multi-byte character, read past the end of the last strings of an
 * event (src/flb_utils.c:920-935, 1255-1268); here such a window counts as "not plain". */
int flbgpu_msgpack_to_json_format(flbgpu_ctx *ctx, const void *data, size_t bytes, int json_format, int date_format,
                                  const char *date_key, int escape_unicode, char **out, size_t *out_size, size_t *undefined_strings);

/* ---- output side: a chunk as GELF messages -------------------------------------------------------------------------
 * flb_msgpack_to_gelf(), src/flb_pack_gelf.c, on every event the log event decoder yields, in order -- the flush loops of
 * out_gelf (plugins/out_gelf/gelf.c:265-392) and out_http `format gelf` (plugins/out_http/http.c:378-440).  Each message is
 * followed by one `separator` byte: '\n' for out_http, 0 for out_gelf over TCP / TLS (it writes the NUL behind each message).
 * struct flbgpu_gelf_fields mirrors struct flb_gelf_fields (include/fluent-bit/flb_pack.h:119); a NULL member, or a NULL
 * `fields`, is the default name.  tag_key (out_gelf's `tag_key`): the body is re-encoded with `tag_key: tag` behind its members
 * first, as inject_tag() does.  Keys are at most 128 bytes, the tag at most 256.
 * An event the reference returns NULL for (no short message, a level that is neither a non-negative integer nor a string, a
 * top-level float longer than 48 characters as "%f") is left out and counted in *failed: out_gelf skips it, out_http fails the
 * whole payload (its caller treats *failed > 0 as FLB_ERROR).  *undefined_strings as for flbgpu_msgpack_to_json_format().
 * Returns 0 with *out = malloc()ed NUL-terminated text of *out_size bytes, 1 when no event was converted, -1 on failure. */
struct flbgpu_gelf_fields {
    const char *timestamp_key;
    const char *host_key;
    const char *short_message_key;
    const char *full_message_key;
    const char *level_key;
};
int flbgpu_msgpack_to_gelf(flbgpu_ctx *ctx, const void *data, size_t bytes, const struct flbgpu_gelf_fields *fields,
                           const char *tag_key, const char *tag, size_t tag_len, int separator,
                           char **out, size_t *out_size, size_t *failed, size_t *undefined_strings);

/* ---- input side: raw text as log events -------------------------------------------------------------------------
 * The line loop of in_tail, plugins/in_tail/tail_file.c process_content() :629-700 and flb_tail_file_pack_line() :338-391, for
 * the plain case (no parser, no docker mode, none of the tail's own multiline modes): the text is cut at '\n'; with
 * skip_empty_lines an empty line and a lone "\r" are stepped over; a line of two bytes or more loses a trailing '\r'; every
 * line becomes one event `[[time, {}], {[path_key: path,] [offset_key: stream_offset + offset of the line,] key: line}]`.
 * The reference stamps each line with the current time; here the caller gives the time of the call.  *consumed = the bytes up
 * to and including the last '\n' (what in_tail's processed_bytes comes to: the rest of the buffer is an unfinished line and
 * stays with the caller), *lines = the lines that became events.  path_key / offset_key may be NULL.  Returns 0 with *out_buf a malloc()ed
 * chunk (NULL when no event came out), -1 on failure. */
int flbgpu_lines_to_events(flbgpu_ctx *ctx, const char *text, size_t bytes, const char *key, int skip_empty_lines,
                           int64_t sec, int64_t nsec, const char *path_key, const char *path, const char *offset_key,
                           uint64_t stream_offset, void **out_buf, size_t *out_size, size_t *consumed, size_t *lines);
/* The same loop with in_tail's `Parser` set (tail_file.c:721-746): arguments and results as flbgpu_lines_to_events(), the
 * context is the parser's.  For every line the loop keeps:
 *   1. the parser gets the line without its trailing '\r' (as the plain event carries it);
 *   2. when it parses (flb_parser_do() >= 0), the event is flb_tail_pack_line_map()'s (:281-336):
 *      `[[time, {}], {<the parsed map's members, each re-encoded as msgpack_pack_object() writes it>, [path_key: path,]
 *      [offset_key: stream_offset + offset of the line]}]` -- path and offset come AFTER the parsed members, and a parsed key
 *      equal to path_key appears twice.  The time is the parsed one; when flb_time_to_nanosec() of it is 0 (no time key, or
 *      exactly the epoch) it is the call's sec / nsec.  Seconds and nanoseconds go out as (uint32_t), like the encoder's;
 *   3. when it does not parse, the event is the plain one with the call's time, but of the line as read: a trailing '\r' stays;
 *   4. the parser is flb_parser_do() whole: every format, Types, Time_Keep, Time_Offset, the decoders, Skip_Empty_Values;
 *   5. a line the device refuses to parse (FLBGPU_E_RXSTACK, RXBUDGET, RXUNICODE, FIELDS, FLOAT, DEEP, ...) fails the call:
 *      -1, flbgpu_last_error() names the bits.  Such a line never becomes a rule-3 event, since the reference would parse it.
 * Calls with the same parser take turns (its flbgpu_parser_do() chain does the work); different parsers run side by side. */
int flbgpu_lines_to_events_parsed(flbgpu_parser *parser, const char *text, size_t bytes, const char *key, int skip_empty_lines,
                                  int64_t sec, int64_t nsec, const char *path_key, const char *path, const char *offset_key,
                                  uint64_t stream_offset, void **out_buf, size_t *out_size, size_t *consumed, size_t *lines);

/* ---- multiline parser definitions ----------------------------------------------------------------------------
 * What a [MULTILINE_PARSER] section becomes (src/flb_parser.c:815-935): flb_ml_parser_create()
 * (src/multiline/flb_ml_parser.c:199-230; type = "regex" | "endswith" | "equal" | "eq", flb_ml_type_lookup()),
 * one flb_ml_rule_create() per `rule "from_state[, from_state]" "/regex/" "to_state"` (src/multiline/flb_ml_rule.c:48-112;
 * the first rule must name start_state) and flb_ml_parser_init() (every to_state must be some rule's from_state).
 * The built-in rule-based parsers java, go, python and ruby exist without being created.  Not built on the device:
 * key_group, a sub-parser (`parser`), and therefore the built-in docker and cri parsers. */
typedef struct flbgpu_ml_parser flbgpu_ml_parser;
flbgpu_ml_parser *flbgpu_ml_parser_create(flbgpu_ctx *ctx, const char *name, const char *type, const char *match_string, int negate,
                                          int flush_ms, const char *key_content, const char *key_group, const char *key_pattern,
                                          const char *parser_name);
int flbgpu_ml_parser_rule(flbgpu_ml_parser *mlp, const char *from_states, const char *regex, const char *to_state);
int flbgpu_ml_parser_init(flbgpu_ml_parser *mlp);
/* config->multiline_buffer_limit (FLB_ML_BUFFER_LIMIT_DEFAULT: 2 MiB), in bytes; read when a multiline filter is initialised.
 * A message that reaches it fails the call (FLBGPU_E_MLLIMIT): the reference truncates it and marks the record. */
int flbgpu_ml_set_buffer_limit(flbgpu_ctx *ctx, size_t bytes);

/* ---- filters ---------------------------------------------------------- */
/* flb_filter_new(), src/flb_filter.c:426: plugin = "parser" | "grep" | "modify" |
 * "record_modifier" | "log_to_metrics" | "rewrite_tag" | "multiline" (the names of the reference's filter_*_plugin structs).
 * "multiline" is plugins/filter_multiline/ml.c in parser mode with `buffer off` (the chunk's lines are concatenated inside
 * the call, cb_ml_filter :833-892); `multiline.parser` names ONE multiline parser, `multiline.key_content` the key. */
flbgpu_filter *flbgpu_filter_new(flbgpu_ctx *ctx, const char *plugin);
/* flb_filter_set_property(), src/flb_filter.c:325: properties keep config order,
 * keys are case-insensitive; "match"/"alias"/"log_level" are accepted and ignored. */
int flbgpu_filter_set_property(flbgpu_filter *f, const char *k, const char *v);
/* the plugin's cb_init (e.g. plugins/filter_grep/grep.c:196): 0 or -1 */
int flbgpu_filter_init(flbgpu_filter *f);
/* the plugin's cb_filter, include/fluent-bit/flb_filter.h:66-73: `data` is a chunk of
 * msgpack log events in HOST memory, not owned; on FLBGPU_FILTER_MODIFIED *out_buf is a
 * malloc()ed chunk owned by the caller (*out_size may be 0: everything dropped). */
int flbgpu_filter_cb(flbgpu_filter *f, const void *data, size_t bytes,
                     const char *tag, int tag_len, void **out_buf, size_t *out_size);
/* the plugin's cb_exit */
void flbgpu_filter_destroy(flbgpu_filter *f);

/* ---- filter "rewrite_tag" (plugins/filter_rewrite_tag/rewrite_tag.c) ---- */
/* Properties: Rule <key> <regex> <new tag> <keep> (several), Emitter_Name, Emitter_Storage.type, Emitter_Mem_Buf_Limit (the
 * emitter itself is the caller's: an input instance of the host pipeline).  The device matches the rules, expands the tag
 * templates ($TAG, $TAG[n], $0..$9, $key['sub'], src/flb_record_accessor.c:483-690) and cuts the matched records out of the
 * chunk; what the reference hands to in_emitter_add_record() one record at a time (rewrite_tag.c:404-413) is returned here
 * grouped by new tag, tags in order of first appearance, records of a tag in chunk order -- the state those calls leave in
 * the emitter (plugins/in_emitter/emitter.c:124: one chunk per tag).  The caller passes each group to its emitter once.
 * The groups belong to the filter and stay valid until its next call (alone or inside a chain) or its destruction.
 * The filter's return value follows the reference: MODIFIED iff at least one record was re-tagged (and the chunk decodes
 * to its end), the result holding the records whose rule says keep plus the ones no rule matched. */
struct flbgpu_emit_group {
    const char *tag;        /* not NUL-terminated */
    size_t tag_len;
    const void *data;       /* the records as the filter saw them, one behind the other */
    size_t size;
    size_t records;
};
int flbgpu_filter_emitted(flbgpu_filter *f, const struct flbgpu_emit_group **groups, size_t *n_groups);

/* ---- fused chain ------------------------------------------------------ */
/* flb_filter_do(), src/flb_filter.c:119-323, over filters that all live on the GPU:
 * one host->device copy, one evaluation pass, one emission pass, one copy back.
 * Filters are applied in the order they were added (config order). */
flbgpu_chain *flbgpu_chain_new(flbgpu_ctx *ctx);
int  flbgpu_chain_add(flbgpu_chain *c, flbgpu_filter *f);     /* f must be initialised */
int  flbgpu_chain_init(flbgpu_chain *c);
/* Same contract as flbgpu_filter_cb.  Returns MODIFIED / NOTOUCH, or -1 on error. */
int  flbgpu_chain_do(flbgpu_chain *c, const void *data, size_t bytes,
                     const char *tag, int tag_len, void **out_buf, size_t *out_size);
void flbgpu_chain_destroy(flbgpu_chain *c);

/* Device-resident variant used for kernel-level measurement: the chunk is already in
 * HBM (d_data) and the result stays in HBM (d_out, capacity out_cap).  *out_size gets
 * the result size; returns MODIFIED / NOTOUCH / -1. */
int flbgpu_chain_do_device(flbgpu_chain *c, const void *d_data, size_t bytes,
                           void *d_out, size_t out_cap, size_t *out_size);

/* per-call statistics of the last flbgpu_chain_do*() on this chain */
struct flbgpu_stats {
    uint64_t records_in;        /* entries of the record index: the decodable records, plus the rare byte runs
                                   inside a record that frame as an event and are kept as "false candidate" */
    uint64_t records_out;       /* records in the result                      */
    uint64_t bytes_in, bytes_out;
    uint64_t kernel_launches;   /* kernels launched by this library so far   */
    uint32_t passes;            /* evaluation passes (1 unless a chunk-level assumption was revised) */
    uint32_t error_bits;        /* FLBGPU_E_* (flbgpu_prog.h) when the call failed */
    /* host wall-clock milliseconds of the call's phases (diagnostic): [0] upload + index + evaluation
     * (until the chunk-level verdicts are settled), [1] size scan, [2] emission + download, [3] total */
    float phase_ms[4];
};
/* ---- several devices in one process ----------------------------------------------------------------------------
 * The path shards by chunk with nothing to agree on (the filters' MODIFIED / NOTOUCH verdicts are per chunk).  A pool is n
 * chains of the same configuration -- one per context / device -- with a worker thread each; flbgpu_pool_do() hands the chunks
 * of a batch to whichever chain is free and returns every chunk's result in its slot: rets[i] as flbgpu_chain_do() returns it,
 * out_bufs[i] malloc()ed on FLBGPU_FILTER_MODIFIED.  The chains stay the caller's (destroy the pool first).  Filters with state
 * across chunks (multiline) keep it per chain; log_to_metrics tables stay per chain until flbgpu_l2m_allreduce(). */
typedef struct flbgpu_pool flbgpu_pool;
flbgpu_pool *flbgpu_pool_new(flbgpu_chain *const *chains, int n);
int flbgpu_pool_do(flbgpu_pool *p, int n_chunks, const void *const *data, const size_t *bytes, const char *tag, int tag_len,
                   void **out_bufs, size_t *out_sizes, int *rets);
void flbgpu_pool_destroy(flbgpu_pool *p);

/* Not part of the reference's contract (a filter returns a buffer the engine frees): an embedding that keeps its own result
 * memory -- reused from call to call, or pinned with flbgpu_host_alloc() -- registers it here.  A result that fits is written
 * there and *out_buf of flbgpu_chain_do() IS that buffer (do not free it); a larger one comes back malloc()ed as before.  With
 * glibc's default malloc a fresh result buffer is fresh pages from the kernel on every call: on the bench's whole-set calls their
 * page faults cost more than the device work (DESIGN.md section 6).  buf NULL: back to malloc() only. */
int flbgpu_chain_set_result_buffer(flbgpu_chain *c, void *buf, size_t cap);
void flbgpu_chain_stats(flbgpu_chain *c, struct flbgpu_stats *out);
/* Every chain (and every filter instance behind flbgpu_filter_cb) owns its device queue -- streams, pinned staging
 * rings, worker threads -- so instances may be called from different threads at the same time, as
 * flb_processor_run() does (src/flb_processor.c:1352-1378); calls on ONE instance are serialised.
 * This is the cudaStream_t the instance launches its kernels on. */
void *flbgpu_chain_stream(flbgpu_chain *c);

/* ---- filter_log_to_metrics state ------------------------------------------------
 * The filter ("log_to_metrics": metric_mode counter | gauge | histogram, Regex/Exclude gates, label_field /
 * add_label, kubernetes_mode, bucket, discard_logs) accumulates into a per-instance table, like ctx->cmt in
 * plugins/filter_log_to_metrics/log_to_metrics.c:964-1148 (cmt_counter_inc / cmt_gauge_set / cmt_histogram_observe).
 * Label sets keep first-seen order.  A multi-GPU deployment merges these tables with flbgpu_l2m_allreduce() below. */
int   flbgpu_l2m_info(flbgpu_filter *f, int *mode, int *n_labels, int *n_buckets, int *n_sets);
/* label set i: 64-bit key, counter value (or histogram count), histogram sum (gauge: the value), cumulative buckets
 * [n_buckets + 1] (last = +Inf), labels = n_labels x 256 bytes (length byte + bytes) */
int   flbgpu_l2m_get(flbgpu_filter *f, int i, uint64_t *hash, uint64_t *count, double *sum, uint64_t *buckets, char *labels);
int   flbgpu_l2m_reset(flbgpu_filter *f);
int   flbgpu_l2m_put(flbgpu_filter *f, uint64_t hash, uint64_t count, double sum, const uint64_t *buckets, const char *labels);
char *flbgpu_l2m_text(flbgpu_filter *f);       /* malloc()ed text dump, free() it */

/* The one exchange step of the path (SURVEY 8e): with one process per GPU, every rank's filter instance holds the table of
 * its record range; flbgpu_l2m_allreduce() leaves on every rank the table cmetrics would hold for the whole input --
 * label sets in first-seen (rank-major) order, counts and buckets summed, gauges from the highest rank that saw the set
 * (lib/cmetrics/src/cmt_cat.c:1032 is the reference's own merge of two contexts).  NCCL over NVLink: an all-gather of the
 * set counts, an all-gather of the label keys, one all-reduce of the value matrix.  The communicator belongs to the context:
 * rank 0 makes the id (ncclGetUniqueId), the embedding process carries the 128 bytes to the other ranks (the engine's
 * own control channel; bench.py uses torch.distributed), every rank calls flbgpu_comm_init.  libnccl is opened at run time. */
int flbgpu_comm_unique_id(uint8_t id[128]);
int flbgpu_comm_init(flbgpu_ctx *ctx, int nranks, int rank, const uint8_t id[128]);
int flbgpu_l2m_allreduce(flbgpu_filter *f);

/* CUDA-event milliseconds of the three kernel groups of the most recent chain call on this
 * context: out[0] record index, out[1] evaluation pass (the regex/interpreter kernel),
 * out[2] emission pass.  Synchronises the library stream. */
int flbgpu_kernel_ms(flbgpu_ctx *ctx, float out[3]);

/* device memory helpers for callers that keep chunks resident (bench, tests) */
void *flbgpu_dev_alloc(flbgpu_ctx *ctx, size_t n);
void  flbgpu_dev_free(flbgpu_ctx *ctx, void *p);
int   flbgpu_dev_upload(flbgpu_ctx *ctx, void *d, const void *h, size_t n);
int   flbgpu_dev_download(flbgpu_ctx *ctx, void *h, const void *d, size_t n);
void *flbgpu_host_alloc(flbgpu_ctx *ctx, size_t n);       /* pinned */
void  flbgpu_host_free(flbgpu_ctx *ctx, void *p);
void *flbgpu_stream(flbgpu_ctx *ctx);                     /* cudaStream_t the library launches on */

#ifdef __cplusplus
}
#endif
#endif
