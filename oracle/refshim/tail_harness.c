/* oracle/_ref/libflbref_tail.so: in_tail's `Parser` branch around the UNMODIFIED reference functions it calls --
 *   flb_parser_do                                      (src/flb_parser.c:1044)
 *   the log event encoder calls of flb_tail_pack_line_map() / flb_tail_repack_map() / flb_tail_file_pack_line()
 *                                                      (plugins/in_tail/tail_file.c:228-391)
 * The line loop itself (process_content(), :629-785) is a static function over struct flb_tail_file and is restated.  Built
 * beside libflbref.so and linked against it (tail.mk), so parsers made by flbref_parser_create() are used as they are.
 * TEST INFRASTRUCTURE ONLY: nothing under fluent-bit_b200/ may link or call this. */
#include <stdlib.h>
#include <string.h>
#include <fluent-bit/flb_info.h>
#include <fluent-bit/flb_mem.h>
#include <fluent-bit/flb_parser.h>
#include <fluent-bit/flb_time.h>
#include <fluent-bit/flb_log_event_encoder.h>
#include <fluent-bit/flb_log_event_decoder.h>
#include <msgpack.h>

/* ---- the same loop with in_tail's `Parser` set (plugins/in_tail/tail_file.c:721-746): the reference's flb_parser_do() on the
 * line without its '\r'; a parsed line through the encoder calls of flb_tail_pack_line_map() / flb_tail_repack_map()
 * (:228-336), a line that does not parse through those of flb_tail_file_pack_line() with the whole line, '\r' included.  Where
 * the reference takes the current time (a parsed time of 0 ns, and every unparsed line), the call's sec / nsec stand in. ---- */
char *flbref_lines_to_events_parsed(void *parser, const char *text, size_t bytes, const char *key, int skip_empty_lines, long long sec,
                                    long long nsec, const char *path_key, const char *path, const char *offset_key,
                                    unsigned long long stream_offset, size_t *out_len, size_t *consumed, size_t *lines)
{
    struct flb_log_event_encoder *enc = flb_log_event_encoder_create(FLB_LOG_EVENT_FORMAT_DEFAULT);
    const char *data = text, *end = text + bytes, *p;
    size_t processed_bytes = 0, n_lines = 0;
    struct flb_time tm, out_time;
    char *out;

    tm.tm.tv_sec = (time_t) sec; tm.tm.tv_nsec = (long) nsec;
    while (data < end && (p = memchr(data, '\n', end - data))) {
        size_t len = (size_t) (p - data), i;
        int crlf = 0, result, ret;
        void *out_buf = NULL;
        size_t out_size = 0;
        if (skip_empty_lines) {
            if (len == 0) { data++; processed_bytes++; continue; }
            else if (len == 1 && data[0] == '\r') { data += 2; processed_bytes += 2; continue; }
        }
        if (len >= 2) crlf = (data[len - 1] == '\r');
        flb_time_zero(&out_time);
        ret = flb_parser_do(parser, data, len - crlf, &out_buf, &out_size, &out_time);
        result = flb_log_event_encoder_begin_record(enc);
        if (ret >= 0) {
            if (flb_time_to_nanosec(&out_time) == 0L) out_time = tm;
            if (result == FLB_EVENT_ENCODER_SUCCESS) result = flb_log_event_encoder_set_timestamp(enc, &out_time);
            if (result == FLB_EVENT_ENCODER_SUCCESS && out_size > 0) {
                msgpack_unpacked map;
                size_t off = 0;
                msgpack_unpacked_init(&map);
                result = msgpack_unpack_next(&map, out_buf, out_size, &off) == MSGPACK_UNPACK_SUCCESS ?
                         FLB_EVENT_ENCODER_SUCCESS : FLB_EVENT_DECODER_ERROR_DESERIALIZATION_FAILURE;
                for (i = 0; i < map.data.via.map.size && result == FLB_EVENT_ENCODER_SUCCESS; i++) {
                    result = flb_log_event_encoder_append_body_msgpack_object(enc, &map.data.via.map.ptr[i].key);
                    if (result == FLB_EVENT_ENCODER_SUCCESS)
                        result = flb_log_event_encoder_append_body_msgpack_object(enc, &map.data.via.map.ptr[i].val);
                }
                msgpack_unpacked_destroy(&map);
            }
        }
        else if (result == FLB_EVENT_ENCODER_SUCCESS) result = flb_log_event_encoder_set_timestamp(enc, &tm);
        if (ret < 0 && path_key && result == FLB_EVENT_ENCODER_SUCCESS)        /* (the plain event: path and offset first) */
            result = flb_log_event_encoder_append_body_values(enc, FLB_LOG_EVENT_CSTRING_VALUE(path_key),
                                                              FLB_LOG_EVENT_STRING_VALUE(path, strlen(path)));
        if (ret < 0 && offset_key && result == FLB_EVENT_ENCODER_SUCCESS)
            result = flb_log_event_encoder_append_body_values(enc, FLB_LOG_EVENT_CSTRING_VALUE(offset_key),
                                                              FLB_LOG_EVENT_UINT64_VALUE(stream_offset + processed_bytes));
        if (ret < 0 && result == FLB_EVENT_ENCODER_SUCCESS)
            result = flb_log_event_encoder_append_body_values(enc, FLB_LOG_EVENT_CSTRING_VALUE(key), FLB_LOG_EVENT_STRING_VALUE(data, len));
        if (ret >= 0 && path_key && result == FLB_EVENT_ENCODER_SUCCESS)      /* (the parsed event: path and offset last) */
            result = flb_log_event_encoder_append_body_values(enc, FLB_LOG_EVENT_CSTRING_VALUE(path_key),
                                                              FLB_LOG_EVENT_STRING_VALUE(path, strlen(path)));
        if (ret >= 0 && offset_key && result == FLB_EVENT_ENCODER_SUCCESS)
            result = flb_log_event_encoder_append_body_values(enc, FLB_LOG_EVENT_CSTRING_VALUE(offset_key),
                                                              FLB_LOG_EVENT_UINT64_VALUE(stream_offset + processed_bytes));
        if (result == FLB_EVENT_ENCODER_SUCCESS) result = flb_log_event_encoder_commit_record(enc);
        else flb_log_event_encoder_rollback_record(enc);
        flb_free(out_buf);
        n_lines++;
        data += len + 1;
        processed_bytes += len + 1;
    }
    *out_len = enc->output_length;
    out = malloc(enc->output_length + 1);
    memcpy(out, enc->output_buffer, enc->output_length);
    *consumed = processed_bytes; *lines = n_lines;
    flb_log_event_encoder_destroy(enc);
    return out;
}

