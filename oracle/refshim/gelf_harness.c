/* oracle/_ref/libflbref_gelf.so: the GELF flush loops around the UNMODIFIED reference converter --
 *   flb_msgpack_to_gelf / flb_msgpack_raw_to_gelf          (src/flb_pack_gelf.c, compiled as it lies by gelf.mk)
 * The loops themselves are restated: out_gelf's cb_gelf_flush() with inject_tag() (plugins/out_gelf/gelf.c:233-392), which
 * out_http's compose_payload_gelf() (plugins/out_http/http.c:378-440) matches byte for byte while no event fails.  Built beside
 * libflbref.so and linked against it (gelf.mk).
 * TEST INFRASTRUCTURE ONLY: nothing under fluent-bit_b200/ may link or call this. */
#include <stdlib.h>
#include <string.h>
#include <fluent-bit/flb_info.h>
#include <fluent-bit/flb_mem.h>
#include <fluent-bit/flb_sds.h>
#include <fluent-bit/flb_pack.h>
#include <fluent-bit/flb_time.h>
#include <fluent-bit/flb_log_event_decoder.h>
#include <msgpack.h>

/* inject_tag() (gelf.c:233-262) with the tag given */
static void inject_tag(msgpack_object *map, const char *tag_key, const char *tag, size_t tag_len, msgpack_sbuffer *sbuf)
{
    msgpack_packer pck;
    uint32_t i;
    msgpack_sbuffer_init(sbuf);
    msgpack_packer_init(&pck, sbuf, msgpack_sbuffer_write);
    msgpack_pack_map(&pck, 1 + map->via.map.size);
    for (i = 0; i < map->via.map.size; i++) {
        msgpack_pack_object(&pck, map->via.map.ptr[i].key);
        msgpack_pack_object(&pck, map->via.map.ptr[i].val);
    }
    msgpack_pack_str(&pck, strlen(tag_key));
    msgpack_pack_str_body(&pck, tag_key, strlen(tag_key));
    msgpack_pack_str(&pck, tag_len);
    msgpack_pack_str_body(&pck, tag, tag_len);
}

static flb_sds_t field(const char *name) { return name ? flb_sds_create(name) : NULL; }

/* Every event of the chunk through the converter, each message followed by `separator` (out_gelf over TCP / TLS writes the
 * sds with its NUL, out_http appends '\n'); an event the converter returns NULL for is left out and counted in *failed.
 * Returns a malloc()ed copy of the text (flbref_cfree), NULL when no event was converted. */
char *flbref_msgpack_to_gelf(const void *data, size_t bytes, const char *timestamp_key, const char *host_key,
                             const char *short_message_key, const char *full_message_key, const char *level_key,
                             const char *tag_key, const char *tag, size_t tag_len, int separator, size_t *out_len, size_t *failed)
{
    struct flb_gelf_fields fields;
    struct flb_log_event_decoder dec;
    struct flb_log_event ev;
    flb_sds_t all = flb_sds_create_size(bytes + 64), s, tmp;
    char sep = (char) separator, *out = NULL;
    size_t prev_off = 0, off, size;

    *out_len = 0; *failed = 0;
    fields.timestamp_key = field(timestamp_key); fields.host_key = field(host_key);
    fields.short_message_key = field(short_message_key); fields.full_message_key = field(full_message_key);
    fields.level_key = field(level_key);
    if (flb_log_event_decoder_init(&dec, (char *) data, bytes) == FLB_EVENT_DECODER_SUCCESS) {
        while (flb_log_event_decoder_next(&dec, &ev) == FLB_EVENT_DECODER_SUCCESS) {
            msgpack_object map = *ev.body;
            off = dec.offset;
            size = off - prev_off;
            prev_off = off;
            s = NULL;
            if (tag_key) {
                msgpack_sbuffer sbuf;
                inject_tag(&map, tag_key, tag, tag_len, &sbuf);
                tmp = flb_msgpack_raw_to_gelf(sbuf.data, sbuf.size, &ev.timestamp, &fields);
                msgpack_sbuffer_destroy(&sbuf);
            }
            else {
                s = flb_sds_create_size((size_t) (size * 1.4));
                tmp = flb_msgpack_to_gelf(&s, &map, &ev.timestamp, &fields);
            }
            if (tmp) {
                s = tmp;
                all = flb_sds_cat(all, s, flb_sds_len(s));
                all = flb_sds_cat(all, &sep, 1);
            }
            else (*failed)++;
            flb_sds_destroy(s);
        }
        flb_log_event_decoder_destroy(&dec);
    }
    if (flb_sds_len(all)) {
        *out_len = flb_sds_len(all);
        out = malloc(*out_len + 1);
        memcpy(out, all, *out_len + 1);
    }
    flb_sds_destroy(all);
    flb_sds_destroy(fields.timestamp_key); flb_sds_destroy(fields.host_key); flb_sds_destroy(fields.short_message_key);
    flb_sds_destroy(fields.full_message_key); flb_sds_destroy(fields.level_key);
    return out;
}
