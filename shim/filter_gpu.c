/* shim/filter_gpu.c -- the reference-side binding of libflbgpu.so: seven Fluent Bit filter plugins
 *
 *     filter_gpu_parser_plugin   filter_gpu_grep_plugin   filter_gpu_modify_plugin
 *     filter_gpu_record_modifier_plugin   filter_gpu_log_to_metrics_plugin
 *     filter_gpu_rewrite_tag_plugin   filter_gpu_multiline_plugin
 *
 * written against Fluent Bit's own headers (struct flb_filter_plugin,
 * include/fluent-bit/flb_filter.h:57-81) and registered exactly like a dynamic plugin: the engine
 * looks up `filter_<name>_plugin` and memcpy's the struct (src/flb_plugin.c:200-324).  Each plugin
 * keeps the stock plugin's config map, so an existing configuration works by renaming the filter
 * (`Name grep` -> `Name gpu_grep`), and forwards its callbacks to the C ABI of include/flbgpu.h:
 *
 *     cb_init    -> flbgpu_filter_new + flbgpu_filter_set_property (config order) + flbgpu_filter_init
 *                   (gpu_parser also mirrors every parser of config->parsers it names: flbgpu_parser_create)
 *     cb_filter  -> flbgpu_filter_cb      (host chunk in, FLB_FILTER_MODIFIED + heap chunk out, or NOTOUCH)
 *     cb_exit    -> flbgpu_filter_destroy
 *
 * libflbgpu.so is opened at run time (FLBGPU_SHIM_LIB, default "libflbgpu.so"): a box without a GPU fails in
 * cb_init with the library's own message -- there is no CPU fallback here either.  flb_filter_do()
 * (src/flb_filter.c:119-323) drives these plugins like any other, so Match / Match_Regex routing and the
 * per-filter framework counters (filter_records_total, filter_bytes_total, filter_drop_records_total, ...) are the
 * engine's own.
 *
 * Built by oracle/refshim/Makefile (target shim) into oracle/_ref/flb-filter_gpu.so and exercised by
 * tests/test_shim.py through the reference's own flb_filter_do().
 */
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <fluent-bit/flb_info.h>
#include <fluent-bit/flb_filter.h>
#include <fluent-bit/flb_filter_plugin.h>
#include <fluent-bit/flb_config.h>
#include <fluent-bit/flb_kv.h>
#include <fluent-bit/flb_mem.h>
#include <fluent-bit/flb_parser.h>
#include <fluent-bit/flb_parser_decoder.h>
#include <fluent-bit/flb_utils.h>
#include <fluent-bit/flb_input.h>
#include <fluent-bit/flb_storage.h>
#include <fluent-bit/flb_metrics.h>
#include <cmetrics/cmetrics.h>
#include <cmetrics/cmt_counter.h>
#include <cfl/cfl_time.h>
#include "../include/flbgpu.h"

/* ---- the C ABI, resolved from the library at run time ---- */
static struct gpu_api {
    void *dso;
    flbgpu_ctx *(*init)(int);
    const char *(*last_error)(void);
    flbgpu_parser *(*parser_create)(flbgpu_ctx *, const char *, const char *, const char *, int, const char *, const char *,
                                    const char *, int, int, int, int, struct flbgpu_parser_types *, int, void *);
    flbgpu_parser *(*parser_get)(flbgpu_ctx *, const char *);
    flbgpu_filter *(*filter_new)(flbgpu_ctx *, const char *);
    int (*filter_set_property)(flbgpu_filter *, const char *, const char *);
    int (*filter_init)(flbgpu_filter *);
    int (*filter_cb)(flbgpu_filter *, const void *, size_t, const char *, int, void **, size_t *);
    void (*filter_destroy)(flbgpu_filter *);
    char *(*l2m_text)(flbgpu_filter *);
    int (*filter_emitted)(flbgpu_filter *, const struct flbgpu_emit_group **, size_t *);
} G;
static flbgpu_ctx *g_ctx;                         /* one context per process and device */
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;
static char g_why[256];

static int api_load(void)
{
    const char *path = getenv("FLBGPU_SHIM_LIB");
    if (G.dso) return 0;
    G.dso = dlopen(path && *path ? path : "libflbgpu.so", RTLD_NOW | RTLD_LOCAL);
    if (!G.dso) { snprintf(g_why, sizeof(g_why), "cannot open libflbgpu: %s", dlerror()); return -1; }
#define SYM(field, name) do { *(void **) &G.field = dlsym(G.dso, name); \
        if (!G.field) { snprintf(g_why, sizeof(g_why), "libflbgpu lacks %s", name); dlclose(G.dso); G.dso = NULL; return -1; } } while (0)
    SYM(init, "flbgpu_init"); SYM(last_error, "flbgpu_last_error"); SYM(parser_create, "flbgpu_parser_create");
    SYM(parser_get, "flbgpu_parser_get"); SYM(filter_new, "flbgpu_filter_new");
    SYM(filter_set_property, "flbgpu_filter_set_property"); SYM(filter_init, "flbgpu_filter_init");
    SYM(filter_cb, "flbgpu_filter_cb"); SYM(filter_destroy, "flbgpu_filter_destroy"); SYM(l2m_text, "flbgpu_l2m_text");
    SYM(filter_emitted, "flbgpu_filter_emitted");
#undef SYM
    return 0;
}

/* errors go to the instance's log (flb_plg_error); FLBGPU_SHIM_DEBUG=1 also copies them to stderr */
#define SHIM_ERROR(ins, ...) do { flb_plg_error(ins, __VA_ARGS__); \
        if (getenv("FLBGPU_SHIM_DEBUG")) { fprintf(stderr, "[flb-filter_gpu] " __VA_ARGS__); fputc('\n', stderr); } } while (0)

static flbgpu_ctx *gpu_context(struct flb_filter_instance *ins)
{
    pthread_mutex_lock(&g_lock);
    if (!g_ctx) {
        const char *dev = getenv("FLBGPU_DEVICE");
        if (api_load() != 0) SHIM_ERROR(ins, "%s", g_why);
        else if (!(g_ctx = G.init(dev ? atoi(dev) : 0))) SHIM_ERROR(ins, "%s", G.last_error());   /* no GPU: fail, never fall back */
    }
    pthread_mutex_unlock(&g_lock);
    return g_ctx;
}

/* struct flb_parser (include/fluent-bit/flb_parser.h:41-68) -> flbgpu_parser_create(): same definition */
static int mirror_parser(struct flb_filter_instance *ins, struct flb_config *config, const char *name)
{
    struct flb_parser *p;
    const char *format;
    char off[16], *offp = NULL;
    if (G.parser_get(g_ctx, name)) return 0;
    p = flb_parser_get(name, config);
    if (!p) return 0;                              /* unknown name: flbgpu_filter_init refuses it like filter_parser.c:135 */
    switch (p->type) {
    case FLB_PARSER_REGEX: format = "regex"; break;
    case FLB_PARSER_JSON: format = "json"; break;
    case FLB_PARSER_LTSV: format = "ltsv"; break;
    case FLB_PARSER_LOGFMT: format = "logfmt"; break;
    default: SHIM_ERROR(ins, "parser '%s': type %d has no GPU form", name, p->type); return -1;
    }
    if (p->time_offset) {                          /* the struct keeps seconds; flb_parser_create() takes "+hhmm" */
        int v = p->time_offset < 0 ? -p->time_offset : p->time_offset;
        snprintf(off, sizeof(off), "%c%02d%02d", p->time_offset < 0 ? '-' : '+', v / 3600, (v % 3600) / 60);
        offp = off;
    }
    {
        /* the decoders as flb_parser_decoder_list_create() built them (one struct flb_parser_dec per key, its rules in order),
         * spelled back as the [PARSER] properties they came from */
        static const char *backend[] = { "json", "escaped", "escaped_utf8", "mysql_quoted" };
        static const char *action[] = { "", " try_next", " do_next" };
        struct flbgpu_parser_decoder dec[65];
        char text[64][320];
        struct mk_list *head, *r_head;
        int n = 0, ok;
        if (p->decoders) {
            mk_list_foreach(head, p->decoders) {
                struct flb_parser_dec *d = mk_list_entry(head, struct flb_parser_dec, _head);
                mk_list_foreach(r_head, &d->rules) {
                    struct flb_parser_dec_rule *r = mk_list_entry(r_head, struct flb_parser_dec_rule, _head);
                    if (n >= 64 || r->backend < 0 || r->backend > 3 || r->action < 0 || r->action > 2) {
                        SHIM_ERROR(ins, "parser '%s': decoder rule outside what the GPU path takes", name);
                        return -1;
                    }
                    snprintf(text[n], sizeof(text[n]), "%s %s%s", backend[r->backend], d->key, action[r->action]);
                    dec[n].property = r->type == FLB_PARSER_DEC_AS ? "decode_field_as" : "decode_field";
                    dec[n].value = text[n];
                    n++;
                }
            }
        }
        dec[n].property = NULL; dec[n].value = NULL;
        ok = G.parser_create(g_ctx, p->name, format, p->p_regex, p->skip_empty, p->time_fmt_full, p->time_key, offp,
                             p->time_keep, p->time_strict, p->time_system_timezone, p->logfmt_no_bare_keys,
                             (struct flbgpu_parser_types *) p->types, p->types_len, n ? dec : NULL) != NULL;
        if (!ok) {
            SHIM_ERROR(ins, "parser '%s': %s", name, G.last_error());
            return -1;
        }
    }
    return 0;
}

static int gpu_init_filter(struct flb_filter_instance *ins, struct flb_config *config, const char *plugin, flbgpu_filter **out);
static int gpu_init(struct flb_filter_instance *ins, struct flb_config *config, const char *plugin)
{
    flbgpu_filter *f;
    if (gpu_init_filter(ins, config, plugin, &f) != 0) return -1;
    flb_filter_set_context(ins, f);
    return 0;
}
static int gpu_init_filter(struct flb_filter_instance *ins, struct flb_config *config, const char *plugin, flbgpu_filter **out)
{
    struct mk_list *head;
    struct flb_kv *kv;
    flbgpu_filter *f;
    if (!gpu_context(ins)) return -1;
    f = G.filter_new(g_ctx, plugin);
    if (!f) { SHIM_ERROR(ins, "%s", G.last_error()); return -1; }
    mk_list_foreach(head, &ins->properties) {       /* config order, as the stock plugins read it (rule order matters) */
        kv = mk_list_entry(head, struct flb_kv, _head);
        if (strcmp(plugin, "parser") == 0 && strcasecmp(kv->key, "parser") == 0 && mirror_parser(ins, config, kv->val) != 0) {
            G.filter_destroy(f);
            return -1;
        }
        G.filter_set_property(f, kv->key, kv->val);
    }
    if (G.filter_init(f) != 0) {
        SHIM_ERROR(ins, "%s", G.last_error());
        G.filter_destroy(f);
        return -1;
    }
    *out = f;
    return 0;
}

static int cb_gpu_filter(const void *data, size_t bytes, const char *tag, int tag_len, void **out_buf, size_t *out_size,
                         struct flb_filter_instance *ins, struct flb_input_instance *i_ins, void *ctx, struct flb_config *config)
{
    int ret = G.filter_cb(ctx, data, bytes, tag, tag_len, out_buf, out_size);
    (void) i_ins; (void) config;
    if (ret < 0) {                                  /* loud, and the chunk passes untouched (the convention of all five stock filters) */
        SHIM_ERROR(ins, "%s", G.last_error());
        return FLB_FILTER_NOTOUCH;
    }
    return ret;
}

static int cb_gpu_exit(void *data, struct flb_config *config)
{
    (void) config;
    if (data && G.filter_destroy) G.filter_destroy(data);
    return 0;
}

/* ---- gpu_rewrite_tag: the device matches the rules, expands the tags and cuts the records out; the emitter -- an input
 * instance of this pipeline -- is created and fed here, the way plugins/filter_rewrite_tag/rewrite_tag.c does it
 * (emitter_create: 38-110, process_record: 404-413), once per new tag instead of once per record ---- */
int in_emitter_add_record(const char *tag, int tag_len, const char *buf_data, size_t buf_size,
                          struct flb_input_instance *in, struct flb_input_instance *i_ins);
struct gpu_rtag {
    flbgpu_filter *f;
    struct flb_input_instance *ins_emitter;
#ifdef FLB_HAVE_METRICS
    struct cmt_counter *cmt_emitted;          /* fluentbit_filter_emit_records_total{name} (rewrite_tag.c:301-311) */
#endif
};
#define GPU_RTAG_METRIC_EMITTED 200             /* FLB_RTAG_METRIC_EMITTED */

static int cb_init_rewrite_tag(struct flb_filter_instance *ins, struct flb_config *config, void *data)
{
    struct gpu_rtag *ctx;
    struct flb_input_instance *em;
    const char *name, *storage, *limit;
    char fallback[128];
    (void) data;
    ctx = flb_calloc(1, sizeof(*ctx));
    if (!ctx) return -1;
    if (gpu_init_filter(ins, config, "rewrite_tag", &ctx->f) != 0) { flb_free(ctx); return -1; }
    name = flb_filter_get_property("emitter_name", ins);
    if (!name) { snprintf(fallback, sizeof(fallback), "emitter_for_%s", flb_filter_name(ins)); name = fallback; }
    storage = flb_filter_get_property("emitter_storage.type", ins);
    limit = flb_filter_get_property("emitter_mem_buf_limit", ins);
    if (flb_input_name_exists(name, config) == FLB_TRUE) {
        SHIM_ERROR(ins, "emitter_name '%s' already exists", name);
        goto fail;
    }
    em = flb_input_new(config, "emitter", NULL, FLB_FALSE);
    if (!em) { SHIM_ERROR(ins, "cannot create emitter instance"); goto fail; }
    if (flb_input_set_property(em, "alias", name) == -1) {
        flb_plg_warn(ins, "cannot set emitter_name, using fallback name '%s'", em->name);
    }
    em->mem_buf_limit = flb_utils_size_to_bytes(limit ? limit : "10M");
    if (flb_input_set_property(em, "storage.type", storage ? storage : "memory") == -1) {
        flb_plg_error(ins, "cannot set storage.type");
    }
    if (flb_input_instance_init(em, config) == -1) { SHIM_ERROR(ins, "cannot initialize emitter instance '%s'", em->name); goto fail; }
    if (flb_storage_input_create(config->cio, em) == -1) { SHIM_ERROR(ins, "cannot initialize storage for stream '%s'", name); goto fail; }
    ctx->ins_emitter = em;
#ifdef FLB_HAVE_METRICS
    ctx->cmt_emitted = cmt_counter_create(ins->cmt, "fluentbit", "filter", "emit_records_total", "Total number of emitted records",
                                          1, (char *[]) {"name"});
    flb_metrics_add(GPU_RTAG_METRIC_EMITTED, "emit_records", ins->metrics);
#endif
    flb_filter_set_context(ins, ctx);
    return 0;
fail:
    G.filter_destroy(ctx->f);
    flb_free(ctx);
    return -1;
}

static int cb_filter_rewrite_tag(const void *data, size_t bytes, const char *tag, int tag_len, void **out_buf, size_t *out_size,
                                 struct flb_filter_instance *ins, struct flb_input_instance *i_ins, void *context, struct flb_config *config)
{
    struct gpu_rtag *ctx = context;
    const struct flbgpu_emit_group *groups = NULL;
    size_t n = 0, i;
    int ret = G.filter_cb(ctx->f, data, bytes, tag, tag_len, out_buf, out_size);
    (void) config;
    if (ret < 0) {
        SHIM_ERROR(ins, "%s", G.last_error());
        return FLB_FILTER_NOTOUCH;
    }
    if (G.filter_emitted(ctx->f, &groups, &n) == 0) {
        size_t emitted = 0;
        for (i = 0; i < n; i++) {
            if (in_emitter_add_record(groups[i].tag, (int) groups[i].tag_len, groups[i].data, groups[i].size, ctx->ins_emitter, i_ins) == -1) {
                flb_plg_warn(ins, "emitter refused %zu records re-tagged '%.*s'", groups[i].records, (int) groups[i].tag_len, groups[i].tag);
            }
            else {
                emitted += groups[i].records;
            }
        }
#ifdef FLB_HAVE_METRICS
        if (emitted > 0) {
            char *name = (char *) flb_filter_name(ins);
            cmt_counter_add(ctx->cmt_emitted, cfl_time_now(), (double) emitted, 1, (char *[]) {name});
            flb_metrics_sum(GPU_RTAG_METRIC_EMITTED, emitted, ins->metrics);
        }
#endif
    }
    return ret;
}

static int cb_exit_rewrite_tag(void *data, struct flb_config *config)
{
    struct gpu_rtag *ctx = data;
    (void) config;
    if (!ctx) return 0;
    if (ctx->f && G.filter_destroy) G.filter_destroy(ctx->f);
    flb_free(ctx);
    return 0;
}

extern struct flb_filter_plugin filter_rewrite_tag_plugin;
struct flb_filter_plugin filter_gpu_rewrite_tag_plugin = {
    .name = "gpu_rewrite_tag", .description = "H100: rewrite_tag on the GPU (libflbgpu)",
    .cb_init = cb_init_rewrite_tag, .cb_filter = cb_filter_rewrite_tag, .cb_exit = cb_exit_rewrite_tag, .flags = 0 };

/* the metric table of a gpu_log_to_metrics instance in cmetrics' text form (what the stock plugin appends to its
 * hidden input from cb_filter / its flush timer, log_to_metrics.c:560-621,1117-1125); free() the result */
char *filter_gpu_l2m_text(struct flb_filter_instance *ins)
{
    return (ins && ins->context && G.l2m_text) ? G.l2m_text(ins->context) : NULL;
}

extern struct flb_filter_plugin filter_parser_plugin, filter_grep_plugin, filter_modify_plugin,
                                filter_record_modifier_plugin, filter_log_to_metrics_plugin, filter_multiline_plugin;

#define GPU_PLUGIN(sym, short_name, gpu_name, stock)                                                        \
    static int cb_init_##sym(struct flb_filter_instance *ins, struct flb_config *config, void *data)         \
    { (void) data; return gpu_init(ins, config, short_name); }                                              \
    struct flb_filter_plugin filter_gpu_##sym##_plugin = {                                                   \
        .name = gpu_name, .description = "H100: " short_name " on the GPU (libflbgpu)",                       \
        .cb_init = cb_init_##sym, .cb_filter = cb_gpu_filter, .cb_exit = cb_gpu_exit, .flags = 0 };

GPU_PLUGIN(parser, "parser", "gpu_parser", filter_parser_plugin)
GPU_PLUGIN(grep, "grep", "gpu_grep", filter_grep_plugin)
GPU_PLUGIN(modify, "modify", "gpu_modify", filter_modify_plugin)
GPU_PLUGIN(record_modifier, "record_modifier", "gpu_record_modifier", filter_record_modifier_plugin)
GPU_PLUGIN(log_to_metrics, "log_to_metrics", "gpu_log_to_metrics", filter_log_to_metrics_plugin)
/* gpu_multiline: plugins/filter_multiline/ml.c in parser mode with `buffer off` (the one mode whose result is the call's own
 * return value: cb_ml_filter :833-892).  The built-in rule-based multiline parsers (java, go, python, ruby) exist on the
 * device side by name.  A parser of a [MULTILINE_PARSER] section is registered by whoever embeds the library with
 * flbgpu_ml_parser_create() / _rule() / _init() -- struct flb_ml_rule keeps the compiled regex, not its text
 * (include/fluent-bit/multiline/flb_ml.h:71-94), so config->multiline_parsers cannot be mirrored from here the way
 * config->parsers is. */
GPU_PLUGIN(multiline, "multiline", "gpu_multiline", filter_multiline_plugin)

/* static initialisers cannot take another object's member: the stock config maps and event types are copied when the
 * library is loaded, before anyone looks the structs up */
__attribute__((constructor)) static void gpu_plugins_adopt_config_maps(void)
{
    filter_gpu_parser_plugin.config_map = filter_parser_plugin.config_map;
    filter_gpu_grep_plugin.config_map = filter_grep_plugin.config_map;
    filter_gpu_modify_plugin.config_map = filter_modify_plugin.config_map;
    filter_gpu_record_modifier_plugin.config_map = filter_record_modifier_plugin.config_map;
    filter_gpu_log_to_metrics_plugin.config_map = filter_log_to_metrics_plugin.config_map;
    filter_gpu_rewrite_tag_plugin.config_map = filter_rewrite_tag_plugin.config_map;
    filter_gpu_multiline_plugin.config_map = filter_multiline_plugin.config_map;
    filter_gpu_multiline_plugin.event_type = filter_multiline_plugin.event_type;
    filter_gpu_rewrite_tag_plugin.event_type = filter_rewrite_tag_plugin.event_type;
    filter_gpu_parser_plugin.event_type = filter_parser_plugin.event_type;
    filter_gpu_grep_plugin.event_type = filter_grep_plugin.event_type;
    filter_gpu_modify_plugin.event_type = filter_modify_plugin.event_type;
    filter_gpu_record_modifier_plugin.event_type = filter_record_modifier_plugin.event_type;
    filter_gpu_log_to_metrics_plugin.event_type = filter_log_to_metrics_plugin.event_type;
}
