/* runtime_ml.h -- host side of filter_multiline (part of runtime.c, included there).
 *
 * Multiline parser definitions: struct flb_ml_parser / flb_ml_parser_create() (src/multiline/flb_ml_parser.c:46-130,
 * :199-230), flb_ml_rule_create() (src/multiline/flb_ml_rule.c:48-112), flb_ml_parser_init() -> flb_ml_rule_init()
 * (:198-300), the built-in java / go / python / ruby parsers (src/multiline/flb_ml_parser_{java,go,python,ruby}.c).
 * The filter: cb_ml_init() / cb_ml_filter() of plugins/filter_multiline/ml.c in `buffer off`, parser mode. */

struct ml_rule_def { char *from, *regex, *to; int start; };
struct flbgpu_ml_parser {
    flbgpu_ctx *ctx;
    char *name;
    int type, negate, inited;
    char *match, *key_content, *key_group, *key_pattern, *parser_name;
    struct ml_rule_def rules[ML_MAX_RULES];
    int n_rules;
    struct flbgpu_ml_parser *next;
};

static char *dup_or_null(const char *s) { return s ? strdup(s) : NULL; }

static void ml_parser_free(struct flbgpu_ml_parser *m)
{
    int i;
    if (!m) return;
    for (i = 0; i < m->n_rules; i++) { free(m->rules[i].from); free(m->rules[i].regex); free(m->rules[i].to); }
    free(m->name); free(m->match); free(m->key_content); free(m->key_group); free(m->key_pattern); free(m->parser_name);
    free(m);
}

static void ml_parsers_free(flbgpu_ctx *ctx)
{
    struct flbgpu_ml_parser *m = ctx->ml_parsers, *nx;
    for (; m; m = nx) { nx = m->next; ml_parser_free(m); }
    ctx->ml_parsers = NULL;
}

flbgpu_ml_parser *flbgpu_ml_parser_create(flbgpu_ctx *ctx, const char *name, const char *type, const char *match_string, int negate,
                                          int flush_ms, const char *key_content, const char *key_group, const char *key_pattern,
                                          const char *parser_name)
{
    struct flbgpu_ml_parser *m, **tail;
    int t;
    (void) flush_ms;                                   /* the timer belongs to the buffered mode */
    g_rt_err[0] = 0;
    if (!ctx || !name || !type) { set_err("[multiline_parser] no 'name' / 'type' defined%s%s", NULL, NULL); return NULL; }
    if (!strcasecmp(type, "regex")) t = ML_T_REGEX;                   /* flb_ml_type_lookup(), src/multiline/flb_ml.c:83-98 */
    else if (!strcasecmp(type, "endswith")) t = ML_T_ENDSWITH;
    else if (!strcasecmp(type, "equal") || !strcasecmp(type, "eq")) t = ML_T_EQ;
    else { set_err("[multiline_parser] invalid type '%s'%s", type, NULL); return NULL; }
    m = calloc(1, sizeof(*m));
    if (!m) { set_err("out of memory%s%s", NULL, NULL); return NULL; }
    m->ctx = ctx; m->type = t; m->negate = negate != 0;
    m->name = strdup(name); m->match = dup_or_null(match_string); m->key_content = dup_or_null(key_content);
    m->key_group = dup_or_null(key_group); m->key_pattern = dup_or_null(key_pattern); m->parser_name = dup_or_null(parser_name);
    if (!m->name) { ml_parser_free(m); set_err("out of memory%s%s", NULL, NULL); return NULL; }
    for (tail = &ctx->ml_parsers; *tail; tail = &(*tail)->next) ;       /* mk_list_add: appended */
    *tail = m;
    return m;
}

/* does the comma-separated list of state names hold `state`?  (flb_slist_split_string(..., ',', -1): entries without the
 * blanks around them) */
static int states_hold(const char *list, const char *state)
{
    const size_t n = strlen(state);
    const char *p = list;
    while (*p) {
        const char *e;
        size_t len;
        while (*p == ' ' || *p == ',') p++;
        e = p;
        while (*e && *e != ',') e++;
        len = (size_t) (e - p);
        while (len && p[len - 1] == ' ') len--;
        if (len == n && !memcmp(p, state, n)) return 1;
        p = e;
    }
    return 0;
}

int flbgpu_ml_parser_rule(flbgpu_ml_parser *m, const char *from_states, const char *regex, const char *to_state)
{
    struct ml_rule_def *r;
    struct rx_compiled c;
    const char *p;
    g_rt_err[0] = 0;
    if (!m || !from_states || !regex) { set_err("[multiline] rule is empty or has invalid 'from_states' tokens%s%s", NULL, NULL); return -1; }
    for (p = from_states; *p == ' ' || *p == ','; p++) ;
    if (!*p) { set_err("[multiline] rule is empty or has invalid 'from_states' tokens%s%s", NULL, NULL); return -1; }
    if (m->n_rules >= ML_MAX_RULES) { set_err("[multiline parser: %s] more rules than the device automaton holds%s", m->name, NULL); return -1; }
    r = &m->rules[m->n_rules];
    r->start = states_hold(from_states, "start_state");
    if (!r->start && m->n_rules == 0) { set_err("[multiline] rule don't contain a 'start_state'%s%s", NULL, NULL); return -1; }
    if (rx_compile(regex, &c) != 0) { set_err("could not compile regex pattern '%s' (%s)", regex, c.err); return -1; }
    rx_compiled_free(&c);
    r->from = strdup(from_states); r->regex = strdup(regex); r->to = dup_or_null(to_state);
    if (!r->from || !r->regex) { free(r->from); free(r->regex); free(r->to); memset(r, 0, sizeof(*r)); set_err("out of memory%s%s", NULL, NULL); return -1; }
    m->n_rules++;
    return 0;
}

int flbgpu_ml_parser_init(flbgpu_ml_parser *m)
{
    int i, j;
    g_rt_err[0] = 0;
    if (!m) return -1;
    for (i = 0; i < m->n_rules; i++) {                 /* set_to_state_map(): every to_state is some rule's from_state */
        int found = 0;
        if (!m->rules[i].to) continue;
        for (j = 0; j < m->n_rules; j++) if (states_hold(m->rules[j].from, m->rules[i].to)) found = 1;
        if (!found) { set_err("[multiline parser: %s] to_state='%s' is not registered", m->name, m->rules[i].to); return -1; }
    }
    m->inited = 1;
    return 0;
}

/* the built-in parsers made of regex rules (flb_ml_parser_builtin_create(), src/multiline/flb_ml_parser.c:143-196) */
static struct flbgpu_ml_parser *ml_builtin(flbgpu_ctx *ctx, const char *name)
{
    static const char *const java[][3] = {
        { "start_state, java_start_exception", "/(.)(?:Exception|Error|Throwable|V8 errors stack trace)[:\\r\\n]/", "java_after_exception" },
        { "java_after_exception", "/^[\\t ]*nested exception is:[\\t ]*/", "java_start_exception" },
        { "java_after_exception", "/^[\\r\\n]*$/", "java_after_exception" },
        { "java_after_exception, java", "/^[\\t ]+(?:eval )?at /", "java" },
        { "java_after_exception, java", "/^[\\t ]+--- End of inner exception stack trace ---$/", "java" },
        { "java_after_exception, java", "/^--- End of stack trace from previous (?x:)location where exception was thrown ---$/", "java" },
        { "java_after_exception, java", "/^[\\t ]*(?:Caused by|Suppressed):/", "java_after_exception" },
        { "java_after_exception, java", "/^[\\t ]*... \\d+ (?:more|common frames omitted)/", "java" }, { 0, 0, 0 } };
    static const char *const go[][3] = {
        { "start_state", "/\\bpanic: /", "go_after_panic" },
        { "start_state", "/http: panic serving/", "go_goroutine" },
        { "go_after_panic", "/^$/", "go_goroutine" },
        { "go_after_panic, go_after_signal, go_frame_1", "/^$/", "go_goroutine" },
        { "go_after_panic", "/^\\[signal /", "go_after_signal" },
        { "go_goroutine", "/^goroutine \\d+ \\[[^\\]]+\\]:$/", "go_frame_1" },
        { "go_frame_1", "/^(?:[^\\s.:]+\\.)*[^\\s.():]+\\(|^created by /", "go_frame_2" },
        { "go_frame_2", "/^\\s/", "go_frame_1" }, { 0, 0, 0 } };
    static const char *const python[][3] = {
        { "start_state", "/^Traceback \\(most recent call last\\):$/", "python" },
        { "python", "/^[\\t ]+File /", "python_code" },
        { "python_code", "/[^\\t ]/", "python" },
        { "python", "/^(?:[^\\s.():]+\\.)*[^\\s.():]+:/", "start_state" }, { 0, 0, 0 } };
    static const char *const ruby[][3] = {
        { "start_state, ruby_start_exception", "/^.+:\\d+:in\\s+.*/", "ruby_after_exception" },
        { "ruby_after_exception, ruby", "/^\\s+from\\s+.*:\\d+:in\\s+.*/", "ruby" }, { 0, 0, 0 } };
    const char *const (*tab)[3] = !strcasecmp(name, "java") ? java : !strcasecmp(name, "go") ? go :
                                  !strcasecmp(name, "python") ? python : !strcasecmp(name, "ruby") ? ruby : NULL;
    struct flbgpu_ml_parser *m;
    int i;
    if (!tab) return NULL;
    m = flbgpu_ml_parser_create(ctx, name, "regex", NULL, 0, 0, NULL, NULL, NULL, NULL);
    if (!m) return NULL;
    for (i = 0; tab[i][0]; i++) if (flbgpu_ml_parser_rule(m, tab[i][0], tab[i][1], tab[i][2])) return NULL;
    if (flbgpu_ml_parser_init(m)) return NULL;
    return m;
}

static struct flbgpu_ml_parser *ml_parser_get(flbgpu_ctx *ctx, const char *name)
{
    struct flbgpu_ml_parser *m;
    for (m = ctx->ml_parsers; m; m = m->next) if (!strcasecmp(m->name, name)) return m;      /* flb_ml_parser_get() */
    return ml_builtin(ctx, name);
}

int flbgpu_ml_set_buffer_limit(flbgpu_ctx *ctx, size_t bytes)
{
    if (!ctx) return -1;
    ctx->ml_limit = bytes; ctx->ml_limit_set = 1;
    return 0;
}

/* the filter's properties -> struct cf_ml in the blob */
static uint32_t emit_ml_filter(flbgpu_filter *f, struct blob *b)
{
    struct kv *p;
    struct cf_ml cf;
    struct cf_ml_rule rules[ML_MAX_RULES];
    struct flbgpu_ml_parser *m = NULL;
    const char *key_content = NULL;
    int use_buffer = 1, n_parsers = 0, i, j;
    memset(&cf, 0, sizeof(cf));
    memset(rules, 0, sizeof(rules));
    for (p = f->props; p; p = p->next) {
        if (!strcasecmp(p->k, "multiline.parser")) {
            /* a comma-separated list (FLB_CONFIG_MAP_CLIST), several entries allowed */
            const char *s = p->v;
            while (*s) {
                const char *e;
                char name[128];
                size_t len;
                while (*s == ' ' || *s == ',') s++;
                if (!*s) break;
                for (e = s; *e && *e != ','; e++) ;
                len = (size_t) (e - s);
                while (len && s[len - 1] == ' ') len--;
                if (len >= sizeof(name)) len = sizeof(name) - 1;
                memcpy(name, s, len); name[len] = 0;
                if (!strcasecmp(name, "docker") || !strcasecmp(name, "cri")) {
                    set_err("[filter multiline] the built-in '%s' parser (sub-parser + key_group) is not built on the device%s", name, NULL);
                    return 0;
                }
                m = ml_parser_get(f->ctx, name);
                if (!m) { if (!g_rt_err[0]) set_err("[multiline] parser '%s' not registered%s", name, NULL); return 0; }
                n_parsers++;
                s = e;
            }
        }
        else if (!strcasecmp(p->k, "multiline.key_content")) key_content = p->v;
        else if (!strcasecmp(p->k, "buffer")) use_buffer = parse_bool(p->v) == 1;       /* flb_utils_bool() */
        else if (!strcasecmp(p->k, "mode")) {
            if (!strcasecmp(p->v, "partial_message")) { set_err("[filter multiline] 'Mode partial_message' is not built on the device%s%s", NULL, NULL); return 0; }
            if (strcasecmp(p->v, "parser")) { set_err("'Mode' must be 'partial_message' or 'parser'%s%s", NULL, NULL); return 0; }
        }
        else if (!strcasecmp(p->k, "emitter_storage.type")) {
            if (strcasecmp(p->v, "memory") && strcasecmp(p->v, "filesystem")) {
                set_err("invalid 'emitter_storage.type' value. Only 'memory' or 'filesystem' types are allowed%s%s", NULL, NULL);
                return 0;
            }
        }
        else if (!strcasecmp(p->k, "debug_flush") || !strcasecmp(p->k, "flush_ms") || !strcasecmp(p->k, "emitter_name") ||
                 !strcasecmp(p->k, "emitter_mem_buf_limit")) continue;
        else { set_err("[filter multiline] unknown configuration property '%s'%s", p->k, NULL); return 0; }
    }
    if (n_parsers == 0) { set_err("The default 'Mode' 'parser' requires at least one 'multiline.parser'%s%s", NULL, NULL); return 0; }
    if (n_parsers > 1) { set_err("[filter multiline] several multiline parsers in one filter are not built on the device%s%s", NULL, NULL); return 0; }
    if (use_buffer) {
        set_err("[filter multiline] only 'buffer off' is built on the device (the buffered mode hands the messages to an emitter input on a timer)%s%s", NULL, NULL);
        return 0;
    }
    if (m->type == ML_T_REGEX && !m->inited) { set_err("[multiline parser: %s] rules not initialised (flbgpu_ml_parser_init)%s", m->name, NULL); return 0; }
    if (m->key_group) { set_err("[multiline parser: %s] key_group is not built on the device%s", m->name, NULL); return 0; }
    if (m->parser_name) { set_err("[multiline parser: %s] a sub-parser is not built on the device%s", m->name, NULL); return 0; }
    if (m->type != ML_T_REGEX && !m->match) { set_err("[multiline parser: %s] no match_string%s", m->name, NULL); return 0; }
    if (!key_content) key_content = m->key_content;    /* the filter's multiline.key_content overrides the parser's */
    /* (key_pattern only changes what the ENDSWITH / EQ types look at, flb_ml.c:243-255) */
    if (m->key_pattern && m->type != ML_T_REGEX) { set_err("[multiline parser: %s] key_pattern is not built on the device%s", m->name, NULL); return 0; }
    cf.type = (uint32_t) m->type; cf.negate = (uint32_t) m->negate; cf.n_rules = (uint32_t) m->n_rules;
    if (key_content) { cf.key_len = (uint32_t) strlen(key_content); cf.key_off = blob_add(b, key_content, cf.key_len ? cf.key_len : 1, 1); }
    else cf.key_len = 0xffffffffu;
    if (m->match) { cf.match_len = (uint32_t) strlen(m->match); cf.match_off = blob_add(b, m->match, cf.match_len ? cf.match_len : 1, 1); }
    cf.limit = (uint32_t) (f->ctx->ml_limit_set ? f->ctx->ml_limit : ((size_t) 2 << 20));       /* FLB_ML_BUFFER_LIMIT_DEFAULT */
    for (i = 0; i < m->n_rules; i++) {
        rules[i].rx_off = emit_rx(b, m->rules[i].regex, NULL);
        if (!rules[i].rx_off) return 0;
        rules[i].start = (uint32_t) m->rules[i].start;
        if (m->rules[i].to)
            for (j = 0; j < m->n_rules; j++) {          /* to_state_map: the rules that list this rule's to_state, in rule order */
                if (!states_hold(m->rules[j].from, m->rules[i].to)) continue;
                if (m->rules[j].start) rules[i].next_start = 1;
                else rules[i].to[rules[i].n_to++] = (uint8_t) j;
            }
    }
    cf.rules_off = blob_add(b, rules, sizeof(rules[0]) * (size_t) (m->n_rules ? m->n_rules : 1), 8);
    return blob_add(b, &cf, sizeof(cf), 8);
}

/* One chunk through the multiline filter of a solo chain.  Same contract as chain_run(). */
static int ml_run(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in_ext, size_t bytes,
                  uint8_t *ext_out, size_t ext_cap, void **host_out, size_t *out_size)
{
    flbgpu_filter *f = c->f[0];
    const struct cf_ml *cf = (const struct cf_ml *) (c->blob.p + c->ml_cfg_off);
    const uint8_t *d_in;
    struct ml_env e;
    uint32_t n_rec, n_ev, h_flags[FLBGPU_MAX_FILTERS + 1];
    size_t off, need, at;
    unsigned long long res[4];
    uint64_t total;
    struct timespec now;

    if (call_start(c, bytes, out_size, NULL) || !(d_in = place_input(c, h_in, d_in_ext, bytes))) return -1;
    if (bk_flags_clear(c->q, c->d_flags) || index_chunk(c, d_in, bytes, &n_rec, &off)) return -1;
    if (refuse_wide_arrays(c, h_in, d_in, off, bytes)) return -1;
    c->st.records_in = n_rec;
    c->st.passes = 1;
    if (n_rec == 0) return FLBGPU_FILTER_NOTOUCH;

    /* ---- work arrays: one allocation, carved ---- */
    memset(&e, 0, sizeof(e));
    e.in = d_in; e.blob = c->d_blob; e.cfg_off = c->ml_cfg_off;
    e.off = c->d_off; e.len = c->d_len; e.kind = c->d_kind; e.n_rec = n_rec;
    e.err = c->d_flags + FLBGPU_MAX_FILTERS;
    e.S = (cf->n_rules + 1) * 4;
    e.nt1 = (n_rec + ML_F1 - 1) / ML_F1;
    e.nt2 = (e.nt1 + ML_F2 - 1) / ML_F2;
    e.state_in = f->ml_state < e.S ? f->ml_state : 0;
    e.time_in[0] = f->ml_time[0]; e.time_in[1] = f->ml_time[1];
    clock_gettime(CLOCK_REALTIME, &now);
    e.now[0] = (int64_t) now.tv_sec; e.now[1] = (int64_t) now.tv_nsec;
#define ML_CARVE(field, type, count) do { at = (at + 15) & ~(size_t) 15; if (base) e.field = (type *) (base + at); at += sizeof(type) * (size_t) (count); } while (0)
    {
        uint8_t *base = NULL;
        int round;
        for (round = 0; round < 2; round++) {
            at = 0;
            ML_CARVE(res, unsigned long long, 4);
            ML_CARVE(feat, struct ml_feat, n_rec);
            ML_CARVE(act, uint8_t, n_rec);
            ML_CARVE(tl, uint32_t, n_rec);
            ML_CARVE(T1, uint8_t, (size_t) e.nt1 * e.S);
            ML_CARVE(T2, uint8_t, (size_t) e.nt2 * e.S);
            ML_CARVE(in1, uint8_t, e.nt1);
            ML_CARVE(in2, uint8_t, e.nt2);
            ML_CARVE(cnt1, uint32_t, e.nt1); ML_CARVE(lt1, uint32_t, e.nt1); ML_CARVE(base1, uint32_t, e.nt1); ML_CARVE(tl1, uint32_t, e.nt1);
            ML_CARVE(cnt2, uint32_t, e.nt2); ML_CARVE(lt2, uint32_t, e.nt2); ML_CARVE(base2, uint32_t, e.nt2); ML_CARVE(tl2, uint32_t, e.nt2);
            ML_CARVE(ev_slot, uint32_t, 2 * (size_t) n_rec + 2);
            ML_CARVE(ev_size, uint32_t, 2 * (size_t) n_rec + 2);
            ML_CARVE(ev_buflen, uint32_t, 2 * (size_t) n_rec + 2);
            ML_CARVE(ev_ctx, uint32_t, 2 * (size_t) n_rec + 2);
            if (round == 0) {
                need = at + 64;
                if (dev_grow(c, (void **) &c->d_mlw, &c->cap_mlw, need, 1, 0)) return -1;
                base = c->d_mlw;
            }
        }
    }
#undef ML_CARVE
    if (bk_ml_plan(c->q, &e)) return -1;
    if (bk_d2h(c->q, res, e.res, sizeof(res)) || bk_sync(c->q)) return -1;
    n_ev = (uint32_t) res[0];
    if (bk_flags_fetch(c->q, c->d_flags, h_flags)) return -1;
    if (refused(c, h_flags[FLBGPU_MAX_FILTERS])) return -1;
    c->st.kernel_launches = bk_launch_count();
    if (n_ev == 0) {                                     /* nothing came out (no decodable event) */
        f->ml_state = (uint32_t) res[1]; f->ml_time[0] = (int64_t) res[2]; f->ml_time[1] = (int64_t) res[3];
        return FLBGPU_FILTER_NOTOUCH;
    }
    /* ---- sizes, offsets ---- */
    if (bk_ml_sizes(c->q, &e, n_ev) || bk_flags_fetch(c->q, c->d_flags, h_flags)) return -1;
    if (refused(c, h_flags[FLBGPU_MAX_FILTERS])) return -1;
    if (sizes_to_offsets(c, e.ev_size, n_ev, NULL, NULL, "result larger than 4 GiB", &total)) return -1;
    c->st.bytes_out = total;
    c->st.records_out = n_ev;
    *out_size = (size_t) total;
    /* the filter's state for the next chunk: flushed, the rule and the group's time stay */
    f->ml_state = (uint32_t) res[1]; f->ml_time[0] = (int64_t) res[2]; f->ml_time[1] = (int64_t) res[3];
    if (total == 0) return FLBGPU_FILTER_NOTOUCH;
    /* ---- emit ---- */
    if (!host_out && !ext_out) {                         /* the result stays in this chain's own device buffer (ml_then_rest) */
        if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_ml_emit(c->q, &e, n_ev, c->d_bsum, c->d_out) || bk_sync(c->q)) return -1;
    }
    else if (!host_out) {
        if (ext_cap < total) { set_err("device output buffer too small%s%s", NULL, NULL); return -1; }
        if (bk_ml_emit(c->q, &e, n_ev, c->d_bsum, ext_out)) return -1;
    }
    else {
        void *out = malloc((size_t) total);
        if (!out) return -1;
        if (dev_grow(c, (void **) &c->d_out, &c->cap_out, total, 1, 0) || bk_ml_emit(c->q, &e, n_ev, c->d_bsum, c->d_out) || bk_d2h(c->q, out, c->d_out, (size_t) total) || bk_sync(c->q)) { free(out); return -1; }
        *host_out = out;
    }
    c->st.kernel_launches = bk_launch_count();
    return FLBGPU_FILTER_MODIFIED;
}

/* `multiline, then other filters`: the multiline chain leaves its result on the device, the chain of the other filters takes it
 * from there.  h_in or d_in_ext is the input; the result goes to host_out (malloc()ed) or to ext_out on the device.
 * flb_filter_do() semantics between the two: NOTOUCH hands the input on unchanged, MODIFIED with nothing left ends the chain. */
static int chain_run(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in_ext, size_t bytes,
                     uint8_t *ext_out, size_t ext_cap, void **host_out, size_t *out_size);
static int ml_then_rest(flbgpu_chain *c, const uint8_t *h_in, const uint8_t *d_in_ext, size_t bytes,
                        uint8_t *ext_out, size_t ext_cap, void **host_out, size_t *out_size)
{
    flbgpu_chain *m = c->ml_solo, *p = c->ml_post;
    size_t n_mid = 0;
    int r = FLBGPU_FILTER_NOTOUCH, k;
    c->ctx->last_q = m->q;                               /* flbgpu_kernel_ms(): the multiline stage's launches */
    p->active = 0;
    for (k = 1; k < c->nf; k++) if ((c->active >> k) & 1) p->active |= 1u << (k - 1);
    if (c->active & 1u) {
        m->active = 1;
        r = ml_run(m, h_in, d_in_ext, bytes, NULL, 0, NULL, &n_mid);
        if (!d_in_ext) bk_upload_end(m->q);
        c->st = m->st;
        if (r < 0) return -1;
    }
    if (r == FLBGPU_FILTER_MODIFIED && n_mid == 0) { *out_size = 0; return FLBGPU_FILTER_MODIFIED; }      /* nothing left: the chain ends */
    if (r != FLBGPU_FILTER_MODIFIED) {
        /* the filters behind it see the chunk as it came */
        if (!p->active) return FLBGPU_FILTER_NOTOUCH;
        r = chain_run(p, h_in, d_in_ext, bytes, ext_out, ext_cap, host_out, out_size);
        if (!d_in_ext) bk_upload_end(p->q);
        if (r >= 0 && !host_out && bk_sync(p->q)) return -1;         /* (the caller waits on the outer chain's queue, not on this one) */
        if (r >= 0) c->st = p->st;
        return r;
    }
    if (p->active) {
        r = chain_run(p, NULL, m->d_out, n_mid, ext_out, ext_cap, host_out, out_size);
        if (r < 0) { c->st.error_bits = p->st.error_bits; return -1; }
        if (!host_out && bk_sync(p->q)) return -1;
        if (r == FLBGPU_FILTER_MODIFIED) {
            c->st.bytes_out = p->st.bytes_out; c->st.records_out = p->st.records_out; c->st.kernel_launches = p->st.kernel_launches;
            return r;
        }
    }
    /* what the multiline filter made is the result */
    *out_size = n_mid;
    if (host_out) {
        void *out = malloc(n_mid);
        if (!out) return -1;
        if (bk_d2h(m->q, out, m->d_out, n_mid) || bk_sync(m->q)) { free(out); return -1; }
        *host_out = out;
    }
    else {
        if (ext_cap < n_mid) { set_err("device output buffer too small%s%s", NULL, NULL); return -1; }
        if (bk_d2d(m->q, ext_out, m->d_out, n_mid) || bk_sync(m->q)) return -1;
    }
    return FLBGPU_FILTER_MODIFIED;
}
