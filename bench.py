#!/usr/bin/env python
"""bench.py -- log lines/s through the parser+filter chain (BASELINE.json metric).

  python bench.py --gpus N --steps K --warmup W            (ours; torchrun for N>1)
  python bench.py --impl reference --gpus N --steps K --warmup W
  python bench.py ... --dump-outputs DIR                  (also writes the last timed step's result, see dump_outputs)

Primary workload (config.workload): BASELINE.json configs[1] -- 10 M JSON lines through filter_parser(json) +
filter_grep + filter_modify, 10 M events per GPU per step (weak scaling).  A step is one pass of the chain over
that batch.  Reported beside it, each with the same fields: the north-star apache chain, configs[0] (10 k apache
lines, parser only, one call), configs[2] (nginx regex parser + record_modifier) and configs[3]
(filter_log_to_metrics histogram over 100 M records in total, metric tables all-reduced over NCCL every step).

  value ....... events/s with the batch resident in HBM (flbgpu_chain_do_device), CUDA events
  e2e ......... the same batch through flbgpu_chain_do() the way flb_filter_do() calls a filter: input in
                ordinary malloc()ed (pageable) memory, default glibc malloc for the result, host<->device copies
                and free() of the result inside the timed region
  e2e_variants  pinned input; and the batch sweep: bytes per call in {64 KB, 2 MB, 64 MB, whole set}, one caller
                thread and 8 caller threads (8 filter instances, what `threaded on` inputs give the engine)
  roofline .... evaluation kernel (k_chain_eval: record decode + parser + filters) timed by CUDA events inside the
                library; algorithmic bytes = chain input + chain output
  cpu_baseline  the UNMODIFIED reference (oracle/_ref) on this box's host cores, bounded sample
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BASE_LINES = 100_000          # distinct synthetic lines; the batch tiles this block

WORKLOADS = {
    # BASELINE.json configs[1]
    "json": {
        "name": "configs[1]: 10M JSON lines -> filter_parser(json)+filter_grep(level ^(warn|error)$)+filter_modify(Add,Rename,Remove)",
        "filters": [("parser", [("Key_Name", "log"), ("Parser", "json")]),
                    ("grep", [("Regex", "level ^(warn|error)$")]),
                    ("modify", [("Add", "env prod"), ("Rename", "msg message"), ("Remove", "debug")])],
    },
    # BASELINE.json north_star
    "apache": {
        "name": "north-star chain: filter_parser(apache regex)+filter_grep(method ^(GET|POST)$)+filter_modify over apache-combined events",
        "filters": [("parser", [("Key_Name", "log"), ("Parser", "apache")]),
                    ("grep", [("Regex", "method ^(GET|POST)$")]),
                    ("modify", [("Add", "env prod"), ("Rename", "code status"), ("Remove", "agent")])],
    },
    # BASELINE.json configs[0]: the reference's own CPU-runnable case, one 10k-line batch per call
    "c0": {
        "name": "configs[0]: 10k-line apache batch -> parser 'apache' (conf/parsers.conf:1-6), one call per batch",
        "filters": [("parser", [("Key_Name", "log"), ("Parser", "apache")])],
    },
    # BASELINE.json configs[2]: the 5xx answers (2 % of the lines) are re-tagged and leave the chunk
    "nginx": {
        "name": "configs[2]: nginx access logs -> regex parser 'nginx' + filter_record_modifier(Record hostname node-1; Remove_key agent) + filter_rewrite_tag(Rule $code ^5 errors.$method false)",
        "filters": [("parser", [("Key_Name", "log"), ("Parser", "nginx")]),
                    ("record_modifier", [("Record", "hostname node-1"), ("Remove_key", "agent")]),
                    ("rewrite_tag", [("Rule", "$code ^5 errors.$method false")])],
    },
    # BASELINE.json configs[3]: 32 label sets, integer-valued observations (exact fp64 sums), logs discarded; with N>1
    # every step ends with the all-reduce of the metric tables (NCCL).
    "l2m": {
        "name": "configs[3]: filter_log_to_metrics histogram(duration) by color,direction over 100M records in total; discard_logs; table all-reduce per step",
        "filters": [("log_to_metrics", [("metric_mode", "histogram"), ("metric_name", "duration"), ("metric_description", "d"),
                                        ("tag", "m"), ("value_field", "duration"), ("label_field", "color"),
                                        ("label_field", "direction"), ("discard_logs", "on")])],
    },
    # BASELINE.json configs[4]: application logs with Java stack traces -> multiline + parser + grep.  filter_multiline (built-in
    # java parser, `buffer off`: the lines of a chunk are concatenated inside the call) leaves its result on the device, the
    # parser (timestamp / level / class of the first line; a stack trace does not match and stays as it is) and the grep
    # (INFO and DEBUG lines go) run on it as one fused chain.
    "ml": {
        "name": "configs[4]: application logs with Java stack traces -> filter_multiline(java, key_content log, buffer off) + filter_parser(regex: time level [class] msg, Reserve_Data) + filter_grep(Exclude level ^(INFO|DEBUG)$)",
        "filters": [("multiline", [("multiline.parser", "java"), ("multiline.key_content", "log"), ("buffer", "off")]),
                    ("parser", [("Key_Name", "log"), ("Parser", "applog"), ("Reserve_Data", "On")]),
                    ("grep", [("Exclude", "level ^(INFO|DEBUG)$")])],
    },
}
NO_PARSER = ("l2m",)
APPLOG_RX = r"^(?<time>\d{4}-\d{2}-\d{2} \d{2}:\d{2}:\d{2}\.\d{3}) (?<level>[A-Z]+) \[(?<class>[^\]]+)\] (?<msg>.*)$"


def java_lines(n, seed):
    """application log lines, about one in eight followed by a Java stack trace of 3-12 frames (some with a cause)"""
    import random
    rng = random.Random(seed)
    pk = ["com.example.app", "org.acme.billing", "io.svc.gateway", "net.corp.auth"]
    cl = ["OrderService", "HttpHandler", "TokenCache", "DbPool", "RetryPolicy", "JsonCodec"]
    ex = ["java.lang.IllegalStateException", "java.io.IOException", "java.lang.NullPointerException", "java.util.concurrent.TimeoutException",
          "org.acme.billing.PaymentError"]
    out = []
    t = 1700000000
    while len(out) < n:
        t += rng.randint(0, 2)
        ts = "2023-11-14 %02d:%02d:%02d.%03d" % ((t // 3600) % 24, (t // 60) % 60, t % 60, rng.randint(0, 999))
        if rng.random() < 0.125:
            out.append(("%s ERROR [%s] request %d failed" % (ts, rng.choice(cl), rng.randint(0, 10 ** 6))).encode())
            out.append(("%s: %s" % (rng.choice(ex), rng.choice(["connection reset", "state is CLOSED", "timed out after 30000 ms", "null"]))).encode())
            for _ in range(rng.randint(3, 12)):
                out.append(("\tat %s.%s.%s(%s.java:%d)" % (rng.choice(pk), rng.choice(cl), rng.choice(["run", "call", "handle", "get", "apply"]),
                                                          rng.choice(cl), rng.randint(1, 900))).encode())
            if rng.random() < 0.4:
                out.append(("Caused by: %s: %s" % (rng.choice(ex), "inner")).encode())
                for _ in range(rng.randint(2, 6)):
                    out.append(("\tat %s.%s.%s(%s.java:%d)" % (rng.choice(pk), rng.choice(cl), "invoke", rng.choice(cl), rng.randint(1, 900))).encode())
                out.append(("\t... %d more" % rng.randint(1, 30)).encode())
        else:
            out.append(("%s INFO [%s] %s in %d ms path=/api/v1/%s/%d" % (ts, rng.choice(cl), rng.choice(["handled", "served", "cached"]),
                                                                        rng.randint(1, 900), rng.choice(["orders", "users", "items"]), rng.randint(1, 99999))).encode())
    return out[:n]


def make_block(wl, rank=0):
    import util
    if wl == "ml":
        return util.chunk_from_lines(java_lines(BASE_LINES, 0xF1B1 + 5 + rank))
    if wl == "l2m":
        import random
        rng = random.Random(0xF1B1 + 4 + rank)
        colors = [b"red", b"green", b"blue", b"cyan", b"black", b"white", b"pink", b"grey"]
        dirs = [b"north", b"south", b"east", b"west"]
        return b"".join(util.event(1700000000 + i, 0, [(b"duration", util.mp_str(str(rng.randint(0, 9999)).encode())),
                                                       (b"color", util.mp_str(rng.choice(colors))),
                                                       (b"direction", util.mp_str(rng.choice(dirs)))]) for i in range(BASE_LINES))
    if wl == "json":
        lines = util.json_lines(BASE_LINES, seed=0xF1B1 + 2 + rank)
    elif wl == "nginx":
        lines = util.apache_lines(BASE_LINES, seed=0xF1B1 + 3 + rank, nginx=True)
    else:
        lines = util.apache_lines(BASE_LINES, seed=0xF1B1 + 1 + rank)
    return util.chunk_from_lines(lines)


def block_offsets(block):
    """offset of every event of a block built by util.chunk_from_lines / util.event (v2 events, 0x80 metadata)"""
    import util
    return [o for o, _ in util.split_records(block)] + [len(block)]


def parser_kw(wl):
    import util
    if wl == "json":
        return dict(name="json", format="json", time_fmt="%d/%b/%Y:%H:%M:%S %z", time_key="time")
    if wl == "nginx":
        return dict(name="nginx", format="regex", regex=util.NGINX_RX, time_fmt=util.APACHE_TIME_FMT, time_key="time")
    if wl == "ml":
        return dict(name="applog", format="regex", regex=APPLOG_RX, time_fmt="%Y-%m-%d %H:%M:%S.%L", time_key="time")
    return dict(name="apache", format="regex", regex=util.APACHE_RX, time_fmt=util.APACHE_TIME_FMT, time_key="time")


def lines_for(args, wl, world=1):
    if wl == "c0":
        return 10_000
    if wl == "l2m":
        return max(BASE_LINES, args.l2m_total // world)      # 100 M records in total: strong scaling
    return args.lines


def host_cores():
    """(usable cores, note): os.cpu_count() capped by the container's CPU quota (cgroup v2 cpu.max / v1 cfs quota) --
    a quota of 16 CPUs makes 128 busy processes run at an eighth of their speed, so the reference gets one pipeline per
    core it can actually have"""
    n = os.cpu_count() or 1
    note = "%d logical CPUs" % n
    try:
        try:
            q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        except OSError:
            q = open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read().strip()
            per = open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read().strip()
        if q != "max" and int(q) > 0:
            lim = max(1, int(int(q) / float(per) + 0.5))
            if lim < n:
                note = "%d logical CPUs, CPU quota of the container %s/%s = %d" % (n, q, per, lim)
                n = lim
    except Exception:
        pass
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    return n, note


# ------------------------------------------------------------------ reference arm
_REF_STATE = {}
_BLOCKS = {}


def _ref_state(wl):
    import util
    st = _REF_STATE.get(wl)
    if st is None and wl == "textpath":
        ref = util.Ref()
        ref.parser(**parser_kw("apache"))
        for p, props in WORKLOADS["apache"]["filters"]:
            ref.filter(p, props)
        st = _REF_STATE[wl] = (ref, textpath_input())
        return st
    if st is None and wl == "tojson":
        ref = util.Ref()                              # the parsed events: the reference's own parser filter over the apache block
        ref.parser(**parser_kw("apache"))
        for p, props in WORKLOADS["c0"]["filters"]:
            ref.filter(p, props)
        ret, out = ref.chain_do(_BLOCKS.get("apache") or make_block("apache"), "bench")
        st = _REF_STATE[wl] = (util.Ref(), C.create_string_buffer(out, len(out)))
        return st
    if st is None:
        ref = util.Ref()
        if wl not in NO_PARSER:
            ref.parser(**parser_kw(wl))
        for p, props in WORKLOADS[wl]["filters"]:
            ref.filter(p, props)
        block = _BLOCKS.get(wl) or make_block(wl)
        buf = C.create_string_buffer(block, len(block))
        st = _REF_STATE[wl] = (ref, buf)
    return st


def _ref_init(workloads):
    """every pool worker: its own reference pipeline per workload and its own copy of the block, built before timing"""
    for wl in workloads:
        ref, buf = _ref_state(wl)
        cut = block_offsets_cached(wl)[200]
        out, n = C.c_void_p(), C.c_size_t()
        nrec = ref.L.flbref_count_records(C.cast(buf, C.c_void_p), cut)
        if ref.L.flbref_filter_do(ref.cfg, C.cast(buf, C.c_void_p), cut, nrec, b"bench", C.byref(out), C.byref(n)) == 1 and out.value:
            ref.L.flbref_free(out)


_OFFS = {}


def block_offsets_cached(wl):
    if wl not in _OFFS:
        _OFFS[wl] = block_offsets(_BLOCKS.get(wl) or make_block(wl))
    return _OFFS[wl]


def _ref_tojson_task(args):
    """one pool task: the reference's flb_pack_msgpack_to_json_format() over this worker's copy of the parsed events, `reps` times"""
    reps = args
    ref, buf = _ref_state("tojson")
    n = C.c_size_t()
    t0 = time.perf_counter()
    for _ in range(reps):
        p = ref.L.flbref_to_json_format(C.cast(buf, C.c_void_p), len(buf), 3, 1, b"date", 1, C.byref(n))
        if p:
            ref.L.flbref_cfree(p)
    return time.perf_counter() - t0, BASE_LINES * reps


def _ref_textpath_task(reps):
    """one pool task: line loop + flb_filter_do + flb_pack_msgpack_to_json_format of the reference over this worker's text"""
    ref, text = _ref_state("textpath")
    t0 = time.perf_counter()
    n = 0
    for _ in range(reps):
        ev, used, n = ref.lines_to_events(text, "log", True, 1700000000, 0)
        ret, out = ref.chain_do(ev, "bench")
        ref.to_json(out, 3, 1, "date", True)
    return time.perf_counter() - t0, n * reps


def _ref_task(args):
    """one pool task: the reference's flb_filter_do over the first `cut` bytes of this worker's block, `reps` times"""
    wl, cut, reps = args
    ref, buf = _ref_state(wl)
    nrec = ref.L.flbref_count_records(C.cast(buf, C.c_void_p), cut)
    t0 = time.perf_counter()
    for _ in range(reps):
        out, n = C.c_void_p(), C.c_size_t()
        r = ref.L.flbref_filter_do(ref.cfg, C.cast(buf, C.c_void_p), cut, nrec, b"bench", C.byref(out), C.byref(n))
        if r == 1 and out.value:
            ref.L.flbref_free(out)
        if wl == "nginx":
            ref.L.flbref_emit_reset(-1)          # (the harness's stand-in for the emitter keeps what it was handed: forget it)
    return time.perf_counter() - t0, nrec * reps


class RefPool:
    """All host cores, each its own reference pipeline (filters are single-threaded per pipeline in the
    reference) over its own copy of the block."""

    def __init__(self, cores, workloads):
        import multiprocessing as mp
        self.cores = cores
        for wl in workloads:                      # generated once; the forked workers inherit them
            _BLOCKS[wl] = make_block(wl)
        self.offs = {wl: block_offsets_cached(wl) for wl in workloads}
        self.pool = mp.get_context("fork").Pool(cores, initializer=_ref_init, initargs=(list(workloads),))
        self.pool.map(time.sleep, [0.01] * cores, chunksize=1)      # every worker is up (initialised) before anything is timed

    def step(self, wl, lines):
        """`lines` events spread evenly over the cores, one task each; returns (events done, seconds): the time of the
        slowest worker inside the reference's calls -- python's pool dispatch is not the reference's cost"""
        offs = self.offs[wl]
        n_tasks = self.cores
        if wl == "c0":                            # configs[0]: whole 10k-line batches, 4 per core
            per, reps = 10_000, 4
        else:
            per = max(1, min(BASE_LINES, -(-lines // n_tasks)))
            reps = max(1, -(-lines // (per * n_tasks)))
        res = self.pool.map(_ref_task, [(wl, offs[per], reps)] * n_tasks, chunksize=1)
        return sum(r[1] for r in res), max(r[0] for r in res)

    def close(self):
        self.pool.close()
        self.pool.join()


def reference_workload(pool, wl, lines, steps, warmup):
    for _ in range(max(1, warmup)):            # first touch builds each worker's pipeline and block
        pool.step(wl, min(lines, pool.cores * 2000))
    done, dt = 0, 0.0
    for _ in range(steps):
        n, wall = pool.step(wl, lines)
        done += n
        dt += wall
    return done / dt, dt / steps, done // steps


def run_reference(args):
    import util
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    if not util.have_ref():
        print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref/libflbref.so missing"}))
        return
    cores, cores_note = host_cores()
    wl = args.workload
    side = [] if args.primary_only else [o for o in ("apache", "c0", "nginx", "ml") if o != wl]
    pool = RefPool(cores, [wl] + side)
    # bounded sample: the reference does 10-50 M lines/s on 128 cores, so a full 10 M-event step is 0.2-1 s
    val, s_per_step, n = reference_workload(pool, wl, lines_for(args, wl), args.steps, args.warmup)
    others = {}
    if not args.primary_only:
        for o in side:
            v, sps, nn = reference_workload(pool, o, lines_for(args, o), max(1, min(args.steps, 3)), 1)
            others[o] = {"workload": WORKLOADS[o]["name"], "value": v, "e2e": v, "unit": "lines/s", "events_per_step": nn,
                         "ms_per_step": 1000 * sps}
    if not args.primary_only:
        try:
            pool.pool.map(_ref_tojson_task, [1] * cores, chunksize=1)                 # builds every worker's input
            res = pool.pool.map(_ref_tojson_task, [3] * cores, chunksize=1)
            v = sum(r[1] for r in res) / max(r[0] for r in res)
            others["tojson"] = {"workload": TOJSON_NAME, "value": v, "e2e": v, "unit": "lines/s", "events_per_step": sum(r[1] for r in res)}
        except Exception as ex:
            others["tojson"] = {"workload": TOJSON_NAME, "error": "%s: %s" % (type(ex).__name__, ex)}
        try:
            pool.pool.map(_ref_textpath_task, [1] * cores, chunksize=1)
            res = pool.pool.map(_ref_textpath_task, [2] * cores, chunksize=1)
            v = sum(r[1] for r in res) / max(r[0] for r in res)
            others["textpath"] = {"workload": TEXTPATH_NAME, "value": v, "e2e": v, "unit": "lines/s", "events_per_step": sum(r[1] for r in res),
                                  "note": "the line loop restated in the harness around the reference's encoder; python ctypes wrappers on this side too"}
        except Exception as ex:
            others["textpath"] = {"workload": TEXTPATH_NAME, "error": "%s: %s" % (type(ex).__name__, ex)}
    pool.close()
    sample = "%d cores (%s), %d events per step in %d-event calls, one pipeline per core, %d steps; time = slowest worker inside the reference's calls" % (
        cores, cores_note, n, min(BASE_LINES, -(-n // cores)), args.steps)
    line = {
        "impl": "reference", "metric": "log lines/sec through parser+filter chain", "value": val, "unit": "lines/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000 * s_per_step,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": WORKLOADS[wl]["name"], "events_per_gpu_per_step": lines_for(args, wl), "distinct_lines": BASE_LINES},
        "host": cores_note,
        "cpu_baseline": {"value": val, "unit": "lines/s", "cores": cores, "kind": "reference", "sample": sample},
        "e2e": {"value": val, "unit": "lines/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    if "apache" in others:
        line["north_star"] = others.pop("apache")
    line["workloads"] = others
    print(json.dumps(line))


# ------------------------------------------------------------------------ our arm
class ClockSampler(threading.Thread):
    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.proc = index, [], None

    def run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap,power.limit")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, text=True)
            for line in self.proc.stdout:
                self.rows.append([x.strip() for x in line.split(",")])
        except Exception:
            pass

    def stop(self):
        if self.proc:
            self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 3 + i and r[3 + i].lower().startswith("active") for r in self.rows)]
        lim = [float(r[7]) for r in self.rows if len(r) > 7 and r[7].replace(".", "").isdigit()]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons,
                "power_limit_w": lim[-1] if lim else None, "samples": len(sm)}


_libc = C.CDLL(None)
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.free.argtypes = [C.c_void_p]
_libc.mallopt.argtypes = [C.c_int, C.c_int]


def tune_malloc():
    """Host allocator policy of an embedding process that keeps freed result buffers in its heap instead of returning them
    to the kernel (no mmap for big blocks, no trimming) -- what Fluent Bit's default jemalloc build does with its retained
    extents.  glibc cannot be switched back afterwards, so this variant is measured last."""
    _libc.mallopt(-4, 0)              # M_MMAP_MAX = 0
    _libc.mallopt(-1, (1 << 31) - 1)  # M_TRIM_THRESHOLD
    _libc.mallopt(-2, 64 << 20)       # M_TOP_PAD


class Workload:
    """one workload on this rank's GPU: chain, host buffers (pageable + pinned), device buffers"""

    def __init__(self, args, wl, L, ctx, rank, world):
        import util
        self.pkg = util.pkg
        self.args, self.wl, self.L, self.ctx, self.rank, self.world = args, wl, L, ctx, rank, world
        if wl not in NO_PARSER:
            kw = parser_kw(wl)
            made = ctx.__dict__.setdefault("_bench_parsers", set())
            if kw["name"] not in made:
                ctx.parser(**kw)
                made.add(kw["name"])
        self.filters = [ctx.filter(p, props) for p, props in WORKLOADS[wl]["filters"]]
        self.chain = ctx.chain(self.filters)
        self.block = make_block(wl, rank)
        self.offs = block_offsets(self.block)
        self.n_lines = lines_for(args, wl, world)
        reps, rem = divmod(self.n_lines, BASE_LINES)
        self.nbytes = len(self.block) * reps + self.offs[rem]
        self.h_page = _libc.malloc(self.nbytes)                 # what Fluent Bit hands a filter: ordinary heap memory
        self.h_pin = None
        for i in range(reps):
            C.memmove(self.h_page + i * len(self.block), self.block, len(self.block))
        if rem:
            C.memmove(self.h_page + reps * len(self.block), self.block, self.offs[rem])
        self.d_in = self.d_out = None
        self.osz = C.c_size_t()
        self.out_p = C.c_void_p()
        # one call takes less than 4 GiB: a bigger batch is a sequence of calls over whole blocks
        seg_blocks = max(1, (2 << 30) // len(self.block))
        self.segs, pos = [], 0
        while pos < self.nbytes:
            n = min(self.nbytes - pos, seg_blocks * len(self.block))
            self.segs.append((pos, n))
            pos += n

    def close(self):
        L, ctx = self.L, self.ctx
        if self.d_in:
            L.flbgpu_dev_free(ctx.h, self.d_in); L.flbgpu_dev_free(ctx.h, self.d_out)
        if self.h_pin:
            L.flbgpu_host_free(ctx.h, self.h_pin)
        _libc.free(self.h_page)
        self.chain.close()

    def exchange(self):
        if self.wl == "l2m" and self.world > 1:
            self.filters[0].l2m_allreduce_lib()      # the one exchange of the path: flbgpu_l2m_allreduce(), NCCL inside the library
            self.L.flbgpu_l2m_reset(self.filters[0].h)    # "flushed": the next interval starts from zero

    # ---- device-resident
    def device_setup(self):
        L, ctx = self.L, self.ctx
        self.d_in = L.flbgpu_dev_alloc(ctx.h, self.nbytes + 64)
        self.out_cap = (self.segs[0][1] + self.segs[0][1] // 2 + 4096 + 4095) & ~4095
        self.d_out = L.flbgpu_dev_alloc(ctx.h, self.out_cap * len(self.segs))     # one result range per call of a step
        assert self.d_in and self.d_out, "device allocation failed"
        L.flbgpu_dev_upload(ctx.h, self.d_in, self.h_page, self.nbytes)

    def step_device(self):
        self.out_sizes = []
        for k, (off, n) in enumerate(self.segs):
            r = self.L.flbgpu_chain_do_device(self.chain.h, self.d_in + off, n, self.d_out + k * self.out_cap, self.out_cap, C.byref(self.osz))
            if r != self.pkg.FILTER_MODIFIED:
                raise RuntimeError("chain_do_device -> %d: %s" % (r, self.ctx.err()))
            self.out_sizes.append(self.osz.value)
        self.out_total = sum(self.out_sizes)
        self.exchange()

    def device_result(self):
        """the chunk the last step_device() returned: its calls' results, in order"""
        buf = C.create_string_buffer(max(1, self.out_total))
        at = 0
        for k, n in enumerate(self.out_sizes):
            if n and self.L.flbgpu_dev_download(self.ctx.h, C.byref(buf, at), self.d_out + k * self.out_cap, n) != 0:
                raise RuntimeError("dev_download: %s" % self.ctx.err())
            at += n
        return buf.raw[:self.out_total]

    # ---- host buffers through the C ABI
    def call(self, chain, ptr, n):
        out, osz = C.c_void_p(), C.c_size_t()
        r = self.L.flbgpu_chain_do(chain.h, ptr, n, b"bench", 5, C.byref(out), C.byref(osz))
        if r < 0:
            raise RuntimeError("chain_do -> %d: %s" % (r, self.ctx.err()))
        if out.value and out.value != getattr(self, "keep", None):
            _libc.free(out)
        return osz.value

    def step_host(self, pinned=False):
        src = self.h_page
        if pinned:
            if not self.h_pin:
                self.h_pin = self.L.flbgpu_host_alloc(self.ctx.h, self.nbytes)
                C.memmove(self.h_pin, self.h_page, self.nbytes)
            src = self.h_pin
        out = sum(self.call(self.chain, src + off, n) for off, n in self.segs)
        self.exchange()
        return out

    def batches(self, bytes_per_call, limit_bytes):
        """[(offset, length)] of consecutive calls of about bytes_per_call, cut at event boundaries"""
        import bisect
        out, pos, blen = [], 0, len(self.block)
        end = min(self.nbytes, limit_bytes)
        while pos < end:
            base, rel = divmod(pos, blen)
            want = pos + bytes_per_call
            if want >= self.nbytes:
                nxt = self.nbytes
            else:
                b2, r2 = divmod(want, blen)
                k = bisect.bisect_right(self.offs, r2) - 1
                nxt = b2 * blen + self.offs[k]
                if nxt <= pos:
                    nxt = b2 * blen + self.offs[min(k + 1, len(self.offs) - 1)]
            out.append((pos, nxt - pos))
            pos = nxt
        return out


DUMP_WINDOW = 4096          # bytes per sampled window of the result
DUMP_WINDOWS = 256
DUMP_BLOCK = 65536          # bytes per checksum block


def dump_outputs(directory, result, out_sizes):
    """What the timed device-resident step returned, as float arrays (at most a few MB for any batch size):
      result_sizes.npy ....... float64, bytes returned by each call of the step
      result_checksums.npy ... float64 [blocks, 2], per 64 KiB block of the result: sum of the bytes, and sum of
                               byte * (position in the block + 1) -- both exact in float64; every byte counts
      result_sample.npy ...... float32, the byte values of 256 windows of 4 KiB at fixed offsets (seeded), or the whole
                               result when it is smaller than that"""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    b = np.frombuffer(result, dtype=np.uint8)
    np.save(os.path.join(directory, "result_sizes.npy"), np.asarray(out_sizes, dtype=np.float64))
    pad = np.zeros(-len(b) % DUMP_BLOCK, dtype=np.uint8)
    blocks = np.concatenate([b, pad]).reshape(-1, DUMP_BLOCK).astype(np.float64)
    weights = np.arange(1, DUMP_BLOCK + 1, dtype=np.float64)
    np.save(os.path.join(directory, "result_checksums.npy"), np.stack([blocks.sum(axis=1), blocks @ weights], axis=1))
    if len(b) <= DUMP_WINDOW * DUMP_WINDOWS:
        sample = b
    else:
        starts = np.sort(np.random.default_rng(0xF1B1).choice(len(b) - DUMP_WINDOW, DUMP_WINDOWS, replace=False))
        sample = np.concatenate([b[s:s + DUMP_WINDOW] for s in starts])
    np.save(os.path.join(directory, "result_sample.npy"), sample.astype(np.float32))


def timed(fn, barrier):
    barrier()
    t0 = time.perf_counter()
    fn()
    barrier()
    return time.perf_counter() - t0


def measure(args, wl, L, ctx, torch, dist, rank, world, local, full=True, dump=None):
    """value / e2e / kernel times of one workload on this rank's GPU; dump: directory for the last timed step's result"""
    w = Workload(args, wl, L, ctx, rank, world)
    n_lines, nbytes = w.n_lines, w.nbytes
    steps = args.steps

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def allmax(x):
        t = torch.tensor([x], device="cuda", dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # ---- device-resident: CUDA events on the instance's stream
    w.device_setup()
    stream = torch.cuda.ExternalStream(w.chain.stream(), device=torch.device("cuda", local))
    for _ in range(args.warmup):
        w.step_device()
    st0 = w.chain.stats()
    sampler = ClockSampler(local)
    sampler.start()
    time.sleep(0.3)
    kms = [0.0, 0.0, 0.0]
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    ev0.record(stream)
    ms3 = (C.c_float * 3)()
    for _ in range(steps):
        w.step_device()
        L.flbgpu_kernel_ms(ctx.h, ms3)
        for k in range(3):
            kms[k] += ms3[k]
    ev1.record(stream)
    barrier()
    dev_ms = allmax(ev0.elapsed_time(ev1))
    clocks = sampler.stop()
    if dump:
        dump_outputs(dump, w.device_result(), w.out_sizes)
    st1 = w.chain.stats()
    launches = int(st1.kernel_launches - st0.kernel_launches)
    out_bytes = w.out_total
    value = world * n_lines * steps / (dev_ms / 1000.0)

    # ---- end to end, the way flb_filter_do() calls: pageable input, glibc's untouched malloc, result freed
    w.step_host()
    e2e_s = allmax(timed(lambda: [w.step_host() for _ in range(steps)], barrier))
    e2e = world * n_lines * steps / e2e_s
    phases = [round(float(x), 2) for x in w.chain.stats().phase_ms]
    variants = {}
    if full:
        # the same calls with the result written into a buffer the caller keeps (flbgpu_chain_set_result_buffer): no fresh pages
        # per call; an ordinary reused heap buffer, then a pinned one
        try:
            if world > 1:
                raise RuntimeError("single-GPU runs only")      # (a failure on one rank between collectives would stall the others)
            cap = int(out_bytes * 1.05) + (1 << 20)
            for name, alloc, release in (("reused_heap_buffer", lambda n: _libc.malloc(n), lambda p: _libc.free(p)),
                                         ("reused_pinned_buffer", lambda n: L.flbgpu_host_alloc(ctx.h, n), lambda p: L.flbgpu_host_free(ctx.h, p))):
                rb = alloc(cap)
                if not rb:
                    continue
                L.flbgpu_chain_set_result_buffer(w.chain.h, rb, cap)
                w.keep = rb
                w.step_host()
                s = allmax(timed(lambda: [w.step_host() for _ in range(steps)], barrier))
                variants[name] = {"value": world * n_lines * steps / s, "unit": "lines/s",
                                  "note": "pageable input; the result goes into a buffer of the caller registered with flbgpu_chain_set_result_buffer()"}
                L.flbgpu_chain_set_result_buffer(w.chain.h, None, 0)
                w.keep = None
                release(rb)
        except Exception as ex:
            if world == 1:
                variants["reused_result_buffer_error"] = "%s: %s" % (type(ex).__name__, ex)
            w.keep = None
        w.step_host(pinned=True)
        s = allmax(timed(lambda: [w.step_host(pinned=True) for _ in range(steps)], barrier))
        variants["pinned_input"] = {"value": world * n_lines * steps / s, "unit": "lines/s", "note": "input in cudaMallocHost memory, glibc's untouched malloc"}
        # batch sweep: bytes per flbgpu_chain_do() call, pageable input, default malloc; 1 caller and 8 callers
        sweep = []
        ncall = 8
        extra = [ctx.chain([ctx.filter(p, props) for p, props in WORKLOADS[wl]["filters"]]) for _ in range(ncall - 1)]
        chains = [w.chain] + extra
        for bpc, limit in ((64 << 10, 96 << 20), (2 << 20, 512 << 20), (64 << 20, 1 << 40)):
            if bpc >= nbytes:
                continue
            bl = w.batches(bpc, limit)
            ev_per_byte = n_lines / float(nbytes)
            for callers in (1, ncall):
                def run_part(t, callers=callers, bl=bl):
                    for i in range(t, len(bl), callers):
                        w.call(chains[t], w.h_page + bl[i][0], bl[i][1])

                def run_all(callers=callers):
                    if callers == 1:
                        run_part(0)
                    else:
                        th = [threading.Thread(target=run_part, args=(t,)) for t in range(callers)]
                        for x in th:
                            x.start()
                        for x in th:
                            x.join()
                run_all()                                   # warm: buffers of every instance grown
                s = allmax(timed(run_all, barrier))
                done = sum(b[1] for b in bl)
                sweep.append({"bytes_per_call": bpc, "callers": callers, "calls": len(bl), "lines_per_s": world * done * ev_per_byte / s,
                              "us_per_call": 1e6 * s * callers / len(bl),
                              "GB_per_s_in": world * done / s / 1e9})
        sweep.append({"bytes_per_call": nbytes, "callers": 1, "calls": 1, "lines_per_s": e2e, "us_per_call": 1e6 * e2e_s / steps,
                      "GB_per_s_in": world * nbytes * steps / e2e_s / 1e9})
        variants["batch_sweep"] = sweep
        for c in extra:
            c.close()
    w.close()
    return {"value": value, "dev_ms": dev_ms, "e2e": e2e, "e2e_steps": steps, "kms": [k / steps for k in kms],
            "launches": launches, "n_lines": n_lines, "nbytes": nbytes, "out_bytes": out_bytes, "clocks": clocks,
            "phases": phases, "variants": variants, "steps": steps}


TOJSON_NAME = ("output side: the parsed apache events of configs[0] as json_lines text -- flb_pack_msgpack_to_json_format(date_key "
               "'date', iso8601, escape_unicode on), what out_stdout / out_http call on the chunk they flush")


def tojson_input(ctx):
    """the events the apache parser makes of the block (our own chain; byte-identical to the reference's by the parity tests)"""
    import util
    made = ctx.__dict__.setdefault("_bench_parsers", set())
    if "apache" not in made:
        ctx.parser(**parser_kw("apache"))
        made.add("apache")
    ch = ctx.chain([ctx.filter(p, props) for p, props in WORKLOADS["c0"]["filters"]])
    ret, out = ch.do(make_block("apache"))
    ch.close()
    assert ret == util.pkg.FILTER_MODIFIED and out
    return out


def measure_tojson(args, L, ctx, torch, world):
    """end to end only (host chunk in, malloc()ed text out): lines/s over `reps` calls on a 100 k-event chunk"""
    chunk = tojson_input(ctx)
    n_ev = BASE_LINES
    buf = C.create_string_buffer(chunk, len(chunk))
    out, n, und = C.c_void_p(), C.c_size_t(), C.c_size_t()
    ms3 = (C.c_float * 3)()

    def call():
        r = L.flbgpu_msgpack_to_json_format(ctx.h, C.cast(buf, C.c_void_p), len(chunk), 3, 1, b"date", 1, C.byref(out), C.byref(n), C.byref(und))
        if r != 0:
            raise RuntimeError("msgpack_to_json_format -> %d: %s" % (r, ctx.err()))
        _libc.free(out)
        return n.value
    for _ in range(max(3, args.warmup)):
        text_bytes = call()
    reps = args.steps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    kms = [0.0, 0.0, 0.0]
    for _ in range(reps):
        call()
        L.flbgpu_kernel_ms(ctx.h, ms3)
        for k in range(3):
            kms[k] += ms3[k]
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    kern = (kms[1] + kms[2]) / reps
    return {"workload": TOJSON_NAME, "e2e": world * n_ev * reps / dt, "unit": "lines/s", "events_per_call": n_ev, "input_bytes_per_call": len(chunk),
            "text_bytes_per_call": text_bytes, "calls": reps, "ms_per_call": 1000 * dt / reps,
            "kernel_ms_per_call": {"index": kms[0] / reps, "size": kms[1] / reps, "emit": kms[2] / reps},
            "value": (n_ev / (kern / 1000.0)) if kern > 0 else None,
            "value_note": "events / (sizing + emission kernel time): the conversion kernels alone, input resident",
            "gpu_launches_per_call": 2, "undefined_strings": und.value}


TEXTPATH_NAME = ("text in, text out: apache access log text -> in_tail's line loop (events) -> filter_parser(apache) + filter_grep(method) + "
                 "filter_modify -> json_lines text; three library calls per 100 k-line buffer, host memory on both ends")


def textpath_input():
    import util
    return b"\n".join(util.apache_lines(BASE_LINES, seed=0xF1B1 + 1)) + b"\n"


def measure_textpath(args, L, ctx, torch, world):
    """the whole path around the filters through the C ABI: flbgpu_lines_to_events + flbgpu_chain_do + flbgpu_msgpack_to_json_format"""
    import util
    text = textpath_input()
    made = ctx.__dict__.setdefault("_bench_parsers", set())
    if "apache" not in made:
        ctx.parser(**parser_kw("apache"))
        made.add("apache")
    ch = ctx.chain([ctx.filter(p, props) for p, props in WORKLOADS["apache"]["filters"]])

    def call():
        ev, used, n = ctx.lines_to_events(text, "log", True, 1700000000, 0)
        ret, out = ch.do(ev, tag="bench")
        js, und = ctx.to_json(out, 3, 1, "date", True)
        return n, len(js)
    for _ in range(max(3, args.warmup)):
        n, nbytes = call()
    reps = args.steps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        call()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    ch.close()
    return {"workload": TEXTPATH_NAME, "e2e": world * n * reps / dt, "unit": "lines/s", "lines_per_call": n, "text_in_bytes": len(text),
            "text_out_bytes": nbytes, "calls": reps, "ms_per_call": 1000 * dt / reps,
            "note": "python ctypes wrappers copy every buffer once more than a C caller would"}


def run_ours(args):
    import torch
    import torch.distributed as dist
    import util
    pkg = util.pkg
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    L = pkg.load()                                  # raises if the CUDA library is missing
    ctx = pkg.Context(local, lib=L)
    if world > 1:
        # the library's own communicator for the metric-table exchange: rank 0 makes the id, torch.distributed (the
        # embedding process's control channel) carries the 128 bytes
        box = [ctx.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        ctx.comm_init(world, rank, box[0])
    WL = args.workload
    m = measure(args, WL, L, ctx, torch, dist, rank, world, local, full=True,
                dump=(args.dump_outputs if world == 1 else os.path.join(args.dump_outputs, "rank%d" % rank)) if args.dump_outputs else None)
    others = {}
    if not args.primary_only:
        for o in ("apache", "c0", "nginx", "l2m", "ml"):
            if o == WL:
                continue
            try:
                others[o] = measure(args, o, L, ctx, torch, dist, rank, world, local, full=(o == "apache"))
            except Exception as ex:                       # a side workload never costs the line its primary numbers
                if o == "apache":
                    raise
                others[o] = {"error": "%s: %s" % (type(ex).__name__, ex)}

    tojson = None
    if not args.primary_only:
        try:
            tojson = measure_tojson(args, L, ctx, torch, world)
        except Exception as ex:
            tojson = {"workload": TOJSON_NAME, "error": "%s: %s" % (type(ex).__name__, ex)}

    textpath = None
    if not args.primary_only:
        try:
            textpath = measure_textpath(args, L, ctx, torch, world)
        except Exception as ex:
            textpath = {"workload": TEXTPATH_NAME, "error": "%s: %s" % (type(ex).__name__, ex)}

    # last: the same end-to-end calls with an allocator that retains freed result buffers (and pinned input)
    tune_malloc()
    retained = {}
    retained_error = None
    try:
        for o in ([WL] if args.primary_only else [WL, "apache"]):
            if o in retained:
                continue
            w = Workload(args, o, L, ctx, rank, world)
            for pinned in (False, True):
                w.step_host(pinned=pinned)
                t0 = time.perf_counter()
                torch.cuda.synchronize()
                for _ in range(args.steps):
                    w.step_host(pinned=pinned)
                torch.cuda.synchronize()
                dt = torch.tensor([time.perf_counter() - t0], device="cuda", dtype=torch.float64)
                if world > 1:
                    dist.all_reduce(dt, op=dist.ReduceOp.MAX)
                retained.setdefault(o, {})["pinned_input" if pinned else "pageable_input"] = world * w.n_lines * args.steps / float(dt.item())
            w.close()
    except Exception as ex:                           # (a device fault inside a side workload above is sticky: keep the line)
        if world > 1:
            raise
        retained_error = "%s: %s" % (type(ex).__name__, ex)
        retained = {}
    for o, v in retained.items():
        tgt = m if o == WL else others.get(o)
        if tgt is not None:
            tgt["variants"]["retaining_malloc"] = dict(v, unit="lines/s", note="glibc tuned to retain freed result buffers (M_MMAP_MAX=0, M_TRIM_THRESHOLD=2GiB): what a jemalloc build of the agent does")

    if retained_error:
        m["variants"]["retaining_malloc"] = {"error": retained_error}
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 3350.0))           # H100 SXM data sheet: 3.35 TB/s of HBM3
    props = torch.cuda.get_device_properties(local)

    def roof(mm):
        eval_ms = mm["kms"][1]
        alg = mm["nbytes"] + mm["out_bytes"]
        ach = alg / (eval_ms / 1000.0) / 1e9 if eval_ms > 0 else None
        return eval_ms, alg, ach

    eval_ms, alg_bytes, achieved = roof(m)

    cpu = None
    if util.have_ref():
        cores, cores_note = host_cores()
        pool = RefPool(cores, [WL])
        sample_lines = min(m["n_lines"], 4_000_000)
        v, sps, n = reference_workload(pool, WL, sample_lines, 2, 1)
        pool.close()
        cpu = {"value": v, "unit": "lines/s", "cores": cores, "kind": "reference",
               "sample": "%d cores (%s), 2 steps of %d events in %d-event calls, one pipeline per core (%.2f s per step: slowest worker inside the reference's calls)" % (cores, cores_note, n, min(BASE_LINES, -(-n // cores)), sps)}

    def side(mm, name):
        if "error" in mm:
            return {"workload": WORKLOADS[name]["name"], "error": mm["error"]}
        e2, a2, ach2 = roof(mm)
        d = {"workload": WORKLOADS[name]["name"], "value": mm["value"], "e2e": mm["e2e"], "unit": "lines/s",
             "events_per_gpu_per_step": mm["n_lines"], "input_bytes_per_gpu": mm["nbytes"], "output_bytes_per_gpu": mm["out_bytes"],
             "steps": mm["steps"], "ms_per_step": mm["dev_ms"] / mm["steps"],
             "kernel_ms_per_step": {"index": mm["kms"][0], "evaluate": e2, "emit": mm["kms"][2]},
             "roofline_frac": (ach2 / peak) if ach2 else None, "gpu_launches": mm["launches"]}
        if mm["variants"]:
            d["e2e_variants"] = mm["variants"]
        if name == "l2m":
            d["scaling"] = "strong"
            d["collective"] = "flbgpu_l2m_allreduce(): the library's own NCCL exchange of the metric tables, every step" if world > 1 else "single GPU: no exchange"
        return d

    line = {
        "metric": "log lines/sec through parser+filter chain", "value": m["value"], "unit": "lines/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": m["dev_ms"] / m["steps"], "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": WORKLOADS[WL]["name"], "events_per_gpu_per_step": m["n_lines"], "distinct_lines": BASE_LINES},
        "config_detail": {"input_bytes_per_gpu": m["nbytes"], "output_bytes_per_gpu": m["out_bytes"],
                          "l2": "input %.0f MB, L2 of the %s %.0f MB" % (m["nbytes"] / 1e6, props.name, props.L2_cache_size / 1e6),
                          "parallelism": ("record shards; one NCCL all-reduce of the metric table per step" if WL == "l2m" else "record shards, no data-path collective"),
                          "e2e_input": "pageable malloc()ed memory", "e2e_host_malloc": "glibc, untouched"},
        "e2e": {"value": m["e2e"], "unit": "lines/s", "h2d_bytes_per_step": m["nbytes"], "d2h_bytes_per_step": m["out_bytes"],
                "steps": m["e2e_steps"], "timing": "wall clock between device-synchronising barriers",
                "host_phase_ms_last_call": dict(zip(["upload+index+evaluate", "size_scan", "emit+download", "total"], m["phases"]))},
        "e2e_variants": m["variants"],
        "gpu_launches": m["launches"],
        "kernel_ms_per_step": {"index": m["kms"][0], "evaluate": eval_ms, "emit": m["kms"][2],
                               "note": "CUDA-event pairs per launch group; index runs on its own priority stream concurrently with evaluate, so the groups are not additive"},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                     "frac": (achieved / peak) if achieved else None,
                     "kernel": "k_chain_eval (evaluation pass)", "algorithmic_bytes_per_launch": alg_bytes,
                     "peak_source": "MEASURED_PEAKS.json hbm_gbs" if peaks else "H100 SXM data sheet, 3350 GB/s"},
        "cpu_baseline": cpu,
        "clocks": m["clocks"],
        "device": props.name,
    }
    if "apache" in others:
        line["north_star"] = side(others.pop("apache"), "apache")
    line["workloads"] = {k: side(v, k) for k, v in others.items()}
    if tojson is not None:
        line["workloads"]["tojson"] = tojson
    if textpath is not None:
        line["workloads"]["textpath"] = textpath
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def main():
    # whatever NCCL has to say (a version banner under NCCL_DEBUG=VERSION, its INFO log) goes to stderr: stdout carries the one JSON line
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--lines", type=int, default=10_000_000, help="events per GPU per step")
    ap.add_argument("--l2m-total", type=int, default=100_000_000, help="records of configs[3] over all GPUs")
    ap.add_argument("--workload", default="json", choices=list(WORKLOADS), help="primary workload (the others are reported beside it)")
    ap.add_argument("--primary-only", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the result of the last timed device-resident step as .npy files")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
