"""f2: filter_multiline in parser mode with `buffer off` (plugins/filter_multiline/ml.c:833-892, src/multiline/flb_ml.c,
flb_ml_rule.c) against the reference's own plugin, chunk after chunk on one filter instance (the rule a group is in and its
time survive from call to call)."""
import random

import pytest

import test_shim
import util

pkg = util.pkg
S = util.mp_str

EXC = [("start_state", r"/(Dec \d+ \d+\:\d+\:\d+)(.*)/", "cont"), ("cont", r"/^\s+at.*/", "cont")]        # conf/parsers_multiline.conf
# a rule whose to_state is a start state flushes right after it matched (try_flushing_buffer); a start rule that also
# continues; an empty-matching start rule; rules sharing a from_state (first in list order wins)
ODD = [("start_state, more", r"/^A/", "more"), ("more", r"/^b/", "more"), ("more", r"/^c/", "start_state"), ("more", r"/^b2/", "more")]
EMPTY = [("start_state", r"/^(S.*)?$/", "c1"), ("c1", r"/^$/", "c1"), ("c1", r"/^ +\S/", "c1")]
RULESETS = {"exc": EXC, "odd": ODD, "empty": EMPTY}

VOCAB = {
    "exc": [b"Dec 14 06:41:08 Exception in thread main", b"Dec 15 01:01:01 again\n", b"    at foo(Foo.java:1)", b"  at x\n", b"\tat tab",
            b"plain line", b"", b"    at orphan", b" ", b"Dec 1 1:1:1"],
    "odd": [b"A start", b"b cont", b"c close", b"b2 never", b"x", b"", b"A", b"b\n", b"cA"],
    "empty": [b"S one", b"", b"  indented", b"S", b"other", b" x\n", b"\n"],
}


# metadata maps of the lines: members repeat across lines (the message keeps the first of each), a bin (it comes out as hex
# text), a nested value, two members that are the same to the reference's flattened hash ("a" + "bc" and "ab" + "c"), a
# duplicate inside one map, values that differ only in type
METAS = [b"\x81" + S(b"src") + S(b"tail"), b"\x82" + S(b"src") + S(b"tail") + S(b"n") + b"\x05", b"\x81" + S(b"n") + b"\x06",
         b"\x81" + S(b"b") + b"\xc4\x03\x00\xab\xff", b"\x81" + S(b"nest") + b"\x82" + S(b"k") + b"\x92\x01\xc0" + S(b"z") + b"\xc3",
         b"\x81" + S(b"a") + S(b"bc"), b"\x81" + S(b"ab") + S(b"c"), b"\x82" + S(b"d") + b"\x01" + S(b"d") + b"\x01",
         b"\x81" + S(b"f") + b"\xcb\x3f\xf0\x00\x00\x00\x00\x00\x00", b"\x81" + S(b"f") + b"\xca\x3f\x80\x00\x00", b"\x80",
         b"\x81" + S(b"e") + b"\xd4\x05\x09", b"\x81" + b"\x07" + S(b"int key")]


def make_chunk(rng, vocab, n, t0, key=b"log", with_meta=0.0):
    evs = []
    for i in range(n):
        r = rng.random()
        line = rng.choice(vocab)
        if r < 0.04:
            fields = [(b"other", S(line))]                                   # no key_content at all
        elif r < 0.08:
            fields = [(key, bytes([rng.randint(0, 100)]))]                   # key_content is not a string
        elif r < 0.12:
            fields = [(key, bytes([7])), (key, S(line)), (b"z", b"\xc3")]    # the first STR key WITH a STR value counts
        elif r < 0.16:
            fields = [(b"a", S(b"x" * rng.randint(0, 40))), (key, S(line)), (key, S(b"second")), (b"n", b"\xcd\x01\x00")]   # duplicate key
        elif r < 0.20:
            fields = [(b"stream", S(b"stdout")), (key, b"\xd9" + bytes([len(line)]) + line), (b"m", b"\x81\xa1k\xcc\x05")]   # str8 spelling, nested map
        else:
            fields = [(key, S(line))]
        if rng.random() < 0.03:
            evs.append(b"\x92\x92\xd7\x00\xff\xff\xff\xff\x00\x00\x00\x00\x80\x80")     # a group marker: the decoder steps over it
        if rng.random() < 0.03:
            evs.append(b"\x92\xce" + (t0 + i).to_bytes(4, "big") + util.mp_map_hdr(1) + S(key) + S(line))     # legacy [ts, body]
        else:
            meta = b"\x80"
            if with_meta and rng.random() < with_meta:
                meta = rng.choice(METAS)
            evs.append(util.event(t0 + i, (i * 7) % 1000, fields, meta=meta))
    return b"".join(evs)


def diff(lib, rules, props, chunks, name="p", **kw):
    ref = util.Ref()
    ctx = pkg.Context(0, lib=lib)
    if rules is not None:
        ref.ml_parser(name, rules=rules, **kw)
        ctx.ml_parser(name, rules=rules, **kw)
    rf = ref.filter("multiline", props)
    ch = ctx.chain([ctx.filter("multiline", props)])
    for i, c in enumerate(chunks):
        want, got = ref.filter_cb(rf, c), ch.do(c)
        if want != got:
            w = [want[1][o:o + l] for o, l in util.split_records(want[1] or b"")]
            g = [got[1][o:o + l] for o, l in util.split_records(got[1] or b"")]
            k = next((k for k in range(max(len(w), len(g))) if (w[k:k + 1] != g[k:k + 1])), -1)
            raise AssertionError("chunk %d: ret %s / %s, %d / %d events, first difference at event %d:\n want %r\n got  %r" %
                                 (i, want[0], got[0], len(w), len(g), k, w[k:k + 1], g[k:k + 1]))


def _regex_rulesets(lib, rounds, n):
    rng = random.Random(11)
    for name, rules in RULESETS.items():
        for key in ("log", "message"):
            props = [("multiline.parser", name), ("multiline.key_content", key), ("buffer", "off")]
            for _ in range(rounds):
                wm = rng.choice([0.0, 0.0, 0.3, 1.0])
                chunks = [make_chunk(rng, VOCAB[name], rng.choice([1, 2, 7, n]), 1700000000 + 1000 * k, key.encode(), with_meta=wm) for k in range(4)]
                diff(lib, rules, props, chunks, name=name)


def _match_types(lib):
    rng = random.Random(12)
    vocab = [b"one, ", b"two, ", b"three\n", b"\n", b"", b"end", b"x end", b"nd", b"three\n\n"]
    for typ, ms in (("endswith", "\n"), ("endswith", "end"), ("equal", "end"), ("eq", "\n")):
        for neg in (False, True):
            props = [("multiline.parser", "m"), ("multiline.key_content", "log"), ("buffer", "off")]
            chunks = [make_chunk(rng, vocab, 60, 1700000000 + 1000 * k, with_meta=0.4 * (k % 2)) for k in range(3)]
            diff(lib, [], props, chunks, name="m", type=typ, match_string=ms, negate=neg)


JAVA = b"""2023-01-01 12:00:00 ERROR request failed
java.lang.RuntimeException: outer problem
\tat com.example.App.run(App.java:10)
\tat com.example.App.main(App.java:5)
Caused by: java.lang.IllegalStateException: inner
\tat com.example.Svc.call(Svc.java:99)
\t... 2 more
2023-01-01 12:00:01 INFO next request
Exception in thread "main" java.lang.Error: boom
    at a.b.C.d(C.java:1)
 nested exception is:
org.x.Y: why
    at q.r(S.java:2)

--- End of stack trace from previous location where exception was thrown ---
Suppressed: z.Q: s
    at eval at foo
done""".split(b"\n")
GO = b"""starting
panic: runtime error: index out of range

goroutine 1 [running]:
main.main()
\t/tmp/x.go:8 +0x1d
created by main.start
\t/tmp/x.go:3 +0x11
exit status 2
2023/01/01 http: panic serving 10.0.0.1:5: oops
goroutine 7 [running]:
net/http.(*conn).serve.func1(0xc0)
\t/usr/lib/go/src/net/http/server.go:1 +0x1
[signal SIGSEGV: segmentation violation]
ok""".split(b"\n")
PY = b"""INFO start
Traceback (most recent call last):
  File "/app/main.py", line 3, in <module>
    run()
  File "/app/main.py", line 1, in run
    raise ValueError("bad")
ValueError: bad
INFO after
Traceback (most recent call last):
  File "x.py", line 1
mod.sub.Err: nope
tail""".split(b"\n")
RUBY = b"""I, [2023] INFO -- : ok
/app/lib/a.rb:12:in `foo': undefined method (NoMethodError)
\tfrom /app/lib/b.rb:3:in `bar'
\tfrom /app/bin/run:1:in `<main>'
next line
x.rb:1:in `y'
  from z.rb:2:in `w'""".split(b"\n")


def _builtins(lib):
    rng = random.Random(13)
    for name, text in (("java", JAVA), ("go", GO), ("python", PY), ("ruby", RUBY)):
        props = [("multiline.parser", name), ("multiline.key_content", "log"), ("buffer", "off")]
        lines = list(text) * 3
        cut = rng.randint(3, len(lines) - 3)
        diff(lib, None, props, [util.chunk_from_lines(lines[:cut]), util.chunk_from_lines(lines[cut:], t0=1700001000),
                                make_chunk(rng, list(text), 50, 1700002000)])
        # no multiline.key_content and none in the parser: every record passes through on its own, re-encoded
        diff(lib, None, [("multiline.parser", name), ("buffer", "off")], [util.chunk_from_lines(lines[:20])])


def _refusals(lib):
    ctx = pkg.Context(0, lib=lib)
    ctx.ml_parser("exc", rules=EXC)
    for bad in ([("multiline.parser", "exc"), ("multiline.key_content", "log")],                         # buffered mode (the default)
                [("multiline.parser", "exc, java"), ("buffer", "off")],                                  # several parsers
                [("multiline.parser", "docker"), ("buffer", "off")], [("multiline.parser", "cri"), ("buffer", "off")],
                [("multiline.parser", "nope"), ("buffer", "off")], [("buffer", "off")],
                [("multiline.parser", "exc"), ("buffer", "off"), ("mode", "partial_message")],
                [("multiline.parser", "exc"), ("buffer", "off"), ("bogus", "1")]):
        with pytest.raises(pkg.FlbGpuError):
            ctx.filter("multiline", bad)
    with pytest.raises(pkg.FlbGpuError):
        ctx.ml_parser("r1", rules=[("cont", "/x/", "cont")])                     # the first rule must name start_state
    with pytest.raises(pkg.FlbGpuError):
        ctx.ml_parser("r2", rules=[("start_state", "/x/", "nowhere")])           # to_state nobody comes from
    with pytest.raises(RuntimeError):
        util.Ref().ml_parser("r2", rules=[("start_state", "/x/", "nowhere")])
    # loud, never approximated: a message at the buffer limit
    ctx2 = pkg.Context(0, lib=lib)
    ctx2.L.flbgpu_ml_set_buffer_limit(ctx2.h, 64)
    ctx2.ml_parser("exc", rules=EXC)
    ch2 = ctx2.chain([ctx2.filter("multiline", [("multiline.parser", "exc"), ("multiline.key_content", "log"), ("buffer", "off")])])
    assert ch2.do(util.chunk_from_lines([b"Dec 1 1:1:1 x", b"  at " + b"y" * 20]))[0] == pkg.FILTER_MODIFIED
    with pytest.raises(pkg.FlbGpuError):
        ch2.do(util.chunk_from_lines([b"Dec 1 1:1:1 x", b"  at " + b"y" * 30, b"  at " + b"z" * 30]))


def _in_a_chain(lib):
    """multiline, then the filters behind it on what it made (the k8s shape of BASELINE configs[4])"""
    lines = list(JAVA) * 4
    ref = util.Ref()
    ctx = pkg.Context(0, lib=lib)
    chain = [("multiline", [("multiline.parser", "java"), ("multiline.key_content", "log"), ("buffer", "off")]),
             ("grep", [("Regex", "log Exception")]),
             ("modify", [("Add", "multiline yes")])]
    fs = []
    for p, props in chain:
        ref.filter(p, props)
        fs.append(ctx.filter(p, props))
    ch = ctx.chain(fs)
    for t0 in (1700000000, 1700005000):
        c = util.chunk_from_lines(lines, t0=t0)
        assert ch.do(c) == ref.chain_do(c)


def _chain_shapes(lib):
    """`multiline, then other filters` runs as two chains with the intermediate chunk on the device: every way the two halves can
    answer (MODIFIED / NOTOUCH / nothing left), Match routing of either half, and the device-resident form of the call"""
    import ctypes as C
    lines = list(JAVA) * 3
    c1 = util.chunk_from_lines(lines)
    no_key = b"".join(util.event(1700000000 + i, 0, [(b"other", S(b"x%d" % i))]) for i in range(20))     # multiline: every record on its own
    ml = ("multiline", [("multiline.parser", "java"), ("multiline.key_content", "log"), ("buffer", "off")])
    shapes = [
        [ml, ("grep", [("Regex", "log Exception")]), ("modify", [("Add", "k v")])],
        [ml, ("grep", [("Regex", "log .")])],                                        # the rest keeps everything: NOTOUCH, the multiline result stands
        [ml, ("grep", [("Regex", "log no_such_text_anywhere")])],                    # the rest drops everything
        [ml, ("modify", [("Add", "k v")]), ("record_modifier", [("Record", "h n1")]), ("grep", [("Exclude", "log INFO")])],
        [ml + ([("match", "other.*")],), ("modify", [("Add", "k v")])],              # the multiline filter is not routed this tag
        [ml, ("modify", [("Add", "k v"), ("match", "other.*")])],                    # ... the rest is not
    ]
    for shape in shapes:
        ref = util.Ref()
        ctx = pkg.Context(0, lib=lib)
        fs = []
        for item in shape:
            p, props = item[0], list(item[1]) + (list(item[2]) if len(item) > 2 else [])
            ref.filter(p, props)
            fs.append(ctx.filter(p, props))
        ch = ctx.chain(fs)
        for c in (c1, no_key, c1[:len(c1) // 2]):
            assert ch.do(c, tag="test") == ref.chain_do(c, "test"), shape
    # device-resident: flbgpu_chain_do_device() on the first shape
    ref = util.Ref()
    ctx = pkg.Context(0, lib=lib)
    fs = []
    for p, props in shapes[0]:
        ref.filter(p, props)
        fs.append(ctx.filter(p, props))
    ch = ctx.chain(fs)
    L = ctx.L
    d_in, d_out = L.flbgpu_dev_alloc(ctx.h, len(c1) + 64), L.flbgpu_dev_alloc(ctx.h, 2 * len(c1) + 4096)
    buf = C.create_string_buffer(c1, len(c1))
    L.flbgpu_dev_upload(ctx.h, d_in, C.cast(buf, C.c_void_p), len(c1))
    n = C.c_size_t()
    r = L.flbgpu_chain_do_device(ch.h, d_in, len(c1), d_out, 2 * len(c1) + 4096, C.byref(n))
    got = C.create_string_buffer(n.value)
    L.flbgpu_dev_download(ctx.h, C.cast(got, C.c_void_p), d_out, n.value)
    assert (r, got.raw[:n.value]) == ref.chain_do(c1, "test")
    L.flbgpu_dev_free(ctx.h, d_in); L.flbgpu_dev_free(ctx.h, d_out)


def _large(lib, n):
    """many automaton blocks and super-blocks: states cross every boundary"""
    rng = random.Random(14)
    props = [("multiline.parser", "exc"), ("multiline.key_content", "log"), ("buffer", "off")]
    diff(lib, EXC, props, [make_chunk(rng, VOCAB["exc"], n, 1700000000), make_chunk(rng, VOCAB["exc"][2:5], n // 4, 1700100000)], name="exc")


GO_PUSHES = [b"panic: my panic", b"\n", b"goroutine 4 [running]:", b"panic(0x45cb40, 0x47ad70)",
             b"  /usr/local/go/src/runtime/panic.go:542 +0x46c fp=0xc42003f7b8 sp=0xc42003f710 pc=0x422f7c", b"main.main.func1(0xc420024120)"]


def _reference_runtime_unbuffered(lib):
    """tests/runtime/filter_multiline.c:345-417 flb_test_multiline_unbuffered: the go parser with `buffer off`, six pushes of one
    record each (timestamp 0: the message's time is "now") -- six records come out, no concatenation, the first holds "panic".
    Compared with the reference's plugin record for record, the eight timestamp bytes apart; then the same six lines in ONE chunk
    (and with real timestamps): one message."""
    props = [("multiline.key_content", "log"), ("multiline.parser", "go"), ("buffer", "off"), ("debug_flush", "off")]
    ref = util.Ref(keep_whole=True)
    rf = ref.filter("multiline", props)
    ctx = pkg.Context(0, lib=lib)
    ch = ctx.chain([ctx.filter("multiline", props)])
    outs = []
    for line in GO_PUSHES:
        c = util.event(0, 0, [(b"log", S(line))])
        want, got = ref.filter_cb(rf, c), ch.do(c)
        assert want[0] == got[0] == pkg.FILTER_MODIFIED
        assert len(util.split_records(got[1])) == 1 and got[1][:4] == want[1][:4] and got[1][12:] == want[1][12:]
        outs.append(got[1])
    assert len(outs) == 6 and b"panic" in outs[0]
    one = util.chunk_from_lines(GO_PUSHES)
    want, got = ref.filter_cb(rf, one), ch.do(one)
    assert want == got and len(util.split_records(got[1])) < 6


def test_reference_runtime_unbuffered_hostsim(sim_lib, ref_available):
    _reference_runtime_unbuffered(sim_lib)


@pytest.mark.gpu
def test_reference_runtime_unbuffered_gpu(gpu_lib, ref_available):
    _reference_runtime_unbuffered(gpu_lib)


def _edge_chunks(lib):
    """nothing decodable, only events the decoder steps over, garbage behind the events, a record without key_content and with a
    zero timestamp (its time is "now": the eight timestamp bytes are left out of the comparison)"""
    mk = b"\x92\x92\xd7\x00\xff\xff\xff\xff\x00\x00\x00\x00\x80\x80"
    props = [("multiline.parser", "java"), ("multiline.key_content", "log"), ("buffer", "off")]
    one = util.event(5, 0, [(b"log", S(b"x"))])
    for c in (mk, mk * 3, mk + one + mk, b"\xc1garbage", one + b"\xc1\xc1", util.event(0, 0, [(b"other", b"\x01")])):
        ref = util.Ref(keep_whole=True)
        rf = ref.filter("multiline", props)
        ctx = pkg.Context(0, lib=lib)
        got, want = ctx.chain([ctx.filter("multiline", props)]).do(c), ref.filter_cb(rf, c)
        assert got[0] == want[0]
        if want[1]:
            assert got[1][:4] == want[1][:4] and got[1][12:] == want[1][12:]
        else:
            assert got[1] == want[1]


def test_multiline_edge_chunks_hostsim(sim_lib, ref_available):
    _edge_chunks(sim_lib)


@pytest.mark.gpu
def test_multiline_edge_chunks_gpu(gpu_lib, ref_available):
    _edge_chunks(gpu_lib)


def test_multiline_rulesets_hostsim(sim_lib, ref_available):
    _regex_rulesets(sim_lib, 6, 300)


def test_multiline_match_types_hostsim(sim_lib, ref_available):
    _match_types(sim_lib)


def test_multiline_builtins_hostsim(sim_lib, ref_available):
    _builtins(sim_lib)


def test_multiline_refusals_hostsim(sim_lib, ref_available):
    _refusals(sim_lib)


def test_multiline_in_a_chain_hostsim(sim_lib, ref_available):
    _in_a_chain(sim_lib)


def test_multiline_chain_shapes_hostsim(sim_lib, ref_available):
    _chain_shapes(sim_lib)


def test_multiline_large_hostsim(sim_lib, ref_available):
    _large(sim_lib, 40000)


@pytest.mark.gpu
def test_multiline_rulesets_gpu(gpu_lib, ref_available):
    _regex_rulesets(gpu_lib, 2, 300)


@pytest.mark.gpu
def test_multiline_match_types_gpu(gpu_lib, ref_available):
    _match_types(gpu_lib)


@pytest.mark.gpu
def test_multiline_builtins_gpu(gpu_lib, ref_available):
    _builtins(gpu_lib)


@pytest.mark.gpu
def test_multiline_refusals_gpu(gpu_lib, ref_available):
    _refusals(gpu_lib)


@pytest.mark.gpu
def test_multiline_in_a_chain_gpu(gpu_lib, ref_available):
    _in_a_chain(gpu_lib)


@pytest.mark.gpu
def test_multiline_chain_shapes_gpu(gpu_lib, ref_available):
    _chain_shapes(gpu_lib)


@pytest.mark.gpu
def test_multiline_large_gpu(gpu_lib, ref_available):
    _large(gpu_lib, 40000)


def _shim_multiline(lib_path):
    """gpu_multiline (built-in java parser, buffer off) in front of gpu_grep and gpu_modify, driven by the reference's own
    flb_filter_do(): the chunks and the per-filter framework counters of the stock chain"""
    filters = [("multiline", [("multiline.parser", "java"), ("multiline.key_content", "log"), ("buffer", "off")]),
               ("grep", [("Regex", "log Exception")]),
               ("modify", [("Add", "multiline yes")])]
    lines = list(JAVA) * 5
    test_shim.same_behaviour(lib_path, [], filters, [util.chunk_from_lines(lines[:37]), util.chunk_from_lines(lines[37:], t0=1700009000)])


def test_shim_multiline_hostsim(ref_available):
    test_shim.need_shim()
    _shim_multiline(util.HOSTSIM_SO)


@pytest.mark.gpu
def test_shim_multiline_gpu(gpu_lib, ref_available):
    test_shim.need_shim()
    _shim_multiline(test_shim.GPU_LIB)


