"""f4 (output side), GELF: flbgpu_msgpack_to_gelf() -- a chunk of log events as the GELF messages out_gelf and out_http
(`format gelf`) send -- against the reference's own flb_msgpack_to_gelf() in the restated flush loop
(oracle/refshim/gelf_harness.c, through tests/gelf_ref.py), and against the reference's own GELF tests as scenarios."""
import base64
import json
import os
import random
import struct

import pytest

import gelf_ref
import util

pkg = util.pkg
FlbGpuError = pkg.FlbGpuError
S = util.mp_str
CUSTOM = dict(timestamp_key="ts", host_key="h", short_message_key="msg", full_message_key="full", level_key="lvl")


@pytest.fixture
def gelf_ref_available():
    if not gelf_ref.have_ref_results():
        pytest.skip("oracle/_ref/libflbref_gelf.so is not built and no stored reference results cover this test")
    return True


def f64(x):
    return b"\xcb" + struct.pack(">d", x)


def f32(x):
    return b"\xca" + struct.pack(">f", x)


def bin_(b):
    return b"\xc4" + bytes([len(b)]) + b


def mp_map(items):
    """items: (encoded key, encoded value) pairs"""
    return util.mp_map_hdr(len(items)) + b"".join(k + v for k, v in items)


def mp_arr(vals):
    return (bytes([0x90 | len(vals)]) if len(vals) < 16 else b"\xdc" + struct.pack(">H", len(vals))) + b"".join(vals)


def ev(body, sec=1700000000, nsec=0, t=None):
    """one v2 event; body: (encoded key, encoded value) pairs; t: an encoded timestamp instead of the ext time"""
    ts = t if t is not None else b"\xd7\x00" + struct.pack(">II", sec & 0xffffffff, nsec & 0xffffffff)
    return b"\x92\x92" + ts + b"\x80" + mp_map(body)


def msg(text=b"m", key=b"short_message"):
    return (S(key), S(text))


# ------------------------------------------------------------------ random chunks
WORDS = [b"", b"a", b"plain text", b'q"z', b"tab\tnl\n", b"h\xc3\xa9llo", b"\xe2\x82\xac" * 7 + b"x" * 9, b"\xf0\x9f\x98\x80 emoji",
         b"bad \xff\xfe utf8", b"x" * 40, b"\x00nul\x01", b"back\\slash" * 3]
KEYS = [b"short_message", b"host", b"timestamp", b"level", b"full_message", b"id", b"msg", b"h", b"ts", b"lvl", b"full", b"k",
        b"a b", b"we/ird:key", b"\xc3\xa9", b"", b"n\x00ul", b"x" * 30]


def rand_value(rng, depth=0):
    r = rng.random()
    if depth < 4 and r < 0.12:
        return mp_map([(S(rng.choice(KEYS)) if rng.random() < 0.9 else rng.choice([b"\x01", bin_(b"bk")]), rand_value(rng, depth + 1))
                       for _ in range(rng.randint(0, 4))])
    if depth < 4 and r < 0.24:
        return mp_arr([rand_value(rng, depth + 1) for _ in range(rng.randint(0, 4))])
    return rng.choice([
        lambda: S(rng.choice(WORDS)), lambda: S(rng.choice(WORDS)), lambda: bin_(rng.choice(WORDS)[:20]), lambda: b"\xc0",
        lambda: rng.choice([b"\xc2", b"\xc3"]), lambda: util.pkg and bytes([rng.randint(0, 127)]),
        lambda: b"\xd0" + struct.pack(">b", rng.randint(-128, 127)), lambda: b"\xd3" + struct.pack(">q", rng.randint(-2 ** 63, 2 ** 63 - 1)),
        lambda: b"\xcf" + struct.pack(">Q", rng.randint(0, 2 ** 64 - 1)),
        lambda: f64(rng.choice([0.5, -2.25, 1e-7, 123456.789, 1.5e39, 1e40, -1e38, 3.3e38, 1e300, float("inf"), float("nan")])),
        lambda: f32(rng.choice([1.5, -0.1, 3.4e38])), lambda: b"\xd4\x05" + bytes([rng.randint(0, 255)]),
        lambda: b"\xc7\x03\x07abc",
        lambda: S(rng.choice([b"0", b"7", b"8", b"info", b"WARNING", b"Err", b"emergency"]))])()


def rand_event(rng):
    body = [(S(rng.choice(KEYS)) if rng.random() < 0.93 else bin_(rng.choice(KEYS)), rand_value(rng)) for _ in range(rng.randint(0, 7))]
    if rng.random() < 0.85:
        body.insert(rng.randint(0, len(body)), msg(rng.choice(WORDS), rng.choice([b"short_message", b"msg"])))
    t = rng.random()
    if t < 0.1:
        return ev(body, t=bytes([rng.randint(0, 127)]))
    if t < 0.2:
        return ev(body, t=f64(rng.choice([1700000000.25, 1.999999, 0.0005, 12345.6789])))
    return ev(body, sec=rng.randint(0, 2 ** 31 - 1), nsec=rng.choice([0, 1, 999999, 12341111, 999999999, 1234111111, -5 * 10 ** 8]))


def rand_chunk(rng, n):
    out = []
    for _ in range(n):
        r = rng.random()
        if r < 0.05:      # a group start and end (seconds -1 / -2): the decoder steps over both
            out.append(b"\x92\x92\xd7\x00" + struct.pack(">II", 0xffffffff, 0) + b"\x80" + mp_map([(S(b"g"), b"\x01")]))
        elif r < 0.08:
            out.append(b"\x92\x92\xd7\x00" + struct.pack(">II", 0xfffffffe, 0) + b"\x80\x80")
        else:
            out.append(rand_event(rng))
    c = b"".join(out)
    if rng.random() < 0.2:
        c += rng.choice([b"\x92\x92\xd7\x00garbage", b"\xc1\xc1", b"\x92"])
    return c


def _diff(lib, n_chunks):
    rng = random.Random(0x6e1f)
    ref = gelf_ref.GelfRef()
    ctx = pkg.Context(0, lib=lib)
    compared = 0
    for r in range(n_chunks):
        chunk = rand_chunk(rng, rng.randint(0, 40))
        kw = dict(fields=CUSTOM if r % 2 else None, separator=b"\n" if r % 3 else b"\0")
        if r % 4 >= 2:
            kw.update(tag_key=rng.choice(["tag", "short_message", "k" * 20]), tag=rng.choice([b"app.log", b"t" * 40, b""]))
        want = ref.to_gelf(chunk, **kw)
        text, failed, undefined = ctx.to_gelf(chunk, **kw)
        assert failed == want[1], (r, kw)
        if undefined == 0:
            assert text == want[0], (r, kw, chunk)
            compared += 1
    assert compared > n_chunks * 0.9


# ------------------------------------------------------------------ one case per rule of src/flb_pack_gelf.c
FLOATS = [(46, 1e39), (47, 1.5e39), (48, 1e40), (49, 1e41), (46, -1e38), (47, -1e39), (48, -9e39), (49, -1e40)]


def _rules(lib):
    ref = gelf_ref.GelfRef()
    ctx = pkg.Context(0, lib=lib)

    def both(events, **kw):
        chunk = b"".join(events)
        want = ref.to_gelf(chunk, **kw)
        got = ctx.to_gelf(chunk, **kw)
        assert got[2] == 0 and got[:2] == want, (kw, chunk)
        return got[0], got[1]

    # top-level floats: "%f" cut to 46 characters plus NUL bytes at 47 / 48, a failed event from 49 on; nested ones never cut
    for n, x in FLOATS:
        assert len("%f" % x) == n
        text, failed = both([ev([msg(), (S(b"f"), f64(x))]), ev([msg(), (S(b"n"), mp_map([(S(b"f"), f64(x))]))])])
        assert failed == (1 if n == 49 else 0)
        if n <= 48:
            assert (b'"_f":' + ("%f" % x).encode()[:46] + b"\0" * (n - 46) + b", ") in text
        assert (b'"_n_f":' + ("%f" % x).encode() + b", ") in text
    # strings inside arrays: raw, unquoted; nested nil is null, top-level nil is left out; booleans quoted outside arrays
    text, _ = both([ev([msg(), (S(b"arr"), mp_arr([S(b'q"z'), b"\xc0", f64(2.5), b"\xc3"])), (S(b"nil"), b"\xc0"), (S(b"b"), b"\xc2")])])
    assert text.startswith(b'{"version":"1.1", "short_message":"m", "_arr":"q"z, null, 2.500000, true", "_b":"false", "timestamp":')
    # timestamps: "%li.%03lu" of seconds and nanoseconds / 10^6, also past 10^9 ns and below 0; integer and float64 times
    for t, nsec, want in [(None, 1234111111, b"100.1234"), (None, 12341111, b"100.012"), (None, -1, b"100.000"),
                          (None, -5 * 10 ** 8, b"100.18446744073709551116"), (bytes([100]), 0, b"100.000"), (f64(100.75), 0, b"100.750")]:
        text, _ = both([ev([msg()], sec=100, nsec=nsec, t=t)])
        assert text.endswith(b'"timestamp":' + want + b"}\n")
    text, _ = both([ev([msg(), (S(b"timestamp"), S(b"then"))])])
    assert text.count(b"timestamp") == 1
    # keys: the first of each field key wins, id goes, others get '_' and valid_char[]; BIN keys count at the top level only;
    # a NUL inside a key with a map value zero-fills the prefix
    text, _ = both([ev([msg(b"one"), msg(b"two"), (S(b"host"), S(b"h1")), (S(b"host"), S(b"h2")), (S(b"id"), b"\x01"),
                        (bin_(b"bk"), b"\x02"), (S(b"we/ird key"), b"\x03"),
                        (S(b"m"), mp_map([(bin_(b"skip"), b"\x04"), (S(b"k"), b"\x05")])), (S(b"a\x00bc"), mp_map([(S(b"d\x00e"), b"\x06")]))])])
    assert (b'"short_message":"one", "host":"h1", "_bk":2, "_we_ird_key":3, "_m_k":5, "_a____d_e":6, "timestamp"') in text
    # level: integers as they are (8 too, int8-encoded too), "0".."7" and syslog names as integers, other strings quoted,
    # other types (a negative integer too) fail the event
    levels = [(b"\x08", b"8"), (b"\xd0\x03", b"3"), (S(b"5"), b"5"), (S(b"DeBuG"), b"7"), (S(b"warning"), b"4"), (S(b"8"), b'"8"'),
              (S(b"verbose"), b'"verbose"')]
    for v, want in levels:
        text, failed = both([ev([msg(), (S(b"level"), v)])])
        assert failed == 0 and b'"level":' + want + b", " in text
    for v in [b"\xff", b"\xd0\xfe", f64(1.0), b"\xc0", bin_(b"1"), mp_arr([b"\x01"]), mp_map([])]:
        assert both([ev([msg(), (S(b"level"), v)])]) == (None, 1)
    # no short message: the event fails and is left out
    assert both([ev([(S(b"x"), S(b"y"))]), ev([msg()])])[1] == 1
    # an empty fixstr before the unpacker's first multi-byte token is a NULL pointer: such a top-level key or value goes
    for tag in (None, b"t"):
        kw = dict(tag_key="tag", tag=tag) if tag else {}
        both([ev([(S(b""), b"\x14"), msg(), (S(b""), b"\x15")]), ev([(S(b"k"), S(b"")), msg()], t=bytes([5])),
              ev([(S(b""), mp_arr([])), (S(b""), mp_map([(S(b"a"), b"\x01")])), msg()], t=bytes([5])),
              ev([(S(b"level"), S(b"")), (S(b"level"), b"\x01"), msg()], t=bytes([5])),
              ev([(S(b""), f64(1e300)), msg()]), ev([(S(b""), f64(1e40)), msg()])], **kw)
    # nesting at msgpack-c's unpack limit: the decoder stops at the event that passes it
    for depth in (30, 31):
        deep = b"\x01"
        for _ in range(depth):
            deep = mp_arr([deep])
        both([ev([msg(), (S(b"d"), deep)]), ev([msg()])])
    # custom field names and tag_key
    text, _ = both([ev([(S(b"msg"), S(b"hi")), (S(b"h"), S(b"box")), (S(b"ts"), f64(1.5)), (S(b"lvl"), S(b"err"))])],
                   fields=CUSTOM, tag_key="tag", tag=b"app")
    assert text == b'{"version":"1.1", "short_message":"hi", "host":"box", "timestamp":1.500000, "level":3, "_tag":"app"}\n'


def _window(lib):
    """strings of every length around the 16-byte window, a multi-byte character at every offset, each followed by a member:
    every byte the reference's writer reads lies inside the chunk"""
    ref = gelf_ref.GelfRef()
    ctx = pkg.Context(0, lib=lib)
    events = []
    for n in range(0, 40):
        for at in (0, 1, 7, 14, 15, 16):
            s = (b"a" * at + "é".encode() + b"b" * 40)[:n]
            events.append(ev([msg(s), (S(b"tail"), S(b"\"\\" + b"z" * 20)), (S(b"after"), b"\x01")]))
    for kw in (dict(), dict(tag_key="tag", tag=b"t")):
        chunk = b"".join(events)
        text, failed, undefined = ctx.to_gelf(chunk, **kw)
        assert undefined == 0 and (text, failed) == ref.to_gelf(chunk, **kw)


def _scenarios(lib):
    sc = json.load(open(os.path.join(util.ROOT, "tests", "golden", "gelf_scenarios.json")))
    assert len(sc) == 8
    ctx = pkg.Context(0, lib=lib)
    for s in sc:
        text, failed, undefined = ctx.to_gelf(base64.b64decode(s["chunk"]), s["fields"])
        assert failed == 0 and undefined == 0, s["test"]
        if s["equals"] is not None:
            assert text == s["equals"].encode() + b"\n", s["test"]
        for p in s["present"]:
            assert p.encode() in text, (s["test"], p)
        assert text == s["ref_out"].encode("latin-1"), s["test"]


def _errors(lib):
    ctx = pkg.Context(0, lib=lib)
    chunk = ev([msg()])
    for kw, what in [(dict(separator=b"\t"), "separator"), (dict(tag_key="tag"), "tag is NULL"),
                     (dict(tag_key="k" * 129, tag=b"t"), "tag_key longer"), (dict(tag_key="tag", tag=b"t" * 257), "tag longer"),
                     (dict(fields=dict(level_key="l" * 129)), "field key longer")]:
        with pytest.raises(FlbGpuError, match=what):
            ctx.to_gelf(chunk, **kw)
    assert ctx.to_gelf(b"") == (None, 0, 0)
    assert ctx.to_gelf(ev([(S(b"x"), b"\x01")])) == (None, 1, 0)
    assert ctx.to_gelf(chunk, fields=dict(short_message_key="k" * 128))[1] == 1


def _large(lib, n, per_event):
    """one chunk of n events (scans across many blocks), against the reference"""
    rng = random.Random(n)
    pool = [rand_event(rng) for _ in range(997)]
    chunk = b"".join(pool[(i * 7919) % len(pool)] for i in range(n))
    want = gelf_ref.GelfRef().to_gelf(chunk, tag_key="tag", tag=b"bulk")
    text, failed, undefined = pkg.Context(0, lib=lib).to_gelf(chunk, tag_key="tag", tag=b"bulk")
    assert undefined == 0 and (text, failed) == want
    return len(chunk)


def test_gelf_diff_hostsim(sim_lib, gelf_ref_available):
    _diff(sim_lib, 160)


def test_gelf_rules_hostsim(sim_lib, gelf_ref_available):
    _rules(sim_lib)


def test_gelf_window_hostsim(sim_lib, gelf_ref_available):
    _window(sim_lib)


def test_gelf_scenarios_hostsim(sim_lib):
    _scenarios(sim_lib)


def test_gelf_errors_hostsim(sim_lib):
    _errors(sim_lib)


@pytest.mark.gpu
def test_gelf_diff_gpu(gpu_lib, gelf_ref_available):
    _diff(gpu_lib, 160)


@pytest.mark.gpu
def test_gelf_rules_gpu(gpu_lib, gelf_ref_available):
    _rules(gpu_lib)


@pytest.mark.gpu
def test_gelf_window_gpu(gpu_lib, gelf_ref_available):
    _window(gpu_lib)


@pytest.mark.gpu
def test_gelf_scenarios_gpu(gpu_lib):
    _scenarios(gpu_lib)


@pytest.mark.gpu
def test_gelf_errors_gpu(gpu_lib):
    _errors(gpu_lib)


@pytest.mark.gpu
def test_gelf_over_8mb_gpu(gpu_lib, gelf_ref_available):
    assert _large(gpu_lib, 200000, 1) > 8 << 20


@pytest.mark.gpu
def test_gelf_million_events_gpu(gpu_lib, gelf_ref_available):
    _large(gpu_lib, 1 << 20, 1)
