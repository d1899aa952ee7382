"""f4 (input side) with a parser: in_tail's `Parser` branch (plugins/in_tail/tail_file.c:721-746) -- raw text to parsed log
events in one call, flbgpu_lines_to_events_parsed() -- against the same loop restated in the reference harness around the
reference's own flb_parser_do() and log event encoder (oracle/refshim/tail_harness.c, through tests/tail_ref.py), and against
committed vectors made from it."""
import base64
import calendar
import json
import os
import random
import threading

import pytest

import tail_ref
import util

pkg = util.pkg
FlbGpuError = pkg.FlbGpuError
TIME_RX = r'^(?:(?<time>\d{4}-\d\d-\d\dT\d\d:\d\d:\d\d) )?(?<msg>.*)$'
PARSERS = {
    "apache2": dict(name="apache2", format="regex", regex=util.APACHE_RX, time_fmt=util.APACHE_TIME_FMT, time_key="time"),
    "json": dict(name="json", format="json", time_key="time", time_fmt="%d/%b/%Y:%H:%M:%S %z"),
    "ltsv": dict(name="ltsv", format="ltsv", time_key="time", time_fmt="%d/%b/%Y:%H:%M:%S %z", types="status:integer size:integer"),
    "logfmt": dict(name="logfmt", format="logfmt", time_key="ts", time_fmt="%Y-%m-%dT%H:%M:%SZ"),
    "typed": dict(name="typed", format="regex", regex=r'^(?<time>[^ ]+) (?<level>[a-z]+) (?<n>-?\d+) (?<f>-?[0-9.]+) (?<msg>.*)$',
                  time_key="time", time_fmt="%Y-%m-%dT%H:%M:%S", time_keep=True, types="n:integer f:float"),
    "decode": dict(name="decode", format="regex", regex=r'^(?<level>[a-z]+) (?<log>.*)$', decoders=[("Decode_Field_As", "json log")]),
    "times": dict(name="times", format="regex", regex=TIME_RX, time_key="time", time_fmt="%Y-%m-%dT%H:%M:%S"),
}
JUNK = [b"", b"\r", b"not a log line", b"\x00\x01bin\xff", b"x" * 300, b"{\"broken\": ", b"crlf junk\r", b" "]


def good_lines(name, n, seed):
    rng = random.Random(seed)
    if name == "apache2":
        return util.apache_lines(n, seed=seed)
    if name == "json":
        out = util.json_lines(n, seed=seed)
        return [l[:-1] + b',"time":"10/Oct/2000:13:55:36 -0700"}' if rng.random() < 0.5 and l.endswith(b"}") else l for l in out]
    if name == "ltsv":
        return util.ltsv_lines(n, seed=seed)
    if name == "logfmt":
        return util.logfmt_lines(n, seed=seed)
    if name == "typed":
        return [("2023-%02d-%02dT%02d:%02d:%02d %s %d %s %s" % (rng.randint(1, 12), rng.randint(1, 28), rng.randint(0, 23), rng.randint(0, 59),
                                                              rng.randint(0, 59), rng.choice(["info", "warn", "error"]), rng.randint(-10 ** 6, 10 ** 6),
                                                              rng.choice(["1.5", "-0.25", "3", "12.125"]), "message %d" % i)).encode()
                for i in range(n)]
    if name == "decode":
        return [rng.choice([b'info {"a": 1, "b": "two", "c": [1, 2]}', b"warn plain text", b'error {"nested": {"k": "v"}}',
                            b'debug "just a string"', b"info [1, 2, 3]"]) for _ in range(n)]
    return [rng.choice([b"no time here", b"2023-10-05T10:11:12 with time", b"1970-01-01T00:00:00 the epoch"]) for _ in range(n)]


def text(name, rng, n, tail=True):
    """parsed lines mixed with lines the parser rejects, CRLF endings, empty lines and lone '\\r'; sometimes an unfinished tail"""
    good = good_lines(name, n, rng.randint(0, 10 ** 6))
    lines = []
    for g in good:
        r = rng.random()
        lines.append(rng.choice(JUNK) if r < 0.15 else g + b"\r" if r < 0.3 else g)
    t = b"\n".join(lines) + (b"\n" if n else b"")
    if tail and rng.random() < 0.5:
        t += rng.choice([b"unfinished", b"\r", good[0] if good else b"x"])
    return t


def kwargs(rng, r):
    kw = dict(key=rng.choice(["log", "message", "m" * 40]), skip_empty_lines=rng.random() < 0.5, sec=1700000000 + r,
              nsec=rng.choice([0, 999999999]))
    if rng.random() < 0.5:
        kw.update(path_key=rng.choice(["file", "path", "host"]), path="/var/log/containers/app-%d.log" % r)
    if rng.random() < 0.5:
        kw.update(offset_key="offset", stream_offset=rng.choice([0, 127, 2 ** 16, 2 ** 32 + 5]))
    return kw


@pytest.fixture
def tail_ref_available():
    if not tail_ref.have_ref_results():
        pytest.skip("oracle/_ref/libflbref_tail.so is not built and no stored reference results cover this test")
    return True


def _pair(lib, names, ref=None):
    ref = ref or tail_ref.TailRef()
    ctx = pkg.Context(0, lib=lib)
    ps = {n: (ctx.parser(**PARSERS[n]), ref.parser(**PARSERS[n])) for n in names}
    return ref, ctx, ps


def _diff(lib, rounds):
    rng = random.Random(51)
    ref, ctx, ps = _pair(lib, ["apache2", "json", "ltsv", "logfmt", "typed", "decode"])
    for r in range(rounds):
        name = rng.choice(sorted(ps))
        t = text(name, rng, rng.choice([0, 1, 2, 5, 40, 300]))
        kw = kwargs(rng, r)
        mine, theirs = ps[name]
        assert mine.lines_to_events(t, **kw) == ref.lines_to_events_parsed(theirs, t, **kw), (r, name, kw, t[:300])


def _time_rules(lib):
    """no time, a parsed time of exactly the epoch (both: the call's time), times before 1970 and after 2106 (32-bit seconds)"""
    ref, ctx, ps = _pair(lib, ["times"], tail_ref.TailRef(keep_whole=True))
    mine, theirs = ps["times"]
    t = b"\n".join([b"no time here", b"1970-01-01T00:00:00 the epoch", b"1960-06-01T12:00:00 before", b"2200-01-01T00:00:01 after",
                    b"2106-02-07T06:28:16 wraps", b"2023-10-05T10:11:12 ordinary"]) + b"\n"
    got = mine.lines_to_events(t, "log", True, 1700000000, 5)
    assert got == ref.lines_to_events_parsed(theirs, t, "log", True, 1700000000, 5)
    recs = util.split_records(got[0])
    assert len(recs) == 6
    stamps = [got[0][o + 4:o + 12] for o, _ in recs]
    call = (1700000000).to_bytes(4, "big") + (5).to_bytes(4, "big")
    assert stamps[0] == call and stamps[1] == call and stamps[5] != call
    assert stamps[2] == (calendar.timegm((1960, 6, 1, 12, 0, 0)) & 0xffffffff).to_bytes(4, "big") + bytes(4)
    assert stamps[3] == (calendar.timegm((2200, 1, 1, 0, 0, 1)) & 0xffffffff).to_bytes(4, "big") + bytes(4)
    assert stamps[4] == bytes(8) and stamps[4] != call          # 2^32 seconds is not 0 ns: kept, and cut to 0 by the (uint32_t)


def _key_rules(lib):
    """a parsed key equal to path_key appears twice; a line holding bytes that frame as an event keeps lines and records paired"""
    ref, ctx, ps = _pair(lib, ["json", "apache2"], tail_ref.TailRef(keep_whole=True))
    fake = b"\x92\x92\xd7\x00" + b"\x01" * 8 + b"\x80\x80"
    t = b"\n".join([b'{"file": "parsed", "a": 1}', b"pre " + fake + b" post", fake, b"x" + fake, b'{"b": 2}',
                    fake + b"\r", b'{"file": 1}' + b" " * 3]) + b"\n"
    for name in ("json", "apache2"):
        mine, theirs = ps[name]
        kw = dict(key="log", skip_empty_lines=True, sec=1700000000, nsec=0, path_key="file", path="/p", offset_key="o", stream_offset=7)
        got = mine.lines_to_events(t, **kw)
        assert got == ref.lines_to_events_parsed(theirs, t, **kw), name
        assert got[2] == 7 and len(util.split_records(got[0])) == 7
    assert got[0].count(b"\xa4file") == 7                        # (apache2 parses none of these: the plain events, path first)


def _large(lib, n, names=("apache2", "json")):
    """megabytes of lines: every tile, block and scan boundary crossed"""
    rng = random.Random(52 + n)
    ref, ctx, ps = _pair(lib, names)
    for name in names:
        t = text(name, rng, n)
        mine, theirs = ps[name]
        kw = dict(key="log", skip_empty_lines=name == "json", sec=1700000000, nsec=1, path_key="file", path="/var/log/a.log", offset_key="o",
                  stream_offset=2 ** 32 - 10)
        got = mine.lines_to_events(t, **kw)
        assert got == ref.lines_to_events_parsed(theirs, t, **kw), name
        assert got[1] == t.rfind(b"\n") + 1 and len(util.split_records(got[0])) == got[2]
    return len(t)


def _refusal(lib):
    """a line the device gives up on (a catastrophically backtracking pattern) fails the call, naming the bit"""
    ctx = pkg.Context(0, lib=lib)
    p = ctx.parser(name="slow", format="regex", regex=r"^(a+)+$")
    assert p.lines_to_events(b"aaaa\n", "log", True, 1, 0)[2] == 1
    with pytest.raises(FlbGpuError, match="RXBUDGET"):
        p.lines_to_events(b"aaaa\n" + b"a" * 40 + b"!\nbbb\n", "log", True, 1, 0)
    assert p.lines_to_events(b"aaaa\n", "log", True, 1, 0)[2] == 1     # (and the parser works on afterwards)


def _runtime_parser(lib):
    """the reference's own runtime test, tests/runtime/in_tail.c flb_test_parser: an apache line through `parser apache2`, then JSON"""
    ref, ctx, ps = _pair(lib, ["apache2"], tail_ref.TailRef(keep_whole=True))
    mine, theirs = ps["apache2"]
    t = b'127.0.0.1 - frank [10/Oct/2000:13:55:36 -0700] "GET /apache_pb.gif HTTP/1.0" 200 2326\n'
    ev = mine.lines_to_events(t, "log", True, 1700000000, 0)
    rev = ref.lines_to_events_parsed(theirs, t, "log", True, 1700000000, 0)
    assert ev == rev and ev[2] == 1
    js, und = ctx.to_json(ev[0], 1, 0, "date", True)
    assert und == 0 and js == ref.to_json(rev[0], 1, 0, "date", True)
    for s in [b'"method":"GET"', b'"host":"127.0.0.1"', b'"user":"frank"', b'"path":"/apache_pb.gif"', b'"code":"200"', b'"size":"2326"']:
        assert s in js, s


def _threads(lib):
    """two threads, two parsers, calls interleaved: every result is the reference's"""
    rng = random.Random(53)
    ref, ctx, ps = _pair(lib, ["apache2", "json"])
    work = {}
    for name in ("apache2", "json"):
        calls = []
        for r in range(12):
            t = text(name, rng, rng.choice([1, 20, 200]))
            kw = kwargs(rng, r)
            calls.append((t, kw, ref.lines_to_events_parsed(ps[name][1], t, **kw)))
        work[name] = calls
    errors = []

    def run(name):
        try:
            for t, kw, want in work[name]:
                got = ps[name][0].lines_to_events(t, **kw)
                if got != want:
                    errors.append((name, kw))
        except Exception as e:                      # (reported by the main thread)
            errors.append((name, repr(e)))

    th = [threading.Thread(target=run, args=(n,)) for n in work]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


def _golden(lib):
    vec = json.load(open(os.path.join(util.ROOT, "tests", "golden", "tail_parser_vectors.json")))
    ctx = pkg.Context(0, lib=lib)
    D = lambda s: None if s is None else base64.b64decode(s)
    assert len(vec) >= 20
    parsers = {}
    for v in vec:
        if v["parser"] not in parsers:
            parsers[v["parser"]] = ctx.parser(**PARSERS[v["parser"]])
        assert parsers[v["parser"]].lines_to_events(D(v["text"]), **v["kw"]) == (D(v["out"]), v["consumed"], v["lines"]), (v["parser"], v["kw"])


def test_tail_parser_diff_hostsim(sim_lib, tail_ref_available):
    _diff(sim_lib, 120)


def test_tail_parser_time_rules_hostsim(sim_lib, tail_ref_available):
    _time_rules(sim_lib)


def test_tail_parser_key_rules_hostsim(sim_lib, tail_ref_available):
    _key_rules(sim_lib)


def test_tail_parser_large_hostsim(sim_lib, tail_ref_available):
    assert _large(sim_lib, 20000) > 2 << 20


def test_tail_parser_bulk_hostsim(sim_lib, tail_ref_available):
    assert _large(sim_lib, 70000, ("apache2",)) > 8 << 20


def test_tail_parser_refusal_hostsim(sim_lib):
    _refusal(sim_lib)


def test_tail_parser_runtime_hostsim(sim_lib, tail_ref_available):
    _runtime_parser(sim_lib)


def test_tail_parser_threads_hostsim(sim_lib, tail_ref_available):
    _threads(sim_lib)


def test_tail_parser_golden_hostsim(sim_lib):
    _golden(sim_lib)


@pytest.mark.gpu
def test_tail_parser_diff_gpu(gpu_lib, tail_ref_available):
    _diff(gpu_lib, 120)


@pytest.mark.gpu
def test_tail_parser_time_rules_gpu(gpu_lib, tail_ref_available):
    _time_rules(gpu_lib)


@pytest.mark.gpu
def test_tail_parser_key_rules_gpu(gpu_lib, tail_ref_available):
    _key_rules(gpu_lib)


@pytest.mark.gpu
def test_tail_parser_large_gpu(gpu_lib, tail_ref_available):
    assert _large(gpu_lib, 20000) > 2 << 20


@pytest.mark.gpu
def test_tail_parser_bulk_gpu(gpu_lib, tail_ref_available):
    assert _large(gpu_lib, 70000, ("apache2",)) > 8 << 20


@pytest.mark.gpu
def test_tail_parser_refusal_gpu(gpu_lib):
    _refusal(gpu_lib)


@pytest.mark.gpu
def test_tail_parser_runtime_gpu(gpu_lib, tail_ref_available):
    _runtime_parser(gpu_lib)


@pytest.mark.gpu
def test_tail_parser_threads_gpu(gpu_lib, tail_ref_available):
    _threads(gpu_lib)


@pytest.mark.gpu
def test_tail_parser_golden_gpu(gpu_lib):
    _golden(gpu_lib)
