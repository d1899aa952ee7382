"""Byte parity of the filter chain against the UNMODIFIED reference (oracle/_ref).

CPU half: the device algorithms compiled for the host (tests/hostsim).  GPU half: the
same cases through libflbgpu.so's C ABI on a real device.  Both compare the returned
code (MODIFIED / NOTOUCH) and every output byte."""
import struct

import pytest

import cases
import util

pkg = util.pkg


def per_filter(fs, chunk):
    """the reference's own loop: one cb_filter per plugin, host buffers in between"""
    cur, modified = chunk, False
    for f in fs:
        r, out = f.cb(cur)
        if r == pkg.FILTER_MODIFIED:
            cur, modified = out, True
            if len(out) == 0:
                break
    return (pkg.FILTER_MODIFIED, cur) if modified else (pkg.FILTER_NOTOUCH, None)


def run_case(lib, parsers, filters, chunk, fused=True):
    ctx = pkg.Context(0, lib=lib)
    ref = util.Ref()
    for kw in parsers:
        ctx.parser(**kw)
        ref.parser(**kw)
    fs = [ctx.filter(p, props) for p, props in filters]
    for p, props in filters:
        ref.filter(p, props)
    want = ref.chain_do(chunk)
    got = ctx.chain(fs).do(chunk) if fused else per_filter(fs, chunk)
    assert got[0] == want[0]
    assert got[1] == want[1]


@pytest.mark.parametrize("case", cases.CASES, ids=[c[0] for c in cases.CASES])
def test_fused_chain_hostsim(case, sim_lib, ref_available):
    _, parsers, filters, mk = case
    run_case(sim_lib, parsers, filters, mk())


@pytest.mark.parametrize("case", cases.CASES[:6], ids=[c[0] for c in cases.CASES[:6]])
def test_per_filter_callbacks_hostsim(case, sim_lib, ref_available):
    _, parsers, filters, mk = case
    run_case(sim_lib, parsers, filters, mk(), fused=False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", cases.CASES, ids=[c[0] for c in cases.CASES])
def test_fused_chain_gpu(case, gpu_lib, ref_available):
    _, parsers, filters, mk = case
    run_case(gpu_lib, parsers, filters, mk())


@pytest.mark.gpu
@pytest.mark.parametrize("case", cases.CASES[:6], ids=[c[0] for c in cases.CASES[:6]])
def test_per_filter_callbacks_gpu(case, gpu_lib, ref_available):
    _, parsers, filters, mk = case
    run_case(gpu_lib, parsers, filters, mk(), fused=False)


def test_edge_chunks_hostsim(sim_lib, ref_available):
    chunk = cases.apache_chunk(50)
    # empty chunk, trailing garbage, garbage at the front, group markers
    marker = util.event(0xffffffff, 0, [(b"g", util.mp_str(b"start"))])
    endm = util.event(0xfffffffe, 0, [])
    for data in [chunk + b"\x01\x02\x03", b"\xc1" + chunk, marker + chunk + endm, marker + endm]:
        for filters in ([("grep", [("Regex", "log GET")])], [cases.P], [("modify", [("Add", "a b")])]):
            run_case(sim_lib, [cases.AP], filters, data)


@pytest.mark.gpu
def test_edge_chunks_gpu(gpu_lib, ref_available):
    chunk = cases.apache_chunk(50)
    marker = util.event(0xffffffff, 0, [(b"g", util.mp_str(b"start"))])
    endm = util.event(0xfffffffe, 0, [])
    for data in [chunk + b"\x01\x02\x03", b"\xc1" + chunk, marker + chunk + endm, marker + endm]:
        for filters in ([("grep", [("Regex", "log GET")])], [cases.P], [("modify", [("Add", "a b")])]):
            run_case(gpu_lib, [cases.AP], filters, data)


def _decoder_forms():
    """the event forms tests/internal/log_event_decoder.c walks through (decode_timestamp, decode_object, the group
    tests): every timestamp spelling in forward and v2 framing with and without metadata, group markers in and out
    of order, truncated and corrupted groups, roots that are not events"""
    S = util.mp_str
    lines = util.apache_lines(40, seed=3)

    def body(i):
        return util.mp_map_hdr(2) + S(b"log") + S(lines[i % 40]) + S(b"n") + bytes([i % 100])

    def ext(s, n):
        return b"\xd7\x00" + struct.pack(">II", s, n)
    ts_forms = [b"\x05", b"\xcc\xc8", b"\xcd\x12\x34", b"\xce\x65\x54\x92\xce", b"\xcf" + struct.pack(">Q", 1700000000),
                b"\xcb" + struct.pack(">d", 1700000000.25), b"\xca" + struct.pack(">f", 1.5), ext(1700000000, 5),
                b"\xd7\x01" + struct.pack(">II", 1, 2), b"\xc7\x08\x00" + struct.pack(">II", 1700000001, 7), b"\xd3" + struct.pack(">q", -5),
                b"\xd0\xfb", b"\xa3abc", b"\xc0", ext(0x80000000, 0), ext(0xfffffffd, 0), ext(0xffffffff, 0), ext(0xfffffffe, 0)]
    out = []
    for k, t in enumerate(ts_forms):
        out.append(b"\x92" + t + body(1) + b"\x92\x92" + t + b"\x80" + body(2) + b"\x92\x92" + t + b"\x81" + S(b"m") + b"\x01" + body(3) +
                   util.event(1700000000, 0, [(b"log", S(lines[k % 5]))]))

    def gs():
        return util.event(0xffffffff, 0, [(b"g", S(b"start"))])

    def ge():
        return util.event(0xfffffffe, 0, [])

    def rec(i):
        return util.event(1700000000 + i, i, [(b"log", S(lines[i % 40]))])
    out += [gs() + rec(1) + rec(2), rec(1) + ge() + rec(2), gs() + gs() + rec(1) + ge() + ge() + rec(2), ge() + gs() + rec(1),
            gs() + rec(1) + ge() + gs() + rec(2) + ge(), gs() + b"\xc1" + rec(1), gs() + rec(1)[:20], b"\x92\x92" + ext(0xffffffff, 0) + b"\x80\x01" + rec(3),
            b"\x93" + ext(1, 1) + b"\x80\x80" + rec(1), b"\x92\x93" + ext(1, 1) + b"\x80\x80\x80" + rec(1), b"\x92\x92" + ext(1, 1) + b"\x90\x80" + rec(1),
            b"\x92\x92" + ext(1, 1) + b"\x80\x90" + rec(2), b"\x91\x80" + rec(1), b"\x80" + rec(1), b"\xa1x" + rec(1)]
    return out


DECODER_FILTERS = ([("grep", [("Regex", "log GET")])], [cases.P], [("modify", [("Add", "a b")])], [("record_modifier", [("Record", "h n1")])],
                   [cases.P, ("grep", [("Regex", "method ^(GET|POST)$")]), ("modify", [("Add", "a b")])])


def _decoder(lib):
    for data in _decoder_forms():
        for filters in DECODER_FILTERS:
            run_case(lib, [cases.AP], filters, data)
    # the same framing spelled with array16 / array32 headers: decodable for the reference, refused -- loudly -- here
    rec = util.event(1700000000, 1, [(b"log", util.mp_str(b"x"))])
    inner = rec[2:]                                                          # ts + meta + body of a v2 event
    for wide in (b"\xdc\x00\x02" + rec[1:], b"\xdd\x00\x00\x00\x02" + rec[1:], b"\x92\xdc\x00\x02" + inner, b"\x92\xdd\x00\x00\x00\x02" + inner):
        for data in (wide, rec + wide + rec):
            ctx = pkg.Context(0, lib=lib)
            with pytest.raises(pkg.FlbGpuError, match="array16/array32"):
                ctx.filter("grep", [("Regex", "log x")]).cb(data)


def test_degenerate_modify_rules_are_refused(sim_lib, ref_available):
    """Hard_copy X X / Hard_rename X X: the reference sizes the new map wrongly and writes a malformed record"""
    for rule in ("Hard_copy", "Hard_rename"):
        ctx = pkg.Context(0, lib=sim_lib)
        with pytest.raises(pkg.FlbGpuError, match="malformed map"):
            ctx.filter("modify", [(rule, "k2 k2")])
        util.Ref().filter("modify", [(rule, "k2 k2")])          # accepted there


def _truncated_tails(lib):
    """a chunk cut at every byte of its last event: grep / modify call it a clean end exactly when msgpack-c's
    streaming parser eats the whole tail (header bytes, complete length fields, complete payloads)"""
    S = util.mp_str
    head = util.chunk_from_lines(util.apache_lines(6, seed=41))
    last = util.event(1700000100, 5, [(b"log", S(b"POST /cut HTTP/1.1 " + b"x" * 40)), (b"n", b"\xcd\x12\x34"), (b"b", b"\xc4\x03abc"), (b"e", b"\xc7\x02\x05hi"),
                                      (b"a", b"\x92\x01\xa0"), (b"m", b"\xde\x00\x01" + S(b"k") + b"\xcb" + struct.pack(">d", 1.5)), (b"s", b"\xda\x00\x04long")],
                      meta=b"\x81" + S(b"t") + b"\xd6\x01abcd")
    for cut in range(0, len(last) + 1):
        data = head + last[:cut]
        for filters in ([("grep", [("Exclude", "log GET")])], [("modify", [("Condition", "Key_value_matches log GET"), ("Add", "m 1")])], [cases.P]):
            run_case(lib, [cases.AP], filters, data)


def test_truncated_tails_hostsim(sim_lib, ref_available):
    _truncated_tails(sim_lib)


@pytest.mark.gpu
def test_truncated_tails_gpu(gpu_lib, ref_available):
    _truncated_tails(gpu_lib)


def test_decoder_forms_hostsim(sim_lib, ref_available):
    _decoder(sim_lib)


@pytest.mark.gpu
def test_decoder_forms_gpu(gpu_lib, ref_available):
    _decoder(gpu_lib)


def _sliced(lib, monkeypatch, n_lines, reps, slice_mb):
    monkeypatch.setenv("FLBGPU_SLICE_MB", str(slice_mb))
    block = util.chunk_from_lines(util.apache_lines(n_lines, seed=33))
    chunk = block * reps
    for name in ("north_star_chain", "grep_regex", "parser_modify_recmod"):
        case = [c for c in cases.CASES if c[0] == name][0]
        run_case(lib, case[1], case[2], chunk)
    # a chunk cut in the middle of a record, and one with garbage in the middle
    case = [c for c in cases.CASES if c[0] == "north_star_chain"][0]
    run_case(lib, case[1], case[2], chunk[:len(chunk) - 37])
    run_case(lib, case[1], case[2], chunk[:len(block) * 2] + b"\xc1garbage" + chunk[len(block) * 2:])


def test_sliced_pipeline_hostsim(sim_lib, ref_available, monkeypatch):
    """several slices per call: slice boundaries fall inside records"""
    _sliced(sim_lib, monkeypatch, 4000, 6, 1)


@pytest.mark.gpu
def test_sliced_pipeline_gpu(gpu_lib, ref_available, monkeypatch):
    _sliced(gpu_lib, monkeypatch, 4000, 6, 1)


@pytest.mark.gpu
def test_large_chunk_gpu(gpu_lib, ref_available):
    """more than one emission range (>512 K records) and more than one upload piece"""
    block = util.chunk_from_lines(util.apache_lines(20000, seed=34))
    case = [c for c in cases.CASES if c[0] == "north_star_chain"][0]
    run_case(gpu_lib, case[1], case[2], block * 30)


def _speculation(lib, monkeypatch):
    """The streaming path speculates on the previous call's chunk-level verdicts: alternate chunks whose
    verdicts differ (grep excludes something / nothing, modify changes something / nothing) on ONE
    chain object and check every call, in both the streaming and the classic form."""
    monkeypatch.setenv("FLBGPU_SLICE_MB", "1")
    lines = util.apache_lines(6000, seed=35)
    gets = [l for l in lines if b'"GET ' in l]
    mixed = util.chunk_from_lines(lines)
    only_get = util.chunk_from_lines(gets)
    has_env = b"".join(util.event(1700000000 + i, 0, [(b"log", util.mp_str(l)), (b"env", util.mp_str(b"x"))]) for i, l in enumerate(gets))
    filters = [("grep", [("Regex", "log GET")]), ("modify", [("Add", "env prod")])]
    for stream, slice_mb in (("1", "1"), ("0", "1"), ("1", "128")):          # streaming slices, classic two-pass, small-chunk form
        monkeypatch.setenv("FLBGPU_STREAM", stream)
        monkeypatch.setenv("FLBGPU_SLICE_MB", slice_mb)
        ctx = pkg.Context(0, lib=lib)
        chain = ctx.chain([ctx.filter(p, props) for p, props in filters])
        for chunk in (mixed, only_get, has_env, mixed, mixed, has_env, only_get, only_get):
            ref = util.Ref()
            for p, props in filters:
                ref.filter(p, props)
            assert chain.do(chunk) == ref.chain_do(chunk)


def test_streaming_speculation_hostsim(sim_lib, ref_available, monkeypatch):
    _speculation(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_streaming_speculation_gpu(gpu_lib, ref_available, monkeypatch):
    _speculation(gpu_lib, monkeypatch)


def _fused_refusal_forms(lib, monkeypatch):
    """A parser whose input an earlier filter of the chain made: the fused chain refuses, and each of its three forms
    (small, streaming, two-pass) hands the call to the filter-by-filter form.  Two calls per chain object; the result is the
    per-filter callbacks' every time."""
    for name in ("docker_then_inner_json", "set_then_parse"):
        _, parsers, filters, mk = [c for c in cases.CASES if c[0] == name][0]
        block = mk()
        chunk = block * ((3 << 20) // len(block) + 1)
        ctx = pkg.Context(0, lib=lib)
        for kw in parsers:
            ctx.parser(**kw)
        want = per_filter([ctx.filter(p, props) for p, props in filters], chunk)
        for env in ({}, {"FLBGPU_SMALL_MB": "0", "FLBGPU_SLICE_MB": "1"}, {"FLBGPU_STREAM": "0"}):     # small, streaming, two-pass
            for k in ("FLBGPU_SMALL_MB", "FLBGPU_SLICE_MB", "FLBGPU_STREAM"):
                monkeypatch.delenv(k, raising=False)
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            chain = ctx.chain([ctx.filter(p, props) for p, props in filters])
            for _ in range(2):
                assert chain.do(chunk) == want, (name, env)
                assert chain.stats().error_bits == 1, (name, env)       # FLBGPU_E_FIELDS: what the fused form refused


def test_fused_refusal_forms_hostsim(sim_lib, monkeypatch):
    _fused_refusal_forms(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_fused_refusal_forms_gpu(gpu_lib, monkeypatch):
    _fused_refusal_forms(gpu_lib, monkeypatch)


def _json_sliced(lib, monkeypatch):
    monkeypatch.setenv("FLBGPU_SLICE_MB", "1")
    chunk = util.chunk_from_lines(util.json_lines(20000, seed=36))
    case = [c for c in cases.CASES if c[0] == "json_chain_config1"][0]
    run_case(lib, case[1], case[2], chunk)
    run_case(lib, case[1], case[2], chunk[:len(chunk) - 11])


def test_json_sliced_hostsim(sim_lib, ref_available, monkeypatch):
    _json_sliced(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_json_sliced_gpu(gpu_lib, ref_available, monkeypatch):
    _json_sliced(gpu_lib, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("name,maker", [("json_chain_config1", lambda: util.json_lines(100000, seed=0xF1B1 + 2)),
                                        ("north_star_chain", lambda: util.apache_lines(100000, seed=0xF1B1 + 1))])
def test_full_size_tiling_gpu(name, maker, gpu_lib, ref_available):
    """BASELINE.json's full size (10 M events, the bench's own data): records are independent, so the
    result of a chunk tiled k times is the block's result tiled k times -- and the block's result is
    checked against the reference."""
    case = [c for c in cases.CASES if c[0] == name][0]
    block = util.chunk_from_lines(maker())
    reps = 100
    ctx = pkg.Context(0, lib=gpu_lib)
    ref = util.Ref()
    for kw in case[1]:
        ctx.parser(**kw); ref.parser(**kw)
    fs = [ctx.filter(p, props) for p, props in case[2]]
    for p, props in case[2]:
        ref.filter(p, props)
    chain = ctx.chain(fs)
    want = ref.chain_do(block)
    one = chain.do(block)
    assert one == want
    big = block * reps
    r, out = chain.do(big)
    del big
    assert r == want[0] and len(out) == len(want[1]) * reps
    n = len(want[1])
    for k in range(reps):
        assert out[k * n:(k + 1) * n] == want[1], "tile %d differs" % k
    st = chain.stats()
    assert 100000 * reps <= st.records_in <= 100000 * reps * 1.001      # index entries: records + the rare kept false candidates


def _deep_nesting(lib):
    """msgpack-c's unpacker holds 32 open containers (MSGPACK_EMBED_STACK_SIZE): an event nested deeper ends the decodable part of
    a chunk for every filter like a malformed byte does -- whether it came in with the chunk or a parser of the same chain made it."""
    S = util.mp_str
    def deep(n, inner=b"\x90"):
        return b"\x91" * n + inner
    # in the input chunk, at every position, for every plugin
    for filt in [("grep", [("Regex", "a x")]), ("grep", [("Exclude", "a y")]), ("modify", [("Add", "env prod")]), ("record_modifier", [("Record", "c d")]),
                 ("parser", [("Key_Name", "a"), ("Parser", "json")])]:
        for depth in (29, 30, 31):
            for pos in (0, 1, 3):
                for inner in (b"\x90", b"\x80", b"\x01"):
                    evs = [util.event(1700000000 + i, 0, [(b"a", S(b"x" if i % 2 else b"y"))]) for i in range(3)]
                    evs.insert(pos, util.event(1700000100, 0, [(b"a", S(b"x")), (b"n", deep(depth, inner))]))
                    chunk = b"".join(evs)
                    ref = util.Ref(); ref.parser(**cases.JS); ref.filter(*filt)
                    ctx = pkg.Context(0, lib=lib); ctx.parser(**cases.JS)
                    assert ctx.chain([ctx.filter(*filt)]).do(chunk) == ref.chain_do(chunk), (filt, depth, pos, inner)
    # metadata nests one level further down
    for depth in (28, 29, 30):
        evs = [util.event(1700000000 + i, 0, [(b"a", S(b"x"))]) for i in range(2)]
        evs.insert(1, util.event(1700000100, 0, [(b"a", S(b"x"))], meta=b"\x81" + S(b"m") + deep(depth)))
        chunk = b"".join(evs)
        ref = util.Ref(); ref.filter("modify", [("Add", "env prod")])
        ctx = pkg.Context(0, lib=lib)
        assert ctx.chain([ctx.filter("modify", [("Add", "env prod")])]).do(chunk) == ref.chain_do(chunk), depth
    # made by the JSON parser of the chain: the parser takes one level more than the filters behind it decode
    for levels in (28, 29, 30, 31, 32):
        for inner in (b"", b"1", b"{}"):
            line = b'{"level":"warn","nested":' + b"[" * levels + inner + b"]" * levels + b"}"
            lines = util.json_lines(40, seed=3) + [line] + util.json_lines(40, seed=4)
            chunk = util.chunk_from_lines(lines)
            for filters in ([cases.PJ, ("grep", [("Regex", "level ^(warn|error)$")]), ("modify", [("Add", "env prod")])],
                            [cases.PJ, ("record_modifier", [("Record", "c d")])], [cases.PJ]):
                ref = util.Ref(); ref.parser(**cases.JS)
                ctx = pkg.Context(0, lib=lib); ctx.parser(**cases.JS)
                for p, props in filters:
                    ref.filter(p, props)
                assert ctx.chain([ctx.filter(p, props) for p, props in filters]).do(chunk) == ref.chain_do(chunk), (levels, inner, filters)


def test_deep_nesting_hostsim(sim_lib, ref_available):
    _deep_nesting(sim_lib)


@pytest.mark.gpu
def test_deep_nesting_gpu(gpu_lib, ref_available):
    _deep_nesting(gpu_lib)
