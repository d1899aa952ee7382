"""f1: filter_rewrite_tag (plugins/filter_rewrite_tag/rewrite_tag.c) -- the result chunk and what goes to the emitter, against
the reference's own plugin (oracle/_ref: in_emitter_add_record() is the harness's log)."""
import struct

import pytest

import cases
import util

pkg = util.pkg
S = util.mp_str


def run(lib, rules, chunk, tag="app.web.x", parsers=(), before=(), after=(), fail_after=-1):
    ref = util.Ref()
    ref.emit_reset(fail_after)
    ctx = pkg.Context(0, lib=lib)
    for kw in parsers:
        ref.parser(**kw); ctx.parser(**kw)
    fs = []
    for p, props in list(before) + [("rewrite_tag", rules)] + list(after):
        ref.filter(p, props)
        fs.append(ctx.filter(p, props))
    want = ref.chain_do(chunk, tag=tag)
    want_emit = ref.emitted_grouped()
    got = ctx.chain(fs).do(chunk, tag=tag)
    got_emit = fs[len(before)].emitted()
    return got, got_emit, want, want_emit


RULES = [
    [("Rule", '$log "^[0-9.]+ .*(GET|POST)" new.$TAG.$1.$TAG[0].$TAG[1] false'), ("Rule", "$log HEAD other true")],
    [("Rule", "$log PUT put.$0 true")],                                   # no capture groups: not even $0 (flb_regex_do)
    [("Rule", "$log (PUT) put.$0.$1.$2.$12 true")],                       # whole match, a group, groups that are not there
    [("Rule", "log ^\\S+ plain.key true")],                               # a key without '$'
    [("Rule", "$nokey . never false")],
    [("Rule", "$log . all.$TAG[7].$TAG[2]x$TAG false")],                  # a part that is not there; $TAG followed by text
    [("Rule", "$log . $TAG[0 false")],                                    # unterminated bracket
    [("Rule", "$log . t.$TAG$0 false")],                                  # the '$' right behind $TAG is literal text
    [("Rule", "$log . k.$log. false")],                                   # a one-character tail behind a key is dropped
    [("Rule", "$log . k.$nokey.z false")],
    [("Rule", "$log . prefix$ false")],                                   # a '$' at the very end is dropped
    [("Rule", "$TAG . x false")],                                         # the key is not a record key: never matches
    [("Rule", "$log . keep.maybe maybe")],                                # not a boolean: keeps nothing
    [("Rule", "$log GET first true"), ("Rule", "$log . second false")],
]


def _rules(lib):
    chunk = util.chunk_from_lines(util.apache_lines(80, seed=12))
    for rules in RULES:
        for tag in ("app.web.x", "nodots", "a.", ".b", ""):
            if tag == "":
                continue                      # (flb_filter_do never runs with an empty tag)
            got, ge, want, we = run(lib, rules, chunk, tag=tag)
            assert got == want, (rules, tag)
            assert ge == we, (rules, tag, [(t, len(b), n) for t, b, n in ge], [(t, len(b), n) for t, b, n in we])


def _values(lib):
    """tag templates over record keys of every type ra_translate_keymap() prints"""
    evs = []
    for i in range(12):
        evs.append(util.event(1700000000 + i, i, [
            (b"s", S(b"str%d" % (i % 3))), (b"i", bytes([i])), (b"neg", b"\xd0" + struct.pack("b", -i - 1)), (b"big", b"\xcf" + struct.pack(">Q", 2 ** 63 + i)),
            (b"t", b"\xc3"), (b"f", b"\xc2"), (b"nil", b"\xc0"), (b"bin", b"\xc4\x03\x00\xab" + bytes([i])),
            (b"arr", b"\x92\x01\x02"), (b"m", b"\x82" + S(b"a") + S(b"in%d" % (i % 2)) + S(b"n") + b"\x81" + S(b"d") + b"\x2a"),
            (b"log", S(b"line %d" % i))]))
    chunk = b"".join(evs)
    for tmpl in ("v.$s", "v.$i.$neg", "v.$big", "v.$t.$f.$nil", "v.$bin", "v.$arr.x", "v.$m['a']", "v.$m['n']['d']", "v.$m['zz'].y", "v.$m['a']['b']"):
        got, ge, want, we = run(lib, [("Rule", "$log . %s false" % tmpl)], chunk)
        assert got == want and ge == we, (tmpl, ge[:2], we[:2])
    # a rule key under a map; a value that is not a string never matches
    for key in ("$m['a']", "$m['n']['d']", "$i", "$m"):
        got, ge, want, we = run(lib, [("Rule", "%s ^in1$ sub.$0 true" % key)], chunk)
        assert got == want and ge == we, key
    # a float or a whole map in the tag: refused loudly (snprintf("%f") / JSON text are not restated)
    fl = b"".join(util.event(1700000000, 0, [(b"log", S(b"x")), (b"d", b"\xcb" + struct.pack(">d", 1.5))]) for _ in range(3))
    ctx = pkg.Context(0, lib=lib)
    f = ctx.filter("rewrite_tag", [("Rule", "$log . v.$d false")])
    with pytest.raises(pkg.FlbGpuError):
        ctx.chain([f]).do(fl)


def _in_chains(lib):
    """behind a parser (the record is re-encoded as that filter left it), before other filters, with routing"""
    chunk = util.chunk_from_lines(util.apache_lines(200, seed=5) + [b"garbage line"] * 3)
    AP = cases.AP
    pf = ("parser", [("Key_Name", "log"), ("Parser", "apache"), ("Reserve_Data", "On")])
    for rules in ([("Rule", "$method ^(GET|PUT)$ by.$method.$code false")], [("Rule", "$code ^5 errors true"), ("Rule", "$log garbage raw.$TAG[1] false")]):
        got, ge, want, we = run(lib, rules, chunk, parsers=[AP], before=[pf])
        assert got == want and ge == we, rules
        got, ge, want, we = run(lib, rules, chunk, parsers=[AP], before=[pf], after=[("modify", [("Add", "env prod")]), ("grep", [("Exclude", "method POST")])])
        assert got == want and ge == we, rules
        got, ge, want, we = run(lib, rules, chunk, parsers=[AP], before=[("grep", [("Regex", "log HTTP")]), pf], after=[("record_modifier", [("Record", "h n1")])])
        assert got == want and ge == we, rules
    # nothing matches: NOTOUCH, nothing emitted
    got, ge, want, we = run(lib, [("Rule", "$log ^nothing$ x false")], chunk)
    assert got == want == (2, None) and ge == we == []
    # two rewrite_tag filters in one chain: run filter by filter
    ref = util.Ref(); ref.emit_reset()
    ctx = pkg.Context(0, lib=lib)
    a = [("Rule", "$log GET g.$TAG true")]; b = [("Rule", "$log POST p.$TAG false")]
    ref.filter("rewrite_tag", a); ref.filter("rewrite_tag", b)
    fa, fb = ctx.filter("rewrite_tag", a), ctx.filter("rewrite_tag", b)
    assert ctx.chain([fa, fb]).do(chunk, tag="t.u") == ref.chain_do(chunk, tag="t.u")
    ours = {}
    for t, d, n in fa.emitted() + fb.emitted():
        ours[t] = (ours.get(t, (b"", 0))[0] + d, ours.get(t, (b"", 0))[1] + n)
    assert [(t, d, n) for t, (d, n) in ours.items()] == ref.emitted_grouped()


def _odd_chunks(lib):
    """events the decoder steps over travel with the next record; a chunk that does not decode to its end"""
    lines = util.apache_lines(9, seed=8)
    evs = [util.event(1700000000 + i, 0, [(b"log", S(l))]) for i, l in enumerate(lines)]
    neg = util.event(-5 & 0xffffffff, 0, [(b"log", S(b"GET negative time"))])      # skipped by flb_log_event_decoder_next
    for pos in (0, 3, 9):
        c = list(evs); c.insert(pos, neg); c.insert(pos, neg)
        chunk = b"".join(c)
        for rules in ([("Rule", "$log . all.$TAG false")], [("Rule", "$log GET g true")]):
            got, ge, want, we = run(lib, rules, chunk)
            assert got == want and ge == we, (pos, rules)
            got, ge, want, we = run(lib, rules, chunk, before=[("modify", [("Add", "a b")])])
            assert got == want and ge == we, (pos, rules, "behind modify")
    whole = b"".join(evs)
    for cut in (1, 5, 13, 40):
        chunk = whole + evs[0][:cut]
        got, ge, want, we = run(lib, [("Rule", "$log . all.$TAG false")], chunk)
        assert got == want and ge == we, cut
    chunk = whole + b"\xc1garbage"
    got, ge, want, we = run(lib, [("Rule", "$log . all.$TAG false")], chunk)
    assert got == want and ge == we


def _config(lib):
    ctx = pkg.Context(0, lib=lib)
    for props in ([("Rule", "$log x")], [("Rule", "$log x y")], [("Rule", "$log ( y false")], [("Rule", "$log x y false"), ("Emitter_Storage.type", "disk")],
                  [("Rule", "$log x y false"), ("Nope", "1")]):
        with pytest.raises(pkg.FlbGpuError):
            ctx.filter("rewrite_tag", props)
        with pytest.raises(Exception):
            util.Ref().filter("rewrite_tag", props)
    ctx.filter("rewrite_tag", [("Rule", "$log x y false extra words"), ("Emitter_Name", "e"), ("Emitter_Mem_Buf_Limit", "5M"), ("Emitter_Storage.type", "filesystem")])
    util.Ref().filter("rewrite_tag", [("Rule", "$log x y false extra words"), ("Emitter_Name", "e"), ("Emitter_Mem_Buf_Limit", "5M"), ("Emitter_Storage.type", "filesystem")])


def _forms(lib, monkeypatch):
    """the three call forms (small chunk, streaming slices, whole chunk) cut the same re-tagged stream"""
    chunk = util.chunk_from_lines(util.apache_lines(30000, seed=21, nginx=True) + [b"junk"] * 5)
    pf = ("parser", [("Key_Name", "log"), ("Parser", "nginx")])
    rules = [("Rule", "$code ^5 errors.$method false"), ("Rule", "$method ^(PUT|HEAD)$ audit.$1.$TAG[1] true")]
    for env in ({}, {"FLBGPU_SMALL_MB": "0", "FLBGPU_SLICE_MB": "1"}, {"FLBGPU_SMALL_MB": "0", "FLBGPU_STREAM": "0"}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        for rep in range(2):                     # the second call speculates on the verdicts of the first
            got, ge, want, we = run(lib, rules, chunk, parsers=[cases.NG], before=[pf], after=[("record_modifier", [("Record", "h n1")])])
            assert got == want and ge == we, (env, rep)
        got, ge, want, we = run(lib, [("Rule", "$code ^9 never false")], chunk, parsers=[cases.NG], before=[pf])
        assert got == want and ge == we == [], env


def test_forms_hostsim(sim_lib, ref_available, monkeypatch): _forms(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_forms_gpu(gpu_lib, ref_available, monkeypatch): _forms(gpu_lib, monkeypatch)


def test_rules_hostsim(sim_lib, ref_available): _rules(sim_lib)
def test_values_hostsim(sim_lib, ref_available): _values(sim_lib)
def test_in_chains_hostsim(sim_lib, ref_available): _in_chains(sim_lib)
def test_odd_chunks_hostsim(sim_lib, ref_available): _odd_chunks(sim_lib)
def test_config_hostsim(sim_lib, ref_available): _config(sim_lib)


@pytest.mark.gpu
def test_rules_gpu(gpu_lib, ref_available): _rules(gpu_lib)
@pytest.mark.gpu
def test_values_gpu(gpu_lib, ref_available): _values(gpu_lib)
@pytest.mark.gpu
def test_in_chains_gpu(gpu_lib, ref_available): _in_chains(gpu_lib)
@pytest.mark.gpu
def test_odd_chunks_gpu(gpu_lib, ref_available): _odd_chunks(gpu_lib)


@pytest.mark.gpu
def test_large_gpu(gpu_lib, ref_available):
    """a chunk of several slices: per-tag buffers equal the reference's, record for record"""
    chunk = util.chunk_from_lines(util.apache_lines(60000, seed=77))
    got, ge, want, we = run(gpu_lib, [("Rule", '$log "^\\S+ \\S+ \\S+ \\[[^\\]]*\\] \\"(\\S+)" m.$1.$TAG[1] false'), ("Rule", "$log . rest true")], chunk, tag="a.b")
    assert got == want and ge == we
