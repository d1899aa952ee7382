"""The split evaluation of a chain `parser(json), then filters that are not grep`.

The head launch parses every record, the tail launch runs the filters behind the parser, and the records the stage-2
JSON walker cannot take (nested values, non-ASCII text, exponents, more than 16 fields, lines that are not JSON) go to a
follow-up launch that runs the whole chain on them.  On the device that follow-up launch runs beside the tail launch, on a
second stream, so either may finish first; the tail must only ever touch the records the head listed for it.  The CPU
emulation runs the two in either order (FLBGPU_SIM_DEFER_FIRST=1: the put-off records first), and each order has to give
the oracle's bytes, return code and metric text.

GPU form: the same chains on chunks of a few hundred thousand records in each call form (small, streaming, two-pass);
the expected result is the block's, checked against the oracle, tiled."""
import random
import re

import pytest

import cases
import l2m_cases
import util

pkg = util.pkg
TS = re.compile(r"^\S+Z ", re.M)

# the kinds of line in a block, in the order they cycle; all but "plain" are handed to the follow-up launch
KINDS = ("plain", "nested", "plain", "non_ascii", "exponent", "wide", "not_json", "plain")
HANDED_OVER = {"nested", "non_ascii", "exponent", "wide", "not_json"}


def _line(kind, i, rng):
    level = rng.choice(["info", "warn", "error", "debug"])
    lat = "%.3f" % (rng.random() * 400)
    if kind == "plain":
        return '{"level":"%s","msg":"req %d ok","latency_ms":%s,"status":200,"trace_id":"%08x"}' % (level, i, lat, rng.getrandbits(32))
    if kind == "nested":
        return '{"level":"%s","msg":"n%d","kube":{"pod":"p-%d","ports":[80,443]},"latency_ms":%s}' % (level, i, i % 97, lat)
    if kind == "non_ascii":
        return '{"level":"%s","msg":"café ☃ %d","latency_ms":%s,"trace_id":"t"}' % (level, i, lat)
    if kind == "exponent":
        return '{"level":"%s","msg":"e%d","latency_ms":%de-1,"big":2.5E3}' % (level, i, rng.randint(1, 4000))
    if kind == "wide":
        return "{" + ",".join(['"level":"%s"' % level, '"latency_ms":%s' % lat] + ['"f%02d":%d' % (j, i + j) for j in range(18)]) + "}"
    return "not json at all %d" % i


def split_block(n=2048, seed=0x5B1):
    """n JSON lines as events, every kind of KINDS throughout -- the last ones included -- and the kind of each record"""
    rng = random.Random(seed)
    kinds = [KINDS[i % len(KINDS)] for i in range(n)]
    kinds[-3:] = ["wide", "not_json", "nested"]          # a block's last records are handed over too
    chunk = util.chunk_from_lines([_line(k, i, rng).encode("utf-8") for i, k in enumerate(kinds)])
    return chunk, kinds


def _check_block(kinds, chunk):
    """what the generator promises, from the chunk's layout"""
    recs = util.split_records(chunk)
    assert len(recs) == len(kinds)
    assert set(kinds) >= HANDED_OVER | {"plain"}
    for lo in range(0, len(kinds), 256):                 # every 256-record block of the chunk holds handed-over records
        assert HANDED_OVER & set(kinds[lo:lo + 256])
    assert kinds[-1] in HANDED_OVER


L2M_BASE = l2m_cases.BASE
SPLIT_CHAINS = [
    # modify under a condition the lines that are not JSON fail: their rows say "raw, untouched"
    ("modify", [cases.PJ, ("modify", [("Condition", "Key_exists level"), ("Add", "env prod"), ("Rename", "msg message")])], None),
    ("record_modifier", [cases.PJ, ("record_modifier", [("Remove_key", "trace_id")])], None),
    ("record_modifier_record", [cases.PJ, ("record_modifier", [("Record", "cluster c1"), ("Remove_key", "big")])], None),
    ("l2m_counter", [cases.PJ, ("log_to_metrics", L2M_BASE + [("metric_mode", "counter"), ("label_field", "level")])], 1),
    ("l2m_histogram", [cases.PJ, ("log_to_metrics", L2M_BASE + [("metric_mode", "histogram"), ("value_field", "latency_ms"),
                                                                ("label_field", "level")])], 1),
]
FORMS = {"small": {}, "streaming": {"FLBGPU_SMALL_MB": "0", "FLBGPU_SLICE_MB": "1"}, "two_pass": {"FLBGPU_STREAM": "0"}}


def _set_env(monkeypatch, env):
    for k in ("FLBGPU_SMALL_MB", "FLBGPU_SLICE_MB", "FLBGPU_STREAM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("FLBGPU_EVAL_SPLIT", "1")          # the split evaluation, whatever the default


def _checkers(filters):
    out = [util.Oracle()] + ([util.Ref()] if util.have_ref_results() else [])
    for c in out:
        c.parser(**cases.JS)
    return out, [[c.filter(p, props) for p, props in filters] for c in out]


def _run_split(lib, filters, k, chunk, calls=2):
    ctx = pkg.Context(0, lib=lib)
    ctx.parser(**cases.JS)
    fs = [ctx.filter(p, props) for p, props in filters]
    chain = ctx.chain(fs)
    checkers, cfs = _checkers(filters)
    for call in range(calls):                            # the metric table accumulates over calls
        got = chain.do(chunk)
        for c, cf in zip(checkers, cfs):
            assert got == c.chain_do(chunk), (type(c).__name__, call)
            if k is not None:
                assert fs[k].l2m_text() == TS.sub("", c.l2m_text(cf[k])), (type(c).__name__, call)
    return got, fs


@pytest.mark.parametrize("order", ["tail_first", "defer_first"])
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("name,filters,k", SPLIT_CHAINS, ids=[c[0] for c in SPLIT_CHAINS])
def test_split_tail_hostsim(name, filters, k, form, order, sim_lib, monkeypatch):
    chunk, kinds = split_block(600)
    _check_block(kinds, chunk)
    _set_env(monkeypatch, FORMS[form])
    monkeypatch.setenv("FLBGPU_SIM_DEFER_FIRST", "1" if order == "defer_first" else "0")
    _run_split(sim_lib, filters, k, chunk)


@pytest.mark.gpu
@pytest.mark.parametrize("name,filters,k", SPLIT_CHAINS, ids=[c[0] for c in SPLIT_CHAINS])
def test_split_tail_gpu(name, filters, k, gpu_lib, monkeypatch):
    """a few hundred thousand records per call: the tail launch takes long enough for the follow-up launch beside it to
    finish records the tail has not reached"""
    block, kinds = split_block()
    _check_block(kinds, block)
    reps = 160                                           # 327 680 records, about 37 MB
    big = block * reps
    for form, env in FORMS.items():
        _set_env(monkeypatch, dict(env, FLBGPU_SMALL_MB="64") if form == "small" else env)
        one, fs = _run_split(gpu_lib, filters, k, block, calls=1)
        ctx2 = pkg.Context(0, lib=gpu_lib)
        ctx2.parser(**cases.JS)
        fs2 = [ctx2.filter(p, props) for p, props in filters]
        r, out = ctx2.chain(fs2).do(big)
        assert r == one[0], form
        if one[1] is None:
            assert out is None, form
        else:
            n = len(one[1])
            assert len(out) == n * reps, form
            for t in range(reps):
                assert out[t * n:(t + 1) * n] == one[1], (form, "tile %d differs" % t)
        if k is not None:
            a, b = fs[k].l2m_sets(), fs2[k].l2m_sets()
            assert [s[:2] for s in a] == [s[:2] for s in b], form
            for sa, sb in zip(a, b):
                assert sb[2] == sa[2] * reps and sb[4] == [x * reps for x in sa[4]], (form, sa[1])
                assert sb[3] == pytest.approx(sa[3] * reps, rel=1e-9), (form, sa[1])
