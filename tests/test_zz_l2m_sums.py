"""filter_log_to_metrics histogram sums, bit for bit.

The reference adds every observation to its label set's sum in record order, across calls: cmt_metric_hist_sum_add()
computes `new = old + val` in IEEE binary64.  The model here is that loop in Python (`float` addition, starting from the
set's previous sum), and each test compares the bits of the sum flbgpu_l2m_get() returns with it, next to the count, the
buckets and the metric text.  Decimal values make the order of the additions visible in the last bits; so do integer sums
that pass 2^53, signed zeros, infinities and NaN payloads.

On the CPU emulation every case runs with the record loops forwards and backwards (FLBGPU_SIM_ORDER=reverse), the two
extremes of what a GPU schedule may do.  Where the reference build is present, a pin test checks that the reference's own
cmetrics context holds the model's bits for every case and call."""
import ctypes as C
import json
import random
import re
import struct

import msgpack
import pytest

import cases
import l2m_cases
import util
from test_zz_split_tail import FORMS, split_block

pkg = util.pkg
TS = re.compile(r"^\S+Z ", re.M)
BOUNDS = [0.5, 10.0, 1000.0]
HIST = l2m_cases.BASE + [("metric_mode", "histogram"), ("value_field", "v"), ("label_field", "c")] + \
    [("bucket", repr(b)) for b in BOUNDS]
TWO53 = 2 ** 53


def bits(x):
    return struct.pack("<d", x).hex()


def f64_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


# ---------------------------------------------------------------- values: (msgpack bytes, what the reference observes)
def v_f64(x):
    return b"\xcb" + struct.pack(">d", x), x


def v_raw64(u):
    """a float64 given by its bits (NaN payloads, the sign bit)"""
    return b"\xcb" + struct.pack(">Q", u), f64_bits(u)


def v_f32(x):
    b = struct.pack(">f", x)
    return b"\xca" + b, struct.unpack(">f", b)[0]


def v_int(n):
    return l2m_cases._mp(n), float(n)


def v_str(s):
    """a string: sscanf("%lf") of its text; None = converts nothing (the call's previous value is observed)"""
    try:
        x = float(s)
    except ValueError:
        x = None
    return util.mp_str(s.encode()), x


class Model:
    """cmetrics' histogram for one label key: sets in first-seen order, each (count, sum, cumulative buckets)"""

    def __init__(self):
        self.sets = {}

    def observe(self, label, v):
        s = self.sets.setdefault(label, [0, 0.0, [0] * (len(BOUNDS) + 1)])
        s[0] += 1
        s[1] = s[1] + v                                 # cmt_metric_hist_sum_add(): new = old + val
        for i in range(len(BOUNDS) - 1, -1, -1):        # cmt_histogram_observe()
            if v > BOUNDS[i]:
                break
            s[2][i] += 1
        s[2][-1] += 1

    def rows(self):
        return [((k,), c, s, list(b)) for k, (c, s, b) in self.sets.items()]


def compare(f, model, what):
    got = [(s[1], s[2], s[3], s[4]) for s in f.l2m_sets()]
    want = model.rows()
    assert [g[0] for g in got] == [w[0] for w in want], what
    assert [(g[1], g[3]) for g in got] == [(w[1], w[3]) for w in want], what
    assert [bits(g[2]) for g in got] == [bits(w[2]) for w in want], (what, [(g[2], w[2]) for g, w in zip(got, want)])


# ---------------------------------------------------------------- cases
# A case: (filters, index of the l2m filter, calls); a call: (chunk, [(label, value) observed in record order]).
def plain_call(recs, t0=1700000000):
    """recs: [(label bytes, (msgpack value, observed value or None))] -> one call; None takes the previous value"""
    evs, obs, prev = [], [], 0.0
    for i, (lab, (mp, x)) in enumerate(recs):
        evs.append(util.event(t0 + i, 0, [(b"c", util.mp_str(lab)), (b"v", mp)]))
        prev = prev if x is None else x
        obs.append((lab, prev))
    return b"".join(evs), obs


def _decimal(rng):
    return rng.randrange(0, 400000) / 1000.0            # three decimals


def _spelled(rng):
    r = rng.random()
    if r < 0.55:
        return v_f64(_decimal(rng))
    if r < 0.75:
        return v_str(rng.choice(["%.3f", " %.3f", "+%.3f", "%.3fe-3", "%.3fE2"]) % _decimal(rng))
    if r < 0.8:
        return v_str(rng.choice(["+.5", " 1.5", "1e-3", "0.123", "-.25"]))
    if r < 0.92:
        return v_int(rng.randrange(-5000, 5000))
    return v_f32(_decimal(rng))


def spellings_case(n_sets, seed, per_call=1000):
    rng = random.Random(seed)
    labs = [b"hot"] + [b"s%02d" % i for i in range(n_sets - 1)]
    calls = []
    for _ in range(3):
        recs = [(labs[0] if rng.random() < 0.5 else rng.choice(labs), _spelled(rng)) for _ in range(per_call)]
        calls.append(plain_call(recs))
    return [("log_to_metrics", HIST)], 0, calls


def cross_call_case():
    """the issue's reproduction: one set, 1000 float64 values with three decimals, three calls"""
    rng = random.Random(1)
    return [("log_to_metrics", HIST)], 0, [plain_call([(b"a", v_f64(_decimal(rng))) for _ in range(1000)]) for _ in range(3)]


def two53_case():
    big = [(b"in_call", v_int(TWO53)), (b"in_call", v_int(1)), (b"in_call", v_int(1)),
           (b"neg", v_int(-TWO53 + 1)), (b"neg", v_int(-1)), (b"neg", v_int(-1)), (b"neg", v_int(-1))]
    return [("log_to_metrics", HIST)], 0, [
        plain_call([(b"across", v_int(TWO53))] + big + [(b"f64", v_f64(float(TWO53 - 2)))]),
        plain_call([(b"across", v_int(1)), (b"across", v_int(1))] + [(b"f64", v_int(1))] * 3),
        plain_call([(b"across", v_int(1)), (b"in_call", v_int(3)), (b"f64", v_f64(1.0))]),
    ]


NAN_NEG_PAYLOAD = 0xfff8000000000123
NAN_POS_PAYLOAD = 0x7ff8000000000456


def specials_case():
    """(one NaN per set: which of two NaN operands an addition passes on is up to the compiler, in the reference too)"""
    inf, ninf = float("inf"), float("-inf")
    c1 = [(b"negzero", v_f64(-0.0)), (b"poszero", v_f64(0.0)), (b"negzero", v_f64(-0.0)), (b"mixzero", v_f64(-0.0)),
          (b"mixzero", v_f64(0.0)), (b"inf", v_f64(1.5)), (b"inf", v_f64(inf)), (b"inf", v_f64(2.25)),
          (b"infs", v_f64(inf)), (b"infs", v_f64(ninf)), (b"nan", v_f64(1.0)), (b"nan", v_raw64(NAN_NEG_PAYLOAD)),
          (b"nan", v_f64(2.5)), (b"nan2", v_raw64(NAN_POS_PAYLOAD)), (b"nan2", v_f64(3.0)),
          (b"ninf", v_f64(ninf)), (b"ninf", v_f64(0.1))]
    c2 = [(b"negzero", v_f64(-0.0)), (b"inf", v_f64(ninf)), (b"nan", v_f64(0.1)), (b"ninf", v_f64(ninf)), (b"poszero", v_f64(-0.0))]
    return [("log_to_metrics", HIST)], 0, [plain_call(c1), plain_call(c2)]


def fixup_case():
    """value texts that convert nothing observe the call's previous value, through the follow-up launch"""
    rng = random.Random(3)
    calls = []
    for c in range(3):
        recs = []
        for i in range(600):
            lab = rng.choice([b"x", b"y", b"z"])
            if (c == 0 and i < 3) or rng.random() < 0.2:
                recs.append((lab, v_str(rng.choice(["fast", "", "-", ".", "x1", " \t"]))))
            else:
                recs.append((lab, v_f64(_decimal(rng)) if rng.random() < 0.6 else v_str("%.3f" % _decimal(rng))))
        calls.append(plain_call(recs))
    return [("log_to_metrics", HIST)], 0, calls


def grouped_case():
    """group markers and negative-timestamp events: skipped by the event decoder, observed by log_to_metrics"""
    rng = random.Random(4)
    calls = []
    for c in range(2):
        evs, obs = [], []
        for g in range(8):
            def add(sec, lab, val):
                mp, x = val
                evs.append(util.event(sec, 0, [(b"c", util.mp_str(lab)), (b"v", mp)]))
                obs.append((lab, x))
            add(0xffffffff, b"marker", v_f64(_decimal(rng)))
            for i in range(rng.randrange(5, 60)):
                add(1700000000 + i, rng.choice([b"a", b"marker"]), v_f64(_decimal(rng)))
            if g % 2 == 0:
                add(0x80000005, b"a", v_f64(_decimal(rng)))
            evs.append(util.event(0xfffffffe, 0, []))
        calls.append((b"".join(evs), obs))
    return [("log_to_metrics", HIST)], 0, calls


def revision_case():
    """grep in front of log_to_metrics: while grep drops nothing it hands the chunk on untouched and log_to_metrics
    observes the group markers in it; once it drops a record it hands on the decoded events it keeps, markers gone.  The
    chain evaluates under an assumed verdict and re-runs when it was wrong, so a record observed by the first pass may be
    missing from the second."""
    rng = random.Random(6)
    calls = []
    for drop in (False, True, False, True):
        evs, obs = [], []
        for g in range(6):
            x = _decimal(rng)
            evs.append(util.event(0xffffffff, 0, [(b"c", util.mp_str(b"a")), (b"v", v_f64(x)[0]), (b"k", util.mp_str(b"y"))]))
            if not drop:
                obs.append((b"a", x))
            for i in range(40):
                x, lab = _decimal(rng), rng.choice([b"a", b"b"])
                keep = not (drop and i == 7)
                evs.append(util.event(1700000000 + i, 0, [(b"c", util.mp_str(lab)), (b"v", v_f64(x)[0]),
                                                          (b"k", util.mp_str(b"y" if keep else b"n"))]))
                if keep:
                    obs.append((lab, x))
        calls.append((b"".join(evs), obs))
    return [("grep", [("Regex", "k ^y$")]), ("log_to_metrics", HIST)], 1, calls


def split_case():
    """parser(json) then log_to_metrics as the split evaluation: the records the head launch puts off are observed by a
    follow-up launch beside the tail launch"""
    chunk, kinds = split_block(600)
    obs = []
    for off, n in util.split_records(chunk):
        body = msgpack.unpackb(chunk[off:off + n], raw=True, strict_map_key=False)[1]
        try:
            rec = json.loads(body[b"log"])
        except ValueError:
            continue                                    # not JSON: kept as it is, no value field
        obs.append((rec["level"].encode(), float(rec["latency_ms"])))
    props = l2m_cases.BASE + [("metric_mode", "histogram"), ("value_field", "latency_ms"), ("label_field", "level")] + \
        [("bucket", repr(b)) for b in BOUNDS]
    return [cases.PJ, ("log_to_metrics", props)], 1, [(chunk, obs)] * 3


CASES = {
    "cross_call": cross_call_case,
    "spellings_hot": lambda: spellings_case(1, 11),
    "spellings_64": lambda: spellings_case(64, 12),
    "two53": two53_case,
    "specials": specials_case,
    "fixup": fixup_case,
    "grouped": grouped_case,
    "revision": revision_case,
    "split": split_case,
}


def _env(monkeypatch, form, order=None):
    for k in ("FLBGPU_SMALL_MB", "FLBGPU_SLICE_MB", "FLBGPU_STREAM", "FLBGPU_EVAL_SPLIT", "FLBGPU_SIM_ORDER"):
        monkeypatch.delenv(k, raising=False)
    for k, v in FORMS[form].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("FLBGPU_EVAL_SPLIT", "1")
    if order:
        monkeypatch.setenv("FLBGPU_SIM_ORDER", order)


def run_case(lib, name, oracle=True):
    filters, k, calls = CASES[name]()
    ctx = pkg.Context(0, lib=lib)
    if filters[0] is cases.PJ:
        ctx.parser(**cases.JS)
    fs = [ctx.filter(p, props) for p, props in filters]
    chain = ctx.chain(fs)
    orc = None
    if oracle:
        orc = util.Oracle()
        if filters[0] is cases.PJ:
            orc.parser(**cases.JS)
        ofs = [orc.filter(p, props) for p, props in filters]
    model = Model()
    for i, (chunk, obs) in enumerate(calls):
        got = chain.do(chunk)
        for lab, x in obs:
            model.observe(lab, x)
        compare(fs[k], model, (name, i))
        if orc is not None:
            assert got == orc.chain_do(chunk), (name, i)
            assert fs[k].l2m_text() == TS.sub("", orc.l2m_text(ofs[k])), (name, i)


@pytest.mark.parametrize("order", ["forward", "reverse"])
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("name", list(CASES))
def test_l2m_sum_hostsim(name, form, order, sim_lib, monkeypatch):
    _env(monkeypatch, form, order)
    run_case(sim_lib, name)


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("name", list(CASES))
def test_l2m_sum_gpu(name, form, gpu_lib, monkeypatch):
    _env(monkeypatch, form)
    run_case(gpu_lib, name, oracle=False)


# ---------------------------------------------------------------- the model against the reference
def _ref_sums(ref, f):
    """{label tuple: (count, sum)} of the reference's own cmetrics context (cmt_encode_msgpack_create)"""
    L = ref.L
    L.flbref_l2m_cmt_msgpack.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    out, n = C.c_void_p(), C.c_size_t()
    assert L.flbref_l2m_cmt_msgpack(f, C.byref(out), C.byref(n)) == 0
    raw = C.string_at(out.value, n.value)
    L.flbref_cfree(out)
    m = msgpack.unpackb(raw, raw=True, strict_map_key=False)
    vals = m[b"metrics"][0][b"values"]
    return [(tuple(v[b"labels"]), v[b"histogram"][b"count"], v[b"histogram"][b"sum"]) for v in vals]


@pytest.mark.parametrize("name", list(CASES))
def test_l2m_sum_model_matches_reference(name):
    if not util.have_ref():
        pytest.skip("the reference build (oracle/_ref) is absent")
    filters, k, calls = CASES[name]()
    ref = util.Ref()
    if filters[0] is cases.PJ:
        ref.parser(**cases.JS)
    rfs = [ref.filter(p, props) for p, props in filters]
    model = Model()
    for i, (chunk, obs) in enumerate(calls):
        ref.chain_do(chunk)
        for lab, x in obs:
            model.observe(lab, x)
        got = sorted((l, c, bits(s)) for l, c, s in _ref_sums(ref, rfs[k]))
        want = sorted((l, c, bits(s)) for l, c, s, _ in model.rows())
        assert got == want, (name, i)


# ---------------------------------------------------------------- flbgpu_l2m_put / flbgpu_l2m_reset
def label_hash(*labels):
    """the hash a set is found by (dev_chain.cuh f_l2m: FNV-1a over the label values run together, as cmetrics does)"""
    h = 1469598103934665603
    for b in b"".join(labels):
        h = ((h ^ b) * 1099511628211) & 0xffffffffffffffff
    return h | 1


def _put_reset(lib):
    ctx = pkg.Context(0, lib=lib)
    f = ctx.filter("log_to_metrics", HIST)
    chain = ctx.chain([f])
    rng = random.Random(9)
    model = Model()
    starts = [(b"dec", 0.1), (b"big", float(TWO53)), (b"negzero", -0.0), (b"int", 7.0), (b"nan", f64_bits(NAN_NEG_PAYLOAD))]
    for lab, s in starts:
        model.sets[lab] = [1, s, [0, 0, 0, 1]]
    f.l2m_replace([(label_hash(lab), (lab,), 1, s, [0, 0, 0, 1]) for lab, s in starts])
    compare(f, model, "put")
    for i in range(3):
        recs = [(b"dec", v_f64(_decimal(rng))) for _ in range(50)] + [(b"big", v_int(1)), (b"big", v_int(1)),
                                                                       (b"negzero", v_f64(-0.0)), (b"int", v_int(5)),
                                                                       (b"nan", v_f64(1.5))]
        chunk, obs = plain_call(recs)
        chain.do(chunk)
        for lab, x in obs:
            model.observe(lab, x)
        compare(f, model, ("after put", i))
    f.l2m_replace([])                                   # flbgpu_l2m_reset(): every set starts again from 0
    model = Model()
    for i in range(2):
        chunk, obs = plain_call([(rng.choice([b"dec", b"int"]), v_f64(_decimal(rng))) for _ in range(300)])
        chain.do(chunk)
        for lab, x in obs:
            model.observe(lab, x)
        compare(f, model, ("after reset", i))


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_l2m_sum_put_reset_hostsim(order, sim_lib, monkeypatch):
    monkeypatch.setenv("FLBGPU_SIM_ORDER", order)
    _put_reset(sim_lib)


@pytest.mark.gpu
def test_l2m_sum_put_reset_gpu(gpu_lib):
    _put_reset(gpu_lib)


# ---------------------------------------------------------------- volume on the GPU
def _volume_calls(n, seed, integers=False):
    """n records per call: one hot set with half of them, 32 others; decimal or integer values"""
    rng = random.Random(seed)
    labs = [b"o%02d" % i for i in range(32)]
    vals = [rng.randrange(0, 10000) for _ in range(4096)]
    out = []
    for c in range(2):
        evs, obs = [], []
        for i in range(n):
            lab = b"hot" if i & 1 else labs[(i >> 1) % 32]
            u = vals[(i * 7 + c) % 4096]
            x = float(u) if integers else u / 1000.0
            evs.append(util.event(1700000000 + (i & 0xffff), 0, [(b"c", util.mp_str(lab)), (b"v", v_f64(x)[0])]))
            obs.append((lab, x))
        out.append((b"".join(evs), obs))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("integers", [False, True], ids=["decimal", "integer"])
@pytest.mark.parametrize("discard", ["off", "on"])
def test_l2m_sum_volume_gpu(discard, integers, gpu_lib):
    """300 000 records a call: the atomics of one hot set meet in every order the schedule makes"""
    ctx = pkg.Context(0, lib=gpu_lib)
    f = ctx.filter("log_to_metrics", HIST + [("discard_logs", discard)])
    chain = ctx.chain([f])
    model = Model()
    for i, (chunk, obs) in enumerate(_volume_calls(300000, 17 + integers, integers)):
        r, out = chain.do(chunk)
        assert r == pkg.FILTER_MODIFIED if discard == "on" else r == pkg.FILTER_NOTOUCH, r
        for lab, x in obs:
            model.observe(lab, x)
        compare(f, model, ("volume", discard, i))
