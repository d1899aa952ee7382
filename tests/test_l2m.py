"""filter_log_to_metrics: metric tables and filter results against the UNMODIFIED reference
(oracle/_ref), on the CPU emulation and on the GPU; plus the cross-rank merge (gloo, world 2)."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import pytest

import l2m_cases
import util

pkg = util.pkg
TS = re.compile(r"^\S+Z ", re.M)


def ref_text(ref, f):
    return TS.sub("", ref.l2m_text(f))


def run_case(lib, parsers, filters, chunk, k, calls=2):
    ctx = pkg.Context(0, lib=lib)
    ref = util.Ref()
    for kw in parsers:
        ctx.parser(**kw)
        ref.parser(**kw)
    fs = [ctx.filter(p, props) for p, props in filters]
    rfs = [ref.filter(p, props) for p, props in filters]
    chain = ctx.chain(fs)
    for _ in range(calls):                       # the table accumulates over calls, like ctx->cmt
        want = ref.chain_do(chunk)
        got = chain.do(chunk)
        assert got[0] == want[0]
        assert got[1] == want[1]
        assert fs[k].l2m_text() == ref_text(ref, rfs[k])


@pytest.mark.parametrize("case", l2m_cases.L2M_CASES, ids=[c[0] for c in l2m_cases.L2M_CASES])
def test_l2m_hostsim(case, sim_lib, ref_available):
    _, parsers, filters, mk, k = case
    run_case(sim_lib, parsers, filters, mk(), k)


@pytest.mark.gpu
@pytest.mark.parametrize("case", l2m_cases.L2M_CASES, ids=[c[0] for c in l2m_cases.L2M_CASES])
def test_l2m_gpu(case, gpu_lib, ref_available):
    _, parsers, filters, mk, k = case
    run_case(gpu_lib, parsers, filters, mk(), k)


def check_golden(lib):
    vec = json.load(open(os.path.join(util.ROOT, "tests", "golden", "l2m_vectors.json")))
    assert len(vec) >= 8
    for v in vec:
        ctx = pkg.Context(0, lib=lib)
        for kw in v["parsers"]:
            ctx.parser(**kw)
        fs = [ctx.filter(p, [tuple(x) for x in props]) for p, props in v["filters"]]
        r, out = ctx.chain(fs).do(bytes.fromhex(v["in_hex"]))
        assert r == v["ret"], v["name"]
        assert (out.hex() if out is not None else None) == v["out_hex"], v["name"]
        assert fs[v["k"]].l2m_text() == v["text"], v["name"]


def test_l2m_golden_hostsim(sim_lib):
    check_golden(sim_lib)


@pytest.mark.gpu
def test_l2m_golden_gpu(gpu_lib):
    check_golden(gpu_lib)


def _forms_count_once(lib, monkeypatch, mode):
    """log_to_metrics behind a filter that grows every record: the small form's result outgrows its output buffer and the
    call moves to the two-pass form.  Each form (small, streaming, two-pass) counts every event of a call once."""
    n = 200
    props = l2m_cases.BASE + [("metric_mode", mode), ("label_field", "c")] + ([("value_field", "v")] if mode == "histogram" else [])
    chunk = b"".join(util.event(1700000000 + i, 0, [(b"c", util.mp_str(b"red")), (b"v", b"\x01")]) for i in range(n))
    texts = []
    for env in ({}, {"FLBGPU_SMALL_MB": "0", "FLBGPU_SLICE_MB": "1"}, {"FLBGPU_STREAM": "0"}):     # small, streaming, two-pass
        for k in ("FLBGPU_SMALL_MB", "FLBGPU_SLICE_MB", "FLBGPU_STREAM"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = pkg.Context(0, lib=lib)
        fs = [ctx.filter("modify", [("Add", "pad " + "p" * 400)]), ctx.filter("log_to_metrics", props)]
        chain = ctx.chain(fs)
        for call in (1, 2):
            r, out = chain.do(chunk)
            assert r == pkg.FILTER_MODIFIED and len(out) > len(chunk) + 400 * n
            assert [s[2] for s in fs[1].l2m_sets()] == [n * call], (env, call)
        texts.append(fs[1].l2m_text())
    assert texts[1] == texts[0] and texts[2] == texts[0]


@pytest.mark.parametrize("mode", ["counter", "histogram"])
def test_l2m_forms_count_once_hostsim(mode, sim_lib, monkeypatch):
    _forms_count_once(sim_lib, monkeypatch, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["counter", "histogram"])
def test_l2m_forms_count_once_gpu(mode, gpu_lib, monkeypatch):
    _forms_count_once(gpu_lib, monkeypatch, mode)


@pytest.mark.parametrize("bad", [
    [("metric_mode", "counter"), ("metric_description", "d")],                              # no tag
    [("metric_mode", "counter"), ("tag", "t")],                                             # no description
    [("metric_mode", "histogram"), ("metric_description", "d"), ("tag", "t")],              # no value_field
    [("metric_mode", "nope"), ("metric_description", "d"), ("tag", "t")],
    [("metric_description", "d"), ("tag", "t"), ("regex", "onlyfield")],
    [("metric_description", "d"), ("tag", "t"), ("add_label", "just_one")],
])
def test_l2m_config_errors(bad, sim_lib, ref_available):
    ctx = pkg.Context(0, lib=sim_lib)
    with pytest.raises(pkg.FlbGpuError):
        ctx.filter("log_to_metrics", bad)
    with pytest.raises(RuntimeError):
        util.Ref().filter("log_to_metrics", bad)


def _previous_value(lib):
    """a value text sscanf("%lf") cannot convert leaves the value of the previous converting record of the call in the
    reference's local variable (log_to_metrics.c:983-984,1060,1090), 0 when there is none: same table, record for record"""
    import random
    S = util.mp_str
    rng = random.Random(5)
    for mode in ("gauge", "histogram"):
        props = [("metric_mode", mode), ("metric_name", "m"), ("value_field", "x"), ("label_field", "c"), ("metric_description", "d"), ("tag", "t"),
                 ("regex", "keep yes")]
        for trial in range(6):
            evs = []
            for i in range(300):
                r = rng.random()
                if trial == 0 and i < 5:
                    v = S(b"fast")                                   # nothing converts before: the local's initial 0
                elif r < 0.15:
                    v = S(rng.choice([b"fast", b"", b"-", b".", b"x1", b"+.e3", b" \t"]))
                elif r < 0.25:
                    v = bytes([rng.randint(0, 100)])                 # integer value
                elif r < 0.30:
                    v = b"\xc3"                                      # a type the filter cannot convert: assigns nothing
                else:
                    v = S(str(rng.randint(0, 999)).encode() + rng.choice([b"", b".5", b"e1", b" tail"]))
                fields = [(b"x", v), (b"c", S(rng.choice([b"red", b"green", b"blue"]))), (b"keep", S(b"yes" if rng.random() < 0.8 else b"no"))]
                if rng.random() < 0.05:
                    fields = fields[1:]                              # no value field at all
                evs.append(util.event(1700000000 + i, 0, fields))
            chunk = b"".join(evs)
            ref = util.Ref()
            rf = ref.filter("log_to_metrics", props)
            want = ref.chain_do(chunk)
            ctx = pkg.Context(0, lib=lib)
            f = ctx.filter("log_to_metrics", props)
            assert ctx.chain([f]).do(chunk) == want
            ts = __import__("re").compile(r"^\S+Z ", __import__("re").M)
            assert f.l2m_text() == ts.sub("", ref.l2m_text(rf)), (mode, trial)
    # what would convert to inf / nan, and hex floats, stay refused (not restated), loudly
    ctx = pkg.Context(0, lib=lib)
    f = ctx.filter("log_to_metrics", [("metric_mode", "gauge"), ("value_field", "x"), ("metric_description", "d"), ("tag", "t")])
    for bad in (b"inf", b"nan", b"0x1p3"):
        with pytest.raises(pkg.FlbGpuError):
            f.cb(util.event(1700000000, 0, [(b"x", S(b"1.5"))]) + util.event(1700000001, 0, [(b"x", S(bad))]))


def test_l2m_previous_value_hostsim(sim_lib, ref_available):
    _previous_value(sim_lib)


@pytest.mark.gpu
def test_l2m_previous_value_gpu(gpu_lib, ref_available):
    _previous_value(gpu_lib)


WORKER = r"""
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import torch.distributed as dist
import util, l2m_cases
pkg = util.pkg
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
name, parsers, filters, mk, k = [c for c in l2m_cases.L2M_CASES if c[0] == {case!r}][0]
chunk = mk()
recs = util.split_records(chunk)
per = (len(recs) + world - 1) // world
mine = recs[rank * per:(rank + 1) * per]
shard = chunk[mine[0][0]: mine[-1][0] + mine[-1][1]]
ctx = pkg.Context(0, lib=pkg.load(util.HOSTSIM_SO))
for kw in parsers:
    ctx.parser(**kw)
fs = [ctx.filter(p, props) for p, props in filters]
ctx.chain(fs).do(shard)
fs[k].l2m_allreduce()
open({out!r} + str(rank), "w").write(fs[k].l2m_text())
dist.destroy_process_group()
"""


@pytest.mark.parametrize("case", ["counter_labels", "histogram_default_buckets", "after_parser_and_grep", "gauge_labels"])
def test_l2m_allreduce_world2(case, sim_lib, ref_available, tmp_path):
    """Two shards of one chunk, one table per rank, merged with the all-reduce: every rank ends
    with exactly the table the reference builds from the whole chunk (same order, same values)."""
    name, parsers, filters, mk, k = [c for c in l2m_cases.L2M_CASES if c[0] == case][0]
    ref = util.Ref()
    for kw in parsers:
        ref.parser(**kw)
    rfs = [ref.filter(p, props) for p, props in filters]
    ref.chain_do(mk())
    want = ref_text(ref, rfs[k])
    out = str(tmp_path / "t")
    script = tmp_path / "w.py"
    script.write_text(WORKER.format(root=util.ROOT, case=case, out=out))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(29600 + os.getpid() % 300), WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r))) for r in range(2)]
    for p in procs:
        assert p.wait(timeout=300) == 0
    for r in range(2):
        assert open(out + str(r)).read() == want


LIB_WORKER = r"""
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import util, l2m_cases
pkg = util.pkg
rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
gpu = {gpu!r}
name, parsers, filters, mk, k = [c for c in l2m_cases.L2M_CASES if c[0] == {case!r}][0]
chunk = mk()
recs = util.split_records(chunk)
per = (len(recs) + world - 1) // world
mine = recs[rank * per:(rank + 1) * per]
shard = chunk[mine[0][0]: mine[-1][0] + mine[-1][1]]
lib = pkg.load() if gpu else pkg.load(util.HOSTSIM_SO)
ctx = pkg.Context(rank if gpu else 0, lib=lib)
# the 128-byte communicator id travels over the embedding process's own channel: here a file
idf = {out!r} + ".id"
if rank == 0:
    uid = ctx.comm_unique_id()
    open(idf + ".tmp", "wb").write(uid); os.rename(idf + ".tmp", idf)
else:
    import time
    while not os.path.exists(idf):
        time.sleep(0.01)
    uid = open(idf, "rb").read()
ctx.comm_init(world, rank, uid)
for kw in parsers:
    ctx.parser(**kw)
fs = [ctx.filter(p, props) for p, props in filters]
ctx.chain(fs).do(shard)
fs[k].l2m_allreduce_lib()              # flbgpu_l2m_allreduce(): the library's own exchange
open({out!r} + str(rank), "w").write(fs[k].l2m_text())
"""


def _lib_allreduce(case, tmp_path, gpu):
    name, parsers, filters, mk, k = [c for c in l2m_cases.L2M_CASES if c[0] == case][0]
    ref = util.Ref()
    for kw in parsers:
        ref.parser(**kw)
    rfs = [ref.filter(p, props) for p, props in filters]
    ref.chain_do(mk())
    want = ref_text(ref, rfs[k])
    out = str(tmp_path / "t")
    script = tmp_path / "w.py"
    script.write_text(LIB_WORKER.format(root=util.ROOT, case=case, out=out, gpu=gpu))
    env = dict(os.environ, WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r))) for r in range(2)]
    for p in procs:
        assert p.wait(timeout=300) == 0
    for r in range(2):
        assert open(out + str(r)).read() == want


@pytest.mark.parametrize("case", ["counter_labels", "histogram_default_buckets", "after_parser_and_grep", "gauge_labels", "counter_no_labels"])
def test_l2m_library_allreduce_world2(case, sim_lib, ref_available, tmp_path):
    """flbgpu_l2m_allreduce() -- the merge logic of the PRODUCT library (runtime.c), two processes; the collectives
    underneath are the CPU emulation's (shared memory) here and NCCL on the GPU box"""
    _lib_allreduce(case, tmp_path, gpu=False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["counter_labels", "histogram_default_buckets", "gauge_labels"])
def test_l2m_library_allreduce_nccl(case, gpu_lib, ref_available, tmp_path):
    """the same over NCCL: needs two GPUs"""
    if gpu_lib.flbgpu_device_count() < 2:
        pytest.skip("one GPU: the NCCL exchange needs two")
    _lib_allreduce(case, tmp_path, gpu=True)
