"""flbgpu_chain_set_result_buffer(): results written into a buffer the caller keeps."""
import os

import pytest

import util

pkg = util.pkg


def _result_buffer(lib):
    """flbgpu_chain_set_result_buffer(): the three call forms write a result that fits into the caller's buffer (the returned
    pointer is that buffer), a larger one comes back malloc()ed; the bytes are the same either way"""
    ctx = pkg.Context(0, lib=lib)
    ap = dict(name="apache", format="regex", regex=util.APACHE_RX, time_fmt=util.APACHE_TIME_FMT, time_key="time")
    ctx.parser(**ap)
    flt = [("parser", [("Key_Name", "log"), ("Parser", "apache")]), ("grep", [("Regex", "method ^(GET|POST)$")]), ("modify", [("Add", "env prod")])]
    plain = ctx.chain([ctx.filter(p, props) for p, props in flt])
    chunk = util.chunk_from_lines(util.apache_lines(3000, seed=3))
    want = plain.do(chunk)
    old = {k: os.environ.get(k) for k in ("FLBGPU_SMALL_MB", "FLBGPU_STREAM", "FLBGPU_SLICE_MB")}
    try:
        for env in ({}, {"FLBGPU_SMALL_MB": "0", "FLBGPU_SLICE_MB": "1"}, {"FLBGPU_SMALL_MB": "0", "FLBGPU_STREAM": "0"}):      # small, streaming, two-pass
            for k in old:
                os.environ.pop(k, None)
            os.environ.update(env)
            for cap in (len(want[1]) + 64, len(want[1]), len(want[1]) - 1, 4096):
                ch = ctx.chain([ctx.filter(p, props) for p, props in flt])
                ch.set_result_buffer(cap)
                for _ in range(2):
                    assert ch.do(chunk) == want, (env, cap)
                ch.set_result_buffer(0)
                assert ch.do(chunk) == want
        # several slices per call: the caller's buffer takes the first slices' result and is outgrown by a later one
        os.environ.update({"FLBGPU_SMALL_MB": "0", "FLBGPU_SLICE_MB": "1"})
        os.environ.pop("FLBGPU_STREAM", None)
        big = chunk * 6
        want_big = plain.do(big)
        for frac in (0.2, 0.5, 0.9, 1.0):
            ch = ctx.chain([ctx.filter(p, props) for p, props in flt])
            ch.set_result_buffer(int(len(want_big[1]) * frac))
            for _ in range(2):
                assert ch.do(big) == want_big, frac
        # grep drops nothing, so the streaming form's speculation (every filter modifies) fails after its result went to the
        # caller's buffer: that buffer stays the caller's and the two-pass form redoes the call
        kept = util.chunk_from_lines([l for l in util.apache_lines(3000, seed=3) if b'"GET ' in l or b'"POST ' in l])
        want_kept = plain.do(kept)
        ch = ctx.chain([ctx.filter(p, props) for p, props in flt])
        ch.set_result_buffer(len(want_kept[1]) + 64)
        for _ in range(2):
            assert ch.do(kept) == want_kept
    finally:
        for k, v in old.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


def test_result_buffer_hostsim(sim_lib):
    _result_buffer(sim_lib)


@pytest.mark.gpu
def test_result_buffer_gpu(gpu_lib):
    _result_buffer(gpu_lib)
