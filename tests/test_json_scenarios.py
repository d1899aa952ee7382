"""The reference's JSON fixtures through filter_parser(json): tests/internal/data/pack/* (the packed
string its pack test expects must come out) and benchmarks/utf8_surrogate_bench_10k.ndjson (two
lines of each of its 11 kinds as golden vectors; all 10 000, stored as tests/golden/utf8_surrogate_bench_10k.ndjson.xz,
against the reference's results).  tests/golden/json_scenarios.json is made by tests/golden/make_json_scenarios.py."""
import json
import lzma
import os

import pytest

import util

pkg = util.pkg
SCENARIOS = json.load(open(os.path.join(util.ROOT, "tests", "golden", "json_scenarios.json")))
KW = dict(name="js", format="json")
PROPS = [("Key_Name", "log"), ("Parser", "js")]
NDJSON = os.path.join(util.ROOT, "tests", "golden", "utf8_surrogate_bench_10k.ndjson.xz")


def run(lib):
    for sc in SCENARIOS:
        ctx = pkg.Context(0, lib=lib)
        ctx.parser(**KW)
        ret, out = ctx.filter("parser", PROPS).cb(util.chunk_from_lines([bytes.fromhex(sc["line_hex"])]))
        assert ret == sc["ret"], sc["name"]
        assert out.hex() == sc["out_hex"], sc["name"]
        if sc["value_hex"]:
            assert bytes.fromhex(sc["value_hex"]) in out, sc["name"]


def test_scenarios_present():
    assert len(SCENARIOS) >= 30
    assert sum(s["name"].startswith("ndjson/") for s in SCENARIOS) == 22


def test_json_scenarios_hostsim(sim_lib):
    run(sim_lib)


@pytest.mark.gpu
def test_json_scenarios_gpu(gpu_lib):
    run(gpu_lib)


def test_whole_surrogate_corpus_live(sim_lib, ref_available):
    lines = [l.rstrip(b"\n") for l in lzma.open(NDJSON, "rb")]
    assert len(lines) == 10000
    chunk = util.chunk_from_lines(lines)
    ctx, ref = pkg.Context(0, lib=sim_lib), util.Ref()
    ctx.parser(**KW); ref.parser(**KW)
    ref.filter("parser", PROPS)
    assert ctx.filter("parser", PROPS).cb(chunk) == ref.chain_do(chunk)
