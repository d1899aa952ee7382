#!/usr/bin/env python
"""Time of the split evaluation (a JSON parser, then other filters) on chunks resident in host memory.

  python tests/tools/splitbench.py [--lib path/to/libflbgpu.so] [--lines 100000] [--reps 4] [--calls 20]

One JSON line per result: per chain, the median wall time of one flbgpu_chain_do() call (host to device, evaluation,
emission, device to host; the call returns after its last device synchronisation).
The chunk is util.json_lines() tiled `reps` times.  Run two builds alternately in one session to compare them."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases  # noqa: E402
import l2m_cases  # noqa: E402
import util  # noqa: E402

CHAINS = {
    "json+modify": [cases.PJ, ("modify", [("Add", "env prod"), ("Rename", "msg message")])],
    "json+record_modifier": [cases.PJ, ("record_modifier", [("Remove_key", "trace_id"), ("Record", "cluster c1")])],
    "json+log_to_metrics": [cases.PJ, ("log_to_metrics", l2m_cases.BASE + [("metric_mode", "counter"), ("label_field", "level")])],
    "json+grep+modify": [cases.PJ, ("grep", [("Regex", "level ^(warn|error)$")]), ("modify", [("Add", "env prod"), ("Rename", "msg message"), ("Remove", "debug")])],
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--lines", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    pkg = util.pkg
    lib = pkg.load(a.lib) if a.lib else pkg.load()
    chunk = util.chunk_from_lines(util.json_lines(a.lines)) * a.reps
    res = {"lib": a.lib or "tree", "records": a.lines * a.reps, "bytes": len(chunk)}
    for name, filters in CHAINS.items():
        ctx = pkg.Context(0, lib=lib)
        ctx.parser(**cases.JS)
        chain = ctx.chain([ctx.filter(p, props) for p, props in filters])
        for _ in range(3):
            chain.do(chunk)
        wall = []
        for _ in range(a.calls):
            t0 = time.perf_counter()
            chain.do(chunk)
            wall.append((time.perf_counter() - t0) * 1e3)
        res[name] = {"call_ms": round(statistics.median(wall), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
