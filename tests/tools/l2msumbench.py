#!/usr/bin/env python
"""Cost of adding log_to_metrics histogram sums up in record order.

  python tests/tools/l2msumbench.py [--lib path/to/libflbgpu.so] [--records 1000000,10000000] [--calls 10]

One JSON line per result.  For a chain of one histogram filter (discard_logs on) over chunks of 1 M and 10 M records, with
1 and 32 label sets, it times flbgpu_chain_do() twice: with three-decimal values, whose sums the host adds up record by
record after the evaluation (the fold), and with integer values 0-9999, which keep the device's atomic sums.  Each
chunk is built from one pre-encoded block of 65 536 records, tiled.

Per case: the median wall time of a call (host to device, evaluation, metric merge; the call returns after its last
device synchronisation), and the median of the call's own phase clock up to the end of the evaluation (stats phase_ms[0]
in the two-pass form) -- the difference is the merge, the fold included.  Run two builds alternately in one session to
compare them."""
import argparse
import json
import os
import random
import statistics
import struct
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import l2m_cases  # noqa: E402
import util  # noqa: E402

BLOCK = 65536


def block(n_sets, decimal, seed=7):
    rng = random.Random(seed)
    labs = [util.mp_str(b"set%02d" % i) for i in range(n_sets)]
    out = []
    for i in range(BLOCK):
        u = rng.randrange(0, 10000)
        v = b"\xcb" + struct.pack(">d", u / 1000.0 if decimal else float(u))
        out.append(util.event(1700000000 + i, 0, [(b"c", labs[i % n_sets]), (b"v", v)]))
    return b"".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--records", default="1000000,10000000")
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()
    os.environ["FLBGPU_STREAM"] = "0"                 # the two-pass form: its phase clock ends with the evaluation
    pkg = util.pkg
    lib = pkg.load(a.lib) if a.lib else pkg.load()
    props = l2m_cases.BASE + [("metric_mode", "histogram"), ("value_field", "v"), ("label_field", "c"), ("discard_logs", "on")]
    for n in [int(x) for x in a.records.split(",")]:
        for n_sets in (1, 32):
            res = {"lib": a.lib or "tree", "records": n, "sets": n_sets}
            for kind in ("decimal", "integer"):
                b = block(n_sets, kind == "decimal")
                chunk = b * (n // BLOCK) + b[:util.split_records(b)[n % BLOCK][0]] if n % BLOCK else b * (n // BLOCK)
                ctx = pkg.Context(0, lib=lib)
                f = ctx.filter("log_to_metrics", props)
                chain = ctx.chain([f])
                for _ in range(2):
                    chain.do(chunk)
                wall, ev = [], []
                for _ in range(a.calls):
                    t0 = time.perf_counter()
                    chain.do(chunk)
                    wall.append((time.perf_counter() - t0) * 1e3)
                    ev.append(chain.stats().phase_ms[0])
                res[kind] = {"call_ms": round(statistics.median(wall), 3), "eval_ms": round(statistics.median(ev), 3),
                             "merge_ms": round(statistics.median(w - e for w, e in zip(wall, ev)), 3)}
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
