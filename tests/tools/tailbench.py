"""in_tail with `Parser` on the device: the one call flbgpu_lines_to_events_parsed() against the two-call composition it replaces
(flbgpu_lines_to_events(), then a one-filter filter_parser chain over its result), on the same text.
   python tests/tools/tailbench.py [--steps N] [--out FILE]
One JSON line per (workload, call size): lines/s end to end (host clock around calls that return host memory), and
flbgpu_kernel_ms() of the last call, with the device name and power limit the numbers were taken at."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import util           # noqa: E402

pkg = util.pkg
SIZES = [("32K", 32 << 10), ("2M", 2 << 20), ("64M", 64 << 20)]
PARSERS = {"apache": dict(name="apache2", format="regex", regex=util.APACHE_RX, time_fmt=util.APACHE_TIME_FMT, time_key="time"),
           "json": dict(name="json", format="json")}


def device():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:      # (the numbers are then reported without it)
        return "unknown (%s)" % e, "unknown"


def text_of(wl, size):
    lines = util.apache_lines(size // 100 + 16, seed=5) if wl == "apache" else util.json_lines(size // 120 + 16, seed=6)
    out, n = [], 0
    for l in lines:
        if n + len(l) + 1 > size:
            break
        out.append(l)
        n += len(l) + 1
    return b"\n".join(out) + b"\n", len(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = pkg.load()
    ctx = pkg.Context(0, lib=L)
    name, power = device()
    vp, sz = C.c_void_p, C.c_size_t
    free = pkg._libc.free
    ms = (C.c_float * 3)()
    rows = []
    for wl, pdef in PARSERS.items():
        p = ctx.parser(**pdef)
        chain = ctx.chain([ctx.filter("parser", [("Key_Name", "log"), ("Parser", pdef["name"])])])
        for label, size in SIZES:
            t, n_lines = text_of(wl, size)
            buf = C.create_string_buffer(t, len(t))
            calls = max(1, (256 << 20) // (len(t) * 8))         # (a step of the small sizes is many calls: enough work to time)
            out, n, used, lines = vp(), sz(), sz(), sz()
            mid, mn = vp(), sz()

            def one_call():
                if L.flbgpu_lines_to_events_parsed(p.h, buf, len(t), b"log", 1, 1700000000, 0, None, None, None, 0, C.byref(out), C.byref(n),
                                                   C.byref(used), C.byref(lines)) != 0:
                    raise RuntimeError(ctx.err())
                free(out)

            def two_calls():
                if L.flbgpu_lines_to_events(ctx.h, buf, len(t), b"log", 1, 1700000000, 0, None, None, None, 0, C.byref(mid), C.byref(mn),
                                            C.byref(used), C.byref(lines)) != 0:
                    raise RuntimeError(ctx.err())
                r = L.flbgpu_chain_do(chain.h, mid, mn.value, b"tail", 4, C.byref(out), C.byref(n))
                free(mid)
                if r < 0:
                    raise RuntimeError(ctx.err())
                free(out)

            res = {}
            for fn in (one_call, two_calls):                     # warm-up of every size and path
                fn(); fn()
            times = {"parsed_call": [], "composition": []}
            for _ in range(a.steps):                             # the two paths alternate, step by step
                for key, fn in (("parsed_call", one_call), ("composition", two_calls)):
                    t0 = time.perf_counter()
                    for _ in range(calls):
                        fn()
                    times[key].append((time.perf_counter() - t0) / calls)
            for key, fn in (("parsed_call", one_call), ("composition", two_calls)):
                fn()
                L.flbgpu_kernel_ms(ctx.h, ms)                    # (the composition: its last call, the chain's)
                best = min(times[key])
                res[key] = {"mlines_s": round(n_lines / best / 1e6, 3), "ms_per_call": round(best * 1e3, 4),
                            "median_ms": round(sorted(times[key])[len(times[key]) // 2] * 1e3, 4),
                            "kernel_ms": [round(x, 4) for x in ms]}
            row = {"workload": wl, "call": label, "bytes": len(t), "lines": n_lines, "calls_per_step": calls, "steps": a.steps,
                   "device": name, "power_limit": power, **res}
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
