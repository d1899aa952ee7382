"""A chunk of log events as GELF messages on the device: flbgpu_msgpack_to_gelf() at out_http's and out_gelf's flush sizes.
   python tests/tools/gelfbench.py [--steps N] [--out FILE]
One JSON line per call size (64 KB, 2 MB, 64 MB of events): events/s end to end (host clock around calls that take and
return host memory), events/s of the two launches alone (flbgpu_kernel_ms() of the sizing and emission passes), and, where
oracle/_ref/libflbref_gelf.so is built, events/s of the reference's flush loop on one host core -- with the device name and
power limit the numbers were taken at."""
import argparse
import ctypes as C
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "tools")]
import gelf_ref       # noqa: E402
import util           # noqa: E402
from tailbench import device   # noqa: E402

pkg = util.pkg
S = util.mp_str
SIZES = [("64K", 64 << 10), ("2M", 2 << 20), ("64M", 64 << 20)]
LEVELS = [b"info", b"info", b"warning", b"err", b"debug", b"6"]


def events(size, seed=11):
    """access-log records as a parser leaves them, with a nested map and an array: (chunk, events)"""
    rng = random.Random(seed)
    lines = util.apache_lines(size // 150 + 16, seed=seed)
    out, n, i = [], 0, 0
    for line in lines:
        host = b"10.0.%d.%d" % (rng.randint(0, 255), rng.randint(0, 255))
        body = [(b"short_message", S(line)), (b"host", S(host)), (b"level", S(rng.choice(LEVELS))),
                (b"code", bytes([0xcd]) + rng.choice([200, 404, 500, 301]).to_bytes(2, "big")),
                (b"size", b"\xce" + rng.randint(0, 10 ** 6).to_bytes(4, "big")),
                (b"http", b"\x82" + S(b"method") + S(rng.choice([b"GET", b"POST"])) + S(b"path") + S(b"/index.html")),
                (b"tags", b"\x92" + S(b"web") + S(b"prod"))]
        e = util.event(1700000000 + i, i * 1000, body)
        if n + len(e) > size:
            break
        out.append(e)
        n += len(e)
        i += 1
    return b"".join(out), len(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = pkg.load()
    ctx = pkg.Context(0, lib=L)
    name, power = device()
    ref = gelf_ref.GelfRef() if gelf_ref.have_ref() else None
    vp, sz = C.c_void_p, C.c_size_t
    free = pkg._libc.free
    ms = (C.c_float * 3)()
    rows = []
    for label, size in SIZES:
        chunk, n_ev = events(size)
        buf = C.create_string_buffer(chunk, len(chunk))
        calls = max(1, (256 << 20) // (len(chunk) * 8))
        out, n, failed, und = vp(), sz(), sz(), sz()

        def one_call():
            if L.flbgpu_msgpack_to_gelf(ctx.h, buf, len(chunk), None, None, None, 0, 10, C.byref(out), C.byref(n), C.byref(failed),
                                        C.byref(und)) != 0:
                raise RuntimeError(ctx.err())
            free(out)

        one_call(); one_call()
        times, kern = [], []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            for _ in range(calls):
                one_call()
            times.append((time.perf_counter() - t0) / calls)
            L.flbgpu_kernel_ms(ctx.h, ms)
            kern.append(ms[1] + ms[2])
        best, kbest = min(times), min(kern)
        row = {"call": label, "bytes": len(chunk), "events": n_ev, "out_bytes": n.value, "calls_per_step": calls, "steps": a.steps,
               "device": name, "power_limit": power,
               "e2e_mevents_s": round(n_ev / best / 1e6, 3), "ms_per_call": round(best * 1e3, 4),
               "median_ms": round(sorted(times)[len(times) // 2] * 1e3, 4),
               "kernel_ms": round(kbest, 4), "kernel_mevents_s": round(n_ev / (kbest / 1e3) / 1e6, 3) if kbest > 0 else None}
        if ref is not None:
            t0 = time.perf_counter()
            ref.to_gelf(chunk)
            row["ref_1core_mevents_s"] = round(n_ev / (time.perf_counter() - t0) / 1e6, 3)
        else:
            row["ref_1core_mevents_s"] = "not measured (oracle/_ref/libflbref_gelf.so absent)"
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
