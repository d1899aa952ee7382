"""The chain's device kernels (kernels.cu) at their tile, warp and list boundaries.

Each generator builds a chunk that crosses one boundary of one kernel and asserts, from the chunk's layout computed here,
that it does -- so that a later change to a generator cannot quietly stop testing the edge.  Each case runs on the CPU
emulation and on the GPU, and is compared with the oracle (and with the reference build where it is present):
  k_index            8192-byte tiles counted from the 16-byte aligned start of a slice; 255 records staged per tile row
  k_index_repair     at most 8192 broken links per slice (BK_MAX_BREAKS)
  stage-1 bitmap     one warp's byte range of at most 8192 bytes (BM_BYTES), 32 flags per word, bm_mask4's false flags
  k_chain_emit_list  one warp's result staged in EMIT_STAGE (8192) bytes of shared memory, +15 bytes of misalignment
  the scans          256 records per block, 256 blocks per scan row"""

import pytest

import cases
import util

pkg = util.pkg
S = util.mp_str

TILE = 8192                 # BK_INDEX_TILE
STAGE_ROW = 255             # BK_STAGE_ROW - 1: kept records one tile stages
MAX_BREAKS = 8192           # BK_MAX_BREAKS
BM_BYTES = 8192             # bytes of one warp's stage-1 bitmap
EMIT_STAGE = 8192           # bytes of one warp's staged result
SMALL, SLICED, TWO_PASS = {}, {"FLBGPU_SMALL_MB": "0"}, {"FLBGPU_STREAM": "0"}
MODIFY = [("modify", [("Add", "env prod")])]


def event_of_size(n, sec=1700000000, fill=b"x", key=b"log"):
    """a v2 event of exactly n bytes: {key: fill * m}"""
    fixed = 13 + 1 + 1 + len(key)
    for hdr, lo, hi in ((1, 0, 31), (2, 32, 255), (3, 256, 65535)):
        m = n - fixed - hdr
        if lo <= m <= hi:
            ev = util.event(sec, 0, [(key, S((fill * m)[:m]))])
            assert len(ev) == n
            return ev
    raise ValueError(n)


def starts(chunk):
    return [o for o, _ in util.split_records(chunk)]


def _checkers(parsers, filters):
    out = [util.Oracle()] + ([util.Ref()] if util.have_ref() else [])
    for c in out:
        for kw in parsers:
            c.parser(**kw)
        for p, props in filters:
            c.filter(p, props)
    return out


def run(lib, monkeypatch, filters, chunk, parsers=(), env=None):
    for k in ("FLBGPU_SMALL_MB", "FLBGPU_SLICE_MB", "FLBGPU_STREAM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    ctx = pkg.Context(0, lib=lib)
    for kw in parsers:
        ctx.parser(**kw)
    got = ctx.chain([ctx.filter(p, props) for p, props in filters]).do(chunk)
    for c in _checkers(parsers, filters):
        assert got == c.chain_do(chunk), (type(c).__name__, env)
    return got


# ---------------------------------------------------------------------------------------------------- k_index
def tile_of(count):
    """sizes of `count` events that fill one tile exactly"""
    base, r = divmod(TILE, count)
    return [base + 1] * r + [base] * (count - r)


def tile_count_chunks():
    """tiles of 253 to 258 records, the sizes chosen so that the records starting in one tile cross 255 (the staging
    row); behind a first event of 0, 19 or 40 bytes, so that the records also straddle the tile boundaries"""
    out, seen = [], set()
    for prefix in (0, 19, 40):
        sizes = [prefix] if prefix else []
        for c in (253, 254, 255, 256, 257, 258, 256, 255):
            sizes += tile_of(c)
        chunk = b"".join(event_of_size(sz, 1700000000 + i) for i, sz in enumerate(sizes))
        per_tile = {}
        for o in starts(chunk):
            per_tile[o // TILE] = per_tile.get(o // TILE, 0) + 1
        seen |= set(per_tile.values())
        out.append(chunk)
    assert {STAGE_ROW - 1, STAGE_ROW, STAGE_ROW + 1, STAGE_ROW + 2} <= seen, sorted(seen)
    return out


def boundary_sweep_chunks():
    """one record's start swept across the 16 bytes on each side of a tile boundary; at TILE - 1 its outer 0x92 is the last
    byte of a tile and its header array, itself a 0x92 that frames a legacy event, sits at rel 0 of the next"""
    out, at = [], set()
    for t in range(TILE - 16, TILE + 17):
        head = event_of_size(t, 1600000000)
        chunk = head + b"".join(event_of_size(40 + i % 7, 1700000000 + i) for i in range(300))
        assert starts(chunk)[1] == t and chunk[t] == 0x92 and chunk[t + 1] == 0x92
        at.add(t)
        out.append(chunk)
    assert TILE - 1 in at and TILE in at
    return out


def all_0x92_chunk():
    """a string of 0x92 bytes longer than a tile: every byte of a tile is a candidate"""
    big = util.event(1700000000, 0, [(b"log", S(b"\x92" * (TILE * 2 + 100)))])
    chunk = b"".join(event_of_size(50, 1700000000 + i) for i in range(10)) + big + b"".join(event_of_size(50, 1700001000 + i) for i in range(10))
    lo = starts(chunk)[10]
    full = [t for t in range(len(chunk) // TILE) if all(b == 0x92 for b in chunk[t * TILE:(t + 1) * TILE])]
    assert full and lo < full[0] * TILE
    return chunk


def _index_cases(lib, monkeypatch):
    for chunk in tile_count_chunks():
        for env in (SMALL, TWO_PASS):
            run(lib, monkeypatch, MODIFY, chunk, env=env)
    for chunk in boundary_sweep_chunks():
        run(lib, monkeypatch, MODIFY, chunk)
    run(lib, monkeypatch, MODIFY, all_0x92_chunk())
    run(lib, monkeypatch, [("grep", [("Exclude", "log ^x")])], all_0x92_chunk(), env=TWO_PASS)
    # chunk lengths of every residue mod 16: the last record cut short, or garbage behind it
    base = b"".join(event_of_size(33 + i % 5, 1700000000 + i) for i in range(700))
    lens = set()
    for cut in range(16):
        for chunk in (base[:len(base) - cut], base + b"\xc1" * cut):
            lens.add(len(chunk) % 16)
            run(lib, monkeypatch, MODIFY, chunk)
    assert lens == set(range(16))


def sliced_unaligned_chunk():
    """records of 37 bytes over three 1 MB slices: every slice after the first starts at a record, off 16-byte alignment"""
    chunk = b"".join(event_of_size(37, 1700000000 + i) for i in range((3 << 20) // 37))
    st = starts(chunk)
    nxt = [min(o for o in st if o >= k << 20) for k in (1, 2)]
    assert all(o % 16 for o in nxt), nxt
    return chunk


def test_index_tiles_hostsim(sim_lib, monkeypatch):
    _index_cases(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_index_tiles_gpu(gpu_lib, monkeypatch):
    _index_cases(gpu_lib, monkeypatch)


def _sliced_unaligned(lib, monkeypatch):
    chunk = sliced_unaligned_chunk()
    run(lib, monkeypatch, MODIFY, chunk, env={"FLBGPU_SLICE_MB": "1", "FLBGPU_SMALL_MB": "0"})
    run(lib, monkeypatch, MODIFY, chunk, env={"FLBGPU_SLICE_MB": "1", "FLBGPU_STREAM": "0"})


def test_index_unaligned_slices_hostsim(sim_lib, monkeypatch):
    _sliced_unaligned(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_index_unaligned_slices_gpu(gpu_lib, monkeypatch):
    _sliced_unaligned(gpu_lib, monkeypatch)


# ---------------------------------------------------------------------------------------------- k_index_repair
def breaks_chunk(n):
    """n records, each with a body value 92 01 80: [1, {}] frames as a legacy event inside the record, one broken link each"""
    chunk = b"".join(util.event(1700000000 + i, 0, [(b"log", S(b"line %d" % i)), (b"a", b"\x92\x01\x80")]) for i in range(n))
    recs = util.split_records(chunk)
    false = [o + chunk[o:o + l].index(b"\x92\x01\x80") for o, l in recs]
    assert len(recs) == n and len(set(false)) == n and all(o < f < o + l for (o, l), f in zip(recs, false))
    return chunk


def _breaks(lib, monkeypatch):
    for n in (MAX_BREAKS, MAX_BREAKS + 1):
        chunk = breaks_chunk(n)
        for env in (SMALL, SLICED):
            run(lib, monkeypatch, [("grep", [("Exclude", "log 7$")])], chunk, env=env)


def test_index_repair_break_limit_hostsim(sim_lib, monkeypatch):
    _breaks(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_index_repair_break_limit_gpu(gpu_lib, monkeypatch):
    _breaks(gpu_lib, monkeypatch)


# --------------------------------------------------------------------------------------------- stage-1 bitmap
JSON_SPLIT = [cases.PJ, ("grep", [("Exclude", "level ^debug$")]), ("modify", [("Add", "env prod")])]
JSON_ONE = [cases.PJ]


def _json_event(sec, line, size):
    """an event of exactly `size` bytes whose log is `line` padded inside its "msg" string"""
    pad = size - len(util.event(sec, 0, [(b"log", S(line))]))
    assert pad >= 0
    for extra in range(0, 4):            # the string header may grow by a byte or two
        l2 = line.replace(b'"msg":"', b'"msg":"' + b"p" * (pad - extra), 1)
        ev = util.event(sec, 0, [(b"log", S(l2))])
        if len(ev) == size:
            return ev
    raise ValueError(size)


LINES = [b'{"level":"warn","msg":"a plain line"}',
         b'{"level":"info","msg":"say \\"#hi\\" and \\\\] x",\t "n":1}',          # "# and \] : bm_mask4 flags the second byte too
         b'{"level":"error","msg":"tab then space",\t "m":2}',                  # a control byte before a space
         b'{"level":"debug","msg":"dropped"}',
         b'{"level":"warn","msg":"nested","k":{"a":[1,2]}}']


def warp_ranges(chunk, first=0):
    """(lo rounded down to 16, hi) of each warp of 32 records, records counted from `first`"""
    st = util.split_records(chunk)[first:]
    out = []
    for w in range(0, len(st), 32):
        grp = st[w:w + 32]
        lo, hi = grp[0][0] & ~15, grp[-1][0] + grp[-1][1]
        out.append((lo, hi))
    return out


def bitmap_chunk(warp_bytes, n_warps=24, tail=5, quote_last=False):
    """records of 256 bytes, so that a warp spans 8192; warp_bytes = 8193 makes every 32nd record a byte longer.  The last
    warp is partial (tail records).  quote_last: the last record of each warp is a JSON string document, its closing quote
    the last byte of the warp's range."""
    evs = []
    n = n_warps * 32 + tail
    for i in range(n):
        size = 256 + (1 if warp_bytes == BM_BYTES + 1 and i % 32 == 31 else 0)
        if quote_last and i % 32 == 31:
            body = b'"' + b"q" * 200 + b'"'
            ev = util.event(1700000000 + i, 0, [(b"log", S(body))])
            ev = util.event(1700000000 + i, 0, [(b"log", S(b'"' + b"q" * (200 + size - len(ev)) + b'"'))])
        else:
            ev = _json_event(1700000000 + i, LINES[i % len(LINES)], size)
        evs.append(ev)
    chunk = b"".join(evs)
    spans = [hi - lo for lo, hi in warp_ranges(chunk)]
    assert warp_bytes in spans, sorted(set(spans))
    if quote_last:
        assert all(chunk[hi - 1] == ord('"') for lo, hi in warp_ranges(chunk)[:-1])
    return chunk


def quote_bits_chunk():
    """closing quotes swept over every bit of a bitmap word (bits 0 and 31 included)"""
    evs, bits = [], set()
    for i in range(32 * 12):
        line = b'{"level":"warn","msg":"' + b"y" * (i % 37) + b'","z":"e"}'
        evs.append(util.event(1700000000 + i, 0, [(b"log", S(line))]))
    chunk = b"".join(evs)
    for w, (lo, hi) in enumerate(warp_ranges(chunk)):
        for o, l in util.split_records(chunk)[w * 32:(w + 1) * 32]:
            rec = chunk[o:o + l]
            q = rec.index(b'","z"') + o
            bits.add((q - lo) % 32)
    assert {0, 31} <= bits
    return chunk


def group_marker_chunk():
    """group markers (events the decoder steps over) inside warps: dead lanes at either end of a warp's range"""
    gs = util.event(0xffffffff, 0, [(b"g", S(b"start"))])
    ge = util.event(0xfffffffe, 0, [])
    evs = []
    for i in range(300):
        if i % 32 in (0, 17):
            evs.append(gs)
        evs.append(_json_event(1700000000 + i, LINES[i % len(LINES)], 120 + i % 50))
        if i % 32 in (31, 18):
            evs.append(ge)
    return b"".join(evs)


def _bitmap(lib, monkeypatch):
    chunks = [bitmap_chunk(BM_BYTES), bitmap_chunk(BM_BYTES + 1), bitmap_chunk(BM_BYTES, quote_last=True), quote_bits_chunk(), group_marker_chunk()]
    for chunk in chunks:
        run(lib, monkeypatch, JSON_SPLIT, chunk, parsers=[cases.JS], env=TWO_PASS)
    for eb in ("128", "1024"):
        monkeypatch.setenv("FLBGPU_EVAL_BLOCK", eb)
        for chunk in chunks[:2] + chunks[4:]:
            run(lib, monkeypatch, JSON_SPLIT, chunk, parsers=[cases.JS], env=TWO_PASS)
    monkeypatch.delenv("FLBGPU_EVAL_BLOCK")
    monkeypatch.setenv("FLBGPU_JSON_BM", "1")               # the bitmap in the single launch of a chain that is not split
    for chunk in chunks:
        run(lib, monkeypatch, JSON_ONE, chunk, parsers=[cases.JS], env=TWO_PASS)


def test_json_bitmap_warps_hostsim(sim_lib, monkeypatch):
    _bitmap(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_json_bitmap_warps_gpu(gpu_lib, monkeypatch):
    _bitmap(gpu_lib, monkeypatch)


# ----------------------------------------------------------------------------------------- k_chain_emit_list
def emit_chunk(first_size, last_size=256, n=32 * 20 + 3, drop_every=0):
    """survivors of 256 bytes (grep keeps them untouched: the result is their bytes), the first of first_size and, from the
    second warp on, the last of each warp of last_size; with drop_every, dropped records between them, and one at the end.
    Returns the chunk and [(total, misalignment)] per emission warp."""
    evs, surv = [], []
    for i in range(n):
        if drop_every and i % drop_every == 1:
            evs.append(event_of_size(60, 1600000000 + i, fill=b"d"))
        sz = first_size if i == 0 else (last_size if i % 32 == 31 and i >= 32 else 256)
        evs.append(event_of_size(sz, 1700000000 + i))
        surv.append(sz)
    evs.append(event_of_size(60, 1600000000, fill=b"d"))
    warps, at = [], 0
    for w in range(0, len(surv), 32):
        tot = sum(surv[w:w + 32])
        warps.append((tot, at % 16))
        at += tot
    return b"".join(evs), warps


def wide_rerun_chunk():
    """modify re-encodes every record; one record per two warps has 20 fields (its cache row says "re-run")"""
    evs = []
    for i in range(32 * 8 + 9):
        items = [(b"log", S(b"line %d" % i))]
        if i % 64 == 40:
            items += [(b"f%02d" % j, bytes([j])) for j in range(19)]
        evs.append(util.event(1700000000 + i, 0, items))
    assert sum(1 for i in range(32 * 8 + 9) if i % 64 == 40) >= 4
    return b"".join(evs)


def one_per_warp_chunk():
    """a grep that keeps one record in 32: every evaluation warp has one survivor, the last emission warp one lane"""
    n = 32 * 33 + 1
    chunk = b"".join(util.event(1700000000 + i, 0, [(b"log", S(b"%s %d" % (b"keep" if i % 32 == 7 else b"drop", i)))]) for i in range(n))
    kept = sum(1 for i in range(n) if i % 32 == 7)
    assert kept % 32 == 1
    return chunk


def _emit(lib, monkeypatch):
    keep_x = [("grep", [("Regex", "log ^x")])]
    seen = set()
    for first, last, drop in ((256, 256, 0), (271, 256, 0), (271, 241, 0), (271, 256, 3)):
        chunk, warps = emit_chunk(first, last, drop_every=drop)
        seen |= set(warps)
        for env in (SMALL, TWO_PASS):
            run(lib, monkeypatch, keep_x, chunk, env=env)
    # exactly EMIT_STAGE aligned; EMIT_STAGE at 15 bytes of misalignment (too large to stage); EMIT_STAGE with the 15 included
    assert (EMIT_STAGE, 0) in seen and (EMIT_STAGE, 15) in seen and (EMIT_STAGE - 15, 15) in seen, sorted(seen)[:8]
    for env in (SMALL, TWO_PASS):
        run(lib, monkeypatch, MODIFY, wide_rerun_chunk(), env=env)
        run(lib, monkeypatch, [("grep", [("Regex", "log ^keep")]), ("modify", [("Add", "env prod")])], one_per_warp_chunk(), env=env)


def test_emit_staging_hostsim(sim_lib, monkeypatch):
    _emit(sim_lib, monkeypatch)


@pytest.mark.gpu
def test_emit_staging_gpu(gpu_lib, monkeypatch):
    _emit(gpu_lib, monkeypatch)


# ------------------------------------------------------------------------------------------------------ scans
@pytest.mark.parametrize("n", [255, 256, 257, 65535, 65536, 65537])
def test_scan_record_counts_hostsim(n, sim_lib, monkeypatch):
    _scan(sim_lib, monkeypatch, n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [255, 256, 257, 65535, 65536, 65537])
def test_scan_record_counts_gpu(n, gpu_lib, monkeypatch):
    _scan(gpu_lib, monkeypatch, n)


def _scan(lib, monkeypatch, n):
    """record counts around one block (256 records) and one row of the block scan (256 blocks)"""
    chunk = b"".join(util.event(1700000000 + i, 0, [(b"log", S(b"%d" % (i % 1000)))]) for i in range(n))
    assert len(util.split_records(chunk)) == n
    for env in (SMALL, TWO_PASS):
        run(lib, monkeypatch, [("grep", [("Exclude", "log 7$")]), ("modify", [("Add", "e p")])], chunk, env=env)
