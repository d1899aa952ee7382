"""The reference side of tests/test_zz_tail_parser.py: in_tail's `Parser` branch restated around the reference's own
flb_parser_do() and log event encoder (oracle/refshim/tail_harness.c, built as oracle/_ref/libflbref_tail.so beside
libflbref.so), with parsers and JSON text from the reference harness (util.Ref).  Its results are stored, in call order per test,
in a transcript of its own (tests/golden/tail_parser_transcript.json.gz, same encoding as util's), so that the tests run where the
reference build is absent; FLBGPU_REF_RECORD=1 with oracle/_ref built rewrites the entries of the tests that ran."""
import atexit
import ctypes as C
import functools
import gzip
import json
import os

import util

TAIL_SO = os.path.join(util.ROOT, "oracle", "_ref", "libflbref_tail.so")
TRANSCRIPT = os.path.join(util.ROOT, "tests", "golden", "tail_parser_transcript.json.gz")


class _Transcript(util._Transcript):
    def __init__(self, path):
        self.path = path
        self.data = {}
        if os.path.exists(path):
            with gzip.open(path, "rt") as f:
                self.data = json.load(f)
        self.fresh = {}
        self.cur, self.seq = None, 0
        if util.RECORD:
            atexit.register(self.save)

    def save(self):
        if not self.fresh:
            return
        self.data.update(self.fresh)
        with open(self.path, "wb") as f:           # mtime 0: the same transcript makes the same file
            with gzip.GzipFile(fileobj=f, mode="wb", mtime=0) as z:
                z.write(json.dumps(self.data, sort_keys=True, separators=(",", ":")).encode())


TRANSCRIPT_DATA = _Transcript(TRANSCRIPT)


def have_ref():
    return util.have_ref() and os.path.exists(TAIL_SO)


def have_ref_results():
    """the reference build is here, or stored results for the running test are"""
    if have_ref():
        if util.RECORD:
            TRANSCRIPT_DATA.fresh.setdefault(TRANSCRIPT_DATA.test_id(), [])
        return True
    return TRANSCRIPT_DATA.has_current_test()


def _recorded(handle=False):
    """util._recorded() with this module's transcript"""
    def deco(fn):
        @functools.wraps(fn)
        def w(self, *a, **k):
            if self.L is None:
                e = TRANSCRIPT_DATA.replay()
                if isinstance(e, dict) and "raise" in e:
                    raise RuntimeError(e["raise"])
                return util.RefHandle() if handle else util._dec(e)
            try:
                r = fn(self, *a, **k)
            except RuntimeError as ex:
                if util.RECORD:
                    TRANSCRIPT_DATA.record({"raise": str(ex)})
                raise
            if util.RECORD:
                TRANSCRIPT_DATA.record("H" if handle else util._enc(r, self.keep_whole))
            return r
        return w
    return deco


class TailRef:
    """The reference's in_tail `Parser` branch (oracle/_ref/libflbref_tail.so), or its stored transcript where that is not built.
    Parsers and JSON text come from util.Ref's functions, called here without util's own transcript."""

    def __init__(self, keep_whole=False):
        self.keep_whole = keep_whole
        if not have_ref():
            self.L = None
            return
        self.ref = util.Ref()                  # (loads libflbref.so first: libflbref_tail.so links against that instance)
        L = C.CDLL(TAIL_SO)
        vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
        L.flbref_lines_to_events_parsed.restype = vp
        L.flbref_lines_to_events_parsed.argtypes = [vp, cp, sz, cp, C.c_int, C.c_longlong, C.c_longlong, cp, cp, cp, C.c_ulonglong,
                                                    C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
        self.L = L

    @_recorded(handle=True)
    def parser(self, **kw):
        return util.Ref.parser.__wrapped__(self.ref, **kw)

    @_recorded()
    def lines_to_events_parsed(self, p, text, key="log", skip_empty_lines=True, sec=0, nsec=0, path_key=None, path=None, offset_key=None,
                               stream_offset=0):
        """in_tail's line loop with parser p as its `Parser`: (chunk bytes or None, bytes consumed, lines seen)"""
        n, used, lines = C.c_size_t(), C.c_size_t(), C.c_size_t()
        b = util.Ref._b
        r = self.L.flbref_lines_to_events_parsed(p, text, len(text), b(key), int(skip_empty_lines), sec, nsec, b(path_key), b(path),
                                                 b(offset_key), stream_offset, C.byref(n), C.byref(used), C.byref(lines))
        out = C.string_at(r, n.value) if n.value else None
        self.ref.L.flbref_cfree(r)
        return out, used.value, lines.value

    @_recorded()
    def to_json(self, data, json_format=3, date_format=0, date_key="date", escape_unicode=True):
        return util.Ref.to_json.__wrapped__(self.ref, data, json_format, date_format, date_key, escape_unicode)
