"""The reference side of tests/test_zz_gelf.py: out_gelf's flush loop (with inject_tag()) restated around the reference's own,
unmodified flb_msgpack_to_gelf() (oracle/refshim/gelf_harness.c, built as oracle/_ref/libflbref_gelf.so beside libflbref.so).
Its results are stored, in call order per test, in a transcript of its own (tests/golden/gelf_transcript.json.gz, tail_ref's
encoding), so that the tests run where the reference build is absent; FLBGPU_REF_RECORD=1 with oracle/_ref built rewrites the
entries of the tests that ran.  The CPU-emulation and GPU forms of a test share one entry: their names differ only in the
trailing _hostsim / _gpu."""
import ctypes as C
import os
import re

import tail_ref
import util

GELF_SO = os.path.join(util.ROOT, "oracle", "_ref", "libflbref_gelf.so")
TRANSCRIPT = os.path.join(util.ROOT, "tests", "golden", "gelf_transcript.json.gz")
FIELDS = ("timestamp_key", "host_key", "short_message_key", "full_message_key", "level_key")


class _Transcript(tail_ref._Transcript):
    @staticmethod
    def test_id():
        return re.sub(r"_(hostsim|gpu)(?=\[|$)", "", util._Transcript.test_id())

    def _next(self):
        t, i = super()._next()
        if i == 0 and util.RECORD:              # the other form of the same test records the same entry again
            self.fresh.pop(t, None)
        return t, i


TRANSCRIPT_DATA = _Transcript(TRANSCRIPT)


def have_ref():
    return os.path.exists(GELF_SO)


def have_ref_results():
    """the reference build is here, or stored results for the running test are"""
    if have_ref():
        return True
    return TRANSCRIPT_DATA.has_current_test()


class GelfRef:
    """The reference's GELF flush loop (oracle/_ref/libflbref_gelf.so), or its stored transcript where that is not built."""

    def __init__(self):
        if not have_ref():
            self.L = None
            return
        C.CDLL(util.REF_SO, mode=C.RTLD_GLOBAL)
        L = C.CDLL(GELF_SO)
        vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
        L.flbref_msgpack_to_gelf.restype = vp
        L.flbref_msgpack_to_gelf.argtypes = [cp, sz, cp, cp, cp, cp, cp, cp, cp, sz, C.c_int, C.POINTER(sz), C.POINTER(sz)]
        self.free = C.CDLL(util.REF_SO).flbref_cfree
        self.free.argtypes = [vp]
        self.L = L

    def to_gelf(self, data, fields=None, tag_key=None, tag=None, separator=b"\n"):
        """what Context.to_gelf() returns, without the undefined count: (text bytes or None, events that failed)"""
        if self.L is None:
            return util._dec(TRANSCRIPT_DATA.replay())
        fields = fields or {}
        n, failed = C.c_size_t(), C.c_size_t()
        tag = util.Ref._b(tag)
        r = self.L.flbref_msgpack_to_gelf(data, len(data), *[util.Ref._b(fields.get(k)) for k in FIELDS], util.Ref._b(tag_key), tag,
                                          len(tag) if tag is not None else 0, separator[0], C.byref(n), C.byref(failed))
        out = C.string_at(r, n.value) if r else None
        if r:
            self.free(r)
        res = (out, failed.value)
        if util.RECORD:
            TRANSCRIPT_DATA.record(util._enc(res))
        return res
