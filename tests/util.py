"""Shared test helpers: reference harness binding (oracle/_ref) with its stored transcript, event encoding,
synthetic line generators (SURVEY.md section 8d)."""
import atexit
import base64
import ctypes as C
import functools
import gzip
import hashlib
import importlib
import json
import os
import random
import struct

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libflbref.so")
SHIM_SO = os.path.join(ROOT, "oracle", "_ref", "flb-filter_gpu.so")
HOSTSIM_SO = os.environ.get("FLBGPU_HOSTSIM_SO") or os.path.join(ROOT, "tests", "hostsim", "libhostsim.so")   # override: a sanitizer build
TRANSCRIPT = os.path.join(ROOT, "tests", "golden", "ref_transcript.json.gz")
RECORD = os.environ.get("FLBGPU_REF_RECORD") == "1"

pkg = importlib.import_module("fluent-bit_b200")


def have_ref():
    """the reference build itself is here (oracle/_ref, made by build() where the reference tree is)"""
    return os.path.exists(REF_SO)


# ------------------------------------------------------------ reference transcript
# What the reference returned to every test that compares with it, in call order per test, so that those tests run
# where the reference build is absent.  FLBGPU_REF_RECORD=1 with oracle/_ref built rewrites the transcript of the tests
# that ran.  Text and outputs up to INLINE bytes are stored whole; longer outputs as their length and a SHA-256 prefix
# (RefDigest), which compares equal to the bytes it was taken of -- unless the Ref was made with
# keep_whole=True, for a test that compares parts of the outputs.  Entries: "s<text>", "b<base64>", "h<digest><length>",
# ["T" or "L", entries...] for a tuple or list, "H" for an object the reference made, {"raise": message}, or a number.
INLINE = 8
DIGEST_HEX = 8


class RefDigest:
    """A stored reference output too long to keep whole: equal to the bytes it was taken of."""

    def __init__(self, digest, n):
        self.digest, self.n = digest, n

    @staticmethod
    def of(b):
        return hashlib.sha256(b).hexdigest()[:DIGEST_HEX]

    def __eq__(self, other):
        if isinstance(other, RefDigest):
            return (self.digest, self.n) == (other.digest, other.n)
        if isinstance(other, (bytes, bytearray)):
            return len(other) == self.n and self.of(bytes(other)) == self.digest
        return NotImplemented

    def __ne__(self, other):
        r = self.__eq__(other)
        return r if r is NotImplemented else not r

    __hash__ = None

    def __len__(self):
        return self.n

    def __repr__(self):
        return "<reference output: %d bytes, sha256 %s...>" % (self.n, self.digest)


class RefHandle:
    """a parser / filter / multiline parser the reference made, in a replayed transcript"""


def _enc(v, whole=False):
    if v is None or isinstance(v, (bool, int, float)):
        return v
    if isinstance(v, str):
        return "s" + v
    if isinstance(v, bytes):
        return "b" + base64.b64encode(v).decode() if whole or len(v) <= INLINE else "h%s%d" % (RefDigest.of(v), len(v))
    if isinstance(v, (tuple, list)):
        return ["T" if isinstance(v, tuple) else "L"] + [_enc(x, whole) for x in v]
    raise TypeError("cannot store %r" % type(v))


def _dec(v):
    if isinstance(v, list):
        items = [_dec(x) for x in v[1:]]
        return tuple(items) if v[0] == "T" else items
    if not isinstance(v, str):
        return v
    if v[0] == "s":
        return v[1:]
    if v[0] == "b":
        return base64.b64decode(v[1:])
    return RefDigest(v[1:1 + DIGEST_HEX], int(v[1 + DIGEST_HEX:]))


class _Transcript:
    def __init__(self):
        self.data = {}
        if os.path.exists(TRANSCRIPT):
            with gzip.open(TRANSCRIPT, "rt") as f:
                self.data = json.load(f)
        self.fresh = {}
        self.cur, self.seq = None, 0
        if RECORD:
            atexit.register(self.save)

    @staticmethod
    def test_id():
        t = os.environ.get("PYTEST_CURRENT_TEST")
        return t.rsplit(" (", 1)[0] if t else "<outside a test>"

    def _next(self):
        t = self.test_id()
        if t != self.cur:
            self.cur, self.seq = t, 0
        self.seq += 1
        return t, self.seq - 1

    def has_current_test(self):
        return self.test_id() in self.data

    def record(self, entry):
        t, i = self._next()
        rows = self.fresh.setdefault(t, [])
        assert len(rows) == i
        rows.append(entry)

    def replay(self):
        t, i = self._next()
        rows = self.data.get(t)
        if rows is None or i >= len(rows):
            raise LookupError("no stored reference result for call %d of %s: rebuild oracle/_ref and record again "
                              "(FLBGPU_REF_RECORD=1)" % (i, t))
        return rows[i]

    def save(self):
        if not self.fresh:
            return
        self.data.update(self.fresh)
        with open(TRANSCRIPT, "wb") as f:          # mtime 0: the same transcript makes the same file
            with gzip.GzipFile(fileobj=f, mode="wb", mtime=0) as z:
                z.write(json.dumps(self.data, sort_keys=True, separators=(",", ":")).encode())


TRANSCRIPT_DATA = _Transcript()


def have_ref_results():
    """the reference build is here (while recording, the running test gets an entry even if it makes no call), or its
    stored results for the running test are"""
    if have_ref():
        if RECORD:
            TRANSCRIPT_DATA.fresh.setdefault(TRANSCRIPT_DATA.test_id(), [])
        return True
    return TRANSCRIPT_DATA.has_current_test()


def _recorded(handle=False):
    """a Ref method whose result (or RuntimeError) goes to the transcript, or comes from it without the reference build"""
    def deco(fn):
        @functools.wraps(fn)
        def w(self, *a, **k):
            if self.L is None:
                e = TRANSCRIPT_DATA.replay()
                if isinstance(e, dict) and "raise" in e:
                    raise RuntimeError(e["raise"])
                return RefHandle() if handle else _dec(e)
            try:
                r = fn(self, *a, **k)
            except RuntimeError as ex:
                if RECORD:
                    TRANSCRIPT_DATA.record({"raise": str(ex)})
                raise
            if RECORD:
                TRANSCRIPT_DATA.record("H" if handle else _enc(r, self.keep_whole))
            return r
        return w
    return deco


class Ref:
    """The UNMODIFIED reference code (oracle/_ref/libflbref.so), or its stored transcript where that is not built."""

    def __init__(self, keep_whole=False):
        self.keep_whole = keep_whole
        if not have_ref():
            self.L = None
            return
        L = C.CDLL(REF_SO)
        vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
        L.flbref_config_create.restype = vp
        L.flbref_parser_create.restype = vp
        L.flbref_parser_create.argtypes = [vp, cp, cp, cp, C.c_int, cp, cp, cp, C.c_int, C.c_int, C.c_int, cp]
        L.flbref_parser_create_dec.restype = vp
        L.flbref_parser_create_dec.argtypes = [vp, cp, cp, cp, C.c_int, cp, cp, cp, C.c_int, C.c_int, C.c_int, cp, cp]
        L.flbref_parser_do.argtypes = [vp, cp, sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
        L.flbref_filter_create.restype = vp; L.flbref_filter_create.argtypes = [vp, cp]
        L.flbref_filter_set.argtypes = [vp, cp, cp]
        L.flbref_filter_init.argtypes = [vp, vp]
        L.flbref_filter_cb.argtypes = [vp, vp, vp, sz, cp, C.POINTER(vp), C.POINTER(sz)]
        L.flbref_filter_do.argtypes = [vp, vp, sz, C.c_int, cp, C.POINTER(vp), C.POINTER(sz)]
        L.flbref_count_records.argtypes = [vp, sz]
        L.flbref_free.argtypes = [vp]
        L.flbref_time_lookup.argtypes = [vp, cp, sz, C.c_longlong, C.POINTER(C.c_longlong), C.POINTER(C.c_double)]
        L.flbref_plugin_load.argtypes = [vp, cp, cp]
        L.flbref_filter_cmt_text.restype = vp; L.flbref_filter_cmt_text.argtypes = [vp]
        L.flbref_l2m_cmt_text.restype = vp; L.flbref_l2m_cmt_text.argtypes = [vp]
        L.flbref_cfree.argtypes = [vp]
        L.flbref_pack_json_state.argtypes = [cp, sz, C.POINTER(vp), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.flbref_lines_to_events.restype = vp
        L.flbref_lines_to_events.argtypes = [cp, sz, cp, C.c_int, C.c_longlong, C.c_longlong, cp, cp, cp, C.c_ulonglong, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
        L.flbref_to_json_format.restype = vp
        L.flbref_to_json_format.argtypes = [vp, sz, C.c_int, C.c_int, cp, C.c_int, C.POINTER(sz)]
        L.flbref_ml_parser_create.restype = vp
        L.flbref_ml_parser_create.argtypes = [vp, cp, cp, cp, C.c_int, C.c_int, cp, cp, cp, cp]
        L.flbref_ml_parser_rule.argtypes = [vp, cp, cp, cp]
        L.flbref_ml_parser_init.argtypes = [vp]
        L.flbref_set_ml_buffer_limit.argtypes = [vp, cp]
        self.L = L
        self.cfg = L.flbref_config_create()

    def load_gpu_plugins(self, gpu_lib_path):
        """register the five filter_gpu_*_plugin structs of the shim (oracle/_ref/flb-filter_gpu.so), bound to the
        given implementation of the C ABI (libflbgpu.so, or the CPU emulation in the not-gpu tests)"""
        if self.L is None:
            raise RuntimeError("the gpu_* plugins are hosted by the reference build (oracle/_ref), which is absent")
        os.environ["FLBGPU_SHIM_LIB"] = gpu_lib_path
        for name in ("parser", "grep", "modify", "record_modifier", "log_to_metrics", "rewrite_tag", "multiline"):
            if self.L.flbref_plugin_load(self.cfg, SHIM_SO.encode(), ("filter_gpu_%s_plugin" % name).encode()) != 0:
                raise RuntimeError("cannot load the gpu_%s plugin from %s" % (name, SHIM_SO))

    @_recorded()
    def pack_json_state(self, js):
        """flb_pack_json_state() on a fresh state: (ret, msgpack bytes or None, last_byte, tokens_count)"""
        out, n, last, cnt = C.c_void_p(), C.c_int(), C.c_int(), C.c_int()
        r = self.L.flbref_pack_json_state(js, len(js), C.byref(out), C.byref(n), C.byref(last), C.byref(cnt))
        data = None
        if r == 0:
            data = C.string_at(out.value, n.value)
            self.L.flbref_free(out)
        return r, data, last.value, cnt.value

    def emit_reset(self, fail_after=-1):
        """forget what filter_rewrite_tag handed to its emitter so far; fail_after >= 0: the emitter refuses from that call on"""
        if self.L is not None:
            self.L.flbref_emit_reset(fail_after)

    @_recorded()
    def emitted(self):
        """[(tag, record bytes)] in the order filter_rewrite_tag called in_emitter_add_record()"""
        return self._emitted()

    @_recorded()
    def emitted_grouped(self):
        """the state those per-record in_emitter_add_record() calls leave in the emitter: [(tag, the records' bytes, count)],
        one buffer per tag in the order the tags first came"""
        d = {}
        for t, b in self._emitted():
            d.setdefault(t, []).append(b)
        return [(t, b"".join(v), len(v)) for t, v in d.items()]

    def _emitted(self):
        log, n = C.c_void_p(), C.c_size_t()
        self.L.flbref_emit_log(C.byref(log), C.byref(n))
        raw = C.string_at(log.value, n.value) if n.value else b""
        out, at = [], 0
        while at < len(raw):
            tl, sz = struct.unpack_from("<II", raw, at)
            out.append((raw[at + 8:at + 8 + tl], raw[at + 8 + tl:at + 8 + tl + sz]))
            at += 8 + tl + sz
        return out

    @_recorded()
    def filter_counters(self, f):
        """the instance's framework counters (src/flb_filter.c:574-616) as {metric line without timestamp}"""
        p = self.L.flbref_filter_cmt_text(f)
        t = C.string_at(p).decode()
        self.L.flbref_cfree(p)
        return sorted(l.split(" ", 1)[1] for l in t.splitlines() if " " in l)

    @_recorded()
    def l2m_text(self, f):
        p = self.L.flbref_l2m_cmt_text(f)
        t = C.string_at(p).decode(errors="replace")
        self.L.flbref_cfree(p)
        return t

    @staticmethod
    def _b(s):
        return s if s is None or isinstance(s, bytes) else s.encode()

    @_recorded(handle=True)
    def parser(self, name, format, regex=None, skip_empty=True, time_fmt=None, time_key=None, time_offset=None,
               time_keep=False, time_strict=True, logfmt_no_bare_keys=False, types=None, decoders=None):
        b = self._b
        if decoders:
            text = "".join("%s\t%s\n" % (k, v) for k, v in decoders)
            p = self.L.flbref_parser_create_dec(self.cfg, b(name), b(format), b(regex), int(skip_empty), b(time_fmt),
                                                b(time_key), b(time_offset), int(time_keep), int(time_strict),
                                                int(logfmt_no_bare_keys), b(types), b(text))
            if not p:
                raise RuntimeError("reference rejected parser " + name)
            return p
        p = self.L.flbref_parser_create(self.cfg, b(name), b(format), b(regex), int(skip_empty), b(time_fmt),
                                        b(time_key), b(time_offset), int(time_keep), int(time_strict),
                                        int(logfmt_no_bare_keys), b(types))
        if not p:
            raise RuntimeError("reference rejected parser " + name)
        return p

    @_recorded()
    def parser_do(self, p, line):
        out, n = C.c_void_p(), C.c_size_t()
        s, ns = C.c_longlong(), C.c_longlong()
        r = self.L.flbref_parser_do(p, line, len(line), C.byref(out), C.byref(n), C.byref(s), C.byref(ns))
        data = C.string_at(out.value, n.value) if (r >= 0 and out.value) else None
        if out.value:
            self.L.flbref_free(out)
        return r, data, (s.value, ns.value)

    @_recorded()
    def lines_to_events(self, text, key="log", skip_empty_lines=True, sec=0, nsec=0, path_key=None, path=None, offset_key=None, stream_offset=0):
        """in_tail's line loop with the reference's encoder: (chunk bytes or None, bytes consumed, lines seen)"""
        n, used, lines = C.c_size_t(), C.c_size_t(), C.c_size_t()
        b = self._b
        p = self.L.flbref_lines_to_events(text, len(text), b(key), int(skip_empty_lines), sec, nsec, b(path_key), b(path), b(offset_key),
                                          stream_offset, C.byref(n), C.byref(used), C.byref(lines))
        out = C.string_at(p, n.value) if n.value else None
        self.L.flbref_cfree(p)
        return out, used.value, lines.value

    @_recorded()
    def to_json(self, data, json_format=3, date_format=0, date_key="date", escape_unicode=True):
        """flb_pack_msgpack_to_json_format(): bytes or None.  json_format 1 json / 2 stream / 3 lines; date_format 0 double /
        1 iso8601 / 2 epoch / 3 java_sql_timestamp / 4 epoch_ms"""
        n = C.c_size_t()
        buf = C.create_string_buffer(data, len(data))
        p = self.L.flbref_to_json_format(C.cast(buf, C.c_void_p), len(data), json_format, date_format, self._b(date_key), int(escape_unicode), C.byref(n))
        if not p:
            return None
        out = C.string_at(p, n.value)
        self.L.flbref_cfree(p)
        return out

    @_recorded(handle=True)
    def ml_parser(self, name, type="regex", rules=(), match_string=None, negate=False, flush_ms=0, key_content=None,
                  key_group=None, key_pattern=None, parser=None):
        """a [MULTILINE_PARSER] section: flb_ml_parser_create() + one flb_ml_rule_create() per rule + flb_ml_parser_init()"""
        b = self._b
        m = self.L.flbref_ml_parser_create(self.cfg, b(name), b(type), b(match_string), int(negate), flush_ms, b(key_content),
                                           b(key_group), b(key_pattern), b(parser))
        if not m:
            raise RuntimeError("reference rejected multiline parser " + name)
        for frm, rx, to in rules:
            if self.L.flbref_ml_parser_rule(m, b(frm), b(rx), b(to)) != 0:
                raise RuntimeError("reference rejected rule %r of multiline parser %s" % ((frm, rx, to), name))
        if type == "regex" and self.L.flbref_ml_parser_init(m) != 0:
            raise RuntimeError("reference rejected the states of multiline parser " + name)
        return m

    @_recorded(handle=True)
    def filter(self, plugin, props):
        f = self.L.flbref_filter_create(self.cfg, self._b(plugin))
        for k, v in props:
            self.L.flbref_filter_set(f, self._b(k), self._b(v))
        if self.L.flbref_filter_init(self.cfg, f) != 0:
            raise RuntimeError("reference filter init failed: %s %r" % (plugin, props))
        return f

    @_recorded()
    def filter_cb(self, f, data, tag="test"):
        out, n = C.c_void_p(), C.c_size_t()
        buf = C.create_string_buffer(data, len(data))
        r = self.L.flbref_filter_cb(self.cfg, f, C.cast(buf, C.c_void_p), len(data), self._b(tag), C.byref(out), C.byref(n))
        res = None
        if r == 1:
            res = C.string_at(out.value, n.value) if n.value else b""
            if out.value:
                self.L.flbref_free(out)
        return r, res

    @_recorded()
    def chain_do(self, data, tag="test"):
        """flb_filter_do over every filter created on this Ref, in creation order."""
        out, n = C.c_void_p(), C.c_size_t()
        buf = C.create_string_buffer(data, len(data))
        nrec = self.L.flbref_count_records(C.cast(buf, C.c_void_p), len(data))
        r = self.L.flbref_filter_do(self.cfg, C.cast(buf, C.c_void_p), len(data), nrec, self._b(tag), C.byref(out), C.byref(n))
        if r == 0:
            return 2, None
        res = C.string_at(out.value, n.value) if n.value else b""
        if out.value:
            self.L.flbref_free(out)
        return 1, res


# ---------------------------------------------------------------- msgpack bits
def mp_str(b):
    n = len(b)
    if n < 32:
        return bytes([0xa0 | n]) + b
    if n < 256:
        return bytes([0xd9, n]) + b
    if n < 65536:
        return b"\xda" + struct.pack(">H", n) + b
    return b"\xdb" + struct.pack(">I", n) + b


def mp_map_hdr(n):
    if n < 16:
        return bytes([0x80 | n])
    if n < 65536:
        return b"\xde" + struct.pack(">H", n)
    return b"\xdf" + struct.pack(">I", n)


def event(sec, nsec, body_items, meta=b"\x80"):
    """One v2 log event; body_items: list of (key bytes, encoded value bytes)."""
    body = mp_map_hdr(len(body_items)) + b"".join(mp_str(k) + v for k, v in body_items)
    return b"\x92\x92\xd7\x00" + struct.pack(">II", sec & 0xffffffff, nsec & 0xffffffff) + meta + body


def chunk_from_lines(lines, key=b"log", t0=1700000000):
    return b"".join(event(t0 + i, i % 1000, [(key, mp_str(l))]) for i, l in enumerate(lines))


def split_records(chunk):
    """[(offset, length)] of the top-level objects of a chunk (pure python walker)."""
    out, i = [], 0
    while i < len(chunk):
        j = _skip(chunk, i)
        out.append((i, j - i))
        i = j
    return out


def _skip(b, i):
    owed = 1
    while owed:
        owed -= 1
        c = b[i]
        if c < 0x80 or c >= 0xe0 or c in (0xc0, 0xc2, 0xc3):
            i += 1
        elif c <= 0x8f:
            owed += 2 * (c & 15); i += 1
        elif c <= 0x9f:
            owed += c & 15; i += 1
        elif c <= 0xbf:
            i += 1 + (c & 31)
        elif c in (0xc4, 0xd9):
            i += 2 + b[i + 1]
        elif c in (0xc5, 0xda):
            i += 3 + struct.unpack(">H", b[i + 1:i + 3])[0]
        elif c in (0xc6, 0xdb):
            i += 5 + struct.unpack(">I", b[i + 1:i + 5])[0]
        elif c == 0xc7:
            i += 3 + b[i + 1]
        elif c == 0xc8:
            i += 4 + struct.unpack(">H", b[i + 1:i + 3])[0]
        elif c == 0xc9:
            i += 6 + struct.unpack(">I", b[i + 1:i + 5])[0]
        elif c in (0xca, 0xce, 0xd2):
            i += 5
        elif c in (0xcb, 0xcf, 0xd3):
            i += 9
        elif c in (0xcc, 0xd0):
            i += 2
        elif c in (0xcd, 0xd1):
            i += 3
        elif c in (0xd4, 0xd5, 0xd6, 0xd7, 0xd8):
            i += 2 + {0xd4: 1, 0xd5: 2, 0xd6: 4, 0xd7: 8, 0xd8: 16}[c]
        elif c == 0xdc:
            owed += struct.unpack(">H", b[i + 1:i + 3])[0]; i += 3
        elif c == 0xdd:
            owed += struct.unpack(">I", b[i + 1:i + 5])[0]; i += 5
        elif c == 0xde:
            owed += 2 * struct.unpack(">H", b[i + 1:i + 3])[0]; i += 3
        elif c == 0xdf:
            owed += 2 * struct.unpack(">I", b[i + 1:i + 5])[0]; i += 5
        else:
            raise ValueError("bad msgpack byte %02x at %d" % (c, i))
    return i


# ------------------------------------------------------------- synthetic logs
APACHE_RX = (r'^(?<host>[^ ]*) [^ ]* (?<user>[^ ]*) \[(?<time>[^\]]*)\] "(?<method>\S+)(?: +(?<path>[^\"]*?)'
             r'(?: +\S*)?)?" (?<code>[^ ]*) (?<size>[^ ]*)(?: "(?<referer>[^\"]*)" "(?<agent>[^\"]*)")?$')
APACHE_TIME_FMT = "%d/%b/%Y:%H:%M:%S %z"
NGINX_RX = (r'^(?<remote>[^ ]*) (?<host>[^ ]*) (?<user>[^ ]*) \[(?<time>[^\]]*)\] "(?<method>\S+)(?: +(?<path>[^\"]*?)'
            r'(?: +\S*)?)?" (?<code>[^ ]*) (?<size>[^ ]*)(?: "(?<referer>[^\"]*)" "(?<agent>[^\"]*)")')
_MON = ["Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"]
_REF = ["-", "http://example.com/", "https://www.google.com/search?q=fluent", "http://10.0.0.1/index.html",
        "https://example.org/a/b/c", "-", "-", "http://intranet/login"]
_AGENT = ["Mozilla/5.0 (X11; Linux x86_64) AppleWebKit/537.36 (KHTML, like Gecko) Chrome/118.0 Safari/537.36",
          "curl/8.1.2", "Mozilla/5.0 (Macintosh; Intel Mac OS X 10_15_7) Gecko/20100101 Firefox/119.0",
          "kube-probe/1.27", "Go-http-client/1.1", "python-requests/2.31.0", "-", "Prometheus/2.45.0"]


def apache_lines(n, seed=0xF1B1 + 1, garbage=0.005, nginx=False):
    rng = random.Random(seed)
    out = []
    t = 1672531200
    for _ in range(n):
        if rng.random() < garbage:
            out.append(("garbage line %d without structure" % rng.randint(0, 10 ** 6)).encode())
            continue
        host = "%d.%d.%d.%d" % (rng.randint(1, 254), rng.randint(0, 255), rng.randint(0, 255), rng.randint(1, 254))
        user = "-" if rng.random() < 0.9 else "".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(3, 8)))
        t += rng.randint(0, 3)
        y, mo, d = 2023, (t // 2678400) % 12, (t // 86400) % 28 + 1
        ts = "%02d/%s/%d:%02d:%02d:%02d %s" % (d, _MON[mo], y, (t // 3600) % 24, (t // 60) % 60, t % 60,
                                               rng.choice(["+0000", "-0300", "+0900", "+0530"]))
        method = rng.choices(["GET", "POST", "PUT", "HEAD"], [70, 20, 5, 5])[0]
        path = "/" + "".join(rng.choice("abcdefghijklmnopqrstuvwxyz0123456789/_-") for _ in range(rng.randint(4, 48)))
        if rng.random() < 0.05:
            path += "?q=" + str(rng.randint(0, 9999))
        code = rng.choices(["200", "304", "404", "500", "301"], [80, 5, 8, 2, 5])[0]
        size = "-" if rng.random() < 0.03 else str(int(10 ** (rng.random() * 6)))
        line = '%s - %s [%s] "%s %s HTTP/1.1" %s %s' % (host, user, ts, method, path, code, size)
        # (an nginx access line is `$remote_addr - $remote_user [...]`: the parser's `host` group takes the "-";
        #  what differs from the apache lines is that referer and agent are always there)
        if nginx or rng.random() >= 0.10:
            line += ' "%s" "%s"' % (rng.choice(_REF), rng.choice(_AGENT))
        out.append(line.encode())
    return out


_LEVELS = ["debug", "info", "info", "info", "warn", "error", "info", "debug"]
_WORDS = ["request", "completed", "failed", "timeout", "connection", "user", "cache", "miss", "hit", "retry",
          "upstream", "queue", "flush", "chunk", "parser", "filter", "ok", "slow", "db", "auth"]


def json_lines(n, seed=0xF1B1 + 2):
    """SURVEY.md section 8d C2: 6-12 keys in the emitting application's field order, str/int/float/bool/null,
    3 % nested map, 2 % escapes, ~150 B."""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        level = rng.choice(_LEVELS)
        msg = " ".join(rng.choice(_WORDS) for _ in range(rng.randint(3, 8)))
        if rng.random() < 0.02:
            msg += ' \\"quoted\\" caf\\u00e9 \\n tab\\t'
        items = ['"level":"%s"' % level, '"msg":"%s"' % msg, '"status":%d' % rng.choice([200, 200, 200, 404, 500, 301]),
                 '"latency_ms":%s' % ("%.3f" % (rng.random() * 500) if rng.random() < 0.8 else str(rng.randint(0, 5000))),
                 '"ok":%s' % rng.choice(["true", "false"]), '"pid":%d' % rng.randint(1, 65535)]
        if rng.random() < 0.5:
            items.append('"debug":"%s"' % rng.choice(_WORDS))
        if rng.random() < 0.5:
            items.append('"trace_id":"%032x"' % rng.getrandbits(128))
        if rng.random() < 0.3:
            items.append('"user":null')
        if rng.random() < 0.4:
            items.append('"bytes":%d' % int(10 ** (rng.random() * 9)))
        if rng.random() < 0.03:
            items.append('"kubernetes":{"pod":"p-%d","labels":{"app":"%s"},"ports":[80,%d]}' % (i % 977, rng.choice(_WORDS), rng.randint(1000, 9999)))
        if rng.random() < 0.2:
            items.append('"neg":-%d' % rng.randint(1, 10 ** 6))
        # one application writes its fields in one order; which optional fields are present varies
        if rng.random() < 0.005:
            out.append(("not json at all %d" % i).encode())
        else:
            out.append(("{" + ",".join(items) + "}").encode())
    return out


def ltsv_lines(n, seed=77):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        out.append(("host:10.0.%d.%d\tident:-\tuser:%s\ttime:%02d/Oct/2023:13:%02d:%02d +0000\treq:GET /p/%d HTTP/1.1\tstatus:%d\tsize:%d\tempty:"
                    % (rng.randint(0, 255), rng.randint(1, 254), rng.choice(["-", "bob", "alice"]), rng.randint(1, 28), rng.randint(0, 59),
                       rng.randint(0, 59), i, rng.choice([200, 404, 500]), rng.randint(0, 10 ** 6))).encode())
    return out


def logfmt_lines(n, seed=78):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        out.append(('ts=2023-10-%02dT10:%02d:%02dZ level=%s msg="%s" dur=%.2f n=%d flag %s'
                    % (rng.randint(1, 28), rng.randint(0, 59), rng.randint(0, 59), rng.choice(_LEVELS),
                       " ".join(rng.choice(_WORDS) for _ in range(rng.randint(1, 5))), rng.random() * 10, i,
                       rng.choice(["", 'empty=""', "k=v"]))).encode())
    return out


ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")


class Oracle:
    """The plain-C restatement under oracle/ (liboracle.so): same driving interface as Ref."""

    def __init__(self, now=None):
        L = C.CDLL(ORACLE_SO)
        vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
        ll = C.POINTER(C.c_longlong)
        L.orc_config_create.restype = vp
        L.orc_parser_create.restype = vp
        L.orc_parser_create.argtypes = [vp, cp, cp, cp, C.c_int, cp, cp, cp, C.c_int, C.c_int, C.c_int, cp]
        L.orc_parser_do_line.argtypes = [vp, cp, sz, C.POINTER(vp), C.POINTER(sz), ll, ll]
        L.orc_time_lookup_str.argtypes = [vp, cp, sz, ll, ll]
        L.orc_filter_create.restype = vp; L.orc_filter_create.argtypes = [vp, cp]
        L.orc_filter_set.argtypes = [vp, cp, cp]
        L.orc_filter_init.argtypes = [vp, vp]
        L.orc_filter_cb.argtypes = [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)]
        L.orc_chain_do.argtypes = [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)]
        L.orc_l2m_text.restype = vp; L.orc_l2m_text.argtypes = [vp]
        L.orc_free.argtypes = [vp]
        L.orc_set_now.argtypes = [C.c_long]
        L.orc_regex_create.restype = vp; L.orc_regex_create.argtypes = [cp, cp, sz]
        L.orc_regex_search.argtypes = [vp, cp, sz, C.POINTER(C.c_int), C.c_int]
        L.orc_regex_ngroups.argtypes = [vp]
        L.orc_regex_nnames.argtypes = [vp]
        L.orc_regex_name.restype = cp; L.orc_regex_name.argtypes = [vp, C.c_int, C.POINTER(C.c_int)]
        self.L = L
        self.cfg = L.orc_config_create()
        L.orc_set_now(now or 0)

    _b = staticmethod(Ref._b)

    def parser(self, name, format, regex=None, skip_empty=True, time_fmt=None, time_key=None, time_offset=None,
               time_keep=False, time_strict=True, logfmt_no_bare_keys=False, types=None):
        b = self._b
        p = self.L.orc_parser_create(self.cfg, b(name), b(format), b(regex), int(skip_empty), b(time_fmt), b(time_key),
                                     b(time_offset), int(time_keep), int(time_strict), int(logfmt_no_bare_keys), b(types))
        if not p:
            raise RuntimeError("oracle rejected parser " + name)
        return p

    def parser_do(self, p, line):
        out, n = C.c_void_p(), C.c_size_t()
        s, ns = C.c_longlong(), C.c_longlong()
        r = self.L.orc_parser_do_line(p, line, len(line), C.byref(out), C.byref(n), C.byref(s), C.byref(ns))
        data = C.string_at(out.value, n.value) if (r >= 0 and out.value) else None
        if out.value:
            self.L.orc_free(out)
        return r, data, (s.value, ns.value)

    def filter(self, plugin, props):
        f = self.L.orc_filter_create(self.cfg, self._b(plugin))
        for k, v in props:
            self.L.orc_filter_set(f, self._b(k), self._b(v))
        if not f or self.L.orc_filter_init(self.cfg, f) != 0:
            raise RuntimeError("oracle filter init failed: %s %r" % (plugin, props))
        return f

    def chain_do(self, data, tag="test"):
        out, n = C.c_void_p(), C.c_size_t()
        buf = C.create_string_buffer(data, len(data))
        r = self.L.orc_chain_do(self.cfg, C.cast(buf, C.c_void_p), len(data), C.byref(out), C.byref(n))
        if r != 1:
            return 2, None
        res = C.string_at(out.value, n.value) if n.value else b""
        if out.value:
            self.L.orc_free(out)
        return 1, res

    def l2m_text(self, f):
        p = self.L.orc_l2m_text(f)
        t = C.string_at(p).decode(errors="replace")
        self.L.orc_free(C.c_void_p(p))
        return t

    def regex_search(self, pattern, subject):
        """None = no match, else [(beg, end)] per group (as flbref_regex_search reports them)."""
        err = C.create_string_buffer(128)
        re = self.L.orc_regex_create(self._b(pattern), err, 128)
        if not re:
            raise RuntimeError("oracle rejects pattern: %s" % err.value.decode())
        ng = self.L.orc_regex_ngroups(re)
        reg = (C.c_int * (2 * ng))()
        r = self.L.orc_regex_search(re, subject, len(subject), reg, ng)
        if r != 1:
            return None
        return [(reg[2 * i], reg[2 * i + 1]) for i in range(ng)]
