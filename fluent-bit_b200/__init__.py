"""fluent-bit_b200 -- Python mirror (ctypes) of the libflbgpu C ABI (include/flbgpu.h).

The product is the C-ABI library `libflbgpu.so` next to this file (CUDA, sm_90a).  This
module only binds it for tests and bench.py; it contains no compute and no fallback:
importing works without a GPU, but `Context()` raises when the library is missing or no
CUDA device is usable.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_LIB = os.path.join(_HERE, "libflbgpu.so")

FILTER_MODIFIED = 1
FILTER_NOTOUCH = 2
TYPE_INT, TYPE_FLOAT, TYPE_BOOL, TYPE_STRING, TYPE_HEX = 1, 2, 3, 4, 5
_TYPE_NAMES = {"integer": TYPE_INT, "float": TYPE_FLOAT, "bool": TYPE_BOOL, "string": TYPE_STRING, "hex": TYPE_HEX}


class FlbGpuError(RuntimeError):
    pass


class ParserTypes(C.Structure):
    _fields_ = [("key", C.c_char_p), ("key_len", C.c_int), ("type", C.c_int)]


class ParserDecoder(C.Structure):
    _fields_ = [("property", C.c_char_p), ("value", C.c_char_p)]


class Time(C.Structure):
    _fields_ = [("tv_sec", C.c_int64), ("tv_nsec", C.c_int64)]


class PackState(C.Structure):
    _fields_ = [("multiple", C.c_int), ("tokens_count", C.c_int), ("last_byte", C.c_int)]


class Stats(C.Structure):
    _fields_ = [("records_in", C.c_uint64), ("records_out", C.c_uint64), ("bytes_in", C.c_uint64),
                ("bytes_out", C.c_uint64), ("kernel_launches", C.c_uint64), ("passes", C.c_uint32),
                ("error_bits", C.c_uint32), ("phase_ms", C.c_float * 4)]


class GelfFields(C.Structure):
    """struct flbgpu_gelf_fields (struct flb_gelf_fields): None = the default name"""
    _fields_ = [("timestamp_key", C.c_char_p), ("host_key", C.c_char_p), ("short_message_key", C.c_char_p),
                ("full_message_key", C.c_char_p), ("level_key", C.c_char_p)]


EXPORTS = [
    "flbgpu_init", "flbgpu_shutdown", "flbgpu_last_error", "flbgpu_backend_name", "flbgpu_device_count",
    "flbgpu_parser_create", "flbgpu_parser_get", "flbgpu_parser_do", "flbgpu_parser_do_batch", "flbgpu_parser_destroy",
    "flbgpu_filter_new", "flbgpu_filter_set_property", "flbgpu_filter_init", "flbgpu_filter_cb",
    "flbgpu_filter_destroy", "flbgpu_chain_new", "flbgpu_chain_add", "flbgpu_chain_init", "flbgpu_chain_do",
    "flbgpu_chain_destroy", "flbgpu_chain_do_device", "flbgpu_chain_stats", "flbgpu_dev_alloc",
    "flbgpu_dev_free", "flbgpu_dev_upload", "flbgpu_dev_download", "flbgpu_host_alloc", "flbgpu_host_free",
    "flbgpu_stream", "flbgpu_kernel_ms", "flbgpu_chain_stream",
    "flbgpu_comm_unique_id", "flbgpu_comm_init", "flbgpu_l2m_allreduce",
    "flbgpu_pack_state_init", "flbgpu_pack_state_reset", "flbgpu_pack_json_state", "flbgpu_pack_json_state_batch",
    "flbgpu_ml_parser_create", "flbgpu_ml_parser_rule", "flbgpu_ml_parser_init", "flbgpu_ml_set_buffer_limit",
    "flbgpu_msgpack_to_json_format", "flbgpu_msgpack_to_gelf", "flbgpu_lines_to_events", "flbgpu_lines_to_events_parsed", "flbgpu_chain_set_result_buffer",
    "flbgpu_pool_new", "flbgpu_pool_do", "flbgpu_pool_destroy",
]


def load(path=None):
    """dlopen the C-ABI library and declare prototypes."""
    path = path or os.environ.get("FLBGPU_LIB") or PRODUCT_LIB      # FLBGPU_LIB: a build variant, for experiments
    if not os.path.exists(path):
        raise FlbGpuError("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)" % path)
    L = C.CDLL(path)
    vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
    L.flbgpu_init.restype = vp; L.flbgpu_init.argtypes = [C.c_int]
    L.flbgpu_shutdown.argtypes = [vp]
    L.flbgpu_last_error.restype = cp
    L.flbgpu_backend_name.restype = cp
    L.flbgpu_parser_create.restype = vp
    L.flbgpu_parser_create.argtypes = [vp, cp, cp, cp, C.c_int, cp, cp, cp, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.POINTER(ParserTypes), C.c_int, vp]
    L.flbgpu_parser_get.restype = vp; L.flbgpu_parser_get.argtypes = [vp, cp]
    L.flbgpu_parser_do.argtypes = [vp, cp, sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(Time)]
    L.flbgpu_parser_do_batch.argtypes = [vp, vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(vp),
                                         C.POINTER(sz), C.POINTER(C.c_uint64), C.POINTER(Time), C.POINTER(C.c_int)]
    L.flbgpu_parser_destroy.argtypes = [vp]
    L.flbgpu_filter_new.restype = vp; L.flbgpu_filter_new.argtypes = [vp, cp]
    L.flbgpu_filter_set_property.argtypes = [vp, cp, cp]
    L.flbgpu_filter_init.argtypes = [vp]
    L.flbgpu_filter_cb.argtypes = [vp, vp, sz, cp, C.c_int, C.POINTER(vp), C.POINTER(sz)]
    L.flbgpu_filter_destroy.argtypes = [vp]
    L.flbgpu_filter_emitted.argtypes = [vp, vp, C.POINTER(sz)]
    L.flbgpu_chain_new.restype = vp; L.flbgpu_chain_new.argtypes = [vp]
    L.flbgpu_chain_add.argtypes = [vp, vp]
    L.flbgpu_chain_init.argtypes = [vp]
    L.flbgpu_chain_do.argtypes = [vp, vp, sz, cp, C.c_int, C.POINTER(vp), C.POINTER(sz)]
    L.flbgpu_chain_destroy.argtypes = [vp]
    L.flbgpu_chain_do_device.argtypes = [vp, vp, sz, vp, sz, C.POINTER(sz)]
    L.flbgpu_chain_stats.argtypes = [vp, C.POINTER(Stats)]
    L.flbgpu_dev_alloc.restype = vp; L.flbgpu_dev_alloc.argtypes = [vp, sz]
    L.flbgpu_dev_free.argtypes = [vp, vp]
    L.flbgpu_dev_upload.argtypes = [vp, vp, vp, sz]
    L.flbgpu_dev_download.argtypes = [vp, vp, vp, sz]
    L.flbgpu_host_alloc.restype = vp; L.flbgpu_host_alloc.argtypes = [vp, sz]
    L.flbgpu_host_free.argtypes = [vp, vp]
    L.flbgpu_stream.restype = vp; L.flbgpu_stream.argtypes = [vp]
    L.flbgpu_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.flbgpu_chain_stream.restype = vp; L.flbgpu_chain_stream.argtypes = [vp]
    L.flbgpu_pack_json_state.argtypes = [vp, cp, sz, C.POINTER(vp), C.POINTER(C.c_int), C.POINTER(PackState)]
    L.flbgpu_pack_json_state_batch.argtypes = [vp, C.c_int, C.POINTER(cp), C.POINTER(sz), C.POINTER(vp), C.POINTER(C.c_int),
                                               C.POINTER(PackState), C.POINTER(C.c_int)]
    L.flbgpu_ml_parser_create.restype = vp
    L.flbgpu_ml_parser_create.argtypes = [vp, cp, cp, cp, C.c_int, C.c_int, cp, cp, cp, cp]
    L.flbgpu_ml_parser_rule.argtypes = [vp, cp, cp, cp]
    L.flbgpu_ml_parser_init.argtypes = [vp]
    L.flbgpu_ml_set_buffer_limit.argtypes = [vp, sz]
    L.flbgpu_msgpack_to_json_format.argtypes = [vp, vp, sz, C.c_int, C.c_int, cp, C.c_int, C.POINTER(vp), C.POINTER(sz), C.POINTER(sz)]
    L.flbgpu_msgpack_to_gelf.argtypes = [vp, vp, sz, C.POINTER(GelfFields), cp, cp, sz, C.c_int, C.POINTER(vp), C.POINTER(sz),
                                         C.POINTER(sz), C.POINTER(sz)]
    L.flbgpu_lines_to_events.argtypes = [vp, vp, sz, cp, C.c_int, C.c_int64, C.c_int64, cp, cp, cp, C.c_uint64, C.POINTER(vp), C.POINTER(sz),
                                         C.POINTER(sz), C.POINTER(sz)]
    L.flbgpu_lines_to_events_parsed.argtypes = [vp, vp, sz, cp, C.c_int, C.c_int64, C.c_int64, cp, cp, cp, C.c_uint64, C.POINTER(vp),
                                                C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
    L.flbgpu_chain_set_result_buffer.argtypes = [vp, vp, sz]
    L.flbgpu_pool_new.restype = vp; L.flbgpu_pool_new.argtypes = [C.POINTER(vp), C.c_int]
    L.flbgpu_pool_do.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz), cp, C.c_int, C.POINTER(vp), C.POINTER(sz), C.POINTER(C.c_int)]
    L.flbgpu_pool_destroy.argtypes = [vp]
    L.flbgpu_comm_unique_id.argtypes = [vp]
    L.flbgpu_comm_init.argtypes = [vp, C.c_int, C.c_int, vp]
    L.flbgpu_l2m_allreduce.argtypes = [vp]
    ip = C.POINTER(C.c_int); u64p = C.POINTER(C.c_uint64)
    L.flbgpu_l2m_info.argtypes = [vp, ip, ip, ip, ip]
    L.flbgpu_l2m_get.argtypes = [vp, C.c_int, u64p, u64p, C.POINTER(C.c_double), u64p, vp]
    L.flbgpu_l2m_reset.argtypes = [vp]
    L.flbgpu_l2m_put.argtypes = [vp, C.c_uint64, C.c_uint64, C.c_double, u64p, vp]
    L.flbgpu_l2m_text.restype = vp; L.flbgpu_l2m_text.argtypes = [vp]
    return L


L2M_LABEL_BYTES = 256

_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


def _b(s):
    if s is None:
        return None
    return s if isinstance(s, bytes) else s.encode()


class Context:
    """flbgpu_ctx: parsers + filters of one device (mirrors struct flb_config for this path)."""

    def __init__(self, device=0, lib=None):
        self.L = lib if lib is not None else load()
        self.h = self.L.flbgpu_init(device)
        if not self.h:
            raise FlbGpuError("flbgpu_init(%d) failed: %s" % (device, self.err()))

    def err(self):
        e = self.L.flbgpu_last_error()
        return e.decode(errors="replace") if e else ""

    def close(self):
        if getattr(self, "h", None):
            self.L.flbgpu_shutdown(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def comm_unique_id(self):
        buf = C.create_string_buffer(128)
        if self.L.flbgpu_comm_unique_id(C.cast(buf, C.c_void_p)) != 0:
            raise FlbGpuError("comm_unique_id: %s" % self.err())
        return buf.raw

    def comm_init(self, nranks, rank, uid):
        buf = C.create_string_buffer(uid, 128)
        if self.L.flbgpu_comm_init(self.h, nranks, rank, C.cast(buf, C.c_void_p)) != 0:
            raise FlbGpuError("comm_init: %s" % self.err())

    def pack_json_state(self, bufs):
        """flb_pack_json_state() over a batch of stream buffers: [(ret, msgpack bytes or None, last_byte, tokens_count)]"""
        n = len(bufs)
        js = (C.c_char_p * n)(*bufs)
        ln = (C.c_size_t * n)(*[len(b) for b in bufs])
        out = (C.c_void_p * n)(); sizes = (C.c_int * n)(); st = (PackState * n)(); rets = (C.c_int * n)()
        if self.L.flbgpu_pack_json_state_batch(self.h, n, js, ln, out, sizes, st, rets) != 0:
            raise FlbGpuError("pack_json_state_batch: %s" % self.err())
        res = []
        for i in range(n):
            data = None
            if rets[i] == 0:
                data = C.string_at(out[i], sizes[i])
            if out[i]:
                _libc.free(out[i])
            res.append((rets[i], data, st[i].last_byte, st[i].tokens_count))
        return res

    def parser(self, name, format, regex=None, skip_empty=True, time_fmt=None, time_key=None, time_offset=None,
               time_keep=False, time_strict=True, logfmt_no_bare_keys=False, types=None, decoders=None):
        """flb_parser_create(); `types` is the Types option text, e.g. "code:integer size:integer"; `decoders` a list of
        (property, value) pairs such as ("Decode_Field_As", "escaped_utf8 log do_next")."""
        arr, n = None, 0
        dec = None
        if decoders:
            dec = (ParserDecoder * (len(decoders) + 1))()
            for i, (k, v) in enumerate(decoders):
                dec[i].property = _b(k); dec[i].value = _b(v)
        if types:
            items = [t.split(":", 1) for t in types.split() if ":" in t]     # flb_parser_conf: entries without a type are skipped
            arr = (ParserTypes * len(items))()
            for i, (k, t) in enumerate(items):
                arr[i].key = _b(k); arr[i].key_len = len(_b(k)); arr[i].type = _TYPE_NAMES.get(t.lower(), TYPE_STRING)
            n = len(items)
        p = self.L.flbgpu_parser_create(self.h, _b(name), _b(format), _b(regex), int(skip_empty), _b(time_fmt),
                                        _b(time_key), _b(time_offset), int(time_keep), int(time_strict), 0,
                                        int(logfmt_no_bare_keys), arr, n, C.cast(dec, C.c_void_p) if dec is not None else None)
        if not p:
            raise FlbGpuError("parser_create(%s): %s" % (name, self.err()))
        return Parser(self, p)

    def lines_to_events(self, text, key="log", skip_empty_lines=True, sec=0, nsec=0, path_key=None, path=None, offset_key=None,
                        stream_offset=0):
        """in_tail's line loop: (chunk bytes or None, bytes consumed, lines seen)"""
        out, n, used, lines = C.c_void_p(), C.c_size_t(), C.c_size_t(), C.c_size_t()
        buf = C.create_string_buffer(text, len(text))
        r = self.L.flbgpu_lines_to_events(self.h, C.cast(buf, C.c_void_p), len(text), _b(key), int(skip_empty_lines), sec, nsec, _b(path_key),
                                          _b(path), _b(offset_key), stream_offset, C.byref(out), C.byref(n), C.byref(used), C.byref(lines))
        if r < 0:
            raise FlbGpuError("lines_to_events: %s" % self.err())
        chunk = None
        if out.value:
            chunk = C.string_at(out.value, n.value)
            _libc.free(out)
        return chunk, used.value, lines.value

    def to_json(self, data, json_format=3, date_format=0, date_key="date", escape_unicode=True):
        """flb_pack_msgpack_to_json_format(): (text bytes or None, strings whose text is undefined in the reference)"""
        out, n, und = C.c_void_p(), C.c_size_t(), C.c_size_t()
        buf = C.create_string_buffer(data, len(data))
        r = self.L.flbgpu_msgpack_to_json_format(self.h, C.cast(buf, C.c_void_p), len(data), json_format, date_format, _b(date_key),
                                                 int(escape_unicode), C.byref(out), C.byref(n), C.byref(und))
        if r < 0:
            raise FlbGpuError("msgpack_to_json_format: %s" % self.err())
        if r == 1:
            return None, und.value
        text = C.string_at(out.value, n.value)
        _libc.free(out)
        return text, und.value

    def to_gelf(self, data, fields=None, tag_key=None, tag=None, separator=b"\n"):
        """flb_msgpack_to_gelf() on every event, as out_gelf / out_http flush a chunk: (text bytes or None, events that failed,
        events with a string whose text is undefined in the reference).  fields: dict of GelfFields' names (missing or None =
        the default name); separator: b"\n" (out_http) or b"\0" (out_gelf over TCP / TLS)."""
        out, n, failed, und = C.c_void_p(), C.c_size_t(), C.c_size_t(), C.c_size_t()
        buf = C.create_string_buffer(data, len(data))
        f = GelfFields(**{k: _b(v) for k, v in (fields or {}).items()}) if fields is not None else None
        tag = _b(tag)
        sep = separator[0] if isinstance(separator, (bytes, bytearray)) else int(separator)
        r = self.L.flbgpu_msgpack_to_gelf(self.h, C.cast(buf, C.c_void_p), len(data), C.byref(f) if f is not None else None, _b(tag_key),
                                          tag, len(tag) if tag is not None else 0, sep, C.byref(out), C.byref(n), C.byref(failed),
                                          C.byref(und))
        if r < 0:
            raise FlbGpuError("msgpack_to_gelf: %s" % self.err())
        if r == 1:
            return None, failed.value, und.value
        text = C.string_at(out.value, n.value)
        _libc.free(out)
        return text, failed.value, und.value

    def ml_parser(self, name, type="regex", rules=(), match_string=None, negate=False, flush_ms=0, key_content=None,
                  key_group=None, key_pattern=None, parser=None):
        """a [MULTILINE_PARSER] section: flb_ml_parser_create + one flb_ml_rule_create per (from_states, regex, to_state) +
        flb_ml_parser_init"""
        m = self.L.flbgpu_ml_parser_create(self.h, _b(name), _b(type), _b(match_string), int(negate), flush_ms, _b(key_content),
                                           _b(key_group), _b(key_pattern), _b(parser))
        if not m:
            raise FlbGpuError("ml_parser_create(%s): %s" % (name, self.err()))
        for frm, rx, to in rules:
            if self.L.flbgpu_ml_parser_rule(m, _b(frm), _b(rx), _b(to)) != 0:
                raise FlbGpuError("ml_parser_rule(%s): %s" % (name, self.err()))
        if type == "regex" and self.L.flbgpu_ml_parser_init(m) != 0:
            raise FlbGpuError("ml_parser_init(%s): %s" % (name, self.err()))
        return m

    def filter(self, plugin, props):
        """flb_filter_new + set_property (props: ordered list of (key, value)) + cb_init."""
        f = self.L.flbgpu_filter_new(self.h, _b(plugin))
        if not f:
            raise FlbGpuError("filter_new(%s): %s" % (plugin, self.err()))
        for k, v in props:
            self.L.flbgpu_filter_set_property(f, _b(k), _b(v))
        if self.L.flbgpu_filter_init(f) != 0:
            e = self.err()
            self.L.flbgpu_filter_destroy(f)
            raise FlbGpuError("filter_init(%s): %s" % (plugin, e))
        return Filter(self, f)

    def chain(self, filters):
        c = self.L.flbgpu_chain_new(self.h)
        for f in filters:
            if self.L.flbgpu_chain_add(c, f.h) != 0:
                raise FlbGpuError("chain_add failed")
        if self.L.flbgpu_chain_init(c) != 0:
            raise FlbGpuError("chain_init: %s" % self.err())
        return Chain(self, c, filters)


class Parser:
    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h

    def do(self, line):
        """flb_parser_do(): returns (ret, msgpack_bytes or None, (sec, nsec))."""
        out, n, t = C.c_void_p(), C.c_size_t(), Time()
        r = self.ctx.L.flbgpu_parser_do(self.h, line, len(line), C.byref(out), C.byref(n), C.byref(t))
        data = None
        if r >= 0 and out.value:
            data = C.string_at(out.value, n.value)
        if out.value:
            _libc.free(out)
        return r, data, (t.tv_sec, t.tv_nsec)

    def lines_to_events(self, text, key="log", skip_empty_lines=True, sec=0, nsec=0, path_key=None, path=None, offset_key=None,
                        stream_offset=0):
        """in_tail's line loop with this parser as its `Parser`: (chunk bytes or None, bytes consumed, lines seen)"""
        out, n, used, lines = C.c_void_p(), C.c_size_t(), C.c_size_t(), C.c_size_t()
        buf = C.create_string_buffer(text, len(text))
        r = self.ctx.L.flbgpu_lines_to_events_parsed(self.h, C.cast(buf, C.c_void_p), len(text), _b(key), int(skip_empty_lines), sec, nsec,
                                                     _b(path_key), _b(path), _b(offset_key), stream_offset, C.byref(out), C.byref(n),
                                                     C.byref(used), C.byref(lines))
        if r < 0:
            raise FlbGpuError("lines_to_events_parsed: %s" % self.ctx.err())
        chunk = None
        if out.value:
            chunk = C.string_at(out.value, n.value)
            _libc.free(out)
        return chunk, used.value, lines.value


def _parser_do_batch(self, lines):
    """flbgpu_parser_do_batch(): [(ret, msgpack map bytes or None, (sec, nsec))] for a list of lines."""
    n = len(lines)
    base = b"".join(lines)
    off = (C.c_uint32 * n)(); ln = (C.c_uint32 * n)()
    at = 0
    for i, l in enumerate(lines):
        off[i] = at; ln[i] = len(l); at += len(l)
    out, osz = C.c_void_p(), C.c_size_t()
    ooff = (C.c_uint64 * (n + 1))(); tm = (Time * n)(); ret = (C.c_int * n)()
    buf = C.create_string_buffer(base, len(base) + 1)
    r = self.ctx.L.flbgpu_parser_do_batch(self.h, C.cast(buf, C.c_void_p), off, ln, n, C.byref(out), C.byref(osz), ooff, tm, ret)
    if r != 0:
        raise FlbGpuError("parser_do_batch failed: %s" % self.ctx.err())
    blob = C.string_at(out.value, osz.value) if osz.value else b""
    if out.value:
        _libc.free(out)
    return [(ret[i], blob[ooff[i]:ooff[i + 1]] if ret[i] >= 0 else None, (tm[i].tv_sec, tm[i].tv_nsec)) for i in range(n)]


Parser.do_batch = _parser_do_batch


def _call_filter(fn, L, handle, data, tag, keep=None):
    """keep: address of a result buffer registered with flbgpu_chain_set_result_buffer (not freed here)"""
    out, n = C.c_void_p(), C.c_size_t()
    buf = C.create_string_buffer(data, len(data)) if not isinstance(data, C.Array) else data
    r = fn(handle, C.cast(buf, C.c_void_p), len(data), _b(tag), len(_b(tag)), C.byref(out), C.byref(n))
    if r < 0:
        e = L.flbgpu_last_error()
        raise FlbGpuError("filter call failed: %s" % (e.decode(errors="replace") if e else "?"))
    res = None
    if r == FILTER_MODIFIED:
        res = C.string_at(out.value, n.value) if n.value else b""
    if out.value and out.value != keep:
        _libc.free(out)
    return r, res


class EmitGroup(C.Structure):
    """struct flbgpu_emit_group (include/flbgpu.h)"""
    _fields_ = [("tag", C.c_void_p), ("tag_len", C.c_size_t), ("data", C.c_void_p), ("size", C.c_size_t), ("records", C.c_size_t)]


class Filter:
    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.L.flbgpu_filter_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def cb(self, data, tag="test"):
        """cb_filter(): (FILTER_MODIFIED, bytes) or (FILTER_NOTOUCH, None)."""
        return _call_filter(self.ctx.L.flbgpu_filter_cb, self.ctx.L, self.h, data, tag)

    # ---- filter_rewrite_tag: what the last call handed to the emitter ----
    def emitted(self):
        """[(new tag, records bytes, record count)]: tags in order of first appearance, records of a tag in chunk order"""
        groups, n = C.POINTER(EmitGroup)(), C.c_size_t()
        if self.ctx.L.flbgpu_filter_emitted(self.h, C.byref(groups), C.byref(n)) != 0:
            raise FlbGpuError("not a rewrite_tag filter")
        return [(C.string_at(groups[i].tag, groups[i].tag_len), C.string_at(groups[i].data, groups[i].size), groups[i].records)
                for i in range(n.value)]

    # ---- filter_log_to_metrics state (the plugin's ctx->cmt) ----
    def l2m_info(self):
        m, nl, nb, ns = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        if self.ctx.L.flbgpu_l2m_info(self.h, C.byref(m), C.byref(nl), C.byref(nb), C.byref(ns)) != 0:
            raise FlbGpuError("not a log_to_metrics filter")
        return m.value, nl.value, nb.value, ns.value

    def l2m_sets(self):
        """[(hash, (label, ...), count, sum, [cumulative buckets..., +Inf])] in first-seen order."""
        _, nl, nb, ns = self.l2m_info()
        out = []
        for i in range(ns):
            h, c, s = C.c_uint64(), C.c_uint64(), C.c_double()
            bk = (C.c_uint64 * (nb + 1))()
            lab = C.create_string_buffer(max(nl, 1) * L2M_LABEL_BYTES)
            self.ctx.L.flbgpu_l2m_get(self.h, i, C.byref(h), C.byref(c), C.byref(s), bk, C.cast(lab, C.c_void_p))
            raw = lab.raw
            labels = tuple(raw[j * L2M_LABEL_BYTES + 1: j * L2M_LABEL_BYTES + 1 + raw[j * L2M_LABEL_BYTES]] for j in range(nl))
            out.append((h.value, labels, c.value, s.value, list(bk)))
        return out

    def l2m_replace(self, sets):
        """Replace the table (used after a cross-rank merge)."""
        _, nl, nb, _ = self.l2m_info()
        self.ctx.L.flbgpu_l2m_reset(self.h)
        for h, labels, c, s, bk in sets:
            lab = bytearray(max(nl, 1) * L2M_LABEL_BYTES)
            for j, v in enumerate(labels):
                lab[j * L2M_LABEL_BYTES] = len(v)
                lab[j * L2M_LABEL_BYTES + 1: j * L2M_LABEL_BYTES + 1 + len(v)] = v
            arr = (C.c_uint64 * (nb + 1))(*bk)
            buf = (C.c_char * len(lab)).from_buffer(lab)
            self.ctx.L.flbgpu_l2m_put(self.h, h, c, s, arr, C.cast(buf, C.c_void_p))

    def l2m_text(self):
        p = self.ctx.L.flbgpu_l2m_text(self.h)
        if not p:
            raise FlbGpuError("not a log_to_metrics filter")
        t = C.string_at(p).decode(errors="replace")
        _libc.free(p)
        return t

    def l2m_allreduce_lib(self):
        """flbgpu_l2m_allreduce(): the library's own exchange (NCCL; the context needs comm_init first)"""
        if self.ctx.L.flbgpu_l2m_allreduce(self.h) != 0:
            raise FlbGpuError("l2m_allreduce: %s" % self.ctx.err())

    def l2m_allreduce(self, device=None):
        """The same merge spelled with torch.distributed (kept as an independent check of the library's exchange).
        Sum this filter's metric table over all ranks of the default process group (the one
        exchange step of the path: cmetrics of N shards -> one table).  Keys travel with one
        all_gather, values with ONE all_reduce (NCCL on GPUs, gloo in the CPU tests).  Label sets
        end up in (rank, first-seen) order on every rank."""
        import torch
        import torch.distributed as dist
        mode, nl, nb, _ = self.l2m_info()
        mine = self.l2m_sets()
        world = dist.get_world_size()
        gathered = [None] * world
        dist.all_gather_object(gathered, [(h, labels) for h, labels, _, _, _ in mine])
        order, seen = [], {}
        for per_rank in gathered:
            for h, labels in per_rank:
                if h not in seen:
                    seen[h] = len(order)
                    order.append((h, labels))
        n = len(order)
        dev = device if device is not None else ("cuda" if dist.get_backend() == "nccl" else "cpu")
        if mode == 1:
            # gauge: the last record wins and shards are consecutive record ranges, so the value of the
            # highest rank that saw the set stays.  Still ONE all_reduce: rank r owns column pair r of an
            # int64 matrix (seen flag, value bits); adding zeros keeps the bits exact.
            import struct
            rank = dist.get_rank()
            buf = torch.zeros((n, 2 * world + 1), dtype=torch.int64)
            for h, _, c, s, _bk in mine:
                i = seen[h]
                buf[i, 0] = c
                buf[i, 1 + 2 * rank] = 1
                buf[i, 2 + 2 * rank] = struct.unpack("<q", struct.pack("<d", s))[0]
            if n:
                buf = buf.to(dev)
                dist.all_reduce(buf)
                buf = buf.cpu()
            merged = []
            for i, (h, labels) in enumerate(order):
                last = max(r for r in range(world) if int(buf[i, 1 + 2 * r]))
                val = struct.unpack("<d", struct.pack("<q", int(buf[i, 2 + 2 * last])))[0]
                merged.append((h, labels, int(buf[i, 0]), val, [0] * (nb + 1)))
            self.l2m_replace(merged)
            return merged
        counts = torch.zeros((n, nb + 2), dtype=torch.int64)
        sums = torch.zeros((n,), dtype=torch.float64)
        for h, _, c, s, bk in mine:
            i = seen[h]
            counts[i, 0] = c
            counts[i, 1:] = torch.tensor(bk, dtype=torch.int64)
            sums[i] = s
        if n:
            # one collective: the float64 sums ride in the same buffer, bit-cast to int64 lanes would
            # not add correctly, so the buffer is [counts | sums] as float64 only when exact (< 2^53)
            counts = counts.to(dev); sums = sums.to(dev)
            if int(counts.max()) < (1 << 52):
                buf = torch.cat([counts.to(torch.float64).reshape(-1), sums])
                dist.all_reduce(buf)
                counts = buf[: n * (nb + 2)].reshape(n, nb + 2).to(torch.int64)
                sums = buf[n * (nb + 2):]
            else:
                dist.all_reduce(counts); dist.all_reduce(sums)
            counts = counts.cpu(); sums = sums.cpu()
        merged = [(h, labels, int(counts[i, 0]), float(sums[i]), [int(x) for x in counts[i, 1:]])
                  for i, (h, labels) in enumerate(order)]
        self.l2m_replace(merged)
        return merged


class Chain:
    def __init__(self, ctx, h, filters):
        self.ctx, self.h, self.filters = ctx, h, filters

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.L.flbgpu_chain_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stream(self):
        """the cudaStream_t this instance launches on"""
        return self.ctx.L.flbgpu_chain_stream(self.h)

    def do(self, data, tag="test"):
        return _call_filter(self.ctx.L.flbgpu_chain_do, self.ctx.L, self.h, data, tag, keep=getattr(self, "_res_addr", None))

    def set_result_buffer(self, nbytes):
        """flbgpu_chain_set_result_buffer() with a buffer of nbytes owned by this object (0: back to malloc only)"""
        self._res = C.create_string_buffer(nbytes) if nbytes else None
        self._res_addr = C.addressof(self._res) if nbytes else None
        self.ctx.L.flbgpu_chain_set_result_buffer(self.h, C.cast(self._res, C.c_void_p) if nbytes else None, nbytes)

    def stats(self):
        s = Stats()
        self.ctx.L.flbgpu_chain_stats(self.h, C.byref(s))
        return s
