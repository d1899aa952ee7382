"""The reference's own GELF tests, as data.

tests/internal/gelf.c packs a record with msgpack_pack_*() calls, sets a time and the short message key, and compares
flb_msgpack_raw_to_gelf()'s text with an expected string.  The five flb_test_format_gelf* cases of tests/runtime/out_http.c push
one JSON event through in_lib into out_http with `format gelf` and gelf_* keys, and look for substrings in the payload.  This
script reads those files where they lie (/root/reference, this container only), extracts per test the record, the time, the
field keys and what the test asserts, runs the UNMODIFIED reference converter on the event (oracle/_ref/libflbref_gelf.so),
and writes tests/golden/gelf_scenarios.json -- which travels, the reference does not.  tests/test_zz_gelf.py then asserts, on
the CPU emulation and on the GPU, the reference test's own expectation AND byte equality with the reference's output.

usage: python tests/golden/make_gelf_scenarios.py"""
import base64
import json
import os
import re
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import gelf_ref
import util
from make_runtime_scenarios import call_args, functions, literals
from scenario_util import chunk_from_json_events

REF = "/root/reference/tests"
FIELD_PROPS = {"gelf_timestamp_key": "timestamp_key", "gelf_host_key": "host_key", "gelf_short_message_key": "short_message_key",
               "gelf_full_message_key": "full_message_key", "gelf_level_key": "level_key"}


def packed(body):
    """the bytes of a sequence of msgpack_pack_*() calls"""
    out = b""
    for m in re.finditer(r"msgpack_pack_(\w+)\(&mp_pck(?:,\s*([^;]*))?\);", body):
        fn, arg = m.group(1), (m.group(2) or "").strip()
        if fn == "map":
            out += util.mp_map_hdr(int(arg))
        elif fn == "array":
            out += bytes([0x90 | int(arg)])
        elif fn == "str":
            n = int(arg)
            out += bytes([0xa0 | n]) if n < 32 else bytes([0xd9, n])
        elif fn == "str_body":
            out += literals(arg.rsplit(",", 1)[0]).encode()
        elif fn == "true":
            out += b"\xc3"
        elif fn == "false":
            out += b"\xc2"
        elif fn == "uint64":
            v = int(arg)
            out += bytes([v]) if v < 128 else b"\xcd" + struct.pack(">H", v) if v < 65536 else b"\xce" + struct.pack(">I", v)
        else:
            raise ValueError("unhandled msgpack_pack_%s" % fn)
    return out


def internal():
    src = open(os.path.join(REF, "internal", "gelf.c")).read()
    macros = {m.group(1): literals(m.group(2)) for m in re.finditer(r"#define (EXPECTED_\w+)\s*\\?\n?((?:\s*\"(?:[^\"\\]|\\.)*\"\s*\\?\n?)+)", src)}
    for name, body in re.findall(r"\nvoid (test_\w+)\(\)\n\{(.*?)\n\}\n", src, re.S):
        sec = int(re.search(r"ts\.tm\.tv_sec\s*=\s*(\d+);", body).group(1))
        nsec = int(re.search(r"ts\.tm\.tv_nsec\s*=\s*(\d+);", body).group(1))
        fields = {k: literals(v) for k, v in re.findall(r"fields\.(\w+)\s*=\s*flb_sds_create\((\"[^\"]*\")\)", body)}
        want = macros[re.search(r"strcmp\(out, (EXPECTED_\w+)\)", body).group(1)]
        chunk = b"\x92\x92\xd7\x00" + struct.pack(">II", sec, nsec) + b"\x80" + packed(body)
        yield dict(source="tests/internal/gelf.c", test=name, fields=fields, chunk=chunk, equals=want, present=[])


def runtime():
    src = open(os.path.join(REF, "runtime", "out_http.c")).read()
    for name, body in functions(src):
        if not name.startswith("flb_test_format_gelf"):
            continue
        props = {}
        for args in call_args(body, "flb_output_set"):
            rest = [literals(a) for a in args[2:] if a != "NULL"]
            props.update(zip(rest[0::2], rest[1::2]))
        assert props.get("format") == "gelf", name
        fields = {FIELD_PROPS[k]: v for k, v in props.items() if k in FIELD_PROPS}
        text = literals(re.search(r"char \*buf1 = (\"(?:[^\"\\]|\\.)*\")", body).group(1))
        # in_lib's tokeniser reads the primitive `6"` of flb_test_format_gelf_level_key as the number 6, as its expectation shows
        text = text.replace(':6"}', ":6}")
        present = [literals(x) for x in re.findall(r"\"(?:[^\"\\]|\\.)*\"", re.search(r"expected_strs\[\] = \{(.*?)\};", body, re.S).group(1))]
        yield dict(source="tests/runtime/out_http.c", test=name, fields=fields, chunk=chunk_from_json_events([text]), equals=None,
                   present=present)


def main():
    if not gelf_ref.have_ref():
        sys.exit("oracle/_ref/libflbref_gelf.so is not built")
    ref = gelf_ref.GelfRef()
    out = []
    for sc in list(internal()) + list(runtime()):
        text, failed = ref.to_gelf(sc["chunk"], sc["fields"])
        assert failed == 0 and text is not None, sc["test"]
        if sc["equals"] is not None:
            assert text == sc["equals"].encode() + b"\n", (sc["test"], text)
        for p in sc["present"]:
            assert p.encode() in text, (sc["test"], p, text)
        sc["chunk"] = base64.b64encode(sc["chunk"]).decode()
        sc["ref_out"] = text.decode("latin-1")
        out.append(sc)
    with open(os.path.join(HERE, "gelf_scenarios.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("%d scenarios" % len(out))


if __name__ == "__main__":
    main()
