"""Golden vectors of in_tail's `Parser` branch, produced from the UNMODIFIED reference (oracle/_ref): the line loop restated in the
harness around the reference's flb_parser_do() and log event encoder (oracle/refshim/tail_harness.c).
  tail_parser_vectors.json -- parser (a name of test_zz_tail_parser.PARSERS), text and arguments in; chunk / consumed / lines out
Run from the repository root with oracle/_ref built: python tests/golden/make_tail_parser_vectors.py"""
import base64
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import tail_ref                  # noqa: E402
import test_zz_tail_parser as TP  # noqa: E402

B = lambda b: base64.b64encode(b).decode()


def vectors():
    rng = random.Random(61)
    ref = tail_ref.TailRef(keep_whole=True)
    handles = {n: ref.parser(**TP.PARSERS[n]) for n in TP.PARSERS}
    out = []
    for r in range(28):
        name = sorted(TP.PARSERS)[r % len(TP.PARSERS)]
        t = TP.text(name, rng, rng.choice([0, 1, 3, 12, 40]))
        kw = dict(key=rng.choice(["log", "message"]), skip_empty_lines=bool(r % 2), sec=1700000000 + r, nsec=r * 1000)
        if r % 3 == 0:
            kw.update(path_key="file", path="/var/log/x-%d.log" % r)
        if r % 4 == 0:
            kw.update(offset_key="offset", stream_offset=2 ** 31 * (r % 8))
        chunk, used, n = ref.lines_to_events_parsed(handles[name], t, **kw)
        out.append({"parser": name, "text": B(t), "kw": kw, "out": B(chunk) if chunk is not None else None, "consumed": used, "lines": n})
    return out


if __name__ == "__main__":
    json.dump(vectors(), open(os.path.join(ROOT, "tests", "golden", "tail_parser_vectors.json"), "w"), indent=0)
