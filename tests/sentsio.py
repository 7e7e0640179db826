"""Reader for the sentence-splitting vectors (tests/golden/docs_sents.jsonl and <prefix>docs_sents.golden.txt.gz, written by
tests/golden/make_docs.py with oracle/ref_build/tools/split_sents.cpp) - test infrastructure."""
import gzip, json, os

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def read_docs():
    with open(os.path.join(HERE, "docs_sents.jsonl"), encoding="utf-8", newline="\n") as f:
        return [json.loads(l) for l in f if l.strip()]


def _ranges(fields):
    return [tuple(int(v) for v in x.split(",")) for x in fields[2:]]


def read_sents_golden(prefix=""):
    """-> per document dict(tokens=[(morph, tag, pos, len, score)], forms=[((word, sent, line, subSent, paired), form)], score,
    ranges=[(begin, end)] in UTF-16 units, byte_ranges=[(begin, end)] in UTF-8 bytes)"""
    out = []
    with gzip.open(os.path.join(HERE, prefix + "docs_sents.golden.txt.gz"), "rb") as f:
        for raw in f.read().split(b"\n"):
            if not raw:
                continue
            line = raw.decode("utf-8")
            p = line.split(" ")
            if p[0] == "S":
                out.append(dict(tokens=[], forms=[], score=float.fromhex(p[3])))
            elif p[0] == "T":
                cur = out[-1]
                cur["tokens"].append((int(p[1]) & 0xFFFFFFFF, int(p[2]), int(p[3]), int(p[4]), float.fromhex(p[5])))
                cur["forms"].append((tuple(int(x) for x in p[6].split(",")), line.split(" ", 7)[7] if len(p) > 7 else ""))
            elif p[0] == "R":
                out[-1]["ranges"] = _ranges(p)
            elif p[0] == "B":
                out[-1]["byte_ranges"] = _ranges(p)
    return out
