#!/usr/bin/env python3
"""Sentence splitting on the GPU: kiwi_b200_split_batch against kiwi_b200_analyze_batch on the same documents, in one process,
alternating the two calls.  Documents: seeded, 4-16 kiwi_b200.synth sentences each (each closed by a final mark), joined by the
separators of tests/golden/docs_sents.jsonl.  Prints one JSON line: per call the device times (ms_sents, ms_total), documents/s and
sentences/s end to end (host clock around the call), and the bytes copied back, with the card's name and power limit.
usage: python scripts/sents_bench.py [--docs 8192] [--reps 5] [--warmup 2] [--out PATH]"""
import argparse, json, os, random, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import kiwi_b200
from kiwi_b200.synth import synth_batch
from tests.orc import IMAGE

SEPS = [" ", "\n", "\r\n", "\n\n", "\r\n\r\n", "\v", "\f", " ", "  ", " \n "]
ENDS = [".", "?", "!", "다.", "요.", "..."]


def make_docs(n, seed=2026):
    rng = random.Random(seed)
    counts = [rng.randint(4, 16) for _ in range(n)]
    sents = synth_batch(sum(counts), seed)
    docs, k = [], 0
    for c in counts:
        parts = [s + rng.choice(ENDS) for s in sents[k:k + c]]
        k += c
        doc = parts[0]
        for p in parts[1:]:
            doc += rng.choice(SEPS) + p
        docs.append(doc)
    return docs


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power = out.strip().splitlines()[0].split(", ")
        return name, power
    except Exception as e:      # (reported, never guessed)
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    docs = make_docs(a.docs)
    blob, off = kiwi_b200.encode_batch(docs)
    kw = kiwi_b200.Kiwi(IMAGE)
    runs = {"split": [], "analyze": []}
    n_sents = None
    for rep in range(a.warmup + a.reps):
        for which in ("split", "analyze"):
            t0 = time.perf_counter()
            r = kw.split_batch((blob, off)) if which == "split" else kw.analyze_batch_arrays(blob, off)
            wall = (time.perf_counter() - t0) * 1e3
            st = kw.last_stats()
            if which == "split":
                n_sents = int(r.sent_offsets[-1])
            if rep >= a.warmup:
                runs[which].append(dict(wall_ms=wall, d2h_bytes=int(st.d2h_bytes), retried=int(st.retried), **{"ms_" + k: float(v) for k, v in r.timings_ms.items()}))
            del r
    med = lambda xs: float(np.median(xs))
    res = {}
    for which, rs in runs.items():
        wall = med([x["wall_ms"] for x in rs])
        res[which] = {k: med([x[k] for x in rs]) for k in rs[0]}
        res[which]["docs_per_s"] = a.docs / wall * 1e3
        res[which]["sents_per_s"] = n_sents / wall * 1e3
        res[which]["wall_ms_all"] = [round(x["wall_ms"], 3) for x in rs]
    name, power = card()
    out = dict(card=name, power_limit=power, docs=a.docs, units=int(off[-1]), sentences=n_sents, reps=a.reps,
               sents_share_of_split_total=res["split"]["ms_sents"] / res["split"]["ms_total"], **res)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    kw.close()


if __name__ == "__main__":
    main()
