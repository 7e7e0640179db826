#!/usr/bin/env python3
"""Cost of the token-joining options: the config-2 batch (8192 synthetic sentences, Knlm model, bench.py) through kiwi_b200_analyze_batch,
alternately without join options (MATCH_ALL_WITH_NORMALIZING) and with J1 (+ joinAffix + joinParticleYo, tests/joinio.py).  Prints one JSON
line: per arm the median over --steps calls of the device milliseconds of the emit / pack phase (emit_kernel or emit_join_kernel, the token
scan and pack, and with J1 the form scan and pack) and of the whole call (H2D to D2H), with the card's name and power limit.
usage: python scripts/join_bench.py [--steps 20] [--warmup 3]"""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kiwi_b200      # noqa: E402
from kiwi_b200.synth import synth_batch      # noqa: E402
from tests.joinio import J1      # noqa: E402
from tests.orc import IMAGE      # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    kw = kiwi_b200.Kiwi(IMAGE, device=0)
    blob, off = kiwi_b200.encode_batch(synth_batch(8192))
    arms = {"plain": kiwi_b200.default_option(kiwi_b200.MATCH_ALL_WITH_NORMALIZING), "J1": kiwi_b200.default_option(J1)}
    times = {a: {"pack": [], "total": []} for a in arms}
    joined = 0
    for step in range(args.warmup + args.steps):
        for a, opt in arms.items():      # (the arms alternate, so drift of the shared machine hits both)
            r = kw.analyze_batch_arrays(blob, off, opt)
            if step >= args.warmup:
                times[a]["pack"].append(r.timings_ms["pack"]); times[a]["total"].append(r.timings_ms["total"])
            if a == "J1":
                joined = int(((r.tokens["morph_id"] & kiwi_b200.JOINED_TOKEN) != 0).sum())
    out = {"card": card(), "batch": 8192, "steps": args.steps, "joined_tokens": joined}
    for a in arms:
        out[a] = {"ms_emit_pack": round(statistics.median(times[a]["pack"]), 4), "ms_total": round(statistics.median(times[a]["total"]), 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
