#!/usr/bin/env python3
"""GPU-box diagnostic: per-sentence Viterbi {start, end} of one 8192-sentence batch (kiwi_b200_debug_timing) ->
gpurun_out/timing_<model>.json: kernel span, the slowest sentences, how much of the span the machine is busy."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import kiwi_b200
from kiwi_b200.synth import synth_batch, u16len
from tests.orc import IMAGE, CONG_IMAGE

model = sys.argv[1] if len(sys.argv) > 1 else "knlm"
tag = sys.argv[2] if len(sys.argv) > 2 else model
kw = kiwi_b200.Kiwi(CONG_IMAGE if model == "cong" else IMAGE)
# resident Viterbi warps per SM (kiwi_b200/csrc/Makefile, viterbi.cu): Knlm 1 block of 12 warps, CoNg 3 blocks of 4 warps
slots = torch.cuda.get_device_properties(0).multi_processor_count * 12
texts = synth_batch(8192)
blob, off = kiwi_b200.encode_batch(texts)
for _ in range(3):
    kw.analyze_batch_arrays(blob, off)
t = kw.debug_timing(len(texts)).astype(np.int64)
start = t[:, 0] - t[:, 0].min(); end = t[:, 1] - t[:, 0].min(); dur = end - start
span = int(end.max())
order = np.argsort(-dur)
lens = np.array([u16len(x) for x in texts])
out = {"model": model, "tag": tag, "span_ms": span / 1e6, "sum_dur_ms": float(dur.sum() / 1e6), "mean_dur_ms": float(dur.mean() / 1e6),
       "p50_ms": float(np.percentile(dur, 50) / 1e6), "p99_ms": float(np.percentile(dur, 99) / 1e6), "max_ms": float(dur.max() / 1e6),
       "warp_slots": slots, "busy_fraction_of_warp_slots": float(dur.sum() / (span * float(slots))),
       "last_start_ms": float(start.max() / 1e6),
       "top": [{"idx": int(i), "len": int(lens[i]), "start_ms": float(start[i] / 1e6), "dur_ms": float(dur[i] / 1e6)} for i in order[:24]],
       "dur_us": (dur // 1000).tolist()}
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "timing_%s.json" % tag), "w"))
print({k: v for k, v in out.items() if k not in ("dur_us", "top")}); print(out["top"][:8])
