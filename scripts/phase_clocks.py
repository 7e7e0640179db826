#!/usr/bin/env python3
"""Diagnostic: where the heaviest sentences of one 8192-sentence Knlm batch spend their Viterbi time.  Needs a library whose
Knlm Viterbi object was built with -DKB_PHASE_CLOCKS (never the shipped one), selected with KIWI_B200_LIB:

  make -C kiwi_b200/csrc variant NAME=phase VFLAGS="<KNLM_FLAGS of the Makefile> -DKB_PHASE_CLOCKS=1"
  KIWI_B200_LIB=kiwi_b200/variants/libkiwi_b200_phase.so python scripts/phase_clocks.py [tag] [output directory, default .]

-> <output directory>/phases_<tag>.json: per-sentence clock64 cycles of each phase (lane 0 of the sentence's warp) and the sentence's `top1`
containers (count, entries, bucket counts, rehashes), for the 24 sentences with the longest Viterbi (%globaltimer).  Inside `evaluate`:
path staging, candidate classification, the candidate walk (`enumeration` = the walk minus the calls it makes: flushItems, the
per-candidate path, the exact redo and the `top1` order), the per-candidate path `evalCand` on `top1` nodes of more than 768 incoming
paths ("big") and on the others, the exact group redo, and how many big nodes and candidates the sentence evaluated."""
import ctypes as C, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import kiwi_b200
from kiwi_b200.synth import synth_batch, u16len
from tests.orc import IMAGE

# the order of the PH_* enum in viterbi.cu
PHASES = ["top1_order", "top1_reorder", "flush_items", "evaluate", "prune", "node_loop", "find_best_path",
          "n_top1", "sum_E", "sum_B", "rehashes",
          "stage_paths", "classify", "walk", "eval_cand_small", "eval_cand_big", "redo_exact", "n_big_nodes", "n_big_cands"]
tag = sys.argv[1] if len(sys.argv) > 1 else "phase"
out_dir = sys.argv[2] if len(sys.argv) > 2 else "."
kw = kiwi_b200.Kiwi(IMAGE)
lib = kiwi_b200.load_library()
if not hasattr(lib, "kiwi_b200_debug_phase_clocks"):
    raise SystemExit("the loaded library has no phase clocks: build a -DKB_PHASE_CLOCKS variant and select it with KIWI_B200_LIB")
lib.kiwi_b200_debug_phase_clocks.argtypes = [C.c_void_p]
buf = np.zeros((8192, len(PHASES)), np.uint64)
texts = synth_batch(8192)
blob, off = kiwi_b200.encode_batch(texts)
for _ in range(2):
    kw.analyze_batch_arrays(blob, off)
assert lib.kiwi_b200_debug_phase_clocks(buf.ctypes.data) == len(PHASES)      # (zeroes the counters)
kw.analyze_batch_arrays(blob, off)
assert lib.kiwi_b200_debug_phase_clocks(buf.ctypes.data) == len(PHASES)
t = kw.debug_timing(len(texts)).astype(np.int64)
dur = t[:, 1] - t[:, 0]
lens = np.array([u16len(x) for x in texts])
ph = buf.astype(np.float64)
P = {k: ph[:, i] for i, k in enumerate(PHASES)}
top = []
for i in np.argsort(-dur)[:24]:
    fb = P["find_best_path"][i]
    rest_eval = P["evaluate"][i] - P["flush_items"][i] - P["top1_reorder"][i] - P["prune"][i]
    share = lambda x: float(x / fb) if fb else 0.0
    top.append({"idx": int(i), "len": int(lens[i]), "dur_ms": float(dur[i] / 1e6), "cycles": int(fb),
                "top1_order": share(P["top1_order"][i]), "top1_reorder": share(P["top1_reorder"][i]), "flush_items": share(P["flush_items"][i]),
                "evaluate_rest": share(rest_eval), "prune": share(P["prune"][i]),
                "end_node_and_setup": share(fb - P["node_loop"][i]), "outside_evaluate": share(P["node_loop"][i] - P["evaluate"][i]),
                "stage_paths": share(P["stage_paths"][i]), "classify": share(P["classify"][i]),
                "enumeration": share(P["walk"][i] - P["flush_items"][i] - P["eval_cand_small"][i] - P["eval_cand_big"][i] - P["redo_exact"][i] - P["top1_reorder"][i]),
                "eval_cand_small": share(P["eval_cand_small"][i]), "eval_cand_big": share(P["eval_cand_big"][i]), "redo_exact": share(P["redo_exact"][i]),
                "n_big_nodes": int(P["n_big_nodes"][i]), "n_big_cands": int(P["n_big_cands"][i]),
                "n_top1": int(P["n_top1"][i]), "sum_E": int(P["sum_E"][i]), "sum_B": int(P["sum_B"][i]), "rehashes": int(P["rehashes"][i])})
tot = {k: float(P[k].sum()) for k in PHASES}
out = {"tag": tag, "span_ms": float((t[:, 1].max() - t[:, 0].min()) / 1e6),
       "batch": {"top1_order_share": tot["top1_order"] / tot["find_best_path"], "top1_reorder_share": tot["top1_reorder"] / tot["find_best_path"],
                 "n_top1": int(tot["n_top1"]), "sum_E": int(tot["sum_E"]), "sentences_with_top1": int((P["n_top1"] > 0).sum())},
       "top": top}
os.makedirs(out_dir, exist_ok=True)
json.dump(out, open(os.path.join(out_dir, "phases_%s.json" % tag), "w"), indent=1)
print(json.dumps(out["batch"]))
for r in top[:8]: print(r)
