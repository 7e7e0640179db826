#!/usr/bin/env python3
"""Serial dependent loads of the LM steps (no GPU).  Runs bench batches through the 32-lane host simulation of the device pipeline and
counts, per sentence, the loads on each LM step's critical path: the loads of the main chain (probe slots, root table reads), its
backoff levels, and the loads the kernels spent after a leaf before the model loader stored the state after every leaf edge in the
edge's table entry (kiwi_b200/csrc/lm_tables.h).  Those come in two kinds, reported apart: the suffix walk after a leaf edge of a
non-root node (`leaf_steps`, `walk_levels`, `walk_loads`), and the one read of the root's empty suffix link after a leaf of the root
(`root_leaf_steps`, one load each).  For every `flushItems` round (32 LM-step items, one per lane) it keeps the largest per-lane sum
three ways: as the kernels were (`round_max_before`), as they are (`round_max_after`), and with the non-root walk only
(`round_max_walk_only`).  A round lasts as long as its slowest lane, so the summed round maxima are the pipeline's critical path in
loads.  The simulator re-does each non-root walk and aborts if it disagrees with the stored state.

Config 2 (Knlm): the rotating bench batches; config 3 (CoNg): the first 8192 sentences of its batch.  The heaviest sentences by LM
steps stand in for the ones that set the Viterbi launch's span.  Build the simulator with the product's staging capacity to see the
shipped split, e.g. `HS32_LIB=<path of a libpipeline_sim32.so compiled with -DKB_STAGE_CAP=1024>`.

  python scripts/lm_chain.py [--batches 4] [--n 8192] [--top 24] [--cong-n 8192] [--jobs J] [--json OUT]"""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
from concurrent.futures import ProcessPoolExecutor
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

FIELDS = ["steps", "chain_loads", "backoff_levels", "leaf_steps", "walk_levels", "walk_loads", "root_leaf_steps", "rounds",
          "round_max_before", "round_max_after", "round_max_walk_only"]
_T = {}


def _texts(cid, r, n):
    if (cid, r, n) not in _T:
        import bench
        from kiwi_b200.synth import SEED
        cfg = bench.CONFIGS[cid]
        nblk = (cfg["batch"] + bench.BLOCK - 1) // bench.BLOCK
        _T[(cid, r, n)] = bench.gen_sentences(cfg, r * nblk, n, SEED)      # bench.py's rotating batch r of rank 0 (its first n sentences)
    return _T[(cid, r, n)]


def work(args):
    cid, r, n, idxs = args
    from hostsim_sweep import _handle, MATCH_ALL
    mode = "cong" if cid == 3 else "plain"
    lib, h = _handle(mode)
    stats = lib.hs32_cg_chain_stats if mode == "cong" else lib.hs32_lm_chain_stats
    stats.argtypes = [C.c_void_p]
    texts = _texts(cid, r, n)
    cap = 8192
    morph = np.zeros(cap, np.uint32); tag = np.zeros(cap, np.uint8); pos = np.zeros(cap, np.uint32); ln = np.zeros(cap, np.uint16); sc = np.zeros(cap, np.float32)
    st = np.zeros(len(FIELDS), np.uint64)
    stats(st.ctypes.data)
    rows = []
    for i in idxs:
        u = np.ascontiguousarray(np.frombuffer(texts[i].encode("utf-16-le", "surrogatepass"), dtype="<u2"))
        s = C.c_float(0); nn = C.c_int(0)
        rc = lib.hs32_analyze(h, u.ctypes.data, len(u), MATCH_ALL, morph.ctypes.data, tag.ctypes.data, pos.ctypes.data, ln.ctypes.data, sc.ctypes.data, cap, C.byref(s), C.byref(nn), None)
        stats(st.ctypes.data)
        rows.append((cid, r, i, int(rc), [int(x) for x in st]))
    return rows


def summary(rows):
    tot = {f: sum(x[4][k] for x in rows) for k, f in enumerate(FIELDS)}
    b, a, w = tot["round_max_before"], tot["round_max_after"], tot["round_max_walk_only"]
    steps = max(1, tot["steps"])
    return {"sentences": len(rows), **tot,
            "loads_per_step_before": (tot["chain_loads"] + tot["walk_loads"] + tot["root_leaf_steps"]) / steps,
            "loads_per_step_after": tot["chain_loads"] / steps,
            "leaf_step_share": tot["leaf_steps"] / steps,
            "root_leaf_step_share": tot["root_leaf_steps"] / steps,
            "walk_loads_per_leaf_step": tot["walk_loads"] / max(1, tot["leaf_steps"]),
            "round_max_cut": (b - a) / max(1, b),                     # both removed (this build against its parent)
            "round_max_cut_walk": (w - a) / max(1, b),                # the part the non-root walk accounts for
            "round_max_cut_root_leaf": (b - w) / max(1, b)}           # the part the root-leaf read accounts for


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--n", type=int, default=8192)
    ap.add_argument("--cong-n", type=int, default=8192, help="config-3 sentences (0: none)")
    ap.add_argument("--top", type=int, default=24)
    ap.add_argument("--sentence", type=int, default=2348, help="a config-2 batch-0 sentence reported on its own")
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 4)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    t0 = time.time()
    tasks = []
    for cid, nb, n in [(2, a.batches, a.n), (3, 1 if a.cong_n else 0, a.cong_n)]:
        per = max(1, n // (a.jobs * 4))
        tasks += [(cid, r, n, list(range(k, min(n, k + per)))) for r in range(nb) for k in range(0, n, per)]
    if a.batches and a.sentence >= a.n:
        tasks.append((2, 0, max(a.n, 8192), [a.sentence]))      # the named sentence beyond the sample (reported on its own only)
    rows = []
    with ProcessPoolExecutor(a.jobs) as ex:
        for x in ex.map(work, tasks): rows += x
    out = {"lib": os.environ.get("HS32_LIB", "libpipeline_sim32.so"), "failed_sentences": sum(1 for x in rows if x[3] < 0), "batches": []}
    for cid, r in sorted({(x[0], x[1]) for x in rows}):
        mine = [x for x in rows if x[0] == cid and x[1] == r and (cid != 2 or x[2] < a.n)]
        heavy = sorted(mine, key=lambda x: -x[4][0])[:a.top]
        b = {"config": cid, "batch": r, "all": summary(mine), "top%d" % a.top: summary(heavy),
             "heaviest": [{"idx": x[2], **{f: x[4][k] for k, f in enumerate(FIELDS)}} for x in heavy]}
        if cid == 2 and r == 0:
            one = [x for x in rows if x[0] == 2 and x[1] == 0 and x[2] == a.sentence]
            if one: b["sentence_%d" % a.sentence] = summary(one)
        out["batches"].append(b)
    out["seconds"] = time.time() - t0
    rnd = lambda d: json.dumps({k: round(v, 4) if isinstance(v, float) else v for k, v in d.items()})
    for b in out["batches"]:
        for k in ["all", "top%d" % a.top, "sentence_%d" % a.sentence]:
            if k in b: print("config %d batch %d  %s: %s" % (b["config"], b["batch"], k, rnd(b[k])))
    if a.json: json.dump(out, open(a.json, "w"), indent=1)
    return 1 if out["failed_sentences"] else 0


if __name__ == "__main__":
    sys.exit(main())
