#!/usr/bin/env python3
"""Where the Knlm kernel takes its LM steps (no GPU).  Runs the rotating config-2 bench batches through the 32-lane host simulation of
the device pipeline and counts, per sentence, the LM steps taken in `flushItems` (the item pipeline), in `evalCand` (the per-candidate
path) on nodes of at most / more than HT_MAX_ENTRIES (768) incoming paths, and elsewhere (end node).  The heaviest sentences by LM steps
stand in for the ones that set the Viterbi launch's span.  Build the simulator with the Knlm build's staging capacity to see the
production split, e.g. `HS32_LIB=<path of a libpipeline_sim32.so compiled with -DKB_STAGE_CAP=1024>`.

  python scripts/lm_sites.py [--batches 4] [--n 8192] [--top 24] [--jobs J] [--json OUT]"""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
from concurrent.futures import ProcessPoolExecutor
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SITES = ["flush_items", "eval_cand_small", "eval_cand_big", "other"]
_T = {}


def _texts(r, n):
    if (r, n) not in _T:
        import bench
        from kiwi_b200.synth import SEED
        cfg = bench.CONFIGS[2]
        nblk = (cfg["batch"] + bench.BLOCK - 1) // bench.BLOCK
        _T[(r, n)] = bench.gen_sentences(cfg, r * nblk, n, SEED)      # bench.py's rotating batch r of rank 0
    return _T[(r, n)]


def work(args):
    r, n, idxs = args
    from hostsim_sweep import _handle, MATCH_ALL
    lib, h = _handle("plain")
    lib.hs32_lm_site_stats.argtypes = [C.c_void_p]
    texts = _texts(r, n)
    cap = 8192
    morph = np.zeros(cap, np.uint32); tag = np.zeros(cap, np.uint8); pos = np.zeros(cap, np.uint32); ln = np.zeros(cap, np.uint16); sc = np.zeros(cap, np.float32)
    st = np.zeros(4, np.uint64)
    lib.hs32_lm_site_stats(st.ctypes.data)
    rows = []
    for i in idxs:
        u = np.ascontiguousarray(np.frombuffer(texts[i].encode("utf-16-le", "surrogatepass"), dtype="<u2"))
        s = C.c_float(0); nn = C.c_int(0)
        rc = lib.hs32_analyze(h, u.ctypes.data, len(u), MATCH_ALL, morph.ctypes.data, tag.ctypes.data, pos.ctypes.data, ln.ctypes.data, sc.ctypes.data, cap, C.byref(s), C.byref(nn), None)
        lib.hs32_lm_site_stats(st.ctypes.data)
        rows.append((r, i, int(rc), [int(x) for x in st]))
    return rows


def summary(rows):
    tot = [sum(x[3][k] for x in rows) for k in range(4)]
    all_ = max(1, sum(tot))
    return {"sentences": len(rows), "lm_steps": sum(tot), **{s: tot[k] for k, s in enumerate(SITES)},
            **{s + "_share": tot[k] / all_ for k, s in enumerate(SITES)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--n", type=int, default=8192)
    ap.add_argument("--top", type=int, default=24)
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 4)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    t0 = time.time()
    per = max(1, a.n // (a.jobs * 4))
    tasks = [(r, a.n, list(range(k, min(a.n, k + per)))) for r in range(a.batches) for k in range(0, a.n, per)]
    rows = []
    with ProcessPoolExecutor(a.jobs) as ex:
        for x in ex.map(work, tasks): rows += x
    out = {"lib": os.environ.get("HS32_LIB", "libpipeline_sim32.so"), "failed_sentences": sum(1 for x in rows if x[2] < 0), "batches": []}
    for r in range(a.batches):
        mine = [x for x in rows if x[0] == r]
        heavy = sorted(mine, key=lambda x: -sum(x[3]))[:a.top]
        out["batches"].append({"batch": r, "all": summary(mine), "top%d" % a.top: summary(heavy),
                               "heaviest": [{"idx": x[1], **{s: x[3][k] for k, s in enumerate(SITES)}} for x in heavy]})
    out["seconds"] = time.time() - t0
    for b in out["batches"]:
        print("batch %d  all: %s" % (b["batch"], json.dumps({k: round(v, 4) if isinstance(v, float) else v for k, v in b["all"].items()})))
        print("batch %d  top%d: %s" % (b["batch"], a.top, json.dumps({k: round(v, 4) if isinstance(v, float) else v for k, v in b["top%d" % a.top].items()})))
        for h in b["heaviest"][:3]: print("   ", h)
    if a.json: json.dump(out, open(a.json, "w"), indent=1)
    return 1 if out["failed_sentences"] else 0


if __name__ == "__main__":
    sys.exit(main())
