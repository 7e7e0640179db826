#!/usr/bin/env python3
"""How often the Knlm kernel repeats an LM step within one sentence (no GPU).  Runs the config-2 bench batch through the 32-lane host
simulation of the device pipeline (tests/hostsim/libpipeline_sim32.so) and reads, per sentence, the kernel's LM steps and the distinct
(lmState, wid) pairs among them: the steps a per-sentence transition cache of unbounded size could answer without walking the Knlm
tables.  The oracle's LM-step count of every sentence rides along as a cross-check (the kernel also steps paths that the reference
filters before its LM step, so it counts somewhat more).

  python scripts/lm_repeat.py [--n 8192] [--top 20] [--jobs J] [--json OUT]"""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
from concurrent.futures import ProcessPoolExecutor
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

_T = {}


def _texts(n):
    if n not in _T:
        import bench
        from kiwi_b200.synth import SEED
        _T[n] = bench.gen_sentences(bench.CONFIGS[2], 0, n, SEED)
    return _T[n]


def work(args):
    n, idxs = args
    import bench
    from hostsim_sweep import _handle, MATCH_ALL
    from tests.orc import Oracle
    lib, h = _handle("plain")
    lib.hs32_lm_repeat_stats.argtypes = [C.c_void_p]
    orc = Oracle(bench.image_path("knlm"))
    texts = _texts(n)
    cap = 8192
    morph = np.zeros(cap, np.uint32); tag = np.zeros(cap, np.uint8); pos = np.zeros(cap, np.uint32); ln = np.zeros(cap, np.uint16); sc = np.zeros(cap, np.float32)
    st = np.zeros(2, np.uint64)
    lib.hs32_lm_repeat_stats(st.ctypes.data)
    rows = []
    for i in idxs:
        u = np.ascontiguousarray(np.frombuffer(texts[i].encode("utf-16-le", "surrogatepass"), dtype="<u2"))
        s = C.c_float(0); nn = C.c_int(0)
        rc = lib.hs32_analyze(h, u.ctypes.data, len(u), MATCH_ALL, morph.ctypes.data, tag.ctypes.data, pos.ctypes.data, ln.ctypes.data, sc.ctypes.data, cap, C.byref(s), C.byref(nn), None)
        lib.hs32_lm_repeat_stats(st.ctypes.data)
        o0 = orc.counters()["lmSteps"]; orc.analyze(texts[i]); o1 = orc.counters()["lmSteps"]
        rows.append((i, int(rc), int(st[0]), int(st[1]), o1 - o0))
    return rows


def summary(rows):
    steps = sum(r[2] for r in rows); distinct = sum(r[3] for r in rows)
    return {"sentences": len(rows), "lm_steps": steps, "distinct_pairs": distinct, "repeat_fraction": 1 - distinct / max(1, steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8192)
    ap.add_argument("--top", type=int, default=20)
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 4)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    idx = list(range(a.n)); per = max(1, len(idx) // (a.jobs * 4))
    t0 = time.time(); rows = []
    with ProcessPoolExecutor(a.jobs) as ex:
        for r in ex.map(work, [(a.n, idx[k:k + per]) for k in range(0, len(idx), per)]): rows += r
    failed = [r for r in rows if r[1] < 0]
    heavy = sorted(rows, key=lambda r: -r[2])[:a.top]
    out = {"batch": "bench.py --config 2, first %d sentences" % a.n, "all": summary(rows), "top%d" % a.top: summary(heavy),
           "heaviest": [{"idx": r[0], "lm_steps": r[2], "distinct_pairs": r[3], "repeat_fraction": 1 - r[3] / max(1, r[2]), "oracle_lm_steps": r[4]} for r in heavy],
           "failed_sentences": len(failed), "seconds": time.time() - t0}
    print(json.dumps({k: v for k, v in out.items() if k != "heaviest"}, indent=1))
    print("%6s %9s %9s %8s %9s" % ("idx", "steps", "distinct", "repeat", "oracle"))
    for r in out["heaviest"]:
        print("%6d %9d %9d %8.3f %9d" % (r["idx"], r["lm_steps"], r["distinct_pairs"], r["repeat_fraction"], r["oracle_lm_steps"]))
    if a.json: json.dump(out, open(a.json, "w"), indent=1)
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
