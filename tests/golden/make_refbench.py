#!/usr/bin/env python3
"""Regenerates tests/golden/refbench_*.npz: the UNMODIFIED reference's tokens for the bench batches (oracle/_ref/ref_bench, built by
oracle/ref_build/Makefile; needs oracle/_ref).  ref_bench analyses the whole batch in the reference's batch mode, as a user of the
reference would; a fixed sample of SAMPLE sentences per batch is stored (the whole dump of a 65 536-sentence batch is tens of MB).
refbench_top1 holds every sentence of the first 2048 config-2 sentences that the oracle sees use the `top1` container or fill a
bucket, analysed as one batch of their own (tests/test_gpu_round2.py)."""
import os, struct, subprocess, sys, tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import bench
from kiwi_b200.synth import SEED
from tests.orc import Oracle, IMAGE

REFDIR = os.path.join(ROOT, "oracle", "_ref")
SAMPLE = 128


def ref_dump(model, texts, typo=None):
    with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False, encoding="utf-8") as f:
        for t in texts: f.write(t + "\n")
        src = f.name
    dump = src + ".bin"
    env = dict(os.environ, KIWI_ARCH_TYPE="avx2", KB_MODEL_TYPE=model, KB_DUMP=dump)
    if typo: env["KB_TYPO"] = typo
    try:
        subprocess.run([os.path.join(REFDIR, "ref_bench"), os.path.join(REFDIR, "models", model + "_small"), src, str(len(os.sched_getaffinity(0))), "1"],
                       check=True, env=env, timeout=3600, capture_output=True)
        raw = open(dump, "rb").read()
    finally:
        for p in (src, dump):
            if os.path.exists(p): os.unlink(p)
    n, = struct.unpack_from("<I", raw, 0)
    assert n == len(texts)
    o = 4; counts = np.zeros(n, np.int64); scores = np.zeros(n, np.float32); rows = []
    for i in range(n):
        nt, sc = struct.unpack_from("<If", raw, o); o += 8
        counts[i] = nt; scores[i] = sc
        rows.append(raw[o:o + 16 * nt]); o += 16 * nt
    return counts, scores, rows


def save(name, idx, counts, scores, rows):
    idx = np.asarray(idx, np.int64)
    np.savez_compressed(os.path.join(HERE, "refbench_%s.npz" % name), index=idx.astype(np.int32), counts=counts[idx].astype(np.int32),
                        scores=scores[idx], tokens=np.frombuffer(b"".join(rows[i] for i in idx), np.uint8))


def sample(n):
    return np.sort(np.random.RandomState(0).choice(n, SAMPLE, replace=False))


for name, cid, model, typo in [("cfg2", 2, "knlm", None), ("cfg3", 3, "cong", None), ("cfg4", 4, "knlm", "basic")]:
    cfg = bench.CONFIGS[cid]
    texts = bench.gen_sentences(cfg, 0, cfg["batch"], SEED)
    save(name, sample(len(texts)), *ref_dump(model, texts, typo))

texts = bench.gen_sentences(bench.CONFIGS[2], 0, 2048, SEED)
orc = Oracle(IMAGE); hard = []; prev = orc.counters2()
for i, t in enumerate(texts):
    orc.analyze(t); c = orc.counters2()
    if c["top1Mode"] > prev["top1Mode"] or c["bucketFull"] > prev["bucketFull"]: hard.append(i)
    prev = c
counts, scores, rows = ref_dump("knlm", [texts[i] for i in hard])
np.savez_compressed(os.path.join(HERE, "refbench_top1.npz"), index=np.asarray(hard, np.int32), counts=counts.astype(np.int32), scores=scores,
                    tokens=np.frombuffer(b"".join(rows), np.uint8))
