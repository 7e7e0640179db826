#!/usr/bin/env python3
"""bench.py — sentences/sec of top-1 analysis (BASELINE.json metric) on N H100s.

  --config 2 (default) : batch=8192 synthetic Korean sentences (web.txt length dist), Knlm model, top-1        [BASELINE.json configs[1]]
  --config 3           : batch=65536, CoNg model (int8 scorer on tensor-core tiles)                            [configs[2]]
  --config 4           : batch=65536, Knlm model + typo lattice (basic typo set, cost weight 6, threshold 2.5), 30 % web_with_typos eojeols [configs[3]]
  --config 5           : 1 M sentences sharded round-robin (sentence i -> GPU i mod N), CoNg model, STRONG scaling   [configs[4]]
One "step" = one pass of the hot path (lattice kernel + Viterbi kernel + emit + pack) over the configuration's batch.
  value  : inputs already resident in HBM, device-timed (CUDA events on the engine stream), whole job.
  e2e    : the same batch through the public C-ABI call kiwi_b200_analyze_batch with HOST buffers
           (pinned staging, H2D of text+offsets and D2H of the packed tokens inside the timed region).
  --impl reference : the UNMODIFIED reference's CPU implementation (oracle/_ref/ref_bench, all host threads, >= 5 passes in ONE
           process, median) on a bounded sample of the same workload; also reports the 1-thread figure (tools/Evaluator.cpp:315-329).
Launch: python bench.py --gpus N --steps K --warmup W   (N > 1: under torchrun, one rank per GPU; or --inproc: ONE process driving
N GPUs through kiwi_b200_init_multi, the library's own ordered fan-out).
--dump-outputs DIR: after the timed steps, write what the last e2e step returned to its caller (token fields, token offsets, sentence
           scores, status) as DIR/<name>.npy; inputs are seeded, so two builds can be compared output for output."""
import argparse, json, math, os, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
REF_BENCH = os.path.join(ROOT, "oracle", "_ref", "ref_bench")
METRIC = "sentences/sec (top-1 analyze, batch=8192)"
UNIT = "sentences/s"
CONFIGS = {
    2: dict(model="knlm", batch=8192, typo=None, typo_frac=0.0, rotate=4, steps=20, scaling="weak"),
    3: dict(model="cong", batch=65536, typo=None, typo_frac=0.0, rotate=1, steps=5, scaling="weak"),
    4: dict(model="knlm", batch=65536, typo="basic", typo_frac=0.3, rotate=1, steps=5, scaling="weak"),
    5: dict(model="cong", batch=1 << 20, typo=None, typo_frac=0.0, rotate=1, steps=3, scaling="strong"),
    # not a BASELINE.json config: the SkipBigram model type (SURVEY 8a row a13).  Its kernel inserts paths one at a time (viterbi.cu
    # exactInsertRound): exact, but slow on path-heavy sentences - no measured line yet
    6: dict(model="sbg", batch=256, typo=None, typo_frac=0.0, rotate=1, steps=1, scaling="weak"),
}
BLOCK = 8192      # synthetic sentences are generated in seeded blocks of 8192 (block b: seed SEED + b)


def image_path(model): return os.path.join(ROOT, "oracle", "_ref", "models", model + "_small.img")
def ref_model_dir(model): return os.path.join(ROOT, "oracle", "_ref", "models", model + "_small")
def typo_image_path(tset): return os.path.join(ROOT, "oracle", "_ref", "models", "typo_%s.img" % tset)


def workload_string(cfg, cid):
    s = "config %d: batch=%d synthetic Korean sentences (web.txt length dist), fabricated %s model (%s_small), top-1" % (
        cid, cfg["batch"], {"knlm": "Knlm", "cong": "CoNg", "sbg": "SkipBigram"}[cfg["model"]], cfg["model"])
    if cfg["typo"]: s += ", typo lattice (%s typo set, typoCostWeight 6, threshold 2.5), %d %% of the sentences from web_with_typos eojeols" % (cfg["typo"], round(100 * cfg["typo_frac"]))
    if cfg["scaling"] == "strong": s += ", sharded round-robin (sentence i -> GPU i mod N)"
    return s


def gen_sentences(cfg, first_block, n, seed_base):
    from kiwi_b200.synth import synth_batch
    out = []
    b = first_block
    while len(out) < n:
        out += synth_batch(min(BLOCK, n - len(out)), seed_base + b, cfg["typo_frac"])
        b += 1
    return out


HBM_PEAK_GBS = 3350.0       # H100 SXM data sheet (HBM3), not a measured figure
INT8_PEAK_TOPS = 1979.0     # H100 SXM data sheet, dense int8 at up to 700 W, not a measured figure
DUMP_SENTENCES = 8192       # --dump-outputs: at most this many sentences (a fixed, seeded sample of larger batches)
DUMP_MAX_BYTES = 64 << 20


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)).get("hbm_gbs", HBM_PEAK_GBS), "measured"
    return HBM_PEAK_GBS, "fallback"


def dump_outputs(out_dir, res):
    """Writes a BatchResult as <name>.npy files: integer fields as float64 (exact), scores as float32.  Batches of more than
    DUMP_SENTENCES sentences are sampled by a seeded choice that depends on the batch size only, so that the same sentences are
    written by every build."""
    import numpy as np
    n = len(res.token_offsets) - 1
    idx = np.arange(n) if n <= DUMP_SENTENCES else np.sort(np.random.RandomState(0).choice(n, DUMP_SENTENCES, replace=False))
    off = res.token_offsets.astype(np.int64)
    counts = off[idx + 1] - off[idx]
    take = np.concatenate([np.arange(off[i], off[i + 1]) for i in idx]) if len(idx) else np.zeros(0, np.int64)
    tok = res.tokens[take]
    arrays = {"sentence_index": idx.astype(np.float64), "token_offsets": np.concatenate([[0], np.cumsum(counts)]).astype(np.float64),
              "sentence_scores": res.scores[idx].astype(np.float32), "status": res.status[idx].astype(np.float64),
              "morph_id": tok["morph_id"].astype(np.float64), "tag": tok["tag"].astype(np.float64), "position": tok["position"].astype(np.float64),
              "length": tok["length"].astype(np.float64), "token_scores": tok["score"].astype(np.float32)}
    total = sum(a.nbytes for a in arrays.values())
    if total > DUMP_MAX_BYTES:
        raise SystemExit("--dump-outputs: %d bytes exceed the %d-byte limit" % (total, DUMP_MAX_BYTES))
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def host_cpus():
    """usable host threads: affinity mask, capped by the cgroup CPU quota when there is one"""
    try: n = len(os.sched_getaffinity(0))
    except Exception: n = os.cpu_count() or 1
    quota = None
    try:
        q, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max": quota = float(q) / float(period)
    except Exception:
        pass
    return n, quota


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons during the timed region (profiling recipe, clocks line)."""
    def __init__(self, index):
        super().__init__(daemon=True)
        self.index = index; self.stop_flag = False; self.samples = []; self.reasons = set(); self.max_mhz = None

    def run(self):
        q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip().split(",")
                self.samples.append(float(out[0])); self.max_mhz = float(out[1])
                for nm, v in zip(names, out[2:]):
                    if v.strip().lower().startswith("active"): self.reasons.add(nm)
            except Exception:
                pass
            time.sleep(0.2)

    def summary(self):
        s = sorted(self.samples)
        return {"sm_mhz": s[len(s) // 2] if s else None, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons), "samples": len(s)}


def work_counters(cfg, cid, texts, seed):
    """Per-sentence algorithmic bytes from the instrumented oracle: committed under profiles/counters_r2.json for the bench batches
    (scripts/make_counters.py, every rotating seed); none committed for the workload: no roofline figure (the oracle is not run here)."""
    from kiwi_b200 import bytemodel
    path = os.path.join(ROOT, "profiles", "counters_r2.json")
    key = "cfg%d" % cid
    if os.path.exists(path):
        d = json.load(open(path))
        if key in d:
            c = d[key]
            return c, c["lattice_bytes_per_sentence"], c["viterbi_bytes_per_sentence"], "profiles/counters_r2.json[%s] (%s)" % (key, c.get("coverage", ""))
    # (no oracle on the product arm: a workload without committed counters reports no algorithmic-byte roofline)
    return {"sentences": 1}, None, None, "no committed work counters for this workload (scripts/make_counters.py writes profiles/counters_r2.json)"


def run_reference_cpu(cfg, texts, threads, repeats, single_sample=0, dump=None):
    """Times the unmodified reference (oracle/_ref/ref_bench) when it travelled with the repo, else the oracle port (1 thread)."""
    if os.path.exists(REF_BENCH) and os.path.exists(ref_model_dir(cfg["model"])):
        with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False, encoding="utf-8") as f:
            for t in texts: f.write(t + "\n")
            tmp = f.name
        try:
            env = dict(os.environ); env.setdefault("KIWI_ARCH_TYPE", "avx2"); env["KB_MODEL_TYPE"] = cfg["model"]
            if cfg["typo"]: env["KB_TYPO"] = cfg["typo"]
            if single_sample: env["KB_SINGLE_SAMPLE"] = str(single_sample)
            if dump: env["KB_DUMP"] = dump
            out = subprocess.run([REF_BENCH, ref_model_dir(cfg["model"]), tmp, str(threads), str(repeats)], capture_output=True, text=True, timeout=3000, env=env)
            lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
            if not lines: raise RuntimeError("ref_bench failed: " + out.stderr[-500:])
            r = json.loads(lines[-1])
            n, quota = host_cpus()
            return {"value": r["sent_per_s_median"], "unit": UNIT, "cores": threads, "kind": "reference",
                    "best": r["sent_per_s"], "single_thread": r["single_thread_sent_per_s"] or None, "single_thread_sample": r["single_thread_sample"],
                    "host": {"affinity_cpus": n, "cgroup_cpu_quota": quota},
                    "sample": "%d sentences of the bench batch, reference Kiwi::analyze batch mode on %d threads, KIWI_ARCH_TYPE=%s, median of %d passes in one process (best %.2f s, median %.2f s)%s" % (
                        r["sentences"], threads, r["arch"], r["repeats"], r["seconds"], r["seconds_median"], "; single thread on the first %d" % r["single_thread_sample"] if r["single_thread_sample"] else "")}
        finally:
            os.unlink(tmp)
    from tests.orc import Oracle, TypoOracle, TYPO_IMAGES
    o = Oracle(image_path(cfg["model"]))
    if cfg["typo"]: o.set_typo(TypoOracle(TYPO_IMAGES[cfg["typo"]]))
    t0 = time.time()
    for t in texts: o.analyze(t)
    dt = time.time() - t0
    return {"value": len(texts) / dt, "unit": UNIT, "cores": 1, "kind": "port", "sample": "%d sentences, oracle restatement single thread, %.2f s" % (len(texts), dt)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours")
    ap.add_argument("--config", type=int, default=2, choices=sorted(CONFIGS))
    ap.add_argument("--batch", type=int, default=None, help="override the configuration's batch size (experiments)")
    ap.add_argument("--model", default=None, choices=["knlm", "cong", "sbg"], help="override the configuration's model (experiments)")
    ap.add_argument("--typo", default=None, choices=["basic", "none"], help="override the configuration's typo set (experiments)")
    ap.add_argument("--cpu-sample", type=int, default=8192)
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg (kernel experiments)")
    ap.add_argument("--inproc", action="store_true", help="one process, --gpus N devices behind ONE handle (kiwi_b200_init_multi) instead of torchrun ranks")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="write the last timed step's results as DIR/<name>.npy")
    args = ap.parse_args()
    cfg = dict(CONFIGS[args.config])
    if args.batch: cfg["batch"] = args.batch
    if args.model: cfg["model"] = args.model
    if args.typo: cfg["typo"] = None if args.typo == "none" else args.typo
    steps = args.steps if args.steps is not None else cfg["steps"]
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    from kiwi_b200.synth import SEED
    workload = workload_string(cfg, args.config)
    strong = cfg["scaling"] == "strong"

    if args.impl == "reference":
        if rank != 0: return 0
        ncpu, quota = host_cpus()
        threads = max(1, min(ncpu, int(math.ceil(quota)) if quota else ncpu))
        texts = gen_sentences(cfg, 0, min(cfg["batch"], args.cpu_sample), SEED)
        # warm-up: one short pass (page cache, model build) that also sizes the run: >= 5 passes, <= ~4 minutes
        w = run_reference_cpu(cfg, texts[:512], threads, 1)
        est = len(texts) / max(w["value"], 1.0)
        repeats = max(5, min(max(steps, 5), int(200 / max(est, 1e-3))))
        last = run_reference_cpu(cfg, texts, threads, repeats, single_sample=min(len(texts), 1024))
        v = last["value"]
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus, "steps": repeats, "warmup": 1,
                          "ms_per_step": 1000.0 * len(texts) / v, "higher_is_better": True, "scaling": cfg["scaling"], "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                          "config": {"workload": workload, "sample": "each step = the first %d sentences of the batch on %d host threads" % (len(texts), threads)},
                          "cpu_baseline": last, "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return 0

    import numpy as np
    import torch
    import kiwi_b200
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a GPU: kiwi_b200 has no CPU fallback")
    inproc = args.inproc and args.gpus > 1
    if inproc: world, rank, local_rank = 1, 0, 0
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    # ---- model: rank 0 reads the image, one NCCL broadcast puts it on every GPU (no collectives afterwards)
    IMAGE = image_path(cfg["model"])
    if rank == 0:
        img = np.fromfile(IMAGE, dtype=np.uint8)
        size = torch.tensor([img.size], dtype=torch.int64, device="cuda")
    else:
        size = torch.zeros(1, dtype=torch.int64, device="cuda")
    if world > 1: dist.broadcast(size, 0)
    buf = torch.from_numpy(img).cuda() if rank == 0 else torch.empty(int(size.item()), dtype=torch.uint8, device="cuda")
    if world > 1: dist.broadcast(buf, 0)
    image_bytes = buf.cpu().numpy().tobytes()
    del buf
    ndev = args.gpus if inproc else world
    kw = kiwi_b200.Kiwi(image_bytes=image_bytes, devices=list(range(args.gpus))) if inproc else kiwi_b200.Kiwi(image_bytes=image_bytes, device=local_rank)
    typo = None
    if cfg["typo"]:
        typo = kiwi_b200.PreparedTypo(path=typo_image_path(cfg["typo"]))      # (a flat typo image next to the model images; nothing of the oracle is imported on the product arm)
    option = kiwi_b200.default_option(typo=typo)

    # ---- synthetic batches.  weak scaling: every rank works on `batch` sentences per step (its own seeds);
    #      strong scaling (config 5): ONE job of `batch` sentences, rank r owns the sentences i = r (mod N)
    R = cfg["rotate"]
    batches = []
    if strong:
        from kiwi_b200.shard import shard_indices
        all_texts = gen_sentences(cfg, 0, cfg["batch"], SEED)
        mine = [all_texts[i] for i in shard_indices(len(all_texts), rank, world)] if world > 1 else all_texts
        cache = os.path.join(tempfile.gettempdir(), "kiwi_b200_cfg%d_%d_r%dof%d.npz" % (args.config, cfg["batch"], rank, world))      # (encoding 1 M strings takes a while)
        if os.path.exists(cache):
            z = np.load(cache); blob, off = z["blob"], z["off"]
        else:
            blob, off = kiwi_b200.encode_batch(mine)
            np.savez(cache, blob=blob, off=off)
        batches.append((mine, blob, off, torch.from_numpy(blob.view(np.int16)).cuda(), torch.from_numpy(off.view(np.int32)).cuda()))
    else:
        nblk = (cfg["batch"] + BLOCK - 1) // BLOCK
        for r in range(R):
            texts = gen_sentences(cfg, (1000 * rank + r) * nblk if (rank or r) else 0, cfg["batch"], SEED)
            blob, off = kiwi_b200.encode_batch(texts)
            batches.append((texts, blob, off, torch.from_numpy(blob.view(np.int16)).cuda(), torch.from_numpy(off.view(np.int32)).cuda()))
    torch.cuda.synchronize()
    n_local = len(batches[0][0])

    def step_device(i):
        _, blob, off, d_blob, d_off = batches[i % R]
        return kw.analyze_device(d_blob.data_ptr(), d_off.data_ptr(), len(off) - 1, int(blob.size), option)

    dev_ms = 0.0; ms_vit = 0.0; ms_lat = 0.0; launches = 0; tokens = 0; retried = 0; wall = 0.0
    sampler = ClockSampler(local_rank)      # (clocks are sampled during the device-timed region only: nvidia-smi polling disturbs the host-timed e2e loop)
    if not inproc:
        for i in range(args.warmup): step_device(i)
        sampler.start()
        if dist: dist.barrier()
        torch.cuda.synchronize()
        t0 = time.time()
        for i in range(steps):
            ms, nt, nl = step_device(i)
            st = kw.last_stats()
            dev_ms += ms; ms_vit += st.ms_viterbi; ms_lat += st.ms_lattice; launches += st.kernel_launches; tokens += nt; retried += st.retried
        torch.cuda.synchronize()
        if dist: dist.barrier()
        wall = time.time() - t0
        sampler.stop_flag = True; sampler.join(timeout=10)     # (nvidia-smi polling disturbs the host-timed e2e loop below: wait out the query in flight)
    else:
        sampler.start()

    # ---- end to end through the public API with host buffers
    for i in range(min(2, args.warmup)): kw.analyze_batch_arrays(batches[i % R][1], batches[i % R][2], option)
    if strong and dist:
        # (the first gather of a process group sets up its point-to-point channels: not part of a steady-state step)
        pad = torch.zeros((len(all_texts) + world - 1) // world, dtype=torch.int32, device="cuda")
        dist.gather(pad, [torch.empty_like(pad) for _ in range(world)] if rank == 0 else None, 0)
    if dist: dist.barrier()
    torch.cuda.synchronize()
    t1 = time.time(); h2d = d2h = 0; e2e_launches = 0; order_ok = None
    res = None
    for i in range(steps):
        res = None      # (the consumer is done with the previous step's result: its holder goes back to the library's pool)
        res = kw.analyze_batch_arrays(batches[i % R][1], batches[i % R][2], option)
        st = kw.last_stats(); h2d += st.h2d_bytes; d2h += st.d2h_bytes; e2e_launches += st.kernel_launches
        if strong and dist:
            # ordered delivery of the sharded job: every rank contributes its per-sentence token counts; rank 0 restores input order
            cnt = torch.from_numpy(np.diff(res.token_offsets.astype(np.int64)).astype(np.int32)).cuda()
            pad = torch.zeros((len(all_texts) + world - 1) // world, dtype=torch.int32, device="cuda"); pad[:cnt.numel()] = cnt
            gathered = [torch.empty_like(pad) for _ in range(world)] if rank == 0 else None
            dist.gather(pad, gathered, 0)
            if rank == 0:
                from kiwi_b200.shard import merge_round_robin
                per_rank = [g.cpu().numpy()[:len(range(r, len(all_texts), world))] for r, g in enumerate(gathered)]
                merged = merge_round_robin(per_rank, len(all_texts)) if i == steps - 1 else None
    torch.cuda.synchronize()
    if dist: dist.barrier()
    e2e_wall = time.time() - t1
    if not sampler.stop_flag:
        sampler.stop_flag = True; sampler.join(timeout=2)
    if strong and rank == 0:
        # order check of the merged job on a sample: sentence i of the merged result must be sentence i of the input
        if dist:
            sample = list(range(0, len(all_texts), 997))
            chk = kw.analyze_batch([all_texts[i] for i in sample], option)
            order_ok = bool(all(int(merged[i]) == int(chk.token_offsets[k + 1] - chk.token_offsets[k]) for k, i in enumerate(sample)))
        elif inproc:
            single = kiwi_b200.Kiwi(image_bytes=image_bytes, device=0)
            sample = list(range(0, len(all_texts), 997))
            chk = single.analyze_batch([all_texts[i] for i in sample], option)
            order_ok = bool(all(np.array_equal(res.sentence(i), chk.sentence(k)) for k, i in enumerate(sample)))
            single.close()

    t = torch.tensor([dev_ms, wall, e2e_wall, ms_vit, ms_lat], dtype=torch.float64, device="cuda")
    if dist: dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, wall, e2e_wall, ms_vit, ms_lat = [float(x) for x in t.tolist()]
    if rank != 0:
        if dist: dist.destroy_process_group()
        return 0

    total_sent = (cfg["batch"] if strong else cfg["batch"] * ndev) * steps
    e2e = total_sent / e2e_wall
    if inproc: dev_ms = e2e_wall * 1000.0; launches = e2e_launches      # (one handle over N devices has no single device timeline: value = the host-timed job)
    value = total_sent / (dev_ms / 1000.0)
    peak, peak_kind = load_peaks()
    c, lat_b, vit_b, csrc = work_counters(cfg, args.config, batches[0][0], SEED)
    kernel = {"knlm": "viterbi_kernel", "cong": "viterbi_cong_kernel", "sbg": "viterbi_sbg_kernel"}[cfg["model"]]
    vit_per_step_ms = ms_vit / steps if steps else 0.0
    achieved = vit_b * n_local / (vit_per_step_ms / 1000.0) / 1e9 if (vit_per_step_ms and vit_b) else None
    prof = {}
    pp = os.path.join(ROOT, "profiles", "ncu_r2.json")
    if os.path.exists(pp): prof = json.load(open(pp)).get(kernel, {})
    cpu = None
    if world == 1 and not inproc and not args.no_cpu:
        ncpu, quota = host_cpus()
        threads = max(1, min(ncpu, int(math.ceil(quota)) if quota else ncpu))
        cpu = run_reference_cpu(cfg, batches[0][0][:args.cpu_sample], threads, 5, single_sample=512)
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": ndev, "steps": steps, "warmup": args.warmup,
        "ms_per_step": dev_ms / steps, "higher_is_better": True, "scaling": cfg["scaling"], "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload,
                   "l2": "per-step scratch working set (GBs) exceeds the 50 MB L2%s; the read-only model stays resident as in steady state" % (" and %d distinct input batches rotate" % R if R > 1 else ""),
                   "parallelism": ("one process, one handle over %d devices (kiwi_b200_init_multi): round-robin shards, one host thread per device, ordered merge" % ndev) if inproc else
                                  "dp%d (sentence sharding, one NCCL broadcast of the model image at init, no steady-state collectives)" % world,
                   "wall_ms_per_step": 1000.0 * wall / steps if steps else None,
                   "retried_sentences_per_step": retried / steps if steps else None,
                   "sentences_per_gpu_per_step": n_local if not inproc else cfg["batch"] // ndev},
        "e2e": {"value": e2e, "unit": UNIT, "h2d_bytes_per_step": h2d // steps, "d2h_bytes_per_step": d2h // steps},
        "gpu_launches": int(launches),
        "clocks": sampler.summary(),
        "roofline": {"bound": "hbm", "kernel": kernel, "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak if achieved else None,
                     "traffic": prof.get("dram_bytes_per_launch"),
                     "peak_kind": peak_kind + " (MEASURED_PEAKS.json hbm_gbs)" if peak_kind == "measured" else "fallback: H100 SXM data sheet HBM3",
                     "algorithmic_bytes_per_sentence": vit_b, "lattice_kernel_bytes_per_sentence": lat_b, "counters": csrc,
                     "kernel_ms_per_step": vit_per_step_ms, "lattice_ms_per_step": ms_lat / steps if steps else None,
                     "kernel_share_of_step": ms_vit / dev_ms if dev_ms and not inproc else None,
                     # the kernels keep their working set in L2: DRAM is not the limiter, so the ncu capture's L2 and issue-slot figures ride along
                     "l2": prof.get("l2"), "issue": prof.get("issue"), "profile": prof.get("source")},
        "tokens_per_step": tokens // steps if steps else None,
    }
    if order_ok is not None: line["config"]["ordered_merge_check"] = order_ok
    if cpu: line["cpu_baseline"] = cpu
    if cfg["model"] == "cong":
        # the int8 gather GEMMs of progressMatrix: 2 * sum(m * n * dim) integer ops per sentence (counted by the instrumented oracle)
        ops = 2.0 * c.get("cgMacs", 0) / max(1, c["sentences"])
        line["roofline"]["tensor"] = {"bound": "tensor", "unit": "TOP/s", "achieved": ops * n_local / (vit_per_step_ms / 1000.0) / 1e12 if vit_per_step_ms else None, "peak": INT8_PEAK_TOPS,
                                      "peak_kind": "H100 SXM data sheet dense int8 (not measured)", "int8_ops_per_sentence": ops,
                                      "note": "the gather GEMMs are a small part of viterbi_cong_kernel's time; the kernel as a whole is latency / L2 bound like the Knlm one"}
    print(json.dumps(line))
    if args.dump_outputs and res is not None:
        dump_outputs(args.dump_outputs, res)
    if dist: dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
