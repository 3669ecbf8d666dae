#!/usr/bin/env python
"""Speaker-embedding extraction: the per-clip loop (one spectrogram + one reference-encoder pass per clip, what
extract_se did before it batched) vs the batched path (extract_se / extract_se_batch: ragged passes shared by all
clips), on the synthetic checkpoint.  Workloads: one voice from a 30 s and from a 60 s reference (3 and 6 segments
of 10 s, as se_extractor.get_se cuts them) and 64 speakers x 3 segments enrolled at once.

Every shape is warmed up first; then the two arms alternate for --reps rounds.  Device time comes from CUDA events
around the arm, host wall time from a clock stopped after a synchronize.  Both arms must return identical
embeddings.  Prints one JSON line per workload, with the card name and its power limit.
    python tools/se_bench.py [--reps 5]"""
import argparse, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle import vc_oracle as O
from openvoice_b200.api import ToneColorConverter, SE_CHUNK_FRAMES

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
args = ap.parse_args()

with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
nat = conv.model.native
SR = 22050
rng = np.random.default_rng(0)


def clip(secs):
    return (0.5 * (2 * rng.random(int(secs * SR), dtype=np.float32) - 1)).astype(np.float32)


def per_clip_se(waves):
    gs = []
    for w in waves:
        y = torch.from_numpy(w).to(conv.device).unsqueeze(0).contiguous()
        n = torch.tensor([y.shape[1]], dtype=torch.int64, device=conv.device)
        y, _ = nat.spectrogram(y, n)
        gs.append(nat.reference_encoder(y).unsqueeze(-1))
    return torch.stack(gs).mean(0)


def timed(fn):
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record(st)
    out = fn()
    e1.record(st)
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1), 1e3 * (time.perf_counter() - t0)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    return name, power


voice30 = [clip(10) for _ in range(3)]
voice60 = [clip(10) for _ in range(6)]
enrol = [[clip(10) for _ in range(3)] for _ in range(64)]
workloads = {
    "voice_30s_3seg": (lambda: per_clip_se(voice30), lambda: conv.extract_se(voice30)),
    "voice_60s_6seg": (lambda: per_clip_se(voice60), lambda: conv.extract_se(voice60)),
    "enrol_64x3seg": (lambda: [per_clip_se(s) for s in enrol], lambda: conv.extract_se_batch(enrol)),
}
name, power = card()
for wl, (loop_fn, batch_fn) in workloads.items():
    for _ in range(2):                                   # warm-up: every shape, both arms
        loop_fn(), batch_fn()
    t = {"loop": ([], []), "batched": ([], [])}
    for r in range(args.reps):
        arms = (("loop", loop_fn), ("batched", batch_fn)) if r % 2 == 0 else (("batched", batch_fn), ("loop", loop_fn))
        outs = {}
        for arm, fn in arms:
            outs[arm], dev_ms, wall_ms = timed(fn)
            t[arm][0].append(dev_ms)
            t[arm][1].append(wall_ms)
        a, b = outs["loop"], outs["batched"]
        a, b = (a, b) if isinstance(a, list) else ([a], [b])
        assert all(torch.equal(x, y) for x, y in zip(a, b)), f"{wl}: the arms disagree"
    res = {"workload": wl, "card": name, "power_limit": power, "reps": args.reps, "chunk_frames": SE_CHUNK_FRAMES}
    for arm, (dev, wall) in t.items():
        res[f"{arm}_device_ms"] = [round(min(dev), 3), round(float(np.median(dev)), 3), round(max(dev), 3)]
        res[f"{arm}_wall_ms"] = [round(min(wall), 3), round(float(np.median(wall)), 3), round(max(wall), 3)]
    res["speedup_wall_median"] = round(float(np.median(t["loop"][1]) / np.median(t["batched"][1])), 3)
    res["speedup_device_median"] = round(float(np.median(t["loop"][0]) / np.median(t["batched"][0])), 3)
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
