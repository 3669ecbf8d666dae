#!/usr/bin/env python
"""Mixed-tau batching (per-item sampling parameters, include/ovc.h: ovc_item_params) on the synthetic checkpoint.

32 x 10 s clips whose requests ask for 4 distinct tau values (8 each) and carry their own seeds.  Two ways to serve them:
    mixed   ONE convert_batch with tau and seeds per item
    split   4 convert_batch calls, one per tau value (what a caller had to do without per-item tau), 8 clips each
Both arms give every request the same audio (checked bit for bit), so only the time differs.  Every arm is warmed up
(graphs captured), then the arms alternate for --reps rounds; host wall time of each call ending in its device sync,
median and spread.  Prints one JSON line with the card name and its power limit.
    python tools/request_params_bench.py [--reps 7] [--precision f16x3]"""
import argparse, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle import vc_oracle as O
from openvoice_b200.api import ToneColorConverter

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--precision", default="f16x3", choices=["fp32", "f16x3", "f16"])
ap.add_argument("--out", default=None, help="also append the JSON line to this file")
args = ap.parse_args()
assert torch.cuda.is_available(), "request_params_bench measures on the GPU"

B, SECS, SR = 32, 10, 22050
TAUS = (0.0, 0.3, 0.6, 1.0)

with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False, precision=args.precision)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
rng = np.random.default_rng(0)
wavs = [(0.5 * (2 * rng.random(SR * SECS, dtype=np.float32) - 1)).astype(np.float32) for _ in range(B)]
taus = [TAUS[i % len(TAUS)] for i in range(B)]
seeds = [int(s) for s in rng.integers(0, 2 ** 63, B)]
gen = torch.Generator().manual_seed(1)
src, tgt = 0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)


def mixed():
    return conv.convert_batch(wavs, src, tgt, tau=taus, seeds=seeds)


def split():
    out = [None] * B
    for t in TAUS:
        idx = [i for i in range(B) if taus[i] == t]
        for i, a in zip(idx, conv.convert_batch([wavs[i] for i in idx], src, tgt, tau=t, seeds=[seeds[i] for i in idx])):
            out[i] = a
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


for _ in range(3):                      # warm up both arms: modules, workspaces, graph capture of each signature
    a, b = mixed(), split()
assert all(np.array_equal(x, y) for x, y in zip(a, b)), "the two arms must give every request the same audio"
t_mixed, t_split = [], []
for _ in range(args.reps):
    t_mixed.append(timed(mixed)[0])
    t_split.append(timed(split)[0])

name = torch.cuda.get_device_name(0)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
except Exception:
    power = "unknown"
audio_s = B * SECS
res = {"bench": "request_params", "gpu": name, "power_limit": power, "precision": args.precision, "clips": B,
       "secs": SECS, "taus": list(TAUS), "reps": args.reps,
       "mixed_ms_median": 1e3 * float(np.median(t_mixed)), "mixed_ms_range": [1e3 * min(t_mixed), 1e3 * max(t_mixed)],
       "split_ms_median": 1e3 * float(np.median(t_split)), "split_ms_range": [1e3 * min(t_split), 1e3 * max(t_split)],
       "speedup_median": float(np.median(t_split) / np.median(t_mixed)),
       "mixed_audio_s_per_s": audio_s / float(np.median(t_mixed)), "split_audio_s_per_s": audio_s / float(np.median(t_split))}
line = json.dumps(res)
print(line, flush=True)
if args.out:
    with open(args.out, "a") as f:
        f.write(line + "\n")
