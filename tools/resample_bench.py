#!/usr/bin/env python
"""On-device sample-rate conversion (ovc_resample) on the synthetic checkpoint's converter.

kernel: one ragged-free batch of 32 x 10 s clips per rate pair (48 k, 44.1 k, 16 k -> 22.05 k and 22.05 k -> 48 k),
    every pair warmed up, then CUDA events around --launches back-to-back launches.  Reports the time per launch, the
    algorithmic bytes 4 (sum L_in + sum L_out) (each input and output sample moved once) and FLOPs 2 * (taps used),
    and the share of the HBM bound: bytes / 3.35 TB/s (H100 SXM data sheet) over the kernel time.
e2e: 32 x 10 s NumPy clips at 48 kHz: host scipy.signal.resample_poly per clip followed by convert_batch, against
    convert_batch(sr=48000).  tau = 0, so both arms are deterministic; the outputs must agree within 1e-4 * rms (scipy
    resamples fp32 input in fp32, the device in fp64).  The arms alternate for --reps rounds; host wall time, median.
Prints one JSON line per measurement, with the card name and its power limit.
    python tools/resample_bench.py [--launches 200] [--reps 5]"""
import argparse, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from scipy.signal import resample_poly
from oracle import vc_oracle as O
from openvoice_b200._native import resample_span
from openvoice_b200.api import ToneColorConverter

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=200)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
args = ap.parse_args()
assert torch.cuda.is_available(), "resample_bench measures on the GPU"

HBM_BPS = 3.35e12
B, SECS, SR = 32, 10, 22050

with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
nat = conv.model.native
rng = np.random.default_rng(0)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    return name, power


def emit(res):
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


def taps_used(a, b, L):
    """Taps summed over the n_out(L) outputs of one clip: j in [ceil((t - N + 1) / up), floor(t / up)] per output."""
    g = np.gcd(a, b)
    up, down = b // g, a // g
    half = 0 if up == down else 10 * max(up, down)
    N, pre_pad = 2 * half + 1, down - half % down
    m = np.arange(resample_span(a, b, L)[0], dtype=np.int64)
    t = (m + (half + pre_pad) // down) * down - pre_pad
    return int((t // up + (-(t - N + 1)) // up + 1).sum())      # floor(t / up) - ceil((t - N + 1) / up) + 1


name, power = card()
for a, b in ((48000, SR), (44100, SR), (16000, SR), (SR, 48000)):
    L = SECS * a
    n = resample_span(a, b, L)[0]
    x = torch.from_numpy((0.5 * (2 * rng.random((B, L), dtype=np.float32) - 1)).astype(np.float32)).cuda()
    lens = torch.full((B,), L, dtype=torch.int64, device="cuda")
    out = torch.empty(B, n, device="cuda")
    for _ in range(5):
        nat.resample(x, lens, a, b, out=out)
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    for _ in range(args.launches):
        nat.resample(x, lens, a, b, out=out)
    e1.record(st)
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / args.launches
    byts = 4.0 * B * (L + n)
    flops = 2.0 * B * taps_used(a, b, L)
    emit({"measure": "kernel", "pair": f"{a}->{b}", "batch": f"{B}x{SECS}s", "card": name, "power_limit": power,
          "launches": args.launches, "us_per_launch": round(us, 2), "bytes": byts, "flops": flops,
          "GB_per_s": round(byts / us * 1e-3, 1), "fp64_GFLOP_per_s": round(flops / us * 1e-3, 1),
          "hbm_bound_share": round(byts / HBM_BPS * 1e6 / us, 3)})

gen = torch.Generator().manual_seed(5)
src, tgt = 0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)
clips = [(0.5 * (2 * rng.random(SECS * 48000, dtype=np.float32) - 1)).astype(np.float32) for _ in range(B)]


def host_arm():
    return conv.convert_batch([resample_poly(c, 147, 320).astype(np.float32) for c in clips], src, tgt, tau=0.0)


def device_arm():
    return conv.convert_batch(clips, src, tgt, tau=0.0, sr=48000)


for _ in range(2):
    host_arm(), device_arm()
t = {"host_resample_poly": [], "device_sr": []}
for r in range(args.reps):
    arms = (("host_resample_poly", host_arm), ("device_sr", device_arm))
    outs = {}
    for arm, fn in (arms if r % 2 == 0 else arms[::-1]):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs[arm] = fn()
        torch.cuda.synchronize()
        t[arm].append(1e3 * (time.perf_counter() - t0))
    for p, q in zip(outs["host_resample_poly"], outs["device_sr"]):
        assert p.shape == q.shape
        err = float(np.abs(p.astype(np.float64) - q).max() / (np.sqrt(np.mean(p.astype(np.float64) ** 2)) + 1e-30))
        assert err <= 1e-4, f"the arms disagree: {err:.3e}"
res = {"measure": "e2e", "workload": f"convert_batch {B}x{SECS}s at 48 kHz", "card": name, "power_limit": power,
       "reps": args.reps}
for arm, ms in t.items():
    res[f"{arm}_wall_ms"] = [round(min(ms), 2), round(float(np.median(ms)), 2), round(max(ms), 2)]
res["speedup_wall_median"] = round(float(np.median(t["host_resample_poly"]) / np.median(t["device_sr"])), 3)
emit(res)
