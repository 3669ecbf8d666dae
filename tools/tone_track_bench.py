#!/usr/bin/env python
"""Cost of time-varying tone colour (include/ovc.h: ovc_convert_waveform_frames, ovc_tone_track_expand) on the
synthetic checkpoint.

For each batch shape (32 x 10 s and 1 x 3 s) three arms run the same conversion through ``convert_waveform`` with every
buffer at a stable address (so each call is a CUDA-graph replay):
    item    one embedding per item on both sides (the existing path)
    tgt     the target embedding per frame ([B, gin, T]), the source per item
    both    both embeddings per frame
plus the expansion of one keyframe track per item into the per-frame target (``tone_track_expand``).  Arms alternate
for --reps rounds; each round times --iters calls between CUDA events.  Then 64 live ``StreamingSessions`` (64-frame
windows, pushes of one window's samples, so every step converts one window per session) step with no retarget and with every 8th session in a target ramp that lasts the whole run
(its windows all overlap a transition); host wall time per step, which ends in the step's device sync, median over the
steps after warm-up.  Prints one JSON line with the card's name and power limit; times are per call, median and range.
    python tools/tone_track_bench.py [--reps 5] [--iters 10] [--precision f16x3]"""
import argparse, json, os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle import vc_oracle as O
from openvoice_b200.api import ToneColorConverter

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--precision", default="f16x3", choices=["fp32", "f16x3", "f16"])
ap.add_argument("--out", default=None, help="also append the JSON line to this file")
args = ap.parse_args()
assert torch.cuda.is_available(), "tone_track_bench measures on the GPU"

SR, HOP, GIN = 22050, 256, 256
with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False, precision=args.precision)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
nat = conv.model.native
dev = torch.device("cuda:0")


def events_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def shape_case(B, secs):
    L = SR * secs // (16 * HOP) * (16 * HOP)
    T = L // HOP
    rng = np.random.default_rng(B)
    wav = torch.from_numpy((0.5 * (2 * rng.random((B, L), dtype=np.float32) - 1)).astype(np.float32)).to(dev)
    wl = torch.full((B,), L, dtype=torch.int64, device=dev)
    g = torch.Generator().manual_seed(2)
    g_item = [(0.1 * torch.randn(B, GIN, generator=g)).to(dev) for _ in range(2)]
    w = torch.linspace(0, 1, T).view(1, 1, T).to(dev)
    g_frames = [(x[:, :, None] + w * (y - x)[:, :, None]).contiguous() for x, y in (g_item, g_item[::-1])]
    out = torch.empty(B, L, device=dev)
    fr = torch.empty(B, dtype=torch.int64, device=dev)
    arms = {
        "item": lambda: nat.convert_waveform(wav, wl, g_item[0], g_item[1], seed=1, out=out, frames_out=fr),
        "tgt": lambda: nat.convert_waveform(wav, wl, g_item[0], g_frames[1], seed=1, out=out, frames_out=fr),
        "both": lambda: nat.convert_waveform(wav, wl, g_frames[0], g_frames[1], seed=1, out=out, frames_out=fr),
    }
    # one track per item: a ramp and a hard switch, expanded into a stable per-frame buffer
    kf = torch.tensor([T // 4, T // 2, T // 2, 3 * T // 4] * B, dtype=torch.int64, device=dev)
    ks = (0.1 * torch.randn(4 * B, GIN, generator=g)).to(dev)
    k0 = torch.arange(0, 4 * B, 4, dtype=torch.int64, device=dev)
    nk = torch.full((B,), 4, dtype=torch.int64, device=dev)
    f0 = torch.zeros(B, dtype=torch.int64, device=dev)
    fT = torch.full((B,), T, dtype=torch.int64, device=dev)
    pf = torch.empty(B, GIN, T, device=dev)
    arms["expand"] = lambda: nat.tone_track_expand(kf, ks, k0, nk, f0, fT, T, out=pf)
    for fn in arms.values():          # workspaces, graph capture of each signature
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            t[k].append(events_ms(fn, args.iters))
    med = {k: float(np.median(v)) for k, v in t.items()}
    res = {f"{k}_ms": med[k] for k in arms}
    res.update({f"{k}_ms_range": [min(v), max(v)] for k, v in t.items()})
    res["tgt_overhead_pct"] = 100 * (med["tgt"] / med["item"] - 1)
    res["both_overhead_pct"] = 100 * (med["both"] / med["item"] - 1)
    res["audio_s_per_s_item"] = B * L / SR / (med["item"] / 1e3)
    res.update({"B": B, "secs": L / SR, "frames": T})
    return res


def sessions_case(S=64, W=64, chunk=64 * 256, steps=16, warm=4):
    import time
    from openvoice_b200.streaming import StreamingSessions
    rng = np.random.default_rng(3)
    audio = (0.5 * (2 * rng.random((S, chunk * steps), dtype=np.float32) - 1)).astype(np.float32)
    g = torch.Generator().manual_seed(4)
    ses = [0.1 * torch.randn(1, GIN, 1, generator=g) for _ in range(S + 1)]
    res = {}
    for arm in ("steady", "transition"):
        ss = StreamingSessions(conv, window_frames=W)
        ids = [ss.open(ses[k], ses[k + 1], seed=k) for k in range(S)]
        t = []
        for step in range(steps):
            if arm == "transition" and step == 1:
                for k in range(0, S, 8):
                    ss.retarget(ids[k], tgt_se=ses[0], ramp_frames=10 ** 6)
            t0 = time.perf_counter()
            ss.push({ids[k]: audio[k, step * chunk:(step + 1) * chunk] for k in range(S)})
            t.append(time.perf_counter() - t0)
        ss.close(ids)
        res[f"{arm}_step_ms"] = 1e3 * float(np.median(t[warm:]))
        res[f"{arm}_step_ms_range"] = [1e3 * min(t[warm:]), 1e3 * max(t[warm:])]
    res.update({"sessions": S, "window_frames": W, "push_samples": chunk, "in_transition": len(range(0, S, 8))})
    return res


name = torch.cuda.get_device_name(0)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
except Exception:
    power = "unknown"
res = {"bench": "tone_track", "gpu": name, "power_limit": power, "precision": args.precision, "reps": args.reps,
       "iters": args.iters, "b32_10s": shape_case(32, 10), "b1_3s": shape_case(1, 3), "sessions": sessions_case()}
line = json.dumps(res)
print(line, flush=True)
if args.out:
    with open(args.out, "a") as f:
        f.write(line + "\n")
