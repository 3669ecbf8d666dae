#!/usr/bin/env python
"""Live sessions at 48 kHz in and out: S sessions of synthetic audio pushed in 20 ms chunks (960 samples) in lockstep.
Three arms: one StreamingSessions(rates=(48000,)) (one batched step per tick, ring resampling on both sides); S
StreamingConverter(input_sr=48000, output_sr=48000, request_seed=...) pushed in turn; and, as the floor, one
StreamingSessions at the model's rate on the same audio duration (441-sample chunks), so the cost of resampling shows.
Prints one JSON line per (S, window) with each arm's audio-s/s (median over rounds, and its range) and the median / p95
wall time of one tick (host clock around work that ends in a device synchronise), plus the card and its power limit.
The arms alternate within each round; one untimed round per arm first warms up every shape.  A separate
torch.profiler pass (--profile) reports the device time of the ovc_resample_rings kernel per step.

python tools/multirate_sessions_bench.py [--sessions 1,8,32,64] [--windows 32,256] [--secs 10] [--rounds 3] [--profile]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import vc_oracle as O  # noqa: E402
from openvoice_b200.api import ToneColorConverter  # noqa: E402
from openvoice_b200.streaming import StreamingConverter, StreamingSessions  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--sessions", default="1,8,32,64")
ap.add_argument("--windows", default="32,256")
ap.add_argument("--secs", type=float, default=10.0)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--rate", type=int, default=48000)
ap.add_argument("--precision", default="f16x3")
ap.add_argument("--profile", action="store_true", help="only the torch.profiler pass")
args = ap.parse_args()
assert torch.cuda.is_available(), "multirate_sessions_bench measures the GPU; there is no CPU arm"

with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False, precision=args.precision)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
SR, R = 22050, args.rate
CH = {R: R // 50, SR: SR // 50}                         # 20 ms chunks


def synth_wave(i, sr):
    """bench.py's synthetic utterance at rate sr: uniform noise in [-0.5, 0.5), seeded per item."""
    rng = np.random.default_rng(1000 + i)
    return (0.5 * (2.0 * rng.random(int(args.secs * sr), dtype=np.float32) - 1.0)).astype(np.float32)


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def run_sessions(waves, ses, W, sr, on_tick=None):
    ss = StreamingSessions(conv, window_frames=W, rates=(R,) if sr != SR else ())
    rate = None if sr == SR else sr
    sids = [ss.open(src, tgt, tau=0.3, seed=i, input_sr=rate, output_sr=rate) for i, (src, tgt) in enumerate(ses)]
    ticks, n = [], 0
    t_all = time.perf_counter()
    for p in range(0, len(waves[0]), CH[sr]):
        t0 = time.perf_counter()
        out = ss.push({sid: w[p:p + CH[sr]] for sid, w in zip(sids, waves)})
        torch.cuda.synchronize()
        ticks.append(time.perf_counter() - t0)
        n += sum(len(v) for v in out.values())
        if on_tick:
            on_tick()
    n += sum(len(v) for v in ss.close(sids).values())
    torch.cuda.synchronize()
    return time.perf_counter() - t_all, ticks, n


def run_converters(waves, ses, W, sr):
    scs = [StreamingConverter(conv, src, tgt, tau=0.3, window_frames=W, input_sr=sr, output_sr=sr, request_seed=i)
           for i, (src, tgt) in enumerate(ses)]
    ticks, n = [], 0
    t_all = time.perf_counter()
    for p in range(0, len(waves[0]), CH[sr]):
        t0 = time.perf_counter()
        for sc, w in zip(scs, waves):
            n += len(sc.push(w[p:p + CH[sr]]))
        torch.cuda.synchronize()
        ticks.append(time.perf_counter() - t0)
    n += sum(len(sc.flush()) for sc in scs)
    torch.cuda.synchronize()
    return time.perf_counter() - t_all, ticks, n


def embeddings(S):
    gen = torch.Generator().manual_seed(S)
    return [(0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)) for _ in range(S)]


def profile_pass(S, W):
    """Device time of the ring resampler per step (both launches), from a torch.profiler run of its own."""
    from torch.profiler import ProfilerActivity, profile
    waves, ses = [synth_wave(i, R) for i in range(S)], embeddings(S)
    run_sessions(waves, ses, W, R)                        # warm-up
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        _, ticks, _ = run_sessions(waves, ses, W, R)
    us, calls = 0.0, 0
    for e in prof.key_averages():
        if "resample_ring_kernel" in e.key:
            us += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            calls += e.count
    steps = len(ticks) + 1
    return {"sessions": S, "window_frames": W, "steps": steps, "resample_rings_launches": calls,
            "resample_rings_us_per_step": us / steps, "resample_rings_us_per_launch": us / max(1, calls)}


name, power = card()
print(json.dumps({"card": name, "power_limit": power, "precision": args.precision, "secs": args.secs, "rate": R,
                  "rounds": args.rounds}), flush=True)
for W in [int(v) for v in args.windows.split(",")]:
    for S in [int(v) for v in args.sessions.split(",")]:
        if args.profile:
            print(json.dumps({**profile_pass(S, W), "card": name, "power_limit": power}), flush=True)
            continue
        w_r, w_m, ses = [synth_wave(i, R) for i in range(S)], [synth_wave(i, SR) for i in range(S)], embeddings(S)
        arms = {"sessions_48k": lambda: run_sessions(w_r, ses, W, R),
                "converters_48k": lambda: run_converters(w_r, ses, W, R),
                "sessions_model_rate": lambda: run_sessions(w_m, ses, W, SR)}
        res = {k: {"rate": [], "ticks": []} for k in arms}
        for r in range(args.rounds + 1):
            order = list(arms) if r % 2 == 0 else list(arms)[::-1]
            for k in order:
                wall, ticks, n = arms[k]()
                if r > 0:                                 # round 0 warms up every shape
                    res[k]["rate"].append(S * args.secs / wall)
                    res[k]["ticks"] += ticks
        line = {"sessions": S, "window_frames": W, "card": name, "power_limit": power}
        for k, v in res.items():
            t = np.asarray(v["ticks"]) * 1e3
            line[k] = {"audio_s_per_s": float(np.median(v["rate"])), "rate_min": float(min(v["rate"])),
                       "rate_max": float(max(v["rate"])), "tick_ms_median": float(np.median(t)),
                       "tick_ms_p95": float(np.percentile(t, 95))}
        print(json.dumps(line), flush=True)
