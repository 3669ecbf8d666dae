#!/usr/bin/env python
"""Live multi-session streaming: S sessions of synthetic audio pushed in 20 ms chunks (441 samples at 22.05 kHz) in
lockstep, through one StreamingSessions (one batched step per tick) or through S StreamingConverter(request_seed=...)
objects pushed in turn.  Prints one JSON line per (S, window) with each arm's audio-s/s (median over rounds) and the
median / p95 wall time of one lockstep tick (host clock around work that ends in a device synchronise), plus the card
and its power limit.  The arms alternate within each round; one untimed round per arm first warms up every shape.

python tools/multistream_bench.py [--sessions 1,8,32,64] [--windows 32,256] [--secs 10] [--rounds 5]"""
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
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--chunk", type=int, default=441)
ap.add_argument("--precision", default="f16x3")
args = ap.parse_args()
assert torch.cuda.is_available(), "multistream_bench measures the GPU; there is no CPU arm"

with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False, precision=args.precision)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
SR = 22050
L = int(args.secs * SR)


def synth_wave(i):
    """bench.py's synthetic utterance: uniform noise in [-0.5, 0.5), seeded per item."""
    rng = np.random.default_rng(1000 + i)
    return (0.5 * (2.0 * rng.random(L, dtype=np.float32) - 1.0)).astype(np.float32)


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def run_sessions(waves, ses, W):
    ss = StreamingSessions(conv, window_frames=W)
    sids = [ss.open(src, tgt, tau=0.3, seed=i) for i, (src, tgt) in enumerate(ses)]
    ticks, n = [], 0
    t_all = time.perf_counter()
    for p in range(0, L, args.chunk):
        t0 = time.perf_counter()
        out = ss.push({sid: w[p:p + args.chunk] for sid, w in zip(sids, waves)})
        torch.cuda.synchronize()
        ticks.append(time.perf_counter() - t0)
        n += sum(len(v) for v in out.values())
    n += sum(len(v) for v in ss.close(sids).values())
    torch.cuda.synchronize()
    return time.perf_counter() - t_all, ticks, n


def run_converters(waves, ses, W):
    scs = [StreamingConverter(conv, src, tgt, tau=0.3, window_frames=W, request_seed=i) for i, (src, tgt) in enumerate(ses)]
    ticks, n = [], 0
    t_all = time.perf_counter()
    for p in range(0, L, args.chunk):
        t0 = time.perf_counter()
        for sc, w in zip(scs, waves):
            n += len(sc.push(w[p:p + args.chunk]))
        torch.cuda.synchronize()
        ticks.append(time.perf_counter() - t0)
    n += sum(len(sc.flush()) for sc in scs)
    torch.cuda.synchronize()
    return time.perf_counter() - t_all, ticks, n


name, power = card()
print(json.dumps({"card": name, "power_limit": power, "precision": args.precision, "secs": args.secs,
                  "chunk": args.chunk, "rounds": args.rounds}), flush=True)
for W in [int(v) for v in args.windows.split(",")]:
    for S in [int(v) for v in args.sessions.split(",")]:
        waves = [synth_wave(i) for i in range(S)]
        gen = torch.Generator().manual_seed(S)
        ses = [(0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen))
               for _ in range(S)]
        arms = {"StreamingSessions": run_sessions, "StreamingConverter": run_converters}
        res = {k: {"rate": [], "ticks": []} for k in arms}
        for r in range(args.rounds + 1):
            order = list(arms) if r % 2 == 0 else list(arms)[::-1]
            for k in order:
                wall, ticks, n = arms[k](waves, ses, W)
                assert n == S * (L // 256) * 256, (k, n)
                if r > 0:                                 # round 0 warms up every shape
                    res[k]["rate"].append(n / SR / wall)
                    res[k]["ticks"] += ticks
        line = {"sessions": S, "window_frames": W, "card": name, "power_limit": power}
        for k, v in res.items():
            t = np.asarray(v["ticks"]) * 1e3
            line[k] = {"audio_s_per_s": float(np.median(v["rate"])), "rate_min": float(min(v["rate"])),
                       "rate_max": float(max(v["rate"])), "tick_ms_median": float(np.median(t)),
                       "tick_ms_p95": float(np.percentile(t, 95))}
        line["speedup"] = line["StreamingSessions"]["audio_s_per_s"] / line["StreamingConverter"]["audio_s_per_s"]
        print(json.dumps(line), flush=True)
