#!/usr/bin/env python
"""Live enrollment cost: S sessions of synthetic audio pushed in 20 ms chunks (441 samples at 22.05 kHz) in lockstep
through one StreamingSessions, with and without ``enroll=Enrollment()`` (the arms alternate within each round; one
untimed round per arm first warms up every shape).  Prints one JSON line per S with each arm's median / p95 tick (host
clock around work that ends in a device synchronise) and the device time of the step's ``reference_encoder_stream`` call
(CUDA events around it, median and p95).  Steps are split into three kinds, each reported on its own for both arms:
steps that take a snapshot, other steps whose new frames complete a GRU step (every 64 frames; in lockstep with a
64-frame window these are also the steps that convert windows), and the rest.  As the
alternative it times ``extract_se`` on the growing prefix (2 s, 5 s and 10 s of audio), which a caller re-encoding the
whole prefix would pay per snapshot.  The card and its power limit are printed with the numbers.

python tools/enroll_bench.py [--sessions 1,8,32,64] [--window 64] [--secs 10] [--rounds 3]"""
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
from openvoice_b200.streaming import Enrollment, StreamingSessions, ready_frames  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--sessions", default="1,8,32,64")
ap.add_argument("--window", type=int, default=64)
ap.add_argument("--secs", type=float, default=10.0)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--chunk", type=int, default=441)
ap.add_argument("--precision", default="f16x3")
args = ap.parse_args()
assert torch.cuda.is_available(), "enroll_bench measures the GPU; there is no CPU arm"

with tempfile.TemporaryDirectory() as td:
    cfg = os.path.join(td, "c.json")
    json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
    conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False, precision=args.precision)
conv.model.load_state_dict(O.synthetic_state_dict(1234))
nat = conv.model.native
SR = 22050
L = int(args.secs * SR)


def synth_wave(i):
    rng = np.random.default_rng(1000 + i)
    return (0.5 * (2.0 * rng.random(L, dtype=np.float32) - 1.0)).astype(np.float32)


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


enc_ms = []
_real = type(nat).reference_encoder_stream


def timed_encoder(self, *a, **k):
    """reference_encoder_stream between two CUDA events; the elapsed time is read after the tick's sync."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = _real(self, *a, **k)
    e1.record()
    enc_ms.append((e0, e1))
    return out


type(nat).reference_encoder_stream = timed_encoder


def kind(n0, n1):
    """What a lockstep step from n0 to n1 samples asks of the encoder: "snapshot", "gru" (a GRU step) or "rows"."""
    if Enrollment().snapshot(n0, n1, 256):
        return "snapshot"
    return "gru" if ready_frames(n1, 256, 1024, False) >> 6 != ready_frames(n0, 256, 1024, False) >> 6 else "rows"


def run(waves, ses, enroll):
    """Ticks of every push step, their kinds, and the encoder events of the push steps (the closing step's dropped)."""
    ss = StreamingSessions(conv, window_frames=args.window)
    sids = [ss.open(src, tgt, tau=0.3, seed=i, enroll=enroll) for i, (src, tgt) in enumerate(ses)]
    ticks, kinds = [], []
    for p in range(0, L, args.chunk):
        t0 = time.perf_counter()
        ss.push({sid: w[p:p + args.chunk] for sid, w in zip(sids, waves)})
        torch.cuda.synchronize()
        ticks.append(time.perf_counter() - t0)
        kinds.append(kind(p, min(L, p + args.chunk)))
    n_push = len(enc_ms)
    ss.close(sids)
    torch.cuda.synchronize()
    return ticks, kinds, enc_ms[:n_push]


name, power = card()
print(json.dumps({"card": name, "power_limit": power, "precision": args.precision, "secs": args.secs,
                  "chunk": args.chunk, "window_frames": args.window, "rounds": args.rounds}), flush=True)
w0 = synth_wave(0)
prefix = {}
for secs in (2, 5, 10):
    n = min(L, int(secs * SR))
    for _ in range(3):
        conv.extract_se(w0[:n])
    torch.cuda.synchronize()
    t = []
    for _ in range(10):
        t0 = time.perf_counter()
        conv.extract_se(w0[:n])
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    prefix[f"{secs}s"] = float(np.median(t) * 1e3)
print(json.dumps({"extract_se_prefix_ms": prefix}), flush=True)
for S in [int(v) for v in args.sessions.split(",")]:
    waves = [synth_wave(i) for i in range(S)]
    gen = torch.Generator().manual_seed(S)
    ses = [(0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen)) for _ in range(S)]
    arms = {"plain": None, "enroll": Enrollment()}
    res = {k: [] for k in arms}
    by_kind = {}                                          # kind -> (plain ticks, enroll ticks, encoder ms)
    for r in range(args.rounds + 1):
        for k in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            enc_ms.clear()
            ticks, kinds, ev = run(waves, ses, arms[k])
            if r > 0:                                     # round 0 warms up every shape
                res[k] += ticks
                for t, kd in zip(ticks, kinds):
                    by_kind.setdefault(kd, ([], [], []))[0 if arms[k] is None else 1].append(t * 1e3)
                if arms[k] is not None:
                    assert len(ev) == len(ticks), (len(ev), len(ticks))
                    by_kind_ev = [a.elapsed_time(b) for a, b in ev]
                    for kd, e in zip(kinds, by_kind_ev):
                        by_kind[kd][2].append(e)
    line = {"sessions": S, "window_frames": args.window, "card": name, "power_limit": power}
    for k, v in res.items():
        t = np.asarray(v) * 1e3
        line[k] = {"tick_ms_median": float(np.median(t)), "tick_ms_p95": float(np.percentile(t, 95))}
    for kd, (tp, t, e) in sorted(by_kind.items()):
        line[kd] = {"steps": len(t), "plain_tick_ms_median": float(np.median(tp)), "tick_ms_median": float(np.median(t)),
                    "tick_ms_p95": float(np.percentile(t, 95)), "encoder_ms_median": float(np.median(e)),
                    "encoder_ms_p95": float(np.percentile(e, 95))}
    print(json.dumps(line), flush=True)
