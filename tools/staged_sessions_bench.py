#!/usr/bin/env python
"""Staged against windowed live sessions: S sessions of synthetic audio pushed in 20 ms chunks (441 samples at
22.05 kHz) in lockstep, through StreamingSessions (every window converted whole with the 2 x 128-frame halo) and
through StagedSessions (latent stack in 16-frame units with a 96-frame halo, generator with a 14-frame halo).  Prints
the arithmetic frames-per-emitted-frame table (device work relative to offline, from the layer shapes), then one JSON
line per (S, window) with each arm's audio-s/s (median over rounds) and the median / p95 wall time of one lockstep tick
(host clock around work that ends in a device synchronise), plus the card and its power limit.  The arms alternate
within each round; round 0 warms up every shape, and its outputs are checked against convert on each whole clip
(<= 2e-6 * rms).

python tools/staged_sessions_bench.py [--sessions 1,8,32,64] [--windows 8,16,32,256] [--secs 5] [--rounds 2]"""
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
from openvoice_b200.streaming import (GEN_HALO_FRAMES, LATENT_HALO_FRAMES, StagedSessions,  # noqa: E402
                                      StreamingSessions)


def macs_per_frame(hp):
    """Multiply-adds per spectrogram frame of the latent stack and of the generator, from the layer shapes."""
    m = hp["model"]
    S, C, Hc = hp["data"]["filter_length"] // 2 + 1, m["inter_channels"], m["hidden_channels"]

    def wn(layers):   # in conv Hc -> 2Hc (kernel 5 in enc_q and the couplings), res/skip Hc -> 2Hc (the last Hc -> Hc)
        return layers * Hc * 2 * Hc * 5 + (layers - 1) * Hc * 2 * Hc + Hc * Hc
    enc = S * Hc + wn(16) + Hc * 2 * C
    coupling = (C // 2) * Hc + wn(4) + Hc * (C // 2)
    latent = enc + 2 * 4 * coupling                       # flow forward and reverse
    ch, up, gen = m["upsample_initial_channel"], 1, 7 * C * m["upsample_initial_channel"]
    for u, k in zip(m["upsample_rates"], m["upsample_kernel_sizes"]):
        cout = ch // 2
        gen += up * u * cout * ch * k // u                # transposed conv: k / u taps per output sample
        up *= u
        gen += up * sum(2 * 3 * cout * cout * ks for ks in m["resblock_kernel_sizes"])
        ch = cout
    gen += up * ch * 7
    return latent, gen


def frames_table(windows):
    lat, gen = macs_per_frame(O.DEFAULT_HPARAMS)
    share = lat / (lat + gen)
    rows = []
    for W in windows:
        U = min(W, 16)
        today = (W + 2 * 128) / W
        staged = share * (U + 2 * LATENT_HALO_FRAMES) / U + (1 - share) * (W + 2 * GEN_HALO_FRAMES) / W
        rows.append({"window_frames": W, "windowed": round(today, 2), "staged": round(staged, 2)})
    return {"latent_share": round(share, 4), "frames_per_emitted_frame": rows}


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,8,32,64")
    ap.add_argument("--windows", default="8,16,32,256")
    ap.add_argument("--secs", type=float, default=5.0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=441)
    ap.add_argument("--precision", default="f16x3")
    args = ap.parse_args()
    windows = [int(v) for v in args.windows.split(",")]
    print(json.dumps(frames_table(windows)), flush=True)
    assert torch.cuda.is_available(), "staged_sessions_bench measures the GPU; there is no CPU arm"
    from openvoice_b200.api import ToneColorConverter
    with tempfile.TemporaryDirectory() as td:
        cfg = os.path.join(td, "c.json")
        json.dump(O.DEFAULT_HPARAMS, open(cfg, "w"))
        conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False, precision=args.precision)
    conv.model.load_state_dict(O.synthetic_state_dict(1234))
    SR, L = 22050, int(args.secs * 22050)

    def synth_wave(i):
        rng = np.random.default_rng(1000 + i)
        return (0.5 * (2.0 * rng.random(L, dtype=np.float32) - 1.0)).astype(np.float32)

    def run(cls, waves, ses, W):
        ss = cls(conv, window_frames=W)
        sids = [ss.open(src, tgt, tau=0.3, seed=i) for i, (src, tgt) in enumerate(ses)]
        ticks, outs = [], [[] for _ in sids]
        t_all = time.perf_counter()
        for p in range(0, L, args.chunk):
            t0 = time.perf_counter()
            out = ss.push({sid: w[p:p + args.chunk] for sid, w in zip(sids, waves)})
            torch.cuda.synchronize()
            ticks.append(time.perf_counter() - t0)
            for k, sid in enumerate(sids):
                outs[k].append(out[sid])
        for k, y in enumerate(ss.close(sids).values()):
            outs[k].append(y)
        torch.cuda.synchronize()
        return time.perf_counter() - t_all, ticks, [np.concatenate(o) for o in outs]

    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "precision": args.precision, "secs": args.secs,
                      "chunk": args.chunk, "rounds": args.rounds}), flush=True)
    refs = {}
    for W in windows:
        for S in [int(v) for v in args.sessions.split(",")]:
            waves = [synth_wave(i) for i in range(S)]
            gen = torch.Generator().manual_seed(S)
            ses = [(0.1 * torch.randn(1, 256, 1, generator=gen), 0.1 * torch.randn(1, 256, 1, generator=gen))
                   for _ in range(S)]
            arms = {"StreamingSessions": StreamingSessions, "StagedSessions": StagedSessions}
            res = {k: {"rate": [], "ticks": [], "err": 0.0} for k in arms}
            for r in range(args.rounds + 1):
                for k in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                    wall, ticks, outs = run(arms[k], waves, ses, W)
                    if r == 0:                            # warm-up round: check every session against convert
                        for i, (y, w) in enumerate(zip(outs, waves)):
                            key = (S, i)
                            if key not in refs:
                                refs[key] = conv.convert(w, ses[i][0], ses[i][1], tau=0.3, seed=i).astype(np.float64)
                            ref = refs[key]
                            assert y.shape == ref.shape, (k, S, W, i)
                            e = float(np.abs(y - ref).max() / np.sqrt((ref ** 2).mean()))
                            res[k]["err"] = max(res[k]["err"], e)
                        assert res[k]["err"] <= 2e-6, (k, S, W, res[k]["err"])
                    else:
                        res[k]["rate"].append(S * L / SR / wall)
                        res[k]["ticks"] += ticks
            line = {"sessions": S, "window_frames": W, "card": name, "power_limit": power}
            for k, v in res.items():
                t = np.asarray(v["ticks"]) * 1e3
                line[k] = {"audio_s_per_s": float(np.median(v["rate"])), "rate_min": float(min(v["rate"])),
                           "rate_max": float(max(v["rate"])), "tick_ms_median": float(np.median(t)),
                           "tick_ms_p95": float(np.percentile(t, 95)), "max_err_rms": v["err"]}
            line["staged_speedup"] = line["StagedSessions"]["audio_s_per_s"] / line["StreamingSessions"]["audio_s_per_s"]
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
