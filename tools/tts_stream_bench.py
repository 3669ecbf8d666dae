#!/usr/bin/env python
"""Streaming base-speaker TTS (BaseSpeakerTTS.tts_stream_batch) against the whole-utterance calls, on the synthetic V1
checkpoint.

Two workloads, each request 4 sentences x 121 tokens (the sentence length SURVEY.md section 8 measured, blanks
included):
    single   one request:   tts_stream         vs tts_from_ids
    batch16  16 requests:   tts_stream_batch   vs tts_batch
For each arm: time to the first chunk (streaming) or to the whole audio (whole-utterance calls, whose first audio IS
the whole audio), and total wall time, host clock around work that ends with the audio on the host (a device sync).
Every arm is warmed up (workspaces, graph capture), then the arms alternate for --reps rounds; medians.  The streamed
audio is checked against the whole call (same length, within 2e-6 of its rms).  Prints one JSON line with the card name
and its power limit.
    python tools/tts_stream_bench.py [--reps 7] [--precision f16x3] [--window 256] [--first 32]"""
import argparse, copy, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle import tts_oracle as T
from oracle import vc_oracle as O
from openvoice_b200.api import BaseSpeakerTTS

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--precision", default="f16x3", choices=["fp32", "f16x3", "f16"])
ap.add_argument("--window", type=int, default=256)
ap.add_argument("--first", type=int, default=32)
ap.add_argument("--out", default=None, help="also append the JSON line to this file")
args = ap.parse_args()
assert torch.cuda.is_available(), "tts_stream_bench measures on the GPU"

SENTS, TOKENS, SR = 4, 121, 22050
with tempfile.TemporaryDirectory() as td:
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1}
    json.dump(hp, open(os.path.join(td, "c.json"), "w"))
    torch.save({"model": T.synthetic_tts_state_dict()}, os.path.join(td, "ckpt.pth"))
    eng = BaseSpeakerTTS(os.path.join(td, "c.json"), device="cuda:0", precision=args.precision)
    eng.load_ckpt(os.path.join(td, "ckpt.pth"))
rng = np.random.default_rng(0)
nv = T.TTS_HPARAMS["n_vocab"]


def request(i):
    return dict(ids=[rng.integers(0, nv, TOKENS).tolist() for _ in range(SENTS)], speaker="default", seed=1000 + i)


reqs = [request(i) for i in range(16)]
one = reqs[0]


def whole_single():
    return [eng.audio_numpy_concat(eng.tts_from_ids(one["ids"], "default", seed=one["seed"]), SR)]


def whole_batch():
    return eng.tts_batch(reqs)


def stream(rs):
    per = [[] for _ in rs]
    t_first = None
    for r, chunk in eng.tts_stream_batch(rs, window_frames=args.window, first_window_frames=args.first):
        if t_first is None:
            t_first = time.perf_counter()
        per[r].append(chunk)
    return t_first, [np.concatenate(p) for p in per]


def timed_whole(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    t = time.perf_counter() - t0
    return t, t, out


def timed_stream(rs):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t_first, out = stream(rs)
    return t_first - t0, time.perf_counter() - t0, out


arms = {"single": (lambda: timed_whole(whole_single), lambda: timed_stream([one])),
        "batch16": (lambda: timed_whole(whole_batch), lambda: timed_stream(reqs))}
for name, (w, s) in arms.items():                # warm-up and the audio check
    for _ in range(3):
        a, b = w()[2], s()[2]
    for x, y in zip(a, b):
        assert x.shape == y.shape
        err = np.abs(x.astype(np.float64) - y).max() / np.sqrt((x.astype(np.float64) ** 2).mean())
        assert err <= 2e-6, (name, err)
times = {k: {"whole_first": [], "whole_total": [], "stream_first": [], "stream_total": []} for k in arms}
for _ in range(args.reps):
    for name, (w, s) in arms.items():
        f, t, _ = w()
        times[name]["whole_first"].append(f)
        times[name]["whole_total"].append(t)
        f, t, _ = s()
        times[name]["stream_first"].append(f)
        times[name]["stream_total"].append(t)

gpu = torch.cuda.get_device_name(0)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
except Exception:
    power = "unknown"
res = {"bench": "tts_stream", "gpu": gpu, "power_limit": power, "precision": args.precision, "sentences": SENTS,
       "tokens": TOKENS, "window_frames": args.window, "first_window_frames": args.first, "reps": args.reps,
       "audio_s_single": len(whole_single()[0]) / SR}
for name, d in times.items():
    for k, v in d.items():
        res[f"{name}_{k}_ms"] = round(1e3 * float(np.median(v)), 2)
line = json.dumps(res)
print(line, flush=True)
if args.out:
    with open(args.out, "a") as f:
        f.write(line + "\n")
