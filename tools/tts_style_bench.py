#!/usr/bin/env python
"""Cost of time-varying speaking style (include/ovc.h: ovc_tts_encode_g) on the synthetic checkpoints.

BASELINE config 3's TTS shape: 16 requests x 3 sentences of 121 tokens, through ``BaseSpeakerTTS.tts_batch`` (the TTS
alone) and ``ToneColorConverter.clone_batch`` (text to cloned voice), in three arms with the same text and seeds:
    sid     speaker ids (the emb_g path)
    blend   one vector per request, 0.7 * style(a) + 0.3 * style(b)
    track   a two-key ToneTrack per request over its token positions (a ramp from one style to another)
Arms alternate for --reps rounds; each round times --iters calls with a host clock that ends in a device sync (the calls
download their audio).  Also reported: the extra decode workspace of per-frame conditioning for the batch's frames,
B * Ymax * (gin + per-frame columns) floats.  Prints one JSON line with the card's name and power limit; times are per
call, median and range.
    python tools/tts_style_bench.py [--reps 5] [--iters 5] [--precision f16x3]"""
import argparse, copy, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle import tts_oracle as T
from oracle import vc_oracle as O
from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter, ToneTrack

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--precision", default="f16x3", choices=["fp32", "f16x3", "f16"])
ap.add_argument("--out", default=None, help="also append the JSON line to this file")
args = ap.parse_args()
assert torch.cuda.is_available(), "tts_style_bench measures on the GPU"

R, S, NTOK, TARGET_COLS = 16, 3, 121, 6656
with tempfile.TemporaryDirectory() as td:
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1, "whispering": 2}
    json.dump(hp, open(os.path.join(td, "tts.json"), "w"))
    torch.save({"model": T.synthetic_tts_state_dict()}, os.path.join(td, "tts.pth"))
    tts = BaseSpeakerTTS(os.path.join(td, "tts.json"), device="cuda:0", precision=args.precision)
    tts.load_ckpt(os.path.join(td, "tts.pth"))
    json.dump(O.DEFAULT_HPARAMS, open(os.path.join(td, "vc.json"), "w"))
    conv = ToneColorConverter(os.path.join(td, "vc.json"), device="cuda:0", enable_watermark=False,
                              precision=args.precision)
conv.model.load_state_dict(O.synthetic_state_dict(1234))

rng = np.random.default_rng(3)
n_spk = T.TTS_HPARAMS["n_speakers"]
text = [[rng.integers(0, T.TTS_HPARAMS["n_vocab"], NTOK).tolist() for _ in range(S)] for _ in range(R)]


def speaker(arm, r):
    a, b = r % n_spk, (r + 1) % n_spk
    if arm == "sid":
        return a
    if arm == "blend":
        return 0.7 * tts.style(a) + 0.3 * tts.style(b)
    return ToneTrack([(0, tts.style(a)), (S * NTOK, tts.style(b))])


def se(seed):
    return 0.1 * torch.randn(1, 256, 1, generator=torch.Generator().manual_seed(seed))


reqs = {arm: [dict(ids=text[r], speaker=speaker(arm, r), seed=100 + r, src_se=se(2 * r), tgt_se=se(2 * r + 1), tau=0.3,
                   convert_seed=r) for r in range(R)] for arm in ("sid", "blend", "track")}
calls = {"tts_batch": lambda q: tts.tts_batch(q), "clone_batch": lambda q: conv.clone_batch(tts, q)}
times = {(c, a): [] for c in calls for a in reqs}
for c, fn in calls.items():
    for a, q in reqs.items():
        fn(q)                                                        # warm-up: modules, workspace sizes, allocator
torch.cuda.synchronize()
for _ in range(args.reps):
    for c, fn in calls.items():
        for a, q in reqs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                fn(q)
            torch.cuda.synchronize()
            times[(c, a)].append((time.perf_counter() - t0) * 1e3 / args.iters)

# decode frames of the track arm (one ragged decode of every sentence): the per-frame workspace it adds
x, lens = tts._pad_ids([s for r in text for s in r])
_, _, _, _, kw = tts._request_sentences(reqs["track"])
frames = tts.model.tts_encode(x, lens, g=kw["g"], seeds=kw["seeds"], streams=kw["streams"]).frames
gin = int(tts.hps.model.gin_channels)
extra = len(frames) * max(frames) * (gin + TARGET_COLS) * 4
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
out = {"bench": "tts_style", "gpu": smi[0] if smi else "unknown", "precision": args.precision,
       "workload": f"{R} requests x {S} sentences x {NTOK} tokens", "reps": args.reps, "iters": args.iters,
       "ms_per_call": {f"{c}/{a}": {"median": round(float(np.median(v)), 3), "min": round(min(v), 3),
                                    "max": round(max(v), 3)} for (c, a), v in times.items()},
       "per_frame_decode_workspace_bytes": extra, "decoded_rows": len(frames), "max_frames": max(frames)}
line = json.dumps(out)
print(line)
if args.out:
    with open(args.out, "a") as f:
        f.write(line + "\n")
