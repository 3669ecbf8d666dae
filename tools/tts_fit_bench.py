#!/usr/bin/env python
"""Cost of the duration fit (include/ovc.h: ovc_tts_encode_fit) on the synthetic checkpoint.

BASELINE config 3's TTS shape: 16 requests x 3 sentences of 121 tokens through ``BaseSpeakerTTS.tts_batch``, in two arms
with the same text and seeds:
    plain     speed 1.0
    duration  each request fitted to its plain length rounded to 0.1 s (one fit group of 3 sentences per request)
and the encode alone (``NativeSynthesizer.tts_encode`` of the 48 sentences, which ends in its host sync) in the same two
arms.  Arms alternate for --reps rounds; each round times --iters calls with a host clock that ends in a device sync.
Prints one JSON line with the card's name and power limit; times are per call, median and range.
    python tools/tts_fit_bench.py [--reps 7] [--iters 5] [--precision f16x3]"""
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
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--precision", default="f16x3", choices=["fp32", "f16x3", "f16"])
ap.add_argument("--out", default=None, help="also append the JSON line to this file")
args = ap.parse_args()
assert torch.cuda.is_available(), "tts_fit_bench measures on the GPU"

R, S, NTOK = 16, 3, 121
with tempfile.TemporaryDirectory() as td:
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    json.dump(hp, open(os.path.join(td, "tts.json"), "w"))
    torch.save({"model": T.synthetic_tts_state_dict()}, os.path.join(td, "tts.pth"))
    tts = BaseSpeakerTTS(os.path.join(td, "tts.json"), device="cuda:0", precision=args.precision)
    tts.load_ckpt(os.path.join(td, "tts.pth"))
sr = int(tts.hps.data.sampling_rate)

rng = np.random.default_rng(3)
text = [[rng.integers(0, T.TTS_HPARAMS["n_vocab"], NTOK).tolist() for _ in range(S)] for _ in range(R)]
plain = [dict(ids=text[r], speaker=r % T.TTS_HPARAMS["n_speakers"], seed=100 + r) for r in range(R)]
lengths = [len(a) for a in tts.tts_batch(plain)]
fitted = [dict(q, duration=round(n / sr, 1)) for q, n in zip(plain, lengths)]
reqs = {"plain": plain, "duration": fitted}
enc = {}
for arm, q in reqs.items():
    seqs, sid, _, _, kw = tts._request_sentences(q)
    x, lens = tts._pad_ids(seqs)
    enc[arm] = (x, lens, torch.as_tensor(sid), kw)
calls = {"tts_batch": lambda arm: tts.tts_batch(reqs[arm]),
         "tts_encode": lambda arm: tts.model.tts_encode(enc[arm][0], enc[arm][1], sid=enc[arm][2], **enc[arm][3])}
times = {(c, a): [] for c in calls for a in reqs}
for c, fn in calls.items():
    for a in reqs:
        fn(a)                                                        # warm-up: modules, workspace sizes, allocator
torch.cuda.synchronize()
for _ in range(args.reps):
    for c, fn in calls.items():
        for a in reqs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                fn(a)
            torch.cuda.synchronize()
            times[(c, a)].append((time.perf_counter() - t0) * 1e3 / args.iters)

out_len = [len(a) for a in tts.tts_batch(fitted)]
want = [int(round(q["duration"] * sr)) for q in fitted]
scales = tts.model.tts_encode(enc["duration"][0], enc["duration"][1], sid=enc["duration"][2], **enc["duration"][3]).length_scale
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
med = {k: float(np.median(v)) for k, v in times.items()}
out = {"bench": "tts_fit", "gpu": smi[0] if smi else "unknown", "precision": args.precision,
       "workload": f"{R} requests x {S} sentences x {NTOK} tokens", "reps": args.reps, "iters": args.iters,
       "ms_per_call": {f"{c}/{a}": {"median": round(med[(c, a)], 3), "min": round(min(v), 3), "max": round(max(v), 3)}
                       for (c, a), v in times.items()},
       "encode_overhead_ms": round(med[("tts_encode", "duration")] - med[("tts_encode", "plain")], 3),
       "tts_batch_overhead_ms": round(med[("tts_batch", "duration")] - med[("tts_batch", "plain")], 3),
       "fitted_samples_minus_target": [n - w for n, w in zip(out_len, want)],
       "scales": sorted({round(s, 6) for s in scales})}
line = json.dumps(out)
print(line)
if args.out:
    with open(args.out, "a") as f:
        f.write(line + "\n")
