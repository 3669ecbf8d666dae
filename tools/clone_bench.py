"""Text to cloned voice, measured as users run it (demo_part1.ipynb: ``tts`` -> ``convert``): whole utterances,
sentences joined with 50 ms / speed gaps, converted as one clip each.

Workload: 16 requests x 3 sentences x ~121 tokens (ragged), synthetic checkpoints (oracle/tts_oracle.py,
oracle/vc_oracle.py), one GPU.  Timed on the host clock around calls that end in a device synchronise (every call
returns host arrays), after warm-up calls of the same shapes:
  clone_batch      ToneColorConverter.clone_batch: host ids in, host audio out, the join on the device
  two_step         BaseSpeakerTTS.tts_batch -> ToneColorConverter.convert_batch on the same requests (host join),
                   timed alternately with clone_batch in the same run
  stream           clone_stream_batch: time to the first chunk and mean time per step
Prints one JSON object with the card's name and power limit (nvidia-smi, read-only).

    python tools/clone_bench.py [--requests 16] [--sentences 3] [--tokens 121] [--iters 5] [--precision f16x3]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build(tmp, precision):
    from oracle import tts_oracle as T
    from oracle import vc_oracle as O
    from openvoice_b200.api import BaseSpeakerTTS, ToneColorConverter
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1}
    with open(os.path.join(tmp, "tts.json"), "w") as f:
        json.dump(hp, f)
    torch.save({"model": T.synthetic_tts_state_dict()}, os.path.join(tmp, "tts.pth"))
    tts = BaseSpeakerTTS(os.path.join(tmp, "tts.json"), device="cuda:0", precision=precision)
    tts.load_ckpt(os.path.join(tmp, "tts.pth"))
    with open(os.path.join(tmp, "vc.json"), "w") as f:
        json.dump(O.DEFAULT_HPARAMS, f)
    conv = ToneColorConverter(os.path.join(tmp, "vc.json"), device="cuda:0", enable_watermark=False, precision=precision)
    conv.model.load_state_dict(O.synthetic_state_dict(1234))
    return tts, conv


def workload(n, k, tokens, seed):
    from oracle import tts_oracle as T
    rng = np.random.default_rng(0)
    gen = torch.Generator().manual_seed(9)
    reqs = []
    for r in range(n):
        ids = [rng.integers(0, T.TTS_HPARAMS["n_vocab"], tokens - (7 * (r * k + j)) % 23).tolist() for j in range(k)]
        reqs.append(dict(ids=ids, speaker=r % T.TTS_HPARAMS["n_speakers"], speed=1.0, seed=seed + r,
                         src_se=0.1 * torch.randn(1, 256, 1, generator=gen), tgt_se=0.1 * torch.randn(1, 256, 1, generator=gen),
                         tau=0.3, convert_seed=seed + 1000 + r))
    return reqs


def measure(n=16, k=3, tokens=121, iters=5, precision="f16x3"):
    assert torch.cuda.is_available(), "clone_bench measures on the GPU"
    with tempfile.TemporaryDirectory() as tmp:
        tts, conv = build(tmp, precision)
    reqs = workload(n, k, tokens, 11)

    def clone():
        return conv.clone_batch(tts, reqs)

    def two_step():
        audio = tts.tts_batch(reqs)
        return conv.convert_batch(audio, [q["src_se"] for q in reqs], [q["tgt_se"] for q in reqs],
                                  tau=[q["tau"] for q in reqs], seeds=[q["convert_seed"] for q in reqs])

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    for _ in range(2):                                    # warm-up: workspaces, pinned buffers, graph captures
        a, b = clone(), two_step()
    same = all(np.array_equal(x, y) for x, y in zip(a, b))
    audio_s = sum(len(x) for x in a) / float(conv.hps.data.sampling_rate)
    t_clone, t_two = [], []
    for _ in range(iters):                                # alternating, so both see the same machine state
        t_clone.append(timed(clone)[0])
        t_two.append(timed(two_step)[0])

    def stream():
        t0 = time.perf_counter()
        first, steps, seen = None, 0, set()
        for r, _ in conv.clone_stream_batch(tts, reqs):
            if first is None:
                first = time.perf_counter() - t0
            if r in seen or not seen:                     # a request yields once per step
                steps += 1
                seen = set()
            seen.add(r)
        torch.cuda.synchronize()
        return first * 1e3, (time.perf_counter() - t0) * 1e3, steps

    stream()
    runs = [stream() for _ in range(iters)]
    med = lambda v: float(np.median(v))  # noqa: E731
    return {
        "workload": f"{n} requests x {k} sentences x ~{tokens} tokens, speed 1.0, synthetic weights, {precision}",
        "card": card(),
        "audio_s_per_call": round(audio_s, 2),
        "clone_batch_ms": round(med(t_clone), 2), "clone_batch_ms_all": [round(v, 2) for v in t_clone],
        "two_step_ms": round(med(t_two), 2), "two_step_ms_all": [round(v, 2) for v in t_two],
        "clone_vs_two_step": round(med(t_two) / med(t_clone), 3),
        "clone_equals_two_step": same,
        "stream_first_chunk_ms": round(med([r[0] for r in runs]), 2),
        "stream_total_ms": round(med([r[1] for r in runs]), 2),
        "stream_steps": runs[0][2],
        "stream_mean_step_ms": round(med([r[1] / r[2] for r in runs]), 2),
        "iters": iters,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--sentences", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=121)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--precision", default="f16x3")
    a = ap.parse_args()
    print(json.dumps(measure(a.requests, a.sentences, a.tokens, a.iters, a.precision)))


if __name__ == "__main__":
    main()
