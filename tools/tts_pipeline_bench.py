"""BASELINE.json config 3: V1 full pipeline BaseSpeakerTTS.tts + ToneColorConverter.convert, batch 16, one H100.

Synthetic checkpoints (no network), token sequences of the length SURVEY.md section 8 measured for a sentence
(T_text = 121 incl. blanks).  Timed with CUDA events after warm-up:
  tts        ids -> waveform (ovc_tts_encode + ovc_tts_decode, ragged batch)          [host ids in, device audio out]
  convert    device audio -> converted audio (ovc_convert_waveform, ragged batch)
  e2e        host ids in -> converted audio on the host (pinned), both stages, one sync for y_lengths
Prints one JSON object.  Not the headline bench (bench.py measures convert at config 2); this is the config-3 companion.

    python tools/tts_pipeline_bench.py [--batch 16] [--tokens 121] [--iters 5] [--cpu]
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def measure(batch=16, tokens=121, iters=5, cpu=False, precision="f16x3"):
    a = argparse.Namespace(batch=batch, tokens=tokens, iters=iters, cpu=cpu, precision=precision)

    from oracle import tts_oracle as T          # synthetic checkpoint recipe + the optional CPU leg only
    from oracle import vc_oracle as V
    from openvoice_b200.api import NativeSynthesizer
    from openvoice_b200.utils import HParams

    dev = torch.device("cuda:0")
    hp_t = copy.deepcopy(V.DEFAULT_HPARAMS)
    hp_t["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    tts = NativeSynthesizer(HParams(**hp_t), "cuda:0", precision=a.precision)
    sd_t = T.synthetic_tts_state_dict()
    tts.load_state_dict(sd_t)
    conv = NativeSynthesizer(HParams(**V.DEFAULT_HPARAMS), "cuda:0", precision=a.precision)
    conv.load_state_dict(V.synthetic_state_dict(1234))

    B, Tn = a.batch, a.tokens
    lens = [Tn - (7 * i) % 23 for i in range(B)]                       # ragged sentences
    tokens, lengths, sid, _ = T.synthetic_tts_inputs(B, Tn, 77, lens)
    tokens_h, lengths_h, sid_h = tokens.pin_memory(), lengths.pin_memory(), sid.pin_memory()
    gen = torch.Generator().manual_seed(9)
    src_se = (0.1 * torch.randn(1, 256, generator=gen)).to(dev).expand(B, -1).contiguous()
    tgt_se = (0.1 * torch.randn(1, 256, generator=gen)).to(dev).expand(B, -1).contiguous()
    hop = 256

    def tts_stage(seed):
        x, xl, s = tokens_h.to(dev, non_blocking=True), lengths_h.to(dev, non_blocking=True), sid_h.to(dev, non_blocking=True)
        yl, _, _ = tts.native.tts_encode(x, xl, s, seed=seed, noise_scale_w=0.6, length_scale=1.0, sdp_ratio=0.2)
        ymax = int(yl.max().item())                                     # the reference syncs here too (models.py:476-478)
        o, _ = tts.native.tts_decode(B, ymax, dev, seed=seed + 1, noise_scale=0.667, ragged=True)
        return o[:, 0], yl

    def convert_stage(wav, yl, seed):
        out, frames = conv.native.convert_waveform(wav.contiguous(), (yl * hop).contiguous(), src_se, tgt_se, tau=0.3, seed=seed)
        return out, frames

    def timed(fn, iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        for i in range(iters):
            r = fn(i)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / iters, r

    for w in range(3):                                                   # warm-up (workspaces, pinned buffers)
        wav, yl = tts_stage(w)
        convert_stage(wav, yl, w)
    torch.cuda.synchronize()

    tts_ms, (wav, yl) = timed(lambda i: tts_stage(100 + i), a.iters)
    audio_s = float(yl.sum().item()) * hop / 22050.0
    conv_ms, _ = timed(lambda i: convert_stage(wav, yl, 200 + i), a.iters)
    host = torch.empty(B, 2 * wav.shape[1], dtype=torch.float32).pin_memory()    # durations vary with the seed

    def e2e(i):
        w, y = tts_stage(300 + i)
        o, _ = convert_stage(w, y, 400 + i)
        host[:, : o.shape[1]].copy_(o, non_blocking=True)
        return y

    e2e_ms, yl2 = timed(e2e, a.iters)
    audio_s2 = float(yl2.sum().item()) * hop / 22050.0
    # stage split of the TTS half (events inside the library)
    tts.native.profile_enable(True)
    x, xl, s = tokens.to(dev), lengths.to(dev), sid.to(dev)
    t0 = time.perf_counter()
    ylp, _, _ = tts.native.tts_encode(x, xl, s, seed=1, noise_scale_w=0.6)
    torch.cuda.synchronize()
    enc_wall_ms = (time.perf_counter() - t0) * 1e3
    enc_launches = tts.native.last_launch_count
    by_kernel = {}
    for name, ms, fl, by, fam in tts.native.profile_detail():
        e = by_kernel.setdefault(name, [0, 0.0])
        e[0] += 1
        e[1] += ms
    tts.native.profile_enable(False)

    res = {
        "workload": f"V1 BaseSpeakerTTS.tts + ToneColorConverter.convert, batch {B}, {Tn} tokens/sentence (ragged), synthetic weights",
        "precision": a.precision,
        "audio_s_per_batch": round(audio_s, 2),
        "tts_ms": round(tts_ms, 2), "convert_ms": round(conv_ms, 2), "e2e_ms": round(e2e_ms, 2),
        "tts_audio_s_per_s": round(audio_s / tts_ms * 1e3, 1),
        "convert_audio_s_per_s": round(audio_s / conv_ms * 1e3, 1),
        "pipeline_audio_s_per_s": round(audio_s2 / e2e_ms * 1e3, 1),
        "text_front_wall_ms": round(enc_wall_ms, 2), "text_front_launches": enc_launches,
        "text_front_kernels_ms": {k: [v[0], round(v[1], 3)] for k, v in sorted(by_kernel.items(), key=lambda kv: -kv[1][1])},
        "frames": [int(v) for v in yl.cpu()],
    }
    if a.cpu:
        from bench import host_cores
        torch.set_num_threads(host_cores())
        n = int(lengths[0])
        with torch.no_grad():
            t0 = time.perf_counter()
            r = T.tts_infer(sd_t, tokens[:1, :n], lengths[:1], sid[:1], torch.randn(1, 2, n), None, noise_scale=0.667,
                            noise_scale_w=0.6)
            t_tts = time.perf_counter() - t0
        secs = int(r["y_lengths"][0]) * hop / 22050.0
        res["cpu_port_tts"] = {"audio_s_per_s": round(secs / t_tts, 2), "sample": "1 sentence", "threads": torch.get_num_threads()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=121)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cpu", action="store_true", help="also time the CPU oracle on one sentence (test infrastructure)")
    ap.add_argument("--precision", default="f16x3")
    a = ap.parse_args()
    print(json.dumps(measure(a.batch, a.tokens, a.iters, a.cpu, a.precision)))


if __name__ == "__main__":
    main()
