"""Live text-to-cloned-voice sessions under staggered arrivals, measured against one stream per request.

Workload: S requests x K sentences x ~TOKENS tokens, synthetic checkpoints (oracle/tts_oracle.py, oracle/vc_oracle.py),
one GPU.  Time advances in ticks (one loop iteration each).  Request r arrives at tick r * STAGGER and its sentence j is
released at tick r * STAGGER + j * GAP.  Two arms run the same schedule, alternately, in the same process:
  sessions     one CloneSessions: a request opens when it arrives, says each sentence when it is released and ends
               after its last; every tick is one ``step()`` for all of them
  per_request  one ``clone_stream_batch(tts, [request])`` generator per request, started when its last sentence is
               released (it needs all of its text); every tick advances every live generator by one step
Per arm: time to first audio per request (from the start of its arrival tick; p50 / p95), audio seconds per wall
second over the whole schedule, and the tick time (median / p95).  Every tick ends in a device synchronise (each step
downloads its audio; the tick adds an explicit one), so the host clock is the measure.  Prints one JSON object with the
card's name and power limit (nvidia-smi, read-only).

    python tools/clone_sessions_bench.py [--sessions 16] [--sentences 3] [--tokens 60] [--stagger 2] [--gap 3]
                                         [--iters 3] [--precision f16x3]
"""
import argparse
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from clone_bench import build, card, workload  # noqa: E402

OPEN = ("speaker", "src_se", "tgt_se", "tau", "seed", "convert_seed", "speed")


def run_sessions(conv, tts, reqs, stagger, gap):
    from openvoice_b200.streaming import CloneSessions
    cs = CloneSessions(conv, tts)
    ids, first, arrive, ticks, samples = {}, {}, {}, [], 0
    t_start = time.perf_counter()
    k = 0
    while k == 0 or cs.sessions or len(ids) < len(reqs):
        t0 = time.perf_counter()
        for r, q in enumerate(reqs):
            a = r * stagger
            if k == a:
                ids[r], arrive[r] = cs.open(**{n: q[n] for n in OPEN}), t0
            if r in ids and ids[r] in cs.sessions:
                j, rem = divmod(k - a, gap)
                if rem == 0 and 0 <= j < len(q["ids"]):
                    cs.say(ids[r], ids=[q["ids"][j]])
                    if j == len(q["ids"]) - 1:
                        cs.end(ids[r])
        out = cs.step()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        back = {sid: r for r, sid in ids.items()}
        for sid, c in out.items():
            first.setdefault(back[sid], t1 - arrive[back[sid]])
            samples += len(c)
        ticks.append(t1 - t0)
        k += 1
    return first, samples, time.perf_counter() - t_start, ticks


def run_per_request(conv, tts, reqs, stagger, gap):
    live, first, arrive, ticks, samples = {}, {}, {}, [], 0
    t_start = time.perf_counter()
    k, started = 0, 0
    while k == 0 or live or started < len(reqs):
        t0 = time.perf_counter()
        for r, q in enumerate(reqs):
            a = r * stagger
            if k == a:
                arrive[r] = t0
            if k == a + (len(q["ids"]) - 1) * gap:      # all of its text is known
                live[r] = conv.clone_stream_batch(tts, [q])
                started += 1
        for r in list(live):
            try:
                _, c = next(live[r])
            except StopIteration:
                del live[r]
                continue
            samples += len(c)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        for r in live:
            first.setdefault(r, t1 - arrive[r])
        ticks.append(t1 - t0)
        k += 1
    return first, samples, time.perf_counter() - t_start, ticks


def summary(runs, sr):
    ttfa = np.concatenate([[v * 1e3 for v in f.values()] for f, _, _, _ in runs])
    ticks = np.concatenate([[v * 1e3 for v in t] for _, _, _, t in runs])
    aps = [s / sr / w for _, s, w, _ in runs]
    return {"ttfa_ms_p50": round(float(np.percentile(ttfa, 50)), 2), "ttfa_ms_p95": round(float(np.percentile(ttfa, 95)), 2),
            "audio_s_per_s": round(float(np.median(aps)), 2), "audio_s_per_s_all": [round(v, 2) for v in aps],
            "tick_ms_median": round(float(np.median(ticks)), 2), "tick_ms_p95": round(float(np.percentile(ticks, 95)), 2),
            "ticks": len(runs[0][3])}


def measure(n=16, k=3, tokens=60, stagger=2, gap=3, iters=3, precision="f16x3"):
    assert torch.cuda.is_available(), "clone_sessions_bench measures on the GPU"
    with tempfile.TemporaryDirectory() as tmp:
        tts, conv = build(tmp, precision)
    reqs = workload(n, k, tokens, 11)
    sr = float(conv.hps.data.sampling_rate)
    run_sessions(conv, tts, reqs, stagger, gap)            # warm-up: workspaces, pinned buffers, graph captures
    run_per_request(conv, tts, reqs, stagger, gap)
    a, b = [], []
    for _ in range(iters):                                  # alternating, so both arms see the same machine state
        a.append(run_sessions(conv, tts, reqs, stagger, gap))
        b.append(run_per_request(conv, tts, reqs, stagger, gap))
    return {"workload": f"{n} requests x {k} sentences x ~{tokens} tokens, arrivals every {stagger} ticks, sentences "
                        f"{gap} ticks apart, synthetic weights, {precision}",
            "card": card(), "sessions": summary(a, sr), "per_request": summary(b, sr), "iters": iters}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, default=16)
    ap.add_argument("--sentences", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=60)
    ap.add_argument("--stagger", type=int, default=2)
    ap.add_argument("--gap", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--precision", default="f16x3")
    a = ap.parse_args()
    import json
    print(json.dumps(measure(a.sessions, a.sentences, a.tokens, a.stagger, a.gap, a.iters, a.precision)))


if __name__ == "__main__":
    main()
