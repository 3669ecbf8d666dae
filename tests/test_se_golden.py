"""extract_se's golden vectors (oracle/make_golden_se.py: the real reference's ``ToneColorConverter.extract_se``)
against the CPU oracle, and the chunk planner of the batched extract_se path.

Tolerance: like tests/test_oracle_golden.py, the oracle must sit within 4x of the reference's own fp32 noise floor
(its fp64 twin), recorded per clip and per mean in tests/golden/REPORT_se.json."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import vc_oracle as O
from openvoice_b200.api import SE_CHUNK_FRAMES, plan_se_chunks

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def clips(seed, lengths):
    rng = np.random.default_rng(int(seed))
    return [(0.5 * (2 * rng.random(int(n), dtype=np.float32) - 1)).astype(np.float32) for n in lengths]


def oracle_se(sd, wav):
    with torch.no_grad():
        return O.reference_encoder(sd, O.spectrogram(torch.from_numpy(wav)[None]).transpose(1, 2))[0].numpy()


@pytest.mark.parametrize("tag", ["a", "b"])
def test_extract_se_golden_matches_oracle(tag, synthetic_sd):
    d = np.load(os.path.join(GOLD, "extract_se.npz"))
    with open(os.path.join(GOLD, "REPORT_se.json")) as f:
        floors = json.load(f)
    got = np.stack([oracle_se(synthetic_sd, w) for w in clips(d[f"{tag}_seed"], d[f"{tag}_lengths"])])
    for i, (g, ref) in enumerate(zip(got, d[f"{tag}_clip"])):
        assert np.abs(g - ref).max() <= 4 * floors[f"{tag}_clip_floor"][i], (tag, i)
    counts = [len(got)] if tag == "a" else [int(n) for n in d["b_counts"]]
    k = 0
    for j, n in enumerate(counts):
        mean = torch.stack([torch.from_numpy(r) for r in got[k: k + n]]).mean(0).numpy()
        assert np.abs(mean - d[f"{tag}_mean"][j]).max() <= 4 * floors[f"{tag}_mean_floor"][j], (tag, j)
        k += n


def check_plan(frames, budget):
    chunks = plan_se_chunks(frames, budget)
    flat = [i for c in chunks for i in c]
    assert sorted(flat) == list(range(len(frames)))                       # every clip exactly once
    for c in chunks:
        padded = len(c) * max(frames[i] for i in c)
        assert padded <= budget or len(c) == 1, (c, padded)
    return chunks


def test_plan_se_chunks():
    rng = np.random.default_rng(0)
    for budget in (1, 100, 1000, SE_CHUNK_FRAMES):
        frames = [int(v) for v in rng.integers(1, 900, size=57)]
        chunks = check_plan(frames, budget)
        order = [i for c in chunks for i in c]
        assert [frames[i] for i in order] == sorted(frames, reverse=True)  # longest first
    assert check_plan([5000, 10, 10], 1000) == [[0], [1, 2]]              # an over-budget clip runs alone
    assert check_plan([861] * 6, SE_CHUNK_FRAMES) == [list(range(6))]       # a 60 s reference is one pass
    assert plan_se_chunks([], 10) == []


def test_plan_restores_caller_order():
    """extract_se puts row j of chunk c back at the caller's index chunks[c][j]."""
    frames = [3, 9, 1, 9, 4, 7, 2]
    rows = [None] * len(frames)
    for c in plan_se_chunks(frames, 12):
        for i in c:
            rows[i] = frames[i]
    assert rows == frames
