"""Generate tests/golden/extract_se.npz by running the REAL reference ``ToneColorConverter.extract_se``.

Run on a machine that has the reference checked out:
``OPENVOICE_REFERENCE=<path to the checkout> python oracle/make_golden_se.py``.  Same method as ``make_golden.py``
(whose reference import and converter construction this reuses): the clips are seeded synthetic waveforms at the
model sampling rate, written as .npy files that the librosa stub loads, so ``extract_se`` (openvoice/api.py:114-139)
runs its own spectrogram_torch and ReferenceEncoder on the seeded synthetic checkpoint.  Two sets:

* ``a_*``: clip lengths that stress the stride-2 chain of the encoder (3 frames + 5 samples, 64, 65 frames + 100
  samples, 140 frames, ...); the solo embedding of every clip and the mean over all of them.
* ``b_*``: a small multi-speaker enrolment (3 speakers of 1, 2 and 4 clips) for ``extract_se_batch``; the solo
  embedding of every clip and each speaker's mean.

Clip i of a set is ``0.5 * (2 * rng.random(L_i, dtype=float32) - 1)`` drawn in order from
``np.random.default_rng(seed)``.  REPORT_se.json records, per clip and per mean, how far the CPU oracle
(``vc_oracle.reference_encoder(spectrogram(...))``) is from the reference and the reference's own fp32 noise floor
(its fp64 twin through the oracle).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True

import vc_oracle as O  # noqa: E402
from make_golden import build_reference_converter, import_reference, maxdiff  # noqa: E402

HOP = 256
SEED_A = 6000
LENGTHS_A = [3 * HOP + 5, 64 * HOP, 65 * HOP + 100, 140 * HOP, 7 * HOP + 200, 33 * HOP + 17, 129 * HOP + 1]
SEED_B = 6001
COUNTS_B = [1, 2, 4]
LENGTHS_B = [20000, 5 * HOP + 131, 12000, 30000, 4 * HOP, 100 * HOP + 3, 2500]


def clips(seed, lengths):
    rng = np.random.default_rng(seed)
    return [(0.5 * (2 * rng.random(n, dtype=np.float32) - 1)).astype(np.float32) for n in lengths]


def oracle_se(sd, wav, dtype=torch.float32):
    w = torch.from_numpy(wav)[None].to(dtype)
    with torch.no_grad():
        return O.reference_encoder(sd, O.spectrogram(w).transpose(1, 2))[0]


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    api, _, _ = import_reference()
    sd = O.synthetic_state_dict(1234)
    sd64 = {k: v.double() for k, v in sd.items()}
    conv = build_reference_converter(api, sd, zero_g=False)
    outdir = os.path.join(ROOT, "tests", "golden")
    report = {}
    out = dict(a_seed=np.array(SEED_A), a_lengths=np.array(LENGTHS_A), b_seed=np.array(SEED_B),
               b_lengths=np.array(LENGTHS_B), b_counts=np.array(COUNTS_B))
    with tempfile.TemporaryDirectory() as td:
        for tag, seed, lengths in (("a", SEED_A, LENGTHS_A), ("b", SEED_B, LENGTHS_B)):
            paths = []
            for i, w in enumerate(clips(seed, lengths)):
                p = os.path.join(td, f"{tag}{i}.npy")
                np.save(p, w)
                paths.append(p)
            solo = torch.stack([conv.extract_se([p])[0, :, 0] for p in paths])          # [k, gin]
            ws = clips(seed, lengths)
            orc = torch.stack([oracle_se(sd, w) for w in ws])
            o64 = torch.stack([oracle_se(sd64, w, torch.float64) for w in ws])
            report[f"{tag}_clip"] = [maxdiff(solo[i], orc[i]) for i in range(len(paths))]
            report[f"{tag}_clip_floor"] = [maxdiff(solo[i].double(), o64[i]) for i in range(len(paths))]
            out[f"{tag}_clip"] = solo.numpy()
            if tag == "a":
                groups = [paths]
            else:
                groups, k = [], 0
                for n in COUNTS_B:
                    groups.append(paths[k: k + n])
                    k += n
            means = torch.stack([conv.extract_se(g)[0, :, 0] for g in groups])          # the reference's own mean
            report[f"{tag}_mean"], report[f"{tag}_mean_floor"], k = [], [], 0
            for j, g in enumerate(groups):
                report[f"{tag}_mean"].append(maxdiff(means[j], orc[k: k + len(g)].mean(0)))
                report[f"{tag}_mean_floor"].append(maxdiff(means[j].double(), o64[k: k + len(g)].mean(0)))
                k += len(g)
            out[f"{tag}_mean"] = means.numpy()
    np.savez_compressed(os.path.join(outdir, "extract_se.npz"), **out)
    with open(os.path.join(outdir, "REPORT_se.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
