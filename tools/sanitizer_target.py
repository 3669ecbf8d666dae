#!/usr/bin/env python
"""One small conversion that exercises every tensor-core kernel for compute-sanitizer: the sequential schedule (fused conv
pairs, tcconv_kernel<C, true>) and the concurrent-branch schedule of small calls, checked against the oracle."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from oracle import vc_oracle as O
from openvoice_b200.api import NativeSynthesizer
from openvoice_b200.utils import HParams

sd = O.synthetic_state_dict(1234)
m = NativeSynthesizer(HParams(**O.DEFAULT_HPARAMS), "cuda:0")
m.load_state_dict(sd)
spec, lengths, gs, gt, noise = O.synthetic_inputs(2, 40, 3, lengths=[40, 23])
with torch.no_grad():
    ro, _, _ = O.voice_conversion_ragged(sd, spec, lengths, gs, gt, noise, 0.3)
for branches in (0, 1):
    m.native.set_option("branches", branches)
    o, _, _ = m.voice_conversion(spec.cuda(), lengths.cuda(), gs.cuda(), gt.cuda(), tau=0.3, noise=noise.cuda(), ragged=True)
    torch.cuda.synchronize()
    err = float((o.cpu() - ro).abs().max() / ro.pow(2).mean().sqrt())
    print(f"branches={branches}: {m.native.last_launch_count} launches, o_hat max|d|/rms = {err:.3e}")
    assert err < 1e-4
print("sanitizer target ok")
