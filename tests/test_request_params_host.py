"""CPU tests of per-request sampling parameters (include/ovc.h: ovc_item_params): the ctypes mirror against the C
layout, the argument checks that run before anything is launched, and seeds travelling with their utterance through
the LPT sharding under gloo (world size 2)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_PROBE = r"""
#include <cstddef>
#include <cstdio>
#include "ovc.h"
int main() {
  std::printf("%zu", sizeof(ovc_item_params));
#define F(n) std::printf(" %s %zu", #n, offsetof(ovc_item_params, n));
  F(seed) F(stream) F(frame0) F(tau) F(noise_scale) F(noise_scale_w) F(length_scale) F(sdp_ratio)
  std::printf("\n");
  return 0;
}
"""


def test_item_params_layout_matches_the_header(tmp_path):
    from openvoice_b200 import _native
    src = tmp_path / "probe.cpp"
    src.write_text(_PROBE)
    exe = tmp_path / "probe"
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert int(out[0]) == C.sizeof(_native.ItemParams)
    got = dict(zip(out[1::2], (int(v) for v in out[2::2])))
    assert list(got) == [f[0] for f in _native.ItemParams._fields_]
    for name, off in got.items():
        assert getattr(_native.ItemParams, name).offset == off, name
    assert set(_native.ITEM_FIELDS) == set(got)


def test_check_seeds_and_per_item_values():
    from openvoice_b200.api import check_per_item, check_seeds, seed_array
    assert check_seeds(None, 3) is None
    assert check_seeds([0, 2 ** 64 - 1, np.uint64(5)], 3) == [0, 2 ** 64 - 1, 5]
    for bad in ([1, 2], [-1, 0, 0], [2 ** 64, 0, 0], [1.5, 0, 0], [True, 0, 0], ["1", 0, 0]):
        with pytest.raises(ValueError):
            check_seeds(bad, 3)
    assert check_per_item(0.3, 4, "tau") == (0.3, None)
    assert check_per_item([0.0, 0.3, 1.0], 3, "tau") == (0.0, [0.0, 0.3, 1.0])
    for bad in ([0.3, 0.3], [0.3, float("nan"), 0.1], [float("inf"), 0.0, 0.0]):
        with pytest.raises(ValueError):
            check_per_item(bad, 3, "tau")
    with pytest.raises(ValueError):
        check_per_item([1.0, 0.0], 2, "length_scale", positive=True)
    a = seed_array([0, 1, 2 ** 63, 2 ** 64 - 1])
    assert a.dtype == np.int64 and a.view(np.uint64).tolist() == [0, 1, 2 ** 63, 2 ** 64 - 1]


def _converter(hps_dict):
    """A ToneColorConverter that never touched a device: every refusal below must happen before one is needed."""
    from openvoice_b200.api import ToneColorConverter
    from openvoice_b200.utils import HParams
    conv = ToneColorConverter.__new__(ToneColorConverter)
    conv.hps = HParams(**hps_dict)
    conv.device = "cuda:0"
    conv.watermark_model = None
    return conv


def test_conversion_refusals_before_any_launch():
    from oracle import vc_oracle as O
    conv = _converter(O.DEFAULT_HPARAMS)
    w = [np.zeros(22050, np.float32), np.zeros(30000, np.float32)]
    se = torch.zeros(1, 256, 1)
    cases = [
        lambda: conv.convert_batch(w, se, se, seeds=[1]),                               # length
        lambda: conv.convert_batch(w, se, se, seeds=[1, -2]),                           # range
        lambda: conv.convert_batch(w, se, se, seeds=[1, 2 ** 64]),
        lambda: conv.convert_batch(w, se, se, tau=[0.3]),                               # length
        lambda: conv.convert_batch(w, se, se, tau=[0.3, float("nan")]),                 # non-finite
        lambda: conv.convert_batch(w, se, se, seeds=[1, 2], noise=[None, None]),        # noise and seeds
        lambda: conv.convert(w[0], se, se, seed=3, noise=torch.zeros(1, 192, 86)),
        lambda: conv.convert_batch_device(w, se, se, seeds=[1, 2, 3]),
        lambda: conv.convert_concurrent(w, se, se, tau=[0.1, 0.2, 0.3]),
        lambda: conv.convert_long(w[0], se, se, seed=3, noise=torch.zeros(192, 86)),
        lambda: conv.convert_long(w[0], se, se, seed=-1),
    ]
    for i, case in enumerate(cases):
        with pytest.raises(ValueError):
            case()
        assert "_dev_cache" not in conv.__dict__ and "_pin_cache" not in conv.__dict__, i


def test_streaming_request_seed_refusals():
    from oracle import vc_oracle as O
    from openvoice_b200.streaming import StreamingConverter
    conv = _converter(O.DEFAULT_HPARAMS)
    se = torch.zeros(1, 256, 1)
    with pytest.raises(ValueError):
        StreamingConverter(conv, se, se, request_seed=1, seed=2)
    with pytest.raises(ValueError):
        StreamingConverter(conv, se, se, request_seed=1, noise_fn=lambda a, b: torch.zeros(192, b - a))
    with pytest.raises(ValueError):
        StreamingConverter(conv, se, se, request_seed=2 ** 64)


def test_synthesizer_refusals_before_any_launch():
    """NativeSynthesizer.voice_conversion / infer check their per-item arguments before touching the device."""
    from openvoice_b200.api import NativeSynthesizer
    m = NativeSynthesizer.__new__(NativeSynthesizer)
    m.device = torch.device("cuda", 0)
    y = torch.zeros(2, 513, 40)
    lens = torch.tensor([40, 30])
    g = torch.zeros(1, 256)
    for kw in (dict(seeds=[1]), dict(seeds=[1, 2], noise=torch.zeros(2, 192, 40)), dict(taus=[0.1, float("inf")]),
               dict(seeds=[1, 2], frame0=[0, 2 ** 32 - 39]), dict(frame0=[0, -1]), dict(seeds=[1, 2], streams=[0])):
        with pytest.raises(ValueError):
            m.voice_conversion(y, lens, g, g, **kw)


_WORKER = r"""
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch, torch.distributed as dist
from openvoice_b200.distributed import convert_sharded, convert_sharded_async, lpt_shard
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
rng = np.random.default_rng(0)
audios = [rng.standard_normal(n).astype(np.float32) for n in (700, 50, 300, 1200, 256, 999, 10, 512)]
seeds = [11, 2 ** 64 - 1, 7, 0, 123456789, 3, 99, 2 ** 40]
taus = [0.0, 0.3, 1.0, 0.3, 0.0, 1.0, 0.3, 0.5]
mine = lpt_shard([len(a) for a in audios], world)[rank]
def mark(a, s, t):       # stands in for the conversion of utterance a with key s and tau t
    n = 256 * (len(a) // 256)
    return (a[:n] * t + (s % 1000003)).astype(np.float32)
def fake_convert(batch, src, tgt, tau=0.3, seeds=None):
    assert len(batch) == len(seeds) == len(tau) == len(mine)
    return [mark(a, s, t) for a, s, t in zip(batch, seeds, tau)]
out = convert_sharded(fake_convert, audios, None, None, tau=taus, seeds=seeds)
if rank == 0:
    for a, s, t, o in zip(audios, seeds, taus, out):
        assert np.array_equal(o, mark(a, s, t))
else:
    assert out is None
class FakeConverter:
    class hps:
        class data:
            hop_length = 256
    device = torch.device("cpu")
    def convert_batch_device(self, batch, src, tgt, tau=0.3, slot=0, seeds=None):
        n = [256 * (len(a) // 256) for a in batch]
        o = torch.zeros(len(batch), max(n))
        for j, a in enumerate(batch):
            o[j, : n[j]] = torch.from_numpy(mark(a, seeds[j], tau[j]))
        return o, n
long = [i for i, a in enumerate(audios) if len(a) >= 256]
res = convert_sharded_async(FakeConverter(), [audios[i] for i in long], None, None, tau=[taus[i] for i in long],
                            seeds=[seeds[i] for i in long]).result()
if rank == 0:
    for i, o in zip(long, res):
        assert np.array_equal(o, mark(audios[i], seeds[i], taus[i]))
dist.barrier()
dist.destroy_process_group()
sys.stdout.write(f"worker-{rank}-ok\n"); sys.stdout.flush()
"""


def test_seeds_follow_their_utterance_through_lpt_sharding_gloo_world2(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script), ROOT],
                       capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "worker-0-ok" in r.stdout and "worker-1-ok" in r.stdout
