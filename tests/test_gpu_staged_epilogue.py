"""The staged epilogue of the TN = 128 tensor-core convs and the C = 128 conv pairs (tcconv_kernel<128, PAIR, 1, 2, true>,
OVC_OPT_STAGED_EPI): the MMA warpgroups stage each tile's conv result in shared memory and a fourth warpgroup runs the
epilogue from there.  Through the kernel harness (tests/kernelcheck/kc_staged.cu) every staged launch must be
bit-identical to the unstaged one, with the sentinel untouched outside the limits; and the library's audio must be
bit-identical with the option on and off."""
import ctypes as C
import importlib.util
import json
import math
import os
import tempfile

import pytest
import torch

from oracle import vc_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# the sentinel helpers, pass modes and single-conv cases of the fp64 kernel tests
G = _load("gpu_kernels_helpers", os.path.join(HERE, "test_gpu_kernels.py"))
KP = _load("kc_pair", os.path.join(HERE, "kernelcheck", "kc_pair.py"))


class StagedHarness(KP.PairHarness):
    """libovc_kc_staged.so: the kc_pair.py harness plus conv and pair launches with the staged epilogue on or off."""

    def __init__(self):
        super().__init__(os.path.join(HERE, "kernelcheck", "libovc_kc_staged.so"))
        self.lib.kc_conv_staged.argtypes = [C.POINTER(KP.kc.KcConv), C.c_int]
        self.lib.kc_pair_fused_staged.argtypes = [C.POINTER(KP.kc.KcConv), C.c_int]
        self.staged = 1

    def conv(self, x, w, bias, y, sync=True, **kw):
        a = self._args(x, w, bias, y, **kw)
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.kc_conv_staged(C.byref(a), self.staged))
        if sync:
            self.sync()

    def pair(self, x, w, bias, w2, bias2, y, sync=True, **kw):
        a = self._args(x, w, bias, y, w2=w2, bias2=bias2, Ntot=x.shape[2], **kw)
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.kc_pair_fused_staged(C.byref(a), self.staged))
        if sync:
            self.sync()


@pytest.fixture(scope="module")
def kc():
    h = StagedHarness()
    assert h.sm_count() > 0
    return h


def bits(t):
    return t.view(torch.int32)


# ------------------------------------------------------------------------------------------------ C = 128 pairs
def check_pair(kc, K, DIL, lens, tmax, seed):
    """Staged against unstaged: torch.equal in both pass modes, with and without MRF accumulate / scale, and the sentinel
    untouched outside each utterance's limit."""
    Cc = 128
    gen = torch.Generator().manual_seed(seed)
    B, L = len(lens), tmax + 3
    x = torch.randn(B, L, Cc, generator=gen)
    w1 = torch.randn(Cc, Cc, K, generator=gen) / math.sqrt(Cc * K)
    w2 = torch.randn(Cc, Cc, K, generator=gen) / math.sqrt(Cc * K)
    b1, b2 = 0.3 * torch.randn(Cc, generator=gen), 0.3 * torch.randn(Cc, generator=gen)
    old = torch.randn(B, L, Cc, generator=gen)
    valid = torch.arange(L)[None, :] < torch.tensor([min(n, tmax) for n in lens])[:, None]
    pw1, pw2 = kc.upload(kc.pack(w1.numpy(), DIL)[0]), kc.upload(kc.pack(w2.numpy(), 1)[0])
    xd, b1d, b2d = x.cuda(), b1.cuda(), b2.cuda()
    lens_t = torch.tensor(lens, dtype=torch.int64, device="cuda")
    for acc in (False, True):
        for p in G.PASSES:
            ys = {}
            for staged in (0, 1):
                kc.staged = staged
                y = G.sentinel_like((B, L, Cc))
                y = (torch.where(valid[..., None], old, y) if acc else y).cuda()
                kc.pair(xd, pw1, b1d, pw2, b2d, y, K=K, DIL=DIL, tmax=tmax, lens=lens_t, slope=0.1,
                        scale=1 / 3 if acc else 1.0, accumulate=acc, passes=p)
                ys[staged] = y.cpu()
            assert torch.equal(bits(ys[0]), bits(ys[1])), (K, DIL, acc, p)
            assert G.is_sent(ys[1][~valid]).all() and not G.is_sent(ys[1][valid]).any(), (K, DIL, acc, p)


@pytest.mark.parametrize("K", [3, 7, 11])
@pytest.mark.parametrize("DIL", [1, 3, 5])
def test_pair_staged_bit_identical(kc, K, DIL):
    """A ragged batch (lengths 0 and 1, around the tile of R = 128 - (k - 1) output steps, past tmax) with more tiles
    than CTAs, so every CTA stages several tiles in a row and the staging handshake wraps its phase."""
    assert kc.pair_fuses(128, K, DIL)
    R = 128 - (K - 1)
    tmax = 3 * R + 5
    lens = (0, 1, R - 1, R, R + 1, 2 * R, tmax, tmax + 40) * (2 * kc.sm_count() // 30 + 1)
    check_pair(kc, K, DIL, lens, tmax, 1000 + K * 10 + DIL)


# ------------------------------------------------------------------------------------------------ single TN = 128 convs
def staged_cases():
    cs = []
    H = 192
    cs.append(G.Case("rb_c256_k7_d3_res_acc", 256, 256, 7, 3, slope=0.1, tmax=700, lens=(700, 466, 1, 0, 129) * 12,
                     res=True, accumulate=True, scale=1 / 3))
    cs.append(G.Case("rb_c128_k3_d1_res", 128, 128, 3, 1, slope=0.1, tmax=600, lens=(600, 128, 127) * 20, res=True))
    cs.append(G.Case("wn_in_gate", H, 2 * H, 5, epi=1, tmax=900, lens=(900, 77, 1) * 20, bias_bs=1))
    for first in (0, 1):
        cs.append(G.Case(f"wn_rs_split192_first{first}", H, 2 * H, 1, epi=2, split=192, first=first, tmax=700,
                         lens=(700, 40) * 30))
    cs.append(G.Case("ups_s8", 512, 8 * 256, 3, slope=0.1, tmax=40, lens=(40, 39) * 4, ups=(8, 16)))
    cs.append(G.Case("rb_c256_k11_d5_grid_div3", 256, 256, 11, 5, slope=0.1, tmax=500, lens=(500, 333, 7) * 10,
                     res=True, accumulate=True, grid_div=3))
    return cs


CASES = {c.name: c for c in staged_cases()}


@pytest.mark.parametrize("name", list(CASES))
def test_conv_staged_bit_identical(kc, name):
    """epi 0 (residual, accumulate, scale), the WaveNet gate (epi 1) and res/skip (epi 2, first and not), a polyphase
    upsampler and a third of the SMs (grid_div = 3): staged equals unstaged bit for bit, y and s."""
    c = CASES[name]
    assert kc.tile_n(c.Ntot, c.Cin, c.K, c.DIL) == 128
    gen = torch.Generator().manual_seed(7)
    d = c.make(gen, False, kc)
    for p in G.PASSES:
        got = {}
        for staged in (0, 1):
            kc.staged = staged
            got[staged] = c.run(kc, d, p, False)
        for k in got[0]:
            assert torch.equal(bits(got[0][k]), bits(got[1][k])), (name, p, k)
        res = G.measure(c, got[1], c.reference(d, False))
        assert G.gate_ok(res, p), (name, p, res)


# ------------------------------------------------------------------------------------------------ the library
@pytest.mark.parametrize("precision", ["f16x3", "f16"])
def test_convert_batch_staged_option(precision):
    """convert_batch at 32 x 10 s: the audio is bit-identical with OVC_OPT_STAGED_EPI 0 and 1."""
    from openvoice_b200.api import ToneColorConverter

    with tempfile.TemporaryDirectory() as td:
        cfg = os.path.join(td, "config.json")
        with open(cfg, "w") as f:
            json.dump(O.DEFAULT_HPARAMS, f)
        conv = ToneColorConverter(cfg, device="cuda:0", enable_watermark=False)
    conv.model.load_state_dict(O.synthetic_state_dict(1234))
    nat = conv.model.native
    nat.set_precision(precision)
    B, L = 32, 10 * 22050
    gen = torch.Generator().manual_seed(0)
    wav = (torch.rand(B, L, generator=gen) - 0.5).cuda()
    wlen = torch.tensor([L - 997 * i for i in range(B)], dtype=torch.int64, device="cuda")
    g = 0.1 * torch.randn(B, 256, generator=gen).cuda()
    out = {}
    for staged in (0, 1):
        nat.set_option("staged_epi", staged)
        out[staged] = nat.convert_waveform(wav, wlen, g, g, tau=0.3, seed=3)[0].clone()
        torch.cuda.synchronize()
    nat.set_option("staged_epi", 1)
    assert torch.isfinite(out[1]).all()
    assert torch.equal(bits(out[0]), bits(out[1]))
