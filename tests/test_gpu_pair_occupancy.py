"""The fused ResBlock conv pairs of the C = 32 / 64 stages at two CTAs per SM (tcconv_kernel<C, true, 2, NAB>, picked by
tc_pair_occ in ovc_tcpack.h).  Each such instantiation runs through the kernel harness (tests/kernelcheck/kc_pair_occ.py)
on ragged batches and must be bit-identical to the one-CTA-per-SM kernel, with nothing written outside the limits;
the device must fit two of its CTAs per SM; and the library's audio is bit-identical with OVC_OPT_PAIR_OCC on and off."""
import importlib.util
import math
import os

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


# the sentinel helpers and pass modes of the single-conv tests
G = _load("gpu_kernels_helpers", os.path.join(HERE, "test_gpu_kernels.py"))


@pytest.fixture(scope="module")
def kc():
    h = _load("kc_pair_occ", os.path.join(HERE, "kernelcheck", "kc_pair_occ.py")).PairOccHarness()
    assert h.sm_count() > 0
    return h


# every generator pair (k 3 / 7 / 11, dilation 1 / 3 / 5) of the C = 32 / 64 stages that runs two CTAs per SM
OCC2_PAIRS = [(32, 3), (32, 7), (64, 7), (64, 11)]


def check_occ(kc, C, K, DIL, lens, tmax, seed):
    """One pair launch at two CTAs per SM against the one-CTA launch: torch.equal in both pass modes, with and without
    MRF accumulate / scale, and the sentinel untouched outside each utterance's limit."""
    gen = torch.Generator().manual_seed(seed)
    B, L = len(lens), tmax + 3
    x = torch.randn(B, L, C, generator=gen)
    w1 = torch.randn(C, C, K, generator=gen) / math.sqrt(C * K)
    w2 = torch.randn(C, C, K, generator=gen) / math.sqrt(C * K)
    b1, b2 = 0.3 * torch.randn(C, generator=gen), 0.3 * torch.randn(C, generator=gen)
    old = torch.randn(B, L, C, generator=gen)
    valid = torch.arange(L)[None, :] < torch.tensor([min(n, tmax) for n in lens])[:, None]
    pw1, pw2 = kc.upload(kc.pack(w1.numpy(), DIL)[0]), kc.upload(kc.pack(w2.numpy(), 1)[0])
    xd, b1d, b2d = x.cuda(), b1.cuda(), b2.cuda()
    lens_t = torch.tensor(lens, dtype=torch.int64, device="cuda")
    for acc in (False, True):
        for p in G.PASSES:
            ys = {}
            for occ in (1, 2):
                y = G.sentinel_like((B, L, C))
                y = (torch.where(valid[..., None], old, y) if acc else y).cuda()
                kc.pair_at(occ, xd, pw1, b1d, pw2, b2d, y, K=K, DIL=DIL, tmax=tmax, lens=lens_t, slope=0.1,
                           scale=1 / 3 if acc else 1.0, accumulate=acc, passes=p)
                ys[occ] = y.cpu()
            assert torch.equal(ys[1].view(torch.int32), ys[2].view(torch.int32)), (C, K, DIL, acc, p)
            assert G.is_sent(ys[2][~valid]).all() and not G.is_sent(ys[2][valid]).any(), (C, K, DIL, acc, p)


@pytest.mark.parametrize("C,K", OCC2_PAIRS)
@pytest.mark.parametrize("DIL", [1, 3, 5])
def test_pair_two_ctas_bit_identical(kc, C, K, DIL):
    """Lengths 0 and 1, around the tile of R = 128 - (k - 1) output steps, and past tmax."""
    cfg = kc.pair_occ(C, K, DIL)
    assert cfg["occ"] == 2, cfg
    R = 128 - (K - 1)
    tmax = 2 * R + 1
    lens = (0, 1, R - 1, R, R + 1, 2 * R, tmax, tmax + 40)
    check_occ(kc, C, K, DIL, lens, tmax, C * 100 + K * 10 + DIL)


@pytest.mark.parametrize("C,K,DIL", [(32, 3, 5), (32, 7, 3), (64, 11, 5)])
def test_pair_two_ctas_many_tiles(kc, C, K, DIL):
    """B * n_tt far above twice the SM count: each CTA walks many tiles, the operand buffers and (C = 64) the streamed
    ring wrap at a different phase every tile, next to a second CTA on the same SM."""
    tmax = 1024
    lens = tuple(tmax - 37 * i for i in range(40))
    check_occ(kc, C, K, DIL, lens, tmax, 7 * C + K)


def test_pair_two_ctas_fit(kc):
    """The device fits two CTAs per SM of every two-CTA config tc_pair_occ picks for a generator pair."""
    configs = {(C, kc.pair_occ(C, K, 1)["nabuf"]) for C, K in OCC2_PAIRS}
    assert configs == {(32, 2), (32, 1), (64, 1)}
    for C, nabuf in sorted(configs):
        assert kc.pair_occupancy(C, 2, nabuf) == 2, (C, nabuf)


def test_pair_occ_bit_identical_end_to_end(native):
    """OVC_OPT_PAIR_OCC on a ragged batch of more than 512 frames (the sequential generator path, where the pair
    kernels run): the same audio with two CTAs per SM as with one, in both tensor-core modes."""
    spec, lengths, gs, gt, noise = O.synthetic_inputs(3, 861, 23, lengths=[861, 500, 37])
    nat = native.native
    try:
        for mode in ("f16x3", "f16"):
            nat.set_precision(mode)
            outs = {}
            for occ in (0, 1):
                nat.set_option("pair_occ", occ)
                o, _, _ = native.voice_conversion(spec.cuda(), lengths.cuda(), gs.cuda(), gt.cuda(), tau=0.3,
                                                  noise=noise.cuda(), ragged=True)
                torch.cuda.synchronize()
                outs[occ] = o.cpu()
            assert torch.isfinite(outs[1]).all()
            assert torch.equal(outs[0], outs[1]), mode
    finally:
        nat.set_option("pair_occ", 1)
