"""The fused ResBlock conv pair (tcconv_kernel<C, true>) where its weights do not stay resident in shared memory: the
C = 128 pairs and the k = 7 / 11 pairs of the C = 64 stage stream both convs' weights through the ring, the C = 32
k = 7 / 11 pairs hold them resident.  Each pair runs through the kernel harness (tests/kernelcheck/kc_pair.py) against
the fp64 composition of test_gpu_kernels.test_conv_pair, with the same gates, and bit-identical to the two single
launches it replaces; end to end, the library's audio is bit-identical with and without pair fusion."""
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


# the reference helpers, gates and sentinel of the single-conv and resident-pair tests
G = _load("gpu_kernels_helpers", os.path.join(HERE, "test_gpu_kernels.py"))


@pytest.fixture(scope="module")
def kc():
    h = _load("kc_pair", os.path.join(HERE, "kernelcheck", "kc_pair.py")).PairHarness()
    assert h.sm_count() > 0
    return h


def check_pair(kc, C, K, DIL, lens, tmax, seed, acc, ref_dev="cpu"):
    """One pair launch on a ragged batch: fp64 gates, sentinel outside the limits, and torch.equal with the two single
    launches, in both pass modes."""
    gen = torch.Generator().manual_seed(seed)
    slope = 0.1
    B, L = len(lens), tmax + 3
    x0 = torch.randn(B, L, C, generator=gen)
    w1c = torch.randn(C, C, K, generator=gen) / math.sqrt(C * K)
    w2c = torch.randn(C, C, K, generator=gen) / math.sqrt(C * K)
    b1c, b2c = 0.3 * torch.randn(C, generator=gen), 0.3 * torch.randn(C, generator=gen)
    old = torch.randn(B, L, C, generator=gen)
    scale = 1 / 3 if acc else 1.0
    m = G.rowmask(list(lens), B, L).to(ref_dev)
    x64, w1, w2 = x0.double().to(ref_dev), w1c.double().to(ref_dev), w2c.double().to(ref_dev)
    b1, b2, old64 = b1c.double().to(ref_dev), b2c.double().to(ref_dev), old.double().to(ref_dev)
    a1 = G.lrelu(x64, slope) * m
    t = (G.conv64(a1, w1, K, DIL) + b1) * m
    s1 = (G.conv64(a1.abs(), w1.abs(), K, DIL) + b1.abs()) * m
    a2 = G.lrelu(t, slope)
    y64 = G.conv64(a2, w2, K, 1) + b2 + x64
    S = G.conv64(a2.abs(), w2.abs(), K, 1) + G.conv64(s1, w2.abs(), K, 1) + b2.abs() + x64.abs()
    if acc:
        y64, S = y64 + old64, S + old64.abs()
    y64, S = (y64 * scale).cpu(), (S * scale).cpu()
    mb = m.bool()[..., 0].cpu()
    dev = "cuda"
    x = x0.to(dev)
    pw1, pw2 = kc.upload(kc.pack(w1c.numpy(), DIL)[0]), kc.upload(kc.pack(w2c.numpy(), 1)[0])
    gb1, gb2 = b1c.to(dev), b2c.to(dev)
    lens_t = torch.tensor(lens, dtype=torch.int64, device=dev)
    for p in G.PASSES:
        def fresh():
            y = G.sentinel_like((B, L, C))
            return (torch.where(mb[..., None], old, y) if acc else y).to(dev)
        y = fresh()
        kc.pair(x, pw1, gb1, pw2, gb2, y, K=K, DIL=DIL, tmax=tmax, lens=lens_t, slope=slope, scale=scale, accumulate=acc,
                passes=p)
        y = y.cpu()
        tb = G.sentinel_like((B, L, C)).to(dev)
        kc.conv(x, pw1, gb1, tb, Ntot=C, K=K, DIL=DIL, tmax=tmax, lens=lens_t, slope=slope, passes=p)
        y2 = fresh()
        kc.conv(tb, pw2, gb2, y2, Ntot=C, K=K, DIL=1, tmax=tmax, lens=lens_t, r=x, slope=slope, scale=scale,
                accumulate=acc, passes=p)
        assert torch.equal(y.view(torch.int32), y2.cpu().view(torch.int32)), (C, K, DIL, acc, p)
        assert G.is_sent(y[~mb]).all() and not G.is_sent(y[mb]).any()
        diff = (y[mb].double() - y64[mb]).abs()
        rms = float(diff.max() / y64[mb].pow(2).mean().sqrt())
        bound = float((diff / S[mb]).max())
        print(f"[kernels] pair_c{C}_k{K}_d{DIL} B={B} acc={int(acc)} passes={p} rms={rms:.3e} bound={bound:.3e}")
        assert rms <= G.GATES[p]["rms"] and bound <= G.GATES[p]["bound"], (rms, bound)


PAIRS = [(128, 3), (128, 7), (128, 11), (64, 7), (64, 11), (32, 7), (32, 11)]


@pytest.mark.parametrize("C,K", PAIRS)
@pytest.mark.parametrize("DIL", [1, 3, 5])
def test_conv_pair_streamed(kc, C, K, DIL):
    """Lengths around the pair's tile of R = 128 - (k - 1) output steps, as in test_conv_pair."""
    assert kc.pair_fuses(C, K, DIL)
    R = 128 - (K - 1)
    lens = (1, R - 1, R, R + 1, 2 * R, 2 * R + 1)
    for acc in (False, True):
        check_pair(kc, C, K, DIL, lens, 2 * R + 1, C * 100 + K * 10 + DIL + int(acc), acc)


@pytest.mark.parametrize("C,K,DIL", [(128, 7, 3), (64, 11, 5)])
def test_conv_pair_many_tiles_ring_wrap(kc, C, K, DIL):
    """B * n_tt far above the SM count: each CTA walks many tiles, and the ring (C 128, k 7: 2 x 56 slots, ring 12;
    C 64, k 11: 2 x 44 slots, ring 24) wraps from conv 1 to conv 2 to the next tile at a different phase every tile."""
    n_w, ring = 2 * (C // 16) * K, kc.ring_slots(C, True)
    assert n_w > ring and n_w % ring
    tmax = 1024
    lens = tuple(tmax - 37 * i for i in range(40))
    check_pair(kc, C, K, DIL, lens, tmax, 7 * C + K, acc=True, ref_dev="cuda")


def test_pair_fusion_bit_identical_end_to_end(native):
    """OVC_OPT_PAIR on a ragged batch of more than 512 frames (the sequential generator path, where the pair kernels
    run): every ResBlock pair of the C = 128 / 64 / 32 stages fused gives the same audio as two launches per pair, in
    both tensor-core modes."""
    spec, lengths, gs, gt, noise = O.synthetic_inputs(3, 861, 23, lengths=[861, 500, 37])
    nat = native.native
    outs, launches = {}, {}
    try:
        for mode in ("f16x3", "f16"):
            nat.set_precision(mode)
            for pair in (0, 1):
                nat.set_option("pair", pair)
                o, _, _ = native.voice_conversion(spec.cuda(), lengths.cuda(), gs.cuda(), gt.cuda(), tau=0.3,
                                                  noise=noise.cuda(), ragged=True)
                torch.cuda.synchronize()
                outs[(mode, pair)], launches[pair] = o.cpu(), nat.last_launch_count
            assert torch.isfinite(outs[(mode, 1)]).all()
            assert torch.equal(outs[(mode, 0)], outs[(mode, 1)]), mode
            # every one of the 27 pairs of the C <= 128 stages runs as one launch instead of two
            assert launches[0] - launches[1] == 27, launches
    finally:
        nat.set_option("pair", 1)
