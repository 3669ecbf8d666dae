"""CPU checks of the tensor-core conv's host side (openvoice_b200/csrc/ovc_tcpack.h), through the kernel harness
tests/kernelcheck/libovc_kc.so: the packed weight format against an independent numpy implementation of the documented
layout, the precision of the hi/lo split, the fit rules, the launch geometry and the polyphase form of the transposed
convs against torch's conv_transpose1d."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))


def load_kc():
    spec = importlib.util.spec_from_file_location("kc", os.path.join(HERE, "kernelcheck", "kc.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def kc():
    return load_kc().Harness()


def np_split(w):
    """hi = fp16(w), lo = fp16((w - hi) * 2^11), in numpy (round to nearest even, like __float2half_rn)."""
    w = np.asarray(w, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = w.astype(np.float16)
        lo = ((w - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
    return hi, lo


def np_pack(w, TN):
    """The documented layout [n_tile][Cin/16][K][column block][hi|lo][TN][8] of W[n][ci][tap]."""
    N, Cin, K = w.shape
    hi, lo = np_split(w)
    parts = np.stack([hi, lo])                                          # [part][N][Cin][K]
    parts = parts.reshape(2, N // TN, TN, Cin // 16, 2, 8, K)           # [part][nt][n][k16][kc][e][tap]
    return np.ascontiguousarray(parts.transpose(1, 3, 6, 4, 0, 2, 5)).reshape(-1).view(np.uint16)


def np_unpack(packed, N, Cin, K, TN):
    """Inverse of np_pack: (hi, lo) as float16 [N][Cin][K]."""
    p = packed.view(np.float16).reshape(N // TN, Cin // 16, K, 2, 2, TN, 8)   # [nt][k16][tap][kc][part][n][e]
    p = p.transpose(4, 0, 5, 1, 3, 6, 2).reshape(2, N, Cin, K)
    return p[0], p[1]


SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 65504.0, -65504.0, 65519.0, 65520.0, -7e4, 2.0 ** -24, -2.0 ** -25, 1e-8, 6.1e-5,
                    1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -12, 3.14159265, -1e-30], np.float32)


@pytest.mark.parametrize("N,Cin,K", [(384, 192, 5), (192, 192, 1), (576, 192, 1), (96, 64, 7), (256, 256, 11), (2048, 512, 3)])
def test_packed_bytes_match_the_documented_layout(kc, N, Cin, K):
    g = np.random.default_rng(N * 7 + K)
    w = (g.standard_normal((N, Cin, K)) * np.exp2(g.uniform(-30, 12, (N, Cin, K)))).astype(np.float32)
    w.reshape(-1)[: SPECIAL.size] = SPECIAL
    packed, TN = kc.pack(w)
    assert TN == (128 if N % 128 == 0 else 64 if N % 64 == 0 else 32)
    assert packed.size == N * Cin * K * 2
    ref = np_pack(w, TN)
    bad = np.flatnonzero(packed != ref)
    assert bad.size == 0, f"{bad.size} halfs differ, first at {bad[:8]}"


def test_split_reconstructs_22_bits(kc):
    g = np.random.default_rng(3)
    n = 32 * 32 * 64
    mag = np.exp2(g.uniform(-40, np.log2(65504.0), n))
    mag[:6] = [65503.9, 65504.0, 65519.99, 2.0 ** -14, 2.0 ** -24, 2.0 ** -36]
    w = (mag * g.choice([-1.0, 1.0], n)).astype(np.float32).reshape(32, 1024, 2)
    packed, TN = kc.pack(w)
    hi, lo = np_unpack(packed, 32, 1024, 2, TN)
    rec = hi.astype(np.float64) + lo.astype(np.float64) / 2048.0
    err = np.abs(rec - w.astype(np.float64))
    a = np.abs(w.astype(np.float64))
    assert np.isfinite(rec).all()
    normal = a >= 2.0 ** -14
    assert (err[normal] <= 2.0 ** -22 * a[normal]).all(), float((err[normal] / a[normal]).max())
    # below fp16's normal range the lo part runs out of exponent: absolute floor 2^-36 (half of lo's 2^-24 step / 2^11)
    assert (err <= 2.0 ** -22 * a + 2.0 ** -36).all()
    # at and above 65520 the hi part rounds to infinity: such a weight (or activation) does not survive the split
    big, _ = kc.pack(np.full((32, 32, 1), 65520.0, np.float32))
    h, l = np_unpack(big, 32, 32, 1, 32)
    assert np.isinf(h).all() and not np.isfinite(h.astype(np.float64) + l.astype(np.float64) / 2048).any()


def test_fit_rules(kc):
    assert kc.tile_n(384, 192, 5) == 128 and kc.tile_n(192, 192, 1) == 64 and kc.tile_n(96, 64, 3) == 32
    assert kc.tile_n(576, 192, 1) == 64 and kc.tile_n(2048, 512, 3) == 128
    assert kc.tile_n(256, 256, 11, 5) == 128                       # halo 25: the largest the A tile holds
    for args in [(80, 64, 3, 1), (64, 48, 3, 1), (64, 64, 11, 6), (64, 64, 13, 5), (64, 64, 53, 1), (0, 64, 3, 1),
                 (64, 0, 3, 1), (64, 64, 0, 1), (64, 64, 3, 0), (64, 64, 3, -1)]:
        assert kc.tile_n(*args) == 0, args
    with pytest.raises(ValueError):
        kc.pack(np.zeros((48, 64, 3), np.float32))
    assert kc.ring_slots(32) == 22 and kc.ring_slots(64) == 12 and kc.ring_slots(128) == 12
    assert kc.ring_slots(32, True) == 44 and kc.ring_slots(64, True) == 24
    for C, K, D in [(32, 3, 1), (32, 3, 5), (64, 3, 1), (64, 3, 3), (64, 3, 5), (32, 5, 1), (32, 5, 3), (32, 5, 5)]:
        assert kc.pair_fits(C, K, D), (C, K, D)
    assert not kc.pair_fits(64, 5, 1)          # 2 * 4 * 5 = 40 weight slots > 24
    assert not kc.pair_fits(32, 7, 1)          # k > 5
    assert not kc.pair_fits(128, 3, 1)         # TN 128 has no pair kernel
    assert not kc.pair_fits(32, 3, 1, D2=2)    # conv 2 has dilation 1
    assert not kc.pair_fits(32, 3, 1, K2=5)
    assert not kc.pair_fits(32, 3, 1, C2=64)
    assert not kc.pair_fits(32, 3, 1, N1=64)


def test_launch_geometry(kc):
    # single conv: 128-step tiles, the SMs split between the column tiles and the concurrent branches
    assert kc.grid(300, 2, 256, 128, 132, 1) == (3, 6, 6, 2)
    assert kc.grid(2048, 16, 256, 128, 132, 1) == (16, 256, 66, 2)
    assert kc.grid(2048, 16, 256, 128, 132, 3) == (16, 256, 22, 2)
    assert kc.grid(100, 1, 2048, 128, 132, 3) == (1, 1, 1, 16)
    assert kc.grid(100, 1, 4096, 128, 16, 1) == (1, 1, 1, 32)   # more column tiles than SMs: still one CTA per column
    # pair: R = 128 - (k - 1) output steps per tile, one CTA per SM
    assert kc.grid(126, 3, 32, 32, 132, pair=True, K=3) == (1, 3, 3, 1)
    assert kc.grid(127, 3, 32, 32, 132, pair=True, K=3) == (2, 6, 6, 1)
    assert kc.grid(124 * 200, 1, 32, 32, 132, pair=True, K=5) == (200, 200, 132, 1)


@pytest.mark.parametrize("s,kk", [(8, 16), (2, 4)])
def test_polyphase_form_equals_conv_transpose(kc, s, kk):
    g = torch.Generator().manual_seed(s)
    cin, cout, B, L = 64, 32, 2, 37
    raw = torch.randn(cin, cout, kk, generator=g, dtype=torch.float64).float()
    x = torch.randn(B, cin, L, generator=g, dtype=torch.float64)
    ref = F.conv_transpose1d(x, raw.double(), stride=s, padding=(kk - s) // 2)          # [B][cout][L*s]
    assert ref.shape[2] == L * s
    wp = kc.ups_weights(raw.numpy(), s).astype(np.float64)                             # [s*cout][cin][3]
    xcl = np.pad(x.transpose(1, 2).numpy(), ((0, 0), (1, 1), (0, 0)))                  # channels-last, zero halo
    y = sum(np.einsum("btc,rc->btr", xcl[:, tap:tap + L], wp[:, :, tap]) for tap in range(3))   # [B][L][s*cout]
    # row = ph * cout + co of input step n is output step s*n + ph of channel co: [B][L][s][cout] = [B][L*s][cout]
    got = y.reshape(B, L * s, cout).transpose(0, 2, 1)
    np.testing.assert_allclose(got, ref.numpy(), rtol=0, atol=1e-12 * float(ref.abs().max()))
