"""CPU checks of the fp32 CUDA-core conv's host side (openvoice_b200/csrc/ovc_convpack.h), through the kernel harness
tests/kernelcheck/libovc_kc_f32.so: the packed weight layout against an independent numpy implementation, the paired-row
interleave of the gate / projection epilogues, and the polyphase form of the transposed convs against torch's
conv_transpose1d."""
import importlib.util
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load_kcf():
    spec = importlib.util.spec_from_file_location("kc_f32", os.path.join(HERE, "kernelcheck", "kc_f32.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def kcf():
    return load_kcf().Harness()


def np_pack(w, CO_T, CI_CH):
    """The documented layout [row_tile][ci_pad][K][CO_T] of W[row][ci][k], zero past cin."""
    rows, cin, K = w.shape
    cin_pad = -(-cin // CI_CH) * CI_CH
    wp = np.zeros((rows, cin_pad, K), np.float32)
    wp[:, :cin] = w
    return np.ascontiguousarray(wp.reshape(rows // CO_T, CO_T, cin_pad, K).transpose(0, 2, 3, 1)).reshape(-1)


def test_variant_table_matches_the_header(kcf):
    src = open(os.path.join(ROOT, "openvoice_b200", "csrc", "ovc_variants.h")).read()
    rows = re.findall(r"X\((\w+), (\d+), (\d+), (\d+), (\d+), (\d+), EPI_(\w+), (\d+), (\d+)\)", src)
    assert len(rows) == len(kcf.variants) == 37
    for name, K, D, WM, WN, CI, epi, NG, XA in rows:
        v = kcf.variants[name]
        assert (v.K, v.DIL, v.CO_T, v.T_T, v.CI_CH, v.epi, v.NG, v.XALIGN) == \
            (int(K), int(D), 32 * int(WM), 64 * int(WN), int(CI), epi, int(NG), int(XA)), name


def test_no_fast_math():
    """The accuracy gates of tests/test_gpu_conv_f32.py rest on IEEE fp32 (no flush to zero, tanhf / expf / division
    within their documented ulp bounds)."""
    mk = open(os.path.join(ROOT, "openvoice_b200", "csrc", "Makefile")).read()
    flags = re.search(r"^NVFLAGS :=(.*)$", mk, re.M).group(1)
    for bad in ("fast-math", "fast_math", "ftz", "prec-div=false", "prec-sqrt=false"):
        assert bad not in flags, bad


@pytest.mark.parametrize("name,rows,cin", [("ENC_PRE", 192, 513), ("FLOW_PRE", 192, 96), ("WN_IN", 384, 192),
                                           ("A_K11D5", 256, 256), ("A_K7D1", 512, 192), ("B_K7D3", 64, 64),
                                           ("C_K11D1", 32, 32), ("FLOW_POST", 96, 192), ("TXT_K3D1", 192, 768),
                                           ("A_K3D1", 128, 13)])
def test_packed_floats_match_the_documented_layout(kcf, name, rows, cin):
    v = kcf.variants[name]
    g = np.random.default_rng(rows * 31 + cin)
    w = g.standard_normal((rows, cin, v.K)).astype(np.float32)
    packed = kcf.pack(name, w)
    cin_pad = -(-cin // v.CI_CH) * v.CI_CH
    assert packed.size == rows * cin_pad * v.K
    ref = np_pack(w, v.CO_T, v.CI_CH)
    bad = np.flatnonzero(packed.view(np.uint32) != ref.view(np.uint32))
    assert bad.size == 0, f"{bad.size} floats differ, first at {bad[:8]}"
    if cin_pad > cin:      # the padding channels of the last chunk are zero (+0.0) in every row tile and tap
        pad = packed.reshape(rows // v.CO_T, cin_pad, v.K, v.CO_T)[:, cin:]
        assert (pad.view(np.uint32) == 0).all()


def test_paired_row_interleave(kcf):
    for half in (192, 96, 64):
        perm = [kcf.paired_row(p, half) for p in range(2 * half)]
        assert sorted(perm) == list(range(2 * half)), half
        for p in range(2 * half):
            q, r = divmod(p, 8)
            assert perm[p] == (4 * q + r if r < 4 else half + 4 * q + r - 4)
    # the packer applies it: packed row p of a paired conv carries natural row paired_row(p, rows / 2)
    w = np.arange(384 * 3 * 1, dtype=np.float32).reshape(384, 3, 1)
    got = kcf.pack("ENC_PROJ", w, paired=True).reshape(384 // 64, 8, 1, 64)[:, 0, 0, :].reshape(-1)
    assert (got == w[[kcf.paired_row(p, 192) for p in range(384)], 0, 0]).all()


@pytest.mark.parametrize("s,kk", [(8, 16), (2, 4)])
def test_polyphase_map_equals_conv_transpose(kcf, s, kk):
    """out[co, s*n + ph] = sum_tap x[n - 1 + tap] . W[:, co, kidx(row = co*s + ph, tap)], with the (row, tap) pairs the
    kernel skips (tap_is_zero) zeroed: equal to conv_transpose1d, and every skipped pair holds no weight."""
    g = torch.Generator().manual_seed(s)
    cin, cout, B, L = 24, 16, 2, 37
    raw = torch.randn(cin, cout, kk, generator=g, dtype=torch.float64)
    x = torch.randn(B, cin, L, generator=g, dtype=torch.float64)
    ref = F.conv_transpose1d(x, raw, stride=s, padding=(kk - s) // 2)          # [B][cout][L*s]
    w3 = torch.zeros(cout * s, cin, 3, dtype=torch.float64)
    for row in range(cout * s):
        for tap in range(3):
            kidx = kcf.ups_kidx(s, kk, row, tap)
            if kcf.tap_is_zero(s, tap, row % 8):
                assert kidx < 0, (row, tap)
                continue
            if kidx >= 0:
                w3[row, :, tap] = raw[:, row // s, kidx]
    y = F.conv1d(x, w3, padding=1)                                              # [B][cout*s][L], row = co*s + ph
    got = y.reshape(B, cout, s, L).permute(0, 1, 3, 2).reshape(B, cout, L * s)
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-12 * float(ref.abs().max()))
    # the packer writes the same map
    name = "UPS8_A" if s == 8 else "UPS2_A"
    v = kcf.variants[name]
    cin_p, cout_p = 16, v.CO_T // s * 2
    rawp = np.random.default_rng(s).standard_normal((cin_p, cout_p, kk)).astype(np.float32)
    packed = kcf.pack_ups(name, rawp, s)
    w3p = np.zeros((cout_p * s, cin_p, 3), np.float32)
    for row in range(cout_p * s):
        for tap in range(3):
            kidx = kcf.ups_kidx(s, kk, row, tap)
            if kidx >= 0:
                w3p[row, :, tap] = rawp[:, row // s, kidx]
    assert (packed == np_pack(w3p, v.CO_T, v.CI_CH)).all()
