"""CPU check of the polyphase resampler arithmetic (openvoice_b200/csrc/ovc_resample.h).

The resample kernel is one thread per output sample around ``output_at``; here the SAME header is compiled with g++
(tests/hostcheck/resample_host.cpp) and its plan, filter bank, span and per-output functions are compared with
``scipy.signal.resample_poly`` at its defaults (Kaiser beta 5, constant padding), the arithmetic the library pins."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.signal import firwin, resample_poly

HERE = os.path.dirname(os.path.abspath(__file__))

PAIRS = [(8000, 22050), (16000, 22050), (24000, 22050), (32000, 22050), (44100, 22050), (48000, 22050),
         (96000, 22050), (192000, 22050), (22050, 44100), (22050, 48000)]
LL = C.c_longlong


@pytest.fixture(scope="module")
def rs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostcheck") / "resample_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "hostcheck", "resample_host.cpp")])
    lib = C.CDLL(so)
    lib.rs_n_out.restype = LL
    lib.rs_n_ready.restype = LL
    return lib


def plan(rs, a, b):
    o = (LL * 7)()
    assert rs.rs_plan(LL(a), LL(b), o) == 0
    return dict(zip(("up", "down", "taps", "K", "half", "pre_pad", "pre_remove"), list(o)))


def filt(rs, a, b):
    p = plan(rs, a, b)
    h = np.empty(p["taps"])
    rs.rs_filter(LL(a), LL(b), h.ctypes.data_as(C.c_void_p))
    return h


def run(rs, a, b, x):
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.empty(rs.rs_n_out(LL(a), LL(b), LL(len(x))))
    rs.rs_run(LL(a), LL(b), x.ctypes.data_as(C.c_void_p), LL(len(x)), y.ctypes.data_as(C.c_void_p))
    return y


@pytest.mark.parametrize("a,b", PAIRS)
def test_plan_and_output_length(rs, a, b):
    p = plan(rs, a, b)
    g = np.gcd(a, b)
    assert (p["up"], p["down"]) == (b // g, a // g)
    M = max(p["up"], p["down"])
    assert p["taps"] == 20 * M + 1 and p["K"] == -(-p["taps"] // p["up"])
    h = firwin(p["taps"], 1.0 / M, window=("kaiser", 5.0))    # passed as the window: only the length logic runs per L
    for L in range(1, 2001):
        assert rs.rs_n_out(LL(a), LL(b), LL(L)) == len(resample_poly(np.zeros(L), p["up"], p["down"], window=h)), L


@pytest.mark.parametrize("a,b", PAIRS)
def test_bank_matches_firwin(rs, a, b):
    p = plan(rs, a, b)
    up, K, N = p["up"], p["K"], p["taps"]
    ref = firwin(N, 1.0 / max(up, p["down"]), window=("kaiser", 5.0)) * up
    h = filt(rs, a, b)
    assert np.abs(h - ref).max() <= 1e-15 * np.abs(ref).max()
    bank = np.empty(up * K)
    rs.rs_bank(LL(a), LL(b), bank.ctypes.data_as(C.c_void_p))
    bank = bank.reshape(up, K)
    for ph in range(up):           # [phase][tap], taps in descending filter index = ascending input index
        n = ph + (K - 1 - np.arange(K)) * up
        ok = n < N
        assert np.array_equal(bank[ph][ok], h[n[ok]]) and not bank[ph][~ok].any()


@pytest.mark.parametrize("a,b", PAIRS)
def test_span_matches_brute_force(rs, a, b):
    p = plan(rs, a, b)
    up, down, N = p["up"], p["down"], p["taps"]
    h = filt(rs, a, b)
    nz = np.nonzero(h)[0]
    lohi = (LL * 2)()

    def support(m):                # input samples j with a nonzero tap h[t - j up]
        t = (m + p["pre_remove"]) * down - p["pre_pad"]
        return [j for j in range((t - N) // up - 1, t // up + 2) if 0 <= t - j * up < N and (t - j * up) in nz_set]
    nz_set = set(nz.tolist())
    for m0, m1 in ((0, 1), (0, 7), (5, 6), (13, 300), (1000, 1001), (12345, 12400)):
        rs.rs_span(LL(a), LL(b), LL(m0), LL(m1), lohi)
        js = [j for m in range(m0, m1) for j in support(m)]
        assert (lohi[0], lohi[1]) == (min(js), max(js) + 1), (m0, m1)
    # a stream of n_in samples can emit exactly the outputs whose support ends inside it
    for n_in in (1, 2, 50, 333, 4000):
        r = rs.rs_n_ready(LL(a), LL(b), LL(n_in))
        if r > 0:
            rs.rs_span(LL(a), LL(b), LL(r - 1), LL(r), lohi)
            assert lohi[1] <= n_in
        rs.rs_span(LL(a), LL(b), LL(r), LL(r + 1), lohi)
        assert lohi[1] > n_in


@pytest.mark.parametrize("a,b", PAIRS)
def test_output_matches_resample_poly(rs, a, b):
    p = plan(rs, a, b)
    rng = np.random.default_rng(a + b)
    for L in (1, 2, p["K"] - 1, p["K"] + 1, 1000, 5003):
        x = (rng.standard_normal(L) * 0.3).astype(np.float32)
        ref = resample_poly(x.astype(np.float64), p["up"], p["down"])
        y = run(rs, a, b, x)
        assert y.shape == ref.shape, L
        rms = np.sqrt(np.mean(ref ** 2)) or 1.0
        assert np.abs(y - ref).max() <= 1e-13 * rms, L
        y32, r32 = y.astype(np.float32), ref.astype(np.float32)
        assert (np.abs(y32 - r32) <= np.spacing(np.maximum(np.abs(y32), np.abs(r32)))).all(), L


def test_refused_rates(rs):
    o = (LL * 7)()
    assert rs.rs_plan(LL(44101), LL(22050), o) == -1        # M = 44 101 > 2048
    assert rs.rs_plan(LL(22050), LL(44101), o) == -1
    for a, b in ((0, 22050), (-48000, 22050), (48000, 0), (48000, -1)):
        assert rs.rs_plan(LL(a), LL(b), o) == -1
    assert rs.rs_plan(LL(2048), LL(1), o) == 0 and rs.rs_plan(LL(2049), LL(1), o) == -1


def test_equal_rates_are_identity(rs):
    x = np.random.default_rng(1).standard_normal(777).astype(np.float32)
    assert np.array_equal(run(rs, 22050, 22050, x).astype(np.float32), x)
