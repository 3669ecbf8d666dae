"""CPU check of the ring form of the resampler (ovc_resample_rings, openvoice_b200/csrc/ovc_resample.h).

The ring kernel clamps each item's descriptor with ``ring_item`` and addresses its input and output rows with
``ring_in_at`` / ``ring_out_at`` around the same ``output_at`` as ``ovc_resample``.  Here the SAME header is compiled with
g++ (tests/hostcheck/resample_ring_host.cpp): the clamp and index rules are compared with a NumPy model, and a host loop
with the kernel's semantics, reading ring rows (with wraparound, open and closed streams) and writing ring rows or a
packed buffer, is compared with the whole-signal result (bit for bit) and scipy.signal.resample_poly (one ulp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.signal import resample_poly

HERE = os.path.dirname(os.path.abspath(__file__))
LL = C.c_longlong
OPEN = 2 ** 63 - 1
MAX_POS = OPEN // (8 * 2048)
PAIRS = [(48000, 22050), (22050, 48000), (8000, 22050), (22050, 16000), (44100, 22050), (22050, 22050)]


@pytest.fixture(scope="module")
def rr(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostcheck") / "resample_ring_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "hostcheck", "resample_ring_host.cpp")])
    lib = C.CDLL(so)
    lib.rr_in_at.restype = LL
    lib.rr_out_at.restype = LL
    return lib


def arr(v):
    return (LL * len(v))(*[int(x) for x in v])


def model_item(d, n_plans, in_rows, out_rows, out_cap, max_count):
    """The clamp rule of ring_item, in NumPy terms."""
    plan, in_row, in_len, m0, count, out_row, out_off = d
    return [int(np.clip(plan, 0, n_plans - 1)), int(np.clip(in_row, 0, in_rows - 1)), max(in_len, 0),
            int(np.clip(m0, 0, MAX_POS)), int(np.clip(count, 0, max_count)), int(np.clip(out_row, 0, out_rows - 1)),
            out_off % out_cap]


def test_clamp_and_index_rules_match_numpy_model(rr):
    rng = np.random.default_rng(0)
    big = [-2 ** 63, -2 ** 40, -1, 0, 1, 2, 7, 1000, 2 ** 40, MAX_POS, MAX_POS + 1, OPEN]
    out7 = (LL * 7)()
    for _ in range(3000):
        d = [int(rng.choice(big)) if rng.random() < 0.5 else int(rng.integers(-50, 50)) for _ in range(7)]
        n_plans, in_rows, out_rows = (int(v) for v in rng.integers(1, 9, 3))
        out_cap, in_cap, max_count = int(rng.integers(1, 5000)), int(rng.integers(1, 5000)), int(rng.integers(0, 3000))
        rr.rr_item(arr(d), n_plans, LL(in_rows), LL(out_rows), LL(out_cap), LL(max_count), out7)
        it = list(out7)
        assert it == model_item(d, n_plans, in_rows, out_rows, out_cap, max_count), d
        assert 0 <= it[0] < n_plans and 0 <= it[4] <= max_count
        for j in (-5, -1, 0, 1, 3 * in_cap + 2, it[2] - 1, it[2], 2 ** 40):
            k = rr.rr_in_at(arr(it), LL(j), LL(in_cap))
            ref = it[1] * in_cap + j % in_cap if 0 <= j < it[2] else -1
            assert k == ref and (k == -1 or 0 <= k < in_rows * in_cap), (it, j)
        for i in (0, 1, max(0, it[4] - 1)):
            k = rr.rr_out_at(arr(it), LL(i), LL(out_cap))
            assert k == it[5] * out_cap + (it[6] + i) % out_cap and 0 <= k < out_rows * out_cap, (it, i)


def span(a, b, n_in=0, m0=0, m1=1):
    from openvoice_b200._native import resample_span
    return resample_span(a, b, n_in, m0, m1)


def whole(rr, a, b, x):
    y = np.empty(span(a, b, len(x))[0], dtype=np.float32)
    rr.rr_whole(LL(a), LL(b), x.ctypes.data_as(C.c_void_p), LL(len(x)), y.ctypes.data_as(C.c_void_p))
    return y


@pytest.mark.parametrize("tile", [256, 37])
def test_ring_items_equal_whole_signal(rr, tile):
    """One call over every pair: per pair an open item (outputs ready so far), a closed item (outputs past n_out, which
    come out as 0), windows that wrap their input ring row, outputs into ring rows (wrapping) and into a packed buffer.
    Input rows hold NaN wherever the item does not read, outputs outside each item's range stay NaN."""
    rng = np.random.default_rng(tile)
    in_cap, out_cap, pk_cap = 3400, 3000, 10 ** 6
    sig, items = [], []                                   # items: (pair, x, in_len, m0, count, packed?)
    for k, (a, b) in enumerate(PAIRS):
        L = int(rng.integers(20000, 40000))
        x = (0.3 * rng.standard_normal(L)).astype(np.float32)
        sig.append(x)
        arrived = L - int(rng.integers(100, 3000))
        ready = span(a, b, arrived)[1]
        n_all = span(a, b, L)[0]
        items.append((k, OPEN, ready - 1500, 1500, k % 2 == 0))               # open: the last ready outputs
        items.append((k, L, n_all - 1400, 1500, k % 2 == 1))                  # closed: the tail and 100 past n_out
        items.append((k, OPEN, 777, 1, False))                                # a single output
    B = len(items)
    rings = np.full((B, in_cap), np.nan, dtype=np.float32)
    out = np.full((B, out_cap), np.nan, dtype=np.float32)
    packed = np.full((1, pk_cap), np.nan, dtype=np.float32)
    desc, at, wrapped = [], 0, 0
    for r, (k, ln, m0, n, pk) in enumerate(items):
        a, b = PAIRS[k]
        x = sig[k]
        _, _, lo, hi = span(a, b, 0, m0, m0 + n)
        lo, hi = max(lo, 0), min(hi, len(x))
        assert hi - lo <= in_cap
        rings[r, np.arange(lo, hi) % in_cap] = x[lo:hi]
        wrapped += (lo // in_cap) != ((hi - 1) // in_cap)
        desc.append((k, r, ln, m0, n, 0 if pk else r, at if pk else m0))
        at += n if pk else 0
    assert wrapped >= 3
    max_count = max(n for *_, n, _ in items)
    rates = [v for p in PAIRS for v in p]
    # ring-row items write `out`, packed items write `packed`: two calls, as a caller with two destinations makes
    for want_pk, dst, cap in ((False, out, out_cap), (True, packed, pk_cap)):
        sel = [d for d, it in zip(desc, items) if it[4] == want_pk]
        flat = arr([v for d in sel for v in d])
        rc = rr.rr_run(len(PAIRS), arr(rates), rings.ctypes.data_as(C.c_void_p), LL(B), LL(in_cap), flat, len(sel),
                       dst.ctypes.data_as(C.c_void_p), LL(dst.shape[0]), LL(cap), LL(max_count), tile)
        assert rc == 0
    written = {0: np.zeros(out.shape, bool), 1: np.zeros(packed.shape, bool)}
    for (k, ln, m0, n, pk), d in zip(items, desc):
        a, b = PAIRS[k]
        x = sig[k]
        ref = whole(rr, a, b, x)
        want = np.zeros(n, dtype=np.float32)
        ms = np.arange(m0, m0 + n)
        inside = ms < len(ref)
        want[inside] = ref[ms[inside]]
        if ln == OPEN:
            assert inside.all()
        if pk:
            got, idx = packed[0, d[6]:d[6] + n], (0, np.arange(d[6], d[6] + n))
        else:
            idx = (d[5], (d[6] + np.arange(n)) % out_cap)
            got = out[idx]
        written[int(pk)][idx] = True
        assert np.array_equal(got, want), (a, b, ln == OPEN, m0)
        poly = resample_poly(x.astype(np.float64), *_updown(a, b)).astype(np.float32)
        g, r = got[inside], poly[ms[inside]]
        assert (np.abs(g - r) <= np.spacing(np.maximum(np.abs(g), np.abs(r)))).all(), (a, b)
    assert np.isnan(out[~written[0]]).all() and np.isnan(packed[~written[1]]).all()
    assert any((d[6] + d[4]) > out_cap for d, it in zip(desc, items) if not it[4])    # a ring output wraps


def _updown(a, b):
    g = np.gcd(a, b)
    return b // g, a // g
