"""CPU checks of the streaming reference encoder (ovc_reference_encoder_stream) and of live-session enrollment.

* The row rules of openvoice_b200/csrc/ovc_refenc_stream.h, compiled with g++ (tests/hostcheck/refenc_stream_host.cpp),
  against a Python model: final frames, layer rows c_l = c0 >> l, the carry rows, the snapshot tail rows and GRU tail
  steps, the descriptor clamps.
* The kernel's schedule replayed in float64 with the oracle's layers applied to row ranges: advancing in any chunking
  and finishing a snapshot from the carry equals the oracle's whole-prefix encoder to 1e-12.
* ``Enrollment`` validation and which step produces which snapshot."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import vc_oracle as O
from openvoice_b200.streaming import Enrollment, ready_frames

HERE = os.path.dirname(os.path.abspath(__file__))
LL = C.c_longlong
HOP, NFFT, PAD = 256, 1024, 384
FILT = [1, 32, 32, 64, 64, 128, 128]


@pytest.fixture(scope="module")
def re(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostcheck") / "refenc_stream_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "hostcheck", "refenc_stream_host.cpp")])
    lib = C.CDLL(so)
    for f in ("re_ready", "re_limit", "re_carry_lo", "re_ws_floats", "re_ws_rows"):
        getattr(lib, f).restype = LL
    lib.re_ready.argtypes = [LL, C.c_int, C.c_int]
    lib.re_limit.argtypes = [LL, C.c_int]
    lib.re_carry_lo.argtypes = [LL]
    lib.re_item.argtypes = [C.POINTER(LL), LL, LL, LL, C.c_int, C.c_int, C.c_int, C.POINTER(LL)]
    return lib


def limit(T, l):
    for _ in range(l):
        T = (T - 1) // 2 + 1
    return T


def model_item(d, c0, state_rows, ring_rows, max_new):
    """The clamp and phase rule of ovc_re::item, in Python terms."""
    cl = lambda v, lo, hi: max(lo, min(v, hi))  # noqa: E731
    c0 = cl(c0, 0, 2 ** 29)
    top = c0 + max(max_new, 0)
    n_adv, n_snap = cl(d[2], 0, 2 ** 50), cl(d[3], 0, 2 ** 50)
    rs, T = ready_frames(n_snap, HOP, NFFT, False), n_snap // HOP
    snap = n_snap > 0
    ok = snap and T >= 1 and n_snap > PAD and c0 <= rs <= top and T - rs <= 2
    a1 = rs if ok else c0
    a2 = cl(ready_frames(n_adv, HOP, NFFT, False), a1, top)
    return [cl(d[0], 0, state_rows - 1), cl(d[1], 0, ring_rows - 1), c0, a1, a2, n_snap, T, T - a1 if ok else 0, int(snap),
            int(ok)]


def item(re, d, c0, state_rows=4, ring_rows=4, max_new=64):
    out = (LL * 10)()
    re.re_item((LL * 4)(*d), c0, state_rows, ring_rows, max_new, HOP, NFFT, out)
    return list(out)


def test_rows_carry_and_tail_for_every_prefix(re):
    for n in range(0, 70001):
        c0 = ready_frames(n, HOP, NFFT, False)
        assert re.re_ready(n, HOP, NFFT) == c0, n
        if n < HOP or n <= PAD:
            continue
        T = n // HOP
        for l in range(7):
            cl, lim = c0 >> l, limit(T, l)
            assert re.re_limit(T, l) == lim
            assert 0 <= lim - cl <= 2, (n, l)                   # tail rows (l = 6: GRU tail steps)
            if l < 6:
                # every input row below c_l that an output row from c_{l+1} on reads is in the carry, in its own slot
                lo = 2 * (c0 >> (l + 1)) - 1
                assert re.re_carry_lo(cl) <= max(lo, 0), (n, l)
                assert cl - re.re_carry_lo(cl) <= 2
        # the descriptor of a snapshot at n against rows consumed up to any earlier point
        for back in (0, 1, 255, 4000):
            cprev = ready_frames(max(0, n - back), HOP, NFFT, False)
            got = item(re, [1, 2, n, n], cprev)
            assert got == model_item([1, 2, n, n], cprev, 4, 4, 64), (n, back)
            if n - cprev * HOP < 64 * HOP:
                assert got[9] == 1 and got[3] == c0 and got[4] == c0 and got[7] == T - c0


def test_geometry_of_the_released_config(re):
    out = (LL * 15)()
    re.re_geom(513, out)
    W = list(out)[:7]
    assert W == [513, 257, 129, 65, 33, 17, 9]
    carry = 2 * sum(FILT[l] * W[l] for l in range(6))
    assert carry == 42626
    assert list(out)[7:13] == [4 + 2 * sum(FILT[i] * W[i] for i in range(l)) for l in range(6)]
    assert out[13] == 4 + carry and out[14] == -(-(4 + carry + 128) // 4) * 4
    for M in (1, 8, 64, 100):
        rows = [re.re_ws_rows(M, l) for l in range(7)]
        assert rows == [max(2, (M >> l) + 1) for l in range(7)]
        n = sum(r * FILT[l] * W[l] for l, r in enumerate(rows)) + rows[6] * 384
        assert re.re_ws_floats(M, 513) == -(-n // 64) * 64


def test_descriptor_clamps(re):
    rng = np.random.default_rng(3)
    big = [-2 ** 63, -2 ** 40, -1, 0, 1, 384, 385, 512, 1000, 2 ** 29 * 256, 2 ** 50, 2 ** 62, 2 ** 63 - 1]
    for _ in range(4000):
        d = [int(rng.choice(big)) if rng.random() < 0.5 else int(rng.integers(-10, 50000)) for _ in range(4)]
        c0 = int(rng.choice(big)) if rng.random() < 0.3 else int(rng.integers(0, 200))
        sr, rr, M = int(rng.integers(1, 9)), int(rng.integers(1, 9)), int(rng.integers(1, 200))
        got = item(re, d, c0, sr, rr, M)
        assert got == model_item(d, c0, sr, rr, M), (d, c0)
        assert 0 <= got[0] < sr and 0 <= got[1] < rr
        assert got[2] <= got[3] <= got[4] <= got[2] + M and 0 <= got[7] <= 2


# ---------------------------------------------------------------------------------------------- float64 replay
class Replay:
    """The kernel's schedule in float64: LayerNorm, the six convs and the GRU applied to row ranges, a carry of the
    <= 2 most recent rows of each conv input, and snapshots finished from the carry plus the prefix's tail frames."""

    def __init__(self, sd, y):
        self.sd, self.y = sd, y
        self.spec = O.spectrogram(y[None])[0]                 # the whole stream's frames: final frames are the same
        self.c0, self.h = 0, torch.zeros(128, dtype=torch.float64)
        self.carry = [dict() for _ in range(6)]

    def ln(self, cols):
        return Fn.layer_norm(cols.T, (cols.shape[0],), self.sd["ref_enc.layernorm.weight"], self.sd["ref_enc.layernorm.bias"])

    def conv(self, l, rows, hin, o0, o1):
        """rows: dict hi -> [C, W]; output rows [o0, o1) of conv l, taps at or past hin (or < 0) read as absent."""
        some = next(iter(rows.values()))
        X = torch.stack([rows[hi] if 0 <= hi < hin else torch.zeros_like(some) for hi in range(2 * o0 - 1, 2 * o1)], 1)
        y = Fn.conv2d(X[None], O._w(self.sd, f"ref_enc.convs.{l}"), self.sd[f"ref_enc.convs.{l}.bias"], stride=2,
                      padding=(0, 1))
        return {o0 + r: t for r, t in enumerate(Fn.relu(y[0]).unbind(1))}

    def gru(self, h, feats):
        sd = self.sd
        for x in feats:
            gi = x.reshape(-1) @ sd["ref_enc.gru.weight_ih_l0"].T + sd["ref_enc.gru.bias_ih_l0"]
            gh = h @ sd["ref_enc.gru.weight_hh_l0"].T + sd["ref_enc.gru.bias_hh_l0"]
            r = torch.sigmoid(gi[:128] + gh[:128])
            u = torch.sigmoid(gi[128:256] + gh[128:256])
            c = torch.tanh(gi[256:] + r * gh[256:])
            h = (1 - u) * c + u * h
        return h

    def layers(self, a, frames, lim):
        """Rows from frame a on (``frames``: their LN inputs), limits lim[l]; returns the GRU inputs of the rows."""
        rows = {a + t: r[None] for t, r in enumerate(self.ln(frames).unbind(0))}
        new = [rows]
        for l in range(6):
            src = dict(self.carry[l])
            src.update(rows)
            o0, o1 = a >> (l + 1), lim[l + 1]
            rows = self.conv(l, src, lim[l], o0, o1) if o1 > o0 else {}
            new.append(rows)
        return new

    def advance(self, n):
        c1 = ready_frames(n, HOP, NFFT, False)
        if c1 <= self.c0:
            return
        a = self.c0
        new = self.layers(a, self.spec[:, a:c1], [c1 >> l for l in range(7)])
        self.h = self.gru(self.h, [new[6][t] for t in sorted(new[6])])
        for l in range(6):
            self.carry[l].update(new[l])
            keep = max(0, (c1 >> l) - 2)
            self.carry[l] = {r: v for r, v in self.carry[l].items() if r >= keep}
        self.c0 = c1

    def snapshot(self, n):
        self.advance(n)
        T, a = n // HOP, self.c0
        tail = O.spectrogram(self.y[None, :n])[0][:, a:T]
        lim = [limit(T, l) for l in range(7)]
        new = self.layers(a, tail, lim) if T > a else [{}] * 7
        h = self.gru(self.h.clone(), [new[6][t] for t in sorted(new[6])])
        return h @ self.sd["ref_enc.proj.weight"].T + self.sd["ref_enc.proj.bias"]


@pytest.fixture(scope="module")
def sd64():
    return {k: v.double() for k, v in O.synthetic_state_dict(1234).items() if k.startswith("ref_enc.")}


def whole(sd, y, n):
    return O.reference_encoder(sd, O.spectrogram(y[None, :n]).transpose(1, 2))[0]


@pytest.mark.parametrize("sizes", [[1], [769], [4000, 1, 769], [50000, 3001]])
def test_incremental_schedule_equals_whole_prefix(sd64, sizes):
    rng = np.random.default_rng(len(sizes) + sizes[0])
    y = torch.from_numpy(0.3 * rng.standard_normal(70000))
    limit_n = 6000 if sizes == [1] else len(y)
    checks = {385, 512, 639, 640, 1023, 1280, 5003} | set(int(v) for v in rng.integers(385, limit_n, 6))
    rp, pos, i = Replay(sd64, y), 0, 0
    with torch.no_grad():
        while pos < limit_n:
            end = min(limit_n, pos + sizes[i % len(sizes)])
            for n in sorted(c for c in checks if pos < c <= end):   # snapshots of prefixes inside the push
                got, ref = rp.snapshot(n), whole(sd64, y, n)
                assert float((got - ref).abs().max() / ref.abs().max()) <= 1e-12, (sizes, n)
            rp.advance(end)
            if sizes[0] >= 769:
                got, ref = rp.snapshot(end), whole(sd64, y, end)
                assert float((got - ref).abs().max() / ref.abs().max()) <= 1e-12, (sizes, end)
            pos, i = end, i + 1


# ---------------------------------------------------------------------------------------------- Enrollment
def test_enrollment_validation():
    e = Enrollment()
    assert (e.every_frames, e.until_frames, e.ramp_frames) == (172, 861, 16)
    for kw in ({"every_frames": 1}, {"every_frames": 10, "until_frames": 9}, {"ramp_frames": -1},
               {"every_frames": 2.5}, {"every_frames": True}):
        with pytest.raises(ValueError):
            Enrollment(**kw)
    Enrollment(2, 2, 0)


def test_snapshot_bookkeeping():
    e = Enrollment(every_frames=10, until_frames=35, ramp_frames=4)
    P = 10 * HOP                                             # samples of one snapshot period
    assert e.snapshot(0, P - 1, HOP) == 0 and e.snapshot(0, P, HOP) == 1
    assert e.snapshot(P, P + 1, HOP) == 0                    # the boundary was already crossed
    assert e.snapshot(P - 1, 3 * P + 5, HOP) == 3            # several boundaries: the last one wins
    assert e.snapshot(0, 100 * P, HOP) == 3                  # 3 * 10 <= 35 < 4 * 10
    assert e.snapshot(3 * P, 100 * P, HOP) == 0              # past until_frames: no more snapshots
    # replaying pushes: each k is produced exactly once, by the push that makes its prefix available
    rng = np.random.default_rng(0)
    for _ in range(200):
        n, seen = 0, []
        for _ in range(40):
            m = n + int(rng.choice([1, 300, P - 1, P, 2 * P + 7]))
            k = e.snapshot(n, m, HOP)
            if k:
                assert n < k * P <= m and not e.snapshot(n, k * P - 1, HOP) >= k
                assert all(k > s for s in seen)
                seen.append(k)
            n = m
        assert not seen or seen[-1] == min(n // P, 3)
