"""CPU checks of the duration fit (include/ovc.h: ovc_tts_fit): the g++ build of the rule in ovc_tts_ops.h against a
brute-force float32 search and the NumPy oracle, the fixtures of oracle/make_golden_tts_fit.py, the target arithmetic
and refusals of BaseSpeakerTTS, the grouping of CloneSessions.say(duration=), and the ctypes mirror of ovc_tts_fit."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import tts_fit_oracle as FO

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
CASES = ["tts_fit_b1_one", "tts_fit_b3_joint", "tts_fit_b2_mixed", "tts_fit_b1_clamp"]


@pytest.fixture(scope="module")
def hc(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostcheck") / "tts_fit_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "hostcheck", "tts_fit_host.cpp")])
    lib = C.CDLL(so)
    lib.hc_group_frames.restype = C.c_longlong
    lib.hc_group_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_float]
    lib.hc_fit_scale.restype = C.c_float
    lib.hc_fit_scale.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_float,
                                 C.c_float]
    return lib


def host_fit(hc, e, lens, target, lo=FO.SCALE_LO, hi=FO.SCALE_HI):
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int64)
    return np.float32(hc.hc_fit_scale(e.ctypes.data, lens.ctypes.data, e.shape[1], 0, e.shape[0], int(target), lo, hi))


def host_frames(hc, e, lens, s):
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int64)
    return int(hc.hc_group_frames(e.ctypes.data, lens.ctypes.data, e.shape[1], 0, e.shape[0], np.float32(s)))


def brute_force(e, lens, target, lo, hi):
    """Every float in [lo, hi] in order; the first whose group frames reach the target, else hi."""
    s = np.arange(FO.bits(lo), FO.bits(hi) + 1, dtype=np.uint32).view(np.float32)
    mask = np.arange(e.shape[1])[None, :] < lens[:, None]
    F = np.zeros(len(s), np.int64)
    for r in range(e.shape[0]):
        w = np.ceil(e[r][mask[r]][None, :] * s[:, None]).astype(np.int64).sum(1)
        F += np.maximum(w, 1)
    hit = np.nonzero(F >= target)[0]
    return s[hit[0]] if len(hit) else np.float32(hi)


def random_group(rng, rows, T):
    lens = rng.integers(0, T + 1, rows)
    logw = rng.normal(1.2, 0.8, (rows, T)).astype(np.float32)
    return np.exp(logw), lens


def test_rule_matches_brute_force_on_narrow_ranges(hc):
    rng = np.random.default_rng(0)
    for trial in range(40):
        e, lens = random_group(rng, int(rng.integers(1, 4)), int(rng.integers(1, 30)))
        lo = np.float32(rng.uniform(0.5, 2.0))
        hi = FO.from_bits(FO.bits(lo) + int(rng.integers(1, 60000)))
        f_lo, f_hi = FO.group_frames(e, lens, lo), FO.group_frames(e, lens, hi)
        for target in (f_lo - 1, f_lo, (f_lo + f_hi) // 2, f_hi, f_hi + 1, int(rng.integers(f_lo, f_hi + 1))):
            want = brute_force(e, lens, target, lo, hi)
            assert host_fit(hc, e, lens, target, lo, hi) == want, (trial, target)
            assert FO.fit_scale(e, lens, target, lo, hi) == want, (trial, target)


def test_rule_matches_the_oracle_and_is_minimal_on_the_full_range(hc):
    rng = np.random.default_rng(1)
    for trial in range(60):
        e, lens = random_group(rng, int(rng.integers(1, 6)), int(rng.integers(1, 130)))
        f1 = FO.group_frames(e, lens, 1.0)
        target = max(1, int(f1 * rng.uniform(0.2, 4.5)))
        s = host_fit(hc, e, lens, target)
        assert s == FO.fit_scale(e, lens, target)
        assert host_frames(hc, e, lens, s) == FO.group_frames(e, lens, s)
        if s < np.float32(FO.SCALE_HI):
            assert FO.group_frames(e, lens, s) >= target
        if s > np.float32(FO.SCALE_LO):
            assert FO.group_frames(e, lens, np.nextafter(s, np.float32(0))) < target


def test_ties_clamps_and_underflow(hc):
    # two equal tokens cross every integer at the same scale: F jumps by 2 and the target between is met there
    e = np.array([[3.0, 3.0, 0.0, 0.0]], np.float32)
    lens = np.array([2])
    s = host_fit(hc, e, lens, 9)                          # F = 8 below s = 4/3, 10 at it
    assert s == FO.fit_scale(e, lens, 9) and FO.group_frames(e, lens, s) == 10
    assert FO.group_frames(e, lens, np.nextafter(s, np.float32(0))) == 8
    # both clamps
    e, lens = np.exp(np.full((2, 10), 1.0, np.float32)), np.array([10, 7])
    assert host_fit(hc, e, lens, 1) == np.float32(FO.SCALE_LO)
    assert host_fit(hc, e, lens, FO.group_frames(e, lens, FO.SCALE_HI) + 1) == np.float32(FO.SCALE_HI)
    assert host_fit(hc, e, lens, FO.group_frames(e, lens, FO.SCALE_HI)) < np.float32(FO.SCALE_HI)
    # tokens whose exp underflows to 0 give no frames; a row of only those still counts one frame
    e = np.exp(np.array([[-200.0, -120.0, 0.5], [-150.0, -300.0, 0.0]], np.float32))
    assert e[0, 0] == 0 and e[1, 1] == 0
    lens = np.array([3, 2])
    for target in (2, 3, 5, 9):
        assert host_fit(hc, e, lens, target) == FO.fit_scale(e, lens, target)
    assert host_frames(hc, e, lens, 4.0) == FO.group_frames(e, lens, 4.0) == int(np.ceil(np.exp(np.float32(0.5)) * 4)) + 1


@pytest.mark.parametrize("name", CASES)
def test_fixtures_follow_the_rule(name, hc):
    d = np.load(os.path.join(GOLD, name + ".npz"))
    meta = json.loads(str(d["meta"]))
    lens = np.array(meta["lengths"] or [meta["T"]] * meta["B"])
    e = np.exp(d["logw"])
    covered = np.zeros(meta["B"], bool)
    for r0, r1, target in d["fit"]:
        s = FO.fit_scale(e[r0:r1], lens[r0:r1], target)
        assert host_fit(hc, e[r0:r1], lens[r0:r1], target) == s
        assert (d["scale"][r0:r1] == s).all()
        assert d["y_lengths"][r0:r1].sum() == FO.group_frames(e[r0:r1], lens[r0:r1], s)
        covered[r0:r1] = True
    assert (d["scale"][~covered] == meta["unfitted_scale"]).all()
    for b in range(meta["B"]):                            # the reference's durations are the rule's per-token frames
        n = lens[b]
        assert np.array_equal(d["w_ceil"][b, :n], FO.token_frames(e[b, :n], d["scale"][b]).astype(np.float32))
    if name == "tts_fit_b1_clamp":
        assert d["scale"][0] == np.float32(FO.SCALE_HI) and d["y_lengths"][0] < d["fit"][0, 2]


# ------------------------------------------------------------------------------------------------ BaseSpeakerTTS
def make_tts():
    from test_clone_sessions_host import make_models
    return make_models()


def test_target_arithmetic_and_refusals():
    from test_clone_sessions_host import HOP, SR
    tts, _ = make_tts()
    gap = int((SR * 0.05) / 1.25)
    for duration, n, speed in ((2.4, 3, 1.25), (0.5, 1, 1.0), (1.0, 2, 0.8)):
        gaps = n * int((SR * 0.05) / speed)
        N = int(round(duration * SR))
        want = -(-(N - gaps) // HOP)
        got = tts.fit_target(duration, n, speed, True, "r")
        assert got == want and HOP * got + gaps >= N > HOP * (got - 1) + gaps
        assert tts.fit_target(duration, n, speed, False, "r") == -(-N // HOP)
    # exactly one frame per sentence is accepted, one sample less is refused
    d_ok = (3 * gap + 3 * HOP) / SR
    assert tts.fit_target(d_ok, 3, 1.25, True, "r") == 3
    with pytest.raises(ValueError, match="request 2: duration .* too short for 3 sentence"):
        tts.fit_target((3 * gap + 2 * HOP) / SR, 3, 1.25, True, "request 2")
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="request 1: duration"):
            tts._request_sentences([dict(ids=[[1, 2]], speaker=0, seed=1),
                                    dict(ids=[[1, 2]], speaker=0, seed=1, duration=bad)])


def test_requests_become_fit_groups():
    tts, _ = make_tts()
    reqs = [dict(ids=[[1, 2, 3], [4, 5]], speaker=0, seed=1, duration=1.5, speed=1.25),
            dict(ids=[[6, 7]], speaker=0, seed=2),
            dict(ids=[[8], [9, 10], [11]], speaker=0, seed=3, duration=2.0)]
    seqs, _, owner, speeds, kw = tts._request_sentences(reqs)
    assert owner == [0, 0, 1, 2, 2, 2]
    assert kw["fit"] == [(0, 2, tts.fit_target(1.5, 2, 1.25, True, "")), (3, 6, tts.fit_target(2.0, 3, 1.0, True, ""))]
    _, _, _, _, kw = tts._request_sentences(reqs[1:2])
    assert "fit" not in kw                                # no duration: the encode runs without fit groups
    with pytest.raises(ValueError, match="request 0: duration 0.01 s is too short"):
        tts._request_sentences([dict(ids=[[1], [2]], speaker=0, seed=1, duration=0.01)])


def test_fit_groups_are_checked_before_any_launch():
    from openvoice_b200.api import FIT_SCALE_RANGE, fit_groups
    assert fit_groups(None, 4, "cpu") is None and fit_groups([], 4, "cpu") is None
    r0, r1, t, lo, hi = fit_groups([(0, 2, 50), (3, 4, 7)], 4, "cpu")
    assert r0.tolist() == [0, 3] and r1.tolist() == [2, 4] and t.tolist() == [50, 7] and (lo, hi) == FIT_SCALE_RANGE
    for bad in ([(0, 0, 5)], [(0, 5, 5)], [(-1, 1, 5)], [(0, 2, 5), (1, 3, 5)], [(2, 3, 5), (0, 1, 5)], [(0, 1, 0)],
                [(0, 1)]):
        with pytest.raises(ValueError, match="fit group"):
            fit_groups(bad, 4, "cpu")


# ------------------------------------------------------------------------------------------------ CloneSessions
def test_say_duration_forms_one_group_per_say():
    from test_clone_sessions_host import keys, sessions, sentences
    tts, conv = make_tts()
    seen = []
    encode = tts.model.tts_encode

    def spy(x, lens, **kw):
        seen.append(kw.get("fit"))
        return encode(x, lens, **kw)
    tts.model.tts_encode = spy
    cs = sessions(tts, conv)
    a, b = cs.open(**keys(0)), cs.open(**keys(1))
    cs.say(a, ids=sentences(0, 2), duration=3.0)
    cs.say(b, ids=sentences(1, 1))
    cs.say(b, ids=sentences(2, 3), duration=4.0)
    cs.say(a, ids=sentences(3, 1), duration=1.0)           # a second say of a: a group of its own
    cs.encode_pending()
    sb = keys(1)["speed"]
    assert seen == [[[0, 2, tts.fit_target(3.0, 2, keys(0)["speed"], True, "")],
                     [3, 6, tts.fit_target(4.0, 3, sb, True, "")],
                     [6, 7, tts.fit_target(1.0, 1, keys(0)["speed"], True, "")]]]
    cs.say(a, ids=sentences(4, 1))
    cs.encode_pending()
    assert seen[-1] is None                               # a step without fitted text: no fit groups
    with pytest.raises(ValueError, match="session 1: duration"):
        cs.say(b, ids=sentences(5, 1), duration=float("nan"))
    with pytest.raises(ValueError, match="session 1: duration 0.001 s is too short"):
        cs.say(b, ids=sentences(5, 1), duration=0.001)
    assert not cs.pending and not cs.pending_fit          # refused text is not queued


def test_cancel_drops_the_fit_of_the_cancelled_session():
    from test_clone_sessions_host import keys, sessions, sentences
    tts, conv = make_tts()
    cs = sessions(tts, conv)
    a, b = cs.open(**keys(0)), cs.open(**keys(1))
    cs.say(a, ids=sentences(0, 2), duration=3.0)
    cs.say(b, ids=sentences(1, 2), duration=2.0)
    cs.cancel(a)
    assert [s for s, _ in cs.pending] == [b, b] and len(cs.pending_fit) == 2
    assert cs.pending_fit[0] == cs.pending_fit[1] is not None


# ------------------------------------------------------------------------------------------------ C layout
_PROBE = r"""
#include <cstddef>
#include <cstdio>
#include "ovc.h"
int main() {
  std::printf("%zu", sizeof(ovc_tts_fit));
#define F(n) std::printf(" %s %zu", #n, offsetof(ovc_tts_fit, n));
  F(row0) F(row1) F(target_frames) F(G) F(scale_lo) F(scale_hi) F(length_scale)
  std::printf("\n");
  return 0;
}
"""


def test_tts_fit_layout_matches_the_header(tmp_path):
    from openvoice_b200 import _native
    src = tmp_path / "probe.cpp"
    src.write_text(_PROBE)
    exe = tmp_path / "probe"
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert int(out[0]) == C.sizeof(_native.TtsFit)
    got = dict(zip(out[1::2], (int(v) for v in out[2::2])))
    assert list(got) == [f[0] for f in _native.TtsFit._fields_]
    for name, off in got.items():
        assert getattr(_native.TtsFit, name).offset == off, name
    assert "ovc_tts_encode_fit" in _native.EXPORTS and _native.ABI_VERSION == 18
