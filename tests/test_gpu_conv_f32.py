"""The fp32 CUDA-core conv family (conv1d_f32<>, openvoice_b200/csrc/ovc_conv.cuh) and the two conv_post kernels on their
own, against plain float64 torch on the CPU.

The convs run through tests/kernelcheck/libovc_kc_f32.so, which calls the library's own compiled instantiations
(launch_<name> of ovc_variants.h) on weights packed by the library's own code (ovc_convpack.h).  The reference uses the
UNPACKED weights: natural [N][Cin][K] weights and conv1d, the raw ConvTranspose1d weight and conv_transpose1d, the gate
and the projection in natural row order.  A packing, interleave or phase bug therefore shows up here even though every
launch of the library shares it.

Gates (proved, not tuned).  u = 2^-24, gamma_m = m u / (1 - m u).  Every output is one sequential fmaf chain of
n = n_chunks * CI_CH * K terms (Cin padded to the chunk) whose activation went through one rounded leaky-relu product,
followed by e <= 4 rounded epilogue operations (bias, residual or old value, the second add, scale).  The standard
bound of recursive summation gives, with S = sum|w||a| + |bias| + |res| + |y_old| (times |scale|) computed in fp64:
  LINEAR, RESSKIP, COUPLE, UPS:  |y - y64| <= gamma_{n+e+1} S
  GATE:  tanh' <= 1, sigmoid' <= 1/4, |tanh|, |sigmoid| <= 1, so the pre-activation errors contribute
         gamma (S_a + S_b / 4); tanhf and expf are within 2 ulp (CUDA C Programming Guide, no fast-math), 1 + e^-z,
         the division (IEEE, -prec-div) and the product add 3 roundings: at most 7 u relative on |y| <= 1, so the
         floor 2^-20 covers them:                                   |Δ| <= gamma (S_a + S_b/4) + 2^-20
  PROJ:  y = m + n tau e^logs: gamma S_m from m; the logs error d <= gamma S_logs scales e^logs by e^d, and expf
         (2 ulp), n * tau and the product (1 rounding each) add 4 u relative, inside the 2^-20 floor; the final add
         rounds once more:                    |Δ| <= gamma S_m + |n tau e^logs| (gamma S_logs + 2^-20) + 2^-23 |y|
  conv_post: 224 terms + lrelu: |Δ| <= gamma_226 S + 2^-21 (tanh' <= 1; tanhf 2 ulp <= 2^-23 on |y| <= 1).
The measured ratios are printed for every case (DESIGN.md section 4.2 records them).

Exactness probe: dyadic data (weights integers / 8, activations integers / 2, slope 0.25, scale 0.5, bias integers / 4)
whose sums need far fewer than 24 bits is computed exactly in any summation order, so a linear epilogue must equal
fp64 bit for bit; a wrong tap, row, column or phase shows up with its position.

Sentinels: every output element outside the compared region holds a NaN with a payload before the launch and must
hold it after; inside, no sentinel may survive.  Mutation controls: corrupted packed weights must fail.
"""
import ctypes
import importlib.util
import math
import os
import re
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SENT = 0x7FC0DEAD
U = 2.0 ** -24
SAME = "same"


def gamma(m):
    return m * U / (1 - m * U)


def load_kcf():
    spec = importlib.util.spec_from_file_location("kc_f32", os.path.join(HERE, "kernelcheck", "kc_f32.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def kcf():
    h = load_kcf().Harness()      # a missing harness is an error, not a skip
    h.setup()
    return h


def sentinel_like(shape):
    return torch.full(shape, SENT, dtype=torch.int32).view(torch.float32)


def is_sent(t):
    return t.view(torch.int32) == SENT


def lrelu(a, slope):
    return torch.where(a >= 0, a, a * slope)


def tmask(lims, T):
    return torch.arange(T)[None, None, :] < torch.as_tensor(lims)[:, None, None]     # [B][1][T] bool


def paired(rows):
    """packed row p -> natural row, the documented interleave (tests/test_convpack_host.py checks the library's)."""
    h = rows // 2
    return [4 * (p // 8) + p % 8 if p % 8 < 4 else h + 4 * (p // 8) + p % 8 - 4 for p in range(rows)]


def r4(n):
    return (n + 3) // 4 * 4


# ------------------------------------------------------------------------------------------------ one conv
class Case:
    def __init__(self, name, variant, cin, rows, tmax, lens, *, lens_out=SAME, mul=1, slope=1.0, bias_bs=False, res=False,
                 accum=False, scale=1.0, split=0, first=False, sign=1.0, ups=None, proj=None, x_pitch=None, tau=0.7):
        self.__dict__.update({k: v for k, v in locals().items() if k != "self"})
        self.lens_out = lens if lens_out is SAME else lens_out
        self.B = len(lens) if lens is not None else (len(self.lens_out) if self.lens_out is not None else 2)
        self.Tt = tmax * mul                                       # the kernel's time axis
        lim = lambda ls: [min(tmax, n) * mul for n in ls] if ls is not None else [self.Tt] * self.B
        self.lim_in, self.lim_out = lim(lens), lim(self.lens_out)
        self.os = ups[0] if ups else 1                             # output steps per kernel step
        self.Tout = self.Tt * self.os
        self.x_pitch = x_pitch or r4(self.Tt + 3)
        self.y_pitch = r4(self.Tout + 5)                           # room for sentinels past the time axis

    def ych(self, v):
        """channels of y (and of s for RESSKIP)."""
        return {"GATE": self.rows // 2, "PROJ": self.rows // 2, "UPS8": self.rows // 8, "UPS2": self.rows // 2,
                "RESSKIP": self.split or self.rows}.get(v.epi, self.rows)

    def slope_for(self, exact):
        return 0.25 if exact and self.slope not in (0.0, 1.0) else self.slope

    def scale_for(self, exact):
        return 0.5 if exact and self.scale != 1.0 else self.scale

    def make(self, v, gen, exact):
        B, cin, rows = self.B, self.cin, self.rows
        K = v.K
        ych = self.ych(v)
        if exact:
            ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=gen).float()
            x = ri(-4, 4, B, cin, self.x_pitch) / 2
            w = ri(-2, 2, rows, cin, K) / 8
            raw = ri(-2, 2, cin, rows // self.os, 2 * self.os) / 8 if self.ups else None
            bias = ri(-8, 8, B if self.bias_bs else 1, rows) / 4
            r, old = ri(-8, 8, B, rows, self.y_pitch) / 2, ri(-8, 8, B, ych, self.y_pitch) / 2
            s_old = ri(-8, 8, B, max(rows - self.split, 1), self.y_pitch) / 2
        else:
            rn = lambda *s: torch.randn(*s, generator=gen)
            x = rn(B, cin, self.x_pitch)
            w = rn(rows, cin, K) / math.sqrt(cin * K)
            raw = rn(cin, rows // self.os, 2 * self.os) / math.sqrt(cin * 2) if self.ups else None
            bias = 0.3 * rn(B if self.bias_bs else 1, rows)
            r = rn(B, rows, self.y_pitch)
            old, s_old = rn(B, ych, self.y_pitch), rn(B, max(rows - self.split, 1), self.y_pitch)
        noise = torch.randn(B, rows // 2, self.Tt, generator=gen) if v.epi == "PROJ" else None
        return dict(x=x, w=w, raw=raw, bias=bias, r=r, old=old, s_old=s_old, noise=noise)

    # ---- fp64 reference
    def reference(self, v, d, exact, noise=None, tau=None):
        """{out: (y64 [B][ch][Tout], allow, S)} -- allow = the proved bound (None for the exactness probe)."""
        B, Tt = self.B, self.Tt
        a = lrelu(d["x"][:, :, :Tt].double(), self.slope_for(exact)) * tmask(self.lim_in, Tt)
        if self.ups:
            s = self.os
            conv = lambda aa, ww: F.conv_transpose1d(aa, ww, stride=s, padding=s // 2)
            w = d["raw"].double()
        else:
            conv = lambda aa, ww: F.conv1d(aa, ww, padding=(v.K - 1) // 2 * v.DIL, dilation=v.DIL)
            w = d["w"].double()
        z = conv(a, w)
        S0 = None if exact else conv(a.abs(), w.abs())
        n = -(-self.cin // v.CI_CH) * v.CI_CH * v.K
        b = d["bias"].double()[:, :, None]
        if self.ups:
            b = b[:, : self.rows // self.os]
        To = self.Tout
        sl = lambda t, ch=None: t[:, :ch, :To].double()
        out = {}

        def lin(key, y, S, e):
            out[key] = (y, None if exact else gamma(n + e + 1) * S, S)

        if v.epi in ("LINEAR", "UPS8", "UPS2"):
            y, S, e = z + b, (None if exact else S0 + b.abs()), 1
            if self.res:
                y, e = y + sl(d["r"], self.rows), e + 1
                S = None if exact else S + sl(d["r"], self.rows).abs()
            if self.accum:
                y, e = y + sl(d["old"]), e + 1
                S = None if exact else S + sl(d["old"]).abs()
            sc = float(np.float32(self.scale_for(exact)))
            if sc != 1.0:
                y, e = y * sc, e + 1
                S = None if exact else S * abs(sc)
            lin("y", y, S, e)
        elif v.epi == "COUPLE":
            lin("y", sl(d["old"]) + self.sign * (z + b), None if exact else sl(d["old"]).abs() + S0 + b.abs(), 2)
        elif v.epi == "RESSKIP":
            sp = self.split
            if sp:
                lin("y", sl(d["old"]) + (z[:, :sp] + b[:, :sp]), None if exact else sl(d["old"]).abs() + S0[:, :sp] + b[:, :sp].abs(), 2)
            base = 0.0 if self.first else sl(d["s_old"])
            lin("s", base + (z[:, sp:] + b[:, sp:]),
                None if exact else (0.0 if self.first else sl(d["s_old"]).abs()) + S0[:, sp:] + b[:, sp:].abs(), 2)
        elif v.epi == "GATE":
            H = self.rows // 2
            za, zb = z[:, :H] + b[:, :H], z[:, H:] + b[:, H:]
            y = torch.tanh(za) * torch.sigmoid(zb)
            S = None if exact else (S0[:, :H] + b[:, :H].abs()) + (S0[:, H:] + b[:, H:].abs()) / 4
            out["y"] = (y, None if exact else gamma(n + 2) * S + 2.0 ** -20, S)
        elif v.epi == "PROJ":
            H = self.rows // 2
            m, logs = z[:, :H] + b[:, :H], z[:, H:] + b[:, H:]
            tau_t = torch.as_tensor(tau, dtype=torch.float64).reshape(-1, 1, 1)
            ne = noise.double() * tau_t * torch.exp(logs)
            y = m + ne
            Sm, Sl = S0[:, :H] + b[:, :H].abs(), S0[:, H:] + b[:, H:].abs()
            g = gamma(n + 2)
            out["y"] = (y, g * Sm + ne.abs() * (g * Sl + 2.0 ** -20) + 2.0 ** -23 * y.abs(), Sm)
        return out

    # ---- the launch
    def run(self, kcf, v, d, exact, w_packed=None, proj=None):
        """Launch on the GPU with sentinel-filled outputs; returns the output buffers on the CPU."""
        dev = "cuda"
        B, rows = self.B, self.rows
        if w_packed is None:
            w_packed = self.pack(kcf, v, d)
        w = torch.from_numpy(w_packed).to(dev)
        perm = paired(rows) if v.epi in ("GATE", "PROJ") else list(range(rows))
        bias = d["bias"][:, perm].contiguous()
        if self.ups:
            bias = d["bias"][:, : rows // self.os].contiguous()
        inside = tmask([l * self.os for l in self.lim_out], self.y_pitch)
        ych = self.ych(v)
        y = sentinel_like((B, ych, self.y_pitch))
        if self.accum or v.epi == "COUPLE" or (v.epi == "RESSKIP" and self.split):
            y = torch.where(inside, d["old"], y)
        s = None
        if v.epi == "RESSKIP" and self.split < rows:
            s = sentinel_like((B, rows - self.split, self.y_pitch))
            if not self.first:
                s = torch.where(inside, d["s_old"], s)
            s = s.to(dev)
        y = y.to(dev)
        lens = lambda ls: torch.tensor(ls, dtype=torch.int64, device=dev) if ls is not None else None
        kw = dict(rows=rows, tmax=self.tmax, mul_in=self.mul, mul_out=self.mul, lens_in=lens(self.lens),
                  lens_out=lens(self.lens_out), slope=self.slope_for(exact), scale=self.scale_for(exact), sign=self.sign,
                  split=self.split, flags=(1 if self.accum else 0) | (2 if self.first else 0),
                  bias_bs=rows if self.bias_bs else 0)
        if self.res:
            kw["r"] = d["r"].to(dev)
        if s is not None:
            kw["s"] = s
        if v.epi == "PROJ":
            kw.update(proj or {})
        kcf.conv(v.name, d["x"].to(dev), w, bias.reshape(-1).to(dev), y, **kw)
        out = {"y": y.cpu()}
        if s is not None:
            out["s"] = s.cpu()
        return out

    def pack(self, kcf, v, d):
        if self.ups:
            return kcf.pack_ups(v.name, d["raw"].numpy(), self.os)
        return kcf.pack(v.name, d["w"].numpy(), paired=v.epi in ("GATE", "PROJ"))


def measure(case, v, got, ref, exact):
    """{out: (max|Δ|/S, max|Δ|/allow, max|Δ|/rms, sentinels ok, exact)} over each item's limit."""
    inside = tmask([l * case.os for l in case.lim_out], case.y_pitch)
    res = {}
    for k, (y64, allow, S) in ref.items():
        g = got[k]
        m = inside.expand_as(g)
        sent_ok = bool(is_sent(g[~m]).all()) and not bool(is_sent(g[m]).any())
        gi = g[:, :, : case.Tout].double()
        mi = m[:, :, : case.Tout]
        diff = (gi - y64).abs()
        diff = torch.where(torch.isnan(gi), torch.full_like(diff, math.inf), diff)[mi]
        yv = y64[mi]
        rms = float(yv.pow(2).mean().sqrt()) if yv.numel() else 1.0
        dmax = float(diff.max()) if diff.numel() else 0.0
        ex = bool((g[:, :, : case.Tout][mi] == yv.float()).all())
        if allow is None:
            res[k] = (math.nan, math.nan, dmax / max(rms, 1e-300), sent_ok, ex)
        else:
            rs = float((diff / S[mi].clamp_min(1e-300)).max()) if diff.numel() else 0.0
            ra = float((diff / allow[mi]).max()) if diff.numel() else 0.0
            res[k] = (rs, ra, dmax / max(rms, 1e-300), sent_ok, ex)
    if v.epi == "RESSKIP" and not case.split:
        res["y_untouched"] = (0.0, 0.0, 0.0, bool(is_sent(got["y"]).all()), True)
    return res


def passes(res, exact):
    return all(s and (e if exact else ra <= 1.0) for _, ra, _, s, e in res.values())


def report(tag, res):
    for k, (rs, ra, rr, s, e) in res.items():
        print(f"[conv_f32] {tag:<34} {k:<11} |d|/S={rs:.3e} |d|/allow={ra:.3e} |d|/rms={rr:.3e} "
              f"sentinel={'ok' if s else 'BAD'} exact={'yes' if e else 'no'}")


# ------------------------------------------------------------------------------------------------ the cases
def edge_lens(T_T):
    """0, 1, the tile edges, one past tmax; tmax = 3 T_T + 3 (four tiles, not a multiple of 4)."""
    tmax = 3 * T_T + 3
    return tmax, (0, 1, T_T - 1, T_T, T_T + 1, tmax + 7)


def library_cases():
    cs = []
    H = 192
    tm, el = edge_lens(128)
    # posterior encoder pre: 4-byte staging for any spectrogram pitch, 16-byte staging when it is a multiple of 4
    cs.append(Case("enc_pre_pitch_odd", "ENC_PRE", 513, H, tm, el, x_pitch=tm + 4 - (tm + 4) % 2 + 1))
    cs.append(Case("enc_pre_pitch4", "ENC_PRE", 513, H, tm, el, x_pitch=r4(tm + 1)))
    cs.append(Case("enc_pre16_pitch4", "FLOW_PRE", 513, H, tm, el, x_pitch=r4(tm + 1)))
    cs.append(Case("flow_pre_nolens", "FLOW_PRE", 96, H, tm, None, lens_out=None))
    cs.append(Case("wn_in_gate", "WN_IN", H, 2 * H, tm, el, bias_bs=True))
    for first in (False, True):
        cs.append(Case(f"wn_rs_split192_first{int(first)}", "WN_RS", H, 2 * H, tm, el, split=H, first=first))
        cs.append(Case(f"wn_rs_split0_first{int(first)}", "WN_RS", H, H, tm, el, split=0, first=first))
    for mode in ("noise", "philox", "items"):
        cs.append(Case(f"enc_proj_{mode}", "ENC_PROJ", H, 2 * H, tm, el, proj=mode))
    tm2, el2 = edge_lens(256)
    for sign in (1.0, -1.0):
        cs.append(Case(f"flow_post_sign{int(sign):+d}", "FLOW_POST", H, 96, tm2, el2, sign=sign))
    # generator: conv_pre (input cut at the frame lengths, output over the whole call), upsamplers, ResBlocks
    cs.append(Case("conv_pre", "A_K7D1", H, 512, 259, (259, 100, 1, 0), lens_out=None, bias_bs=True))
    cs.append(Case("ups0_s8_mul1", "UPS8_A", 512, 8 * 256, 259, (0, 1, 127, 128, 129, 266), slope=0.1, ups=(8, 16)))
    cs.append(Case("ups1_s8_mul8", "UPS8_A", 256, 8 * 128, 33, (33, 11, 0, 1, 35), mul=8, slope=0.1, ups=(8, 16)))
    cs.append(Case("ups2_s2_mul64", "UPS2_A", 128, 2 * 64, 5, (5, 2, 0, 1, 7), mul=64, slope=0.1, ups=(2, 4)))
    cs.append(Case("ups3_s2_mul128", "UPS2_B", 64, 2 * 32, 7, (7, 3, 0, 1, 9), mul=128, slope=0.1, ups=(2, 4)))
    for vn, C, T_T in (("UPS2_A", 128, 128), ("UPS2_B", 64, 256)):
        t, l = edge_lens(T_T)
        cs.append(Case(f"{vn.lower()}_mul1_edges", vn, C, C, t, l, slope=0.1, ups=(2, 4)))
    n = 0
    for cls, C, mul, tmax, T_T in (("A", 256, 8, 50, 128), ("A", 128, 64, 7, 128), ("B", 64, 128, 7, 256),
                                   ("C", 32, 256, 7, 512)):
        for K in (3, 7, 11):
            for D in (1, 3, 5):
                kw = dict(slope=0.1, res=D == 1 or n % 2 == 0, accum=n % 3 == 1, scale=1 / 3 if n % 4 == 0 else 1.0)
                cs.append(Case(f"rb_c{C}_k{K}_d{D}_mul{mul}", f"{cls}_K{K}D{D}", C, C, tmax,
                               (tmax, tmax // 3 + 1, 0, 1, tmax + 2), mul=mul, **kw))
                if C != 256:      # every ResBlock variant once more at mul 1 with limits that are not multiples of 4
                    t, l = edge_lens(T_T)
                    cs.append(Case(f"rb_c{C}_k{K}_d{D}_mul1_edges", f"{cls}_K{K}D{D}", C, C, t, l, **kw))
                n += 1
    # TTS text side: FFN conv_1 / conv_2 (relu as the second conv's input activation) and the duration predictor
    t, l = edge_lens(128)
    cs.append(Case("tts_ffn1", "A_K3D1", H, 768, 121, (121, 37, 1, 0)))
    cs.append(Case("tts_ffn2_relu", "TXT_K3D1", 768, H, t, l, slope=0.0))
    cs.append(Case("tts_dp_conv2_relu", "A_K3D1", 256, 256, 121, (121, 37, 1, 0), slope=0.0))
    return cs


CASES = {c.name: c for c in library_cases()}
_CACHE = {}


def skipped(kcf, name, exact):
    """the exactness probe needs a linear epilogue"""
    return exact and kcf.variants[CASES[name].variant].epi in ("GATE", "PROJ")


def prepared(kcf, name, exact):
    """(case, variant, data, reference), computed once per case and data kind."""
    key = (name, exact)
    if key not in _CACHE:
        c = CASES[name]
        v = kcf.variants[c.variant]
        gen = torch.Generator().manual_seed(zlib.crc32(name.encode()) + int(exact))
        d = c.make(v, gen, exact)
        proj, noise, tau = None, None, None
        if v.epi == "PROJ":
            proj, noise, tau = proj_inputs(c, d, gen)
        _CACHE[key] = (c, v, d, c.reference(v, d, exact, noise, tau), proj)
    return _CACHE[key]


def proj_inputs(c, d, gen):
    """Launch arguments and the expected noise of one PROJ case: an explicit noise tensor, or in-kernel Philox draws
    with the call's key (stream b, frame t) or with per-item seed / stream / frame0 / tau."""
    from openvoice_b200 import _native
    B, H, Tt = c.B, c.rows // 2, c.Tt
    if c.proj == "noise":
        return dict(r=d["noise"].to("cuda"), tau=c.tau), d["noise"], [float(np.float32(c.tau))] * B
    if c.proj == "philox":
        seed, tau = 0x5EED1234ABCD, 0.6
        noise = torch.stack([_native.philox_normals(seed, b, 0, H, 0, Tt).cpu() for b in range(B)])
        return dict(callp=dict(seed=seed, tau=tau), seed=777, tau=9.0), noise, [float(np.float32(tau))] * B
    seeds = [int(s) for s in torch.randint(0, 2 ** 62, (B,), generator=gen)]
    streams = [int(s) for s in torch.randint(0, 1000, (B,), generator=gen)]
    frames = [int(s) for s in torch.randint(0, 2 ** 20, (B,), generator=gen)]
    taus = [float(np.float32(0.2 + 0.15 * b)) for b in range(B)]
    noise = torch.stack([_native.philox_normals(seeds[b], streams[b], 0, H, frames[b], Tt).cpu() for b in range(B)])
    dev = "cuda"
    items = dict(seed=torch.tensor(seeds, dtype=torch.int64, device=dev),
                 stream=torch.tensor(streams, dtype=torch.int64, device=dev),
                 frame0=torch.tensor(frames, dtype=torch.int64, device=dev),
                 tau=torch.tensor(taus, dtype=torch.float32, device=dev))
    return dict(callp=dict(seed=1, tau=5.0, items=items)), noise, taus


def test_every_variant_is_covered(kcf):
    src = open(os.path.join(HERE, "..", "openvoice_b200", "csrc", "ovc_variants.h")).read()
    names = set(re.findall(r"^\s*X\((\w+),", src, re.M))
    assert len(names) == 37 and names == set(kcf.variants)
    assert {c.variant for c in CASES.values()} == names


@pytest.mark.parametrize("name", list(CASES))
def test_library_layer(kcf, name):
    """Each conv1d_f32 launch the library makes for the default and the TTS checkpoints, at its own geometry and mul,
    plus every generator variant at mul 1 with limits at the tile edges: random data against the proved gate, dyadic
    data bit for bit (linear epilogues), sentinels around every output."""
    for exact in (False, True):
        if skipped(kcf, name, exact):
            continue
        c, v, d, ref, proj = prepared(kcf, name, exact)
        got = c.run(kcf, v, d, exact, proj=proj)
        res = measure(c, v, got, ref, exact)
        report(name + (" exact" if exact else ""), res)
        assert passes(res, exact), (name, exact, res)


@pytest.mark.parametrize("name", ["rb_c256_k11_d5_mul8", "ups0_s8_mul1", "enc_pre_pitch_odd", "wn_in_gate"])
def test_mutation_controls_fail(kcf, name):
    """Corrupted packed weights must fail the gate (random data) and the exactness probe (dyadic data, linear
    epilogues): taps 0 and K-1 swapped (ENC_PRE has one tap: no swap), the last ci-chunk of the last row tile zeroed
    (for ENC_PRE the partial chunk that holds channel 512 alone)."""
    for exact in (False, True):
        if skipped(kcf, name, exact):
            continue
        c, v, d, ref, proj = prepared(kcf, name, exact)
        packed = c.pack(kcf, v, d)
        n_chunks = -(-c.cin // v.CI_CH)
        muts = {"chunk": kcf.corrupt(v.name, packed, c.rows, c.cin, "chunk", n_chunks - 1, c.rows // v.CO_T - 1)}
        if v.K > 1:
            muts["swap"] = kcf.corrupt(v.name, packed, c.rows, c.cin, "swap", 0, v.K - 1)
        for kind, mp in muts.items():
            res = measure(c, v, c.run(kcf, v, d, exact, w_packed=mp, proj=proj), ref, exact)
            report(f"{name} mutant {kind}" + (" exact" if exact else ""), res)
            assert not passes(res, exact), (name, kind, exact)


# ------------------------------------------------------------------------------------------------ conv_post
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("mul,tmax,lens,y_len", [(256, 5, (5, 2, 0, 1, 7), 5 * 256 + 256),
                                                 (1, 1031, (1031, 517, 0, 1, 2000, 255), 1035)])
def test_conv_post(kcf, channels_last, mul, tmax, lens, y_len):
    """tanh(conv1d(lrelu_0.01(x), w, pad 3)) in the kernel's own layout: within the gate inside each limit, exactly 0
    in [lim, y_len), the sentinel past y_len."""
    gen = torch.Generator().manual_seed(mul + int(channels_last))
    B, T, dev = len(lens), tmax * mul, "cuda"
    if not channels_last:
        y_len = y_len if y_len % 4 == 0 else r4(y_len)
    y_pitch = r4(y_len + 9)
    lim = [min(tmax, n) * mul for n in lens]
    x = torch.randn(B, 32, r4(T + 3), generator=gen)                   # [C][pitch]
    w = torch.randn(1, 32, 7, generator=gen) / math.sqrt(32 * 7) * 3
    a = lrelu(x[:, :, :T].double(), 0.01) * tmask(lim, T)
    z = F.conv1d(a, w.double(), padding=3)[:, 0]
    S = F.conv1d(a.abs(), w.double().abs(), padding=3)[:, 0]
    y64, allow = torch.tanh(z), gamma(226) * S + 2.0 ** -21
    xin = x[:, :, :T].transpose(1, 2).contiguous() if channels_last else x
    y = sentinel_like((B, y_pitch)).to(dev)
    kcf.conv_post(xin.to(dev), w.reshape(-1).to(dev), y, y_len=y_len, tmax=tmax, mul=mul,
                  lens=torch.tensor(lens, dtype=torch.int64, device=dev), channels_last=channels_last)
    y = y.cpu()
    t = torch.arange(y_pitch)[None, :]
    li = torch.tensor(lim)[:, None]
    inside, zero, past = t < torch.minimum(li, torch.tensor(y_len)), (t >= li) & (t < y_len), (t >= y_len).expand(B, -1)
    d = (y[:, :T].double() - y64).abs()[inside[:, :T]]
    ratio = float((d / allow[inside[:, :T]]).max())
    print(f"[conv_f32] conv_post cl={int(channels_last)} mul={mul} |d|/S={float((d / S[inside[:, :T]].clamp_min(1e-300)).max()):.3e} "
          f"|d|/allow={ratio:.3e} |d|/rms={float(d.max() / y64[inside[:, :T]].pow(2).mean().sqrt()):.3e}")
    assert ratio <= 1.0
    assert (y[zero].view(torch.int32) == 0).all(), "[lim, y_len) must be +0"
    assert is_sent(y[past]).all(), "a store past y_len"


def test_conv_post_refuses_a_partial_vector(kcf):
    """The [C][pitch] kernel stores whole float4s: a y_len that is not a multiple of 4 is refused on the host."""
    dev = "cuda"
    x = torch.zeros(1, 32, 16, device=dev)
    y = torch.zeros(1, 32, device=dev)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        kcf.conv_post(x, torch.zeros(224, device=dev), y, y_len=13, tmax=13, mul=1)


def test_bad_launches_are_refused(kcf):
    """Argument mistakes come back as errors from the host checks, never as a device fault."""
    dev = "cuda"
    x = torch.zeros(1, 192, 132, device=dev)
    w = torch.zeros(kcf.packed_floats("WN_RS", 384, 192), device=dev)
    b = torch.zeros(384, device=dev)
    y = torch.zeros(1, 192, 132, device=dev)
    s = torch.zeros(1, 192, 132, device=dev)
    ok = dict(rows=384, tmax=128, s=s, split=192)
    kcf.conv("WN_RS", x, w, b, y, **ok)
    for bad, match in ((dict(split=100), "split"), (dict(tmax=140), "pitch"), (dict(rows=400), "rows"),
                       (dict(s=None), "null")):
        with pytest.raises(RuntimeError, match=match):
            kcf.conv("WN_RS", x, w, b, y, **{**ok, **bad})
    with pytest.raises(RuntimeError, match="w:"):
        kcf.conv("WN_RS", x, w[:-4].contiguous(), b, y, **ok)
    xo = torch.zeros(1, 192, 131, device=dev)                 # pitch 131: no 16-byte cp.async
    with pytest.raises(RuntimeError, match="16-byte"):
        kcf.conv("FLOW_PRE", xo, torch.zeros(kcf.packed_floats("FLOW_PRE", 192, 192), device=dev), b, y, rows=192, tmax=128)
    a = kcf.lib.kc_conv.argtypes[0]._type_()
    a.variant = 1000
    assert kcf.lib.kc_conv(ctypes.byref(a)) != 0 and "unknown variant" in kcf.lib.kc_error().decode()
