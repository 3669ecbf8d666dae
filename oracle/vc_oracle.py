"""CPU oracle for the OpenVoice tone-colour-converter hot path.

TEST INFRASTRUCTURE ONLY.  This file is the *checker*: a functional, module-free
restatement (torch CPU, fp32 or fp64) of what the reference computes on
``ToneColorConverter.convert -> SynthesizerTrn.voice_conversion``.  Only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` leg may import it.  The product (``openvoice_b200``) never
does: its only compute path is the sm_90a CUDA library and it fails loudly
without it.

Parity pinning: ``oracle/make_golden.py`` imports the real reference from the
checkout named by ``OPENVOICE_REFERENCE``, drives the reference's own
``SynthesizerTrn.voice_conversion`` / ``ToneColorConverter.convert`` /
``spectrogram_torch`` / ``ReferenceEncoder`` on the seeded synthetic checkpoint
below and commits the results under ``tests/golden/``;
``tests/test_oracle_golden.py`` checks this file against those vectors (the
reference ships no tests / golden vectors of its own -- SURVEY.md section 8c).

Every function cites the reference lines it follows (paths relative to
the reference repository's root).  Tensors are ``[B, C, T]`` like the reference.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F

StateDict = Dict[str, torch.Tensor]

LRELU_SLOPE = 0.1  # openvoice/modules.py:14

# Released converter hyper-parameters (SURVEY.md appendix A.1; the json that ships
# with checkpoints/converter/config.json).  V2 = same + zero_g + _version_.
DEFAULT_HPARAMS = {
    "data": {
        "sampling_rate": 22050,
        "filter_length": 1024,
        "hop_length": 256,
        "win_length": 1024,
        "n_speakers": 0,
    },
    "model": {
        "zero_g": False,
        "inter_channels": 192,
        "hidden_channels": 192,
        "filter_channels": 768,
        "n_heads": 2,
        "n_layers": 6,
        "kernel_size": 3,
        "p_dropout": 0.1,
        "resblock": "1",
        "resblock_kernel_sizes": [3, 7, 11],
        "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
        "upsample_rates": [8, 8, 2, 2],
        "upsample_initial_channel": 512,
        "upsample_kernel_sizes": [16, 16, 4, 4],
        "n_layers_q": 3,
        "use_spectral_norm": False,
        "gin_channels": 256,
    },
}

ENC_Q_LAYERS = 16  # openvoice/models.py:438-446 (hard-coded k=5, dilation_rate=1, n_layers=16)
FLOW_LAYERS = 4  # openvoice/models.py:448
N_FLOWS = 4  # openvoice/models.py:375
WN_KERNEL = 5


# --------------------------------------------------------------------------------------
# parameters
# --------------------------------------------------------------------------------------
def state_dict_schema(hp: Optional[dict] = None, with_ref_enc: bool = True) -> Dict[str, tuple]:
    """Names and shapes of the converter checkpoint (SURVEY.md appendix A.2).

    Follows the constructors at openvoice/models.py:182-211 (PosteriorEncoder),
    :224-270 (Generator), :367-388 (ResidualCouplingBlock), :301-338 (ReferenceEncoder),
    openvoice/modules.py:133-183 (WN), :221-294 (ResBlock1), :402-435 (coupling layer).
    Old-style weight-norm stores ``weight_g`` / ``weight_v``.
    """
    hp = hp or DEFAULT_HPARAMS
    m = hp["model"]
    spec = hp["data"]["filter_length"] // 2 + 1
    H = m["hidden_channels"]
    C = m["inter_channels"]
    gin = m["gin_channels"]
    out: Dict[str, tuple] = {}

    def wn(prefix: str, n_layers: int) -> None:
        out[f"{prefix}.cond_layer.bias"] = (2 * H * n_layers,)
        out[f"{prefix}.cond_layer.weight_g"] = (2 * H * n_layers, 1, 1)
        out[f"{prefix}.cond_layer.weight_v"] = (2 * H * n_layers, gin, 1)
        for i in range(n_layers):
            out[f"{prefix}.in_layers.{i}.bias"] = (2 * H,)
            out[f"{prefix}.in_layers.{i}.weight_g"] = (2 * H, 1, 1)
            out[f"{prefix}.in_layers.{i}.weight_v"] = (2 * H, H, WN_KERNEL)
            rs = 2 * H if i < n_layers - 1 else H
            out[f"{prefix}.res_skip_layers.{i}.bias"] = (rs,)
            out[f"{prefix}.res_skip_layers.{i}.weight_g"] = (rs, 1, 1)
            out[f"{prefix}.res_skip_layers.{i}.weight_v"] = (rs, H, 1)

    out["enc_q.pre.weight"] = (H, spec, 1)
    out["enc_q.pre.bias"] = (H,)
    wn("enc_q.enc", ENC_Q_LAYERS)
    out["enc_q.proj.weight"] = (2 * C, H, 1)
    out["enc_q.proj.bias"] = (2 * C,)

    for f in range(N_FLOWS):
        p = f"flow.flows.{2 * f}"
        out[f"{p}.pre.weight"] = (H, C // 2, 1)
        out[f"{p}.pre.bias"] = (H,)
        wn(f"{p}.enc", FLOW_LAYERS)
        out[f"{p}.post.weight"] = (C // 2, H, 1)
        out[f"{p}.post.bias"] = (C // 2,)

    U = m["upsample_initial_channel"]
    out["dec.conv_pre.weight"] = (U, C, 7)
    out["dec.conv_pre.bias"] = (U,)
    out["dec.cond.weight"] = (U, gin, 1)
    out["dec.cond.bias"] = (U,)
    ch = U
    for i, (u, k) in enumerate(zip(m["upsample_rates"], m["upsample_kernel_sizes"])):
        cin, cout = U // (2 ** i), U // (2 ** (i + 1))
        out[f"dec.ups.{i}.bias"] = (cout,)
        out[f"dec.ups.{i}.weight_g"] = (cin, 1, 1)
        out[f"dec.ups.{i}.weight_v"] = (cin, cout, k)
        ch = cout
        for j, ks in enumerate(m["resblock_kernel_sizes"]):
            rb = f"dec.resblocks.{i * len(m['resblock_kernel_sizes']) + j}"
            for cv in ("convs1", "convs2"):
                for d in range(3):
                    out[f"{rb}.{cv}.{d}.bias"] = (ch,)
                    out[f"{rb}.{cv}.{d}.weight_g"] = (ch, 1, 1)
                    out[f"{rb}.{cv}.{d}.weight_v"] = (ch, ch, ks)
    out["dec.conv_post.weight"] = (1, ch, 7)

    if with_ref_enc:
        filters = [1, 32, 32, 64, 64, 128, 128]
        for i in range(6):
            out[f"ref_enc.convs.{i}.bias"] = (filters[i + 1],)
            out[f"ref_enc.convs.{i}.weight_g"] = (filters[i + 1], 1, 1, 1)
            out[f"ref_enc.convs.{i}.weight_v"] = (filters[i + 1], filters[i], 3, 3)
        L = spec
        for _ in range(6):
            L = (L - 3 + 2) // 2 + 1
        out["ref_enc.gru.weight_ih_l0"] = (384, 128 * L)
        out["ref_enc.gru.weight_hh_l0"] = (384, 128)
        out["ref_enc.gru.bias_ih_l0"] = (384,)
        out["ref_enc.gru.bias_hh_l0"] = (384,)
        out["ref_enc.proj.weight"] = (gin, 128)
        out["ref_enc.proj.bias"] = (gin,)
        out["ref_enc.layernorm.weight"] = (spec,)
        out["ref_enc.layernorm.bias"] = (spec,)
    return out


def synthetic_state_dict(seed: int = 1234, hp: Optional[dict] = None) -> StateDict:
    """Seeded synthetic checkpoint (no released checkpoint is reachable offline).

    Recipe of SURVEY.md appendix B.3: N(0,1)*gain/sqrt(fan_in) for weights, small
    biases, weight_g = ||weight_v|| so the effective weight equals v.  It gives O(1)
    activations in every block, a non-trivial flow (``post`` is NOT zero as the
    default init at openvoice/modules.py:434-435 would make it) and an unsaturated
    final tanh.
    """
    hp = hp or DEFAULT_HPARAMS
    rates = hp["model"]["upsample_rates"]
    schema = state_dict_schema(hp)
    gen = torch.Generator().manual_seed(seed)
    sd: StateDict = {}
    for name in sorted(schema):
        shape = schema[name]
        if name.endswith("weight_g"):
            continue
        if name.endswith("bias") or name.startswith("ref_enc.gru.bias"):
            sd[name] = torch.randn(shape, generator=gen) * 0.02
            continue
        if name == "ref_enc.layernorm.weight":
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=gen)
            continue
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        gain = 1.0
        if name.startswith("dec.ups."):
            i = int(name.split(".")[2])
            fan_in = shape[0] * shape[2] / rates[i]
        elif name.startswith("enc_q.proj"):
            gain = 0.3
        elif name.startswith("enc_q.pre"):
            gain = 0.5
        elif ".res_skip_layers." in name:
            gain = 0.5
        elif name.startswith("dec.resblocks."):
            gain = 0.35
        elif name.startswith("dec.conv_post"):
            gain = 0.5
        elif name.endswith(".post.weight"):
            gain = 0.5
        sd[name] = torch.randn(shape, generator=gen) * (gain / math.sqrt(fan_in))
    for name, shape in schema.items():
        if name.endswith("weight_g"):
            v = sd[name[:-1] + "v"]
            sd[name] = v.reshape(v.shape[0], -1).norm(dim=1).reshape(shape)
    return sd


def synthetic_inputs(B: int, T: int, seed: int = 0, spec_channels: int = 513, gin: int = 256,
                     inter: int = 192, lengths: Optional[Sequence[int]] = None):
    """Seeded (spec, lengths, g_src, g_tgt, noise) -- SURVEY.md appendix B.3 input recipe."""
    gen = torch.Generator().manual_seed(10_000 + seed)
    spec = 8.0 * torch.rand(B, spec_channels, T, generator=gen) ** 4
    g_src = 0.1 * torch.randn(B, gin, 1, generator=gen)
    g_tgt = 0.1 * torch.randn(B, gin, 1, generator=gen)
    noise = torch.randn(B, inter, T, generator=gen)
    if lengths is None:
        lengths = [T] * B
    return spec, torch.tensor(list(lengths), dtype=torch.int64), g_src, g_tgt, noise


# --------------------------------------------------------------------------------------
# building blocks
# --------------------------------------------------------------------------------------
def fold_weight_norm(v: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """w = g * v / ||v||, norm over every dim except 0 (torch.nn.utils.weight_norm, dim=0;
    used at openvoice/modules.py:160,172,182 and openvoice/models.py:247 -- for
    ConvTranspose1d dim 0 is Cin)."""
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(g.shape)
    return v * (g / n)


def _w(sd: StateDict, prefix: str) -> torch.Tensor:
    if f"{prefix}.weight" in sd:
        return sd[f"{prefix}.weight"]
    return fold_weight_norm(sd[f"{prefix}.weight_v"], sd[f"{prefix}.weight_g"])


def sequence_mask(lengths: torch.Tensor, T: int, dtype) -> torch.Tensor:
    """[B,1,T] float mask, t < length (openvoice/commons.py:121-125, models.py:213)."""
    return (torch.arange(T, device=lengths.device)[None, :] < lengths[:, None]).unsqueeze(1).to(dtype)


def wn_forward(sd: StateDict, prefix: str, x: torch.Tensor, mask: torch.Tensor,
               g: torch.Tensor, n_layers: int) -> torch.Tensor:
    """Gated conv stack (openvoice/modules.py:185-210; gate = commons.py:100-107)."""
    H = x.shape[1]
    cond = F.conv1d(g, _w(sd, f"{prefix}.cond_layer"), sd[f"{prefix}.cond_layer.bias"])
    skip = torch.zeros_like(x)
    for i in range(n_layers):
        a = F.conv1d(x, _w(sd, f"{prefix}.in_layers.{i}"), sd[f"{prefix}.in_layers.{i}.bias"],
                     padding=(WN_KERNEL - 1) // 2)
        a = a + cond[:, 2 * H * i: 2 * H * (i + 1), :]
        acts = torch.tanh(a[:, :H]) * torch.sigmoid(a[:, H:])
        rs = F.conv1d(acts, _w(sd, f"{prefix}.res_skip_layers.{i}"),
                      sd[f"{prefix}.res_skip_layers.{i}.bias"])
        if i < n_layers - 1:
            x = (x + rs[:, :H]) * mask
            skip = skip + rs[:, H:]
        else:
            skip = skip + rs
    return skip * mask


def posterior_encoder(sd: StateDict, spec: torch.Tensor, lengths: torch.Tensor, g: torch.Tensor,
                      noise: torch.Tensor, tau: float):
    """openvoice/models.py:212-221; ``noise`` stands in for randn_like at :220."""
    mask = sequence_mask(lengths, spec.shape[2], spec.dtype)
    x = F.conv1d(spec, sd["enc_q.pre.weight"], sd["enc_q.pre.bias"]) * mask
    x = wn_forward(sd, "enc_q.enc", x, mask, g, ENC_Q_LAYERS)
    stats = F.conv1d(x, sd["enc_q.proj.weight"], sd["enc_q.proj.bias"]) * mask
    C = stats.shape[1] // 2
    m, logs = stats[:, :C], stats[:, C:]
    z = (m + noise * tau * torch.exp(logs)) * mask
    return z, m, logs, mask


def coupling_layer(sd: StateDict, prefix: str, x: torch.Tensor, mask: torch.Tensor,
                   g: torch.Tensor, reverse: bool) -> torch.Tensor:
    """Mean-only additive coupling (openvoice/modules.py:437-456 with mean_only=True)."""
    half = x.shape[1] // 2
    x0, x1 = x[:, :half], x[:, half:]
    h = F.conv1d(x0, sd[f"{prefix}.pre.weight"], sd[f"{prefix}.pre.bias"]) * mask
    h = wn_forward(sd, f"{prefix}.enc", h, mask, g, FLOW_LAYERS)
    m = F.conv1d(h, sd[f"{prefix}.post.weight"], sd[f"{prefix}.post.bias"]) * mask
    if not reverse:
        x1 = m + x1 * mask
    else:
        x1 = (x1 - m) * mask
    return torch.cat([x0, x1], dim=1)


def flow(sd: StateDict, x: torch.Tensor, mask: torch.Tensor, g: torch.Tensor,
         reverse: bool) -> torch.Tensor:
    """[coupling, channel-flip] x4, or the reversed list (openvoice/models.py:390-397,
    Flip = openvoice/modules.py:374-381)."""
    if not reverse:
        for f in range(N_FLOWS):
            x = coupling_layer(sd, f"flow.flows.{2 * f}", x, mask, g, False)
            x = torch.flip(x, [1])
    else:
        for f in reversed(range(N_FLOWS)):
            x = torch.flip(x, [1])
            x = coupling_layer(sd, f"flow.flows.{2 * f}", x, mask, g, True)
    return x


def resblock1(sd: StateDict, prefix: str, x: torch.Tensor, k: int,
              dilations: Sequence[int]) -> torch.Tensor:
    """openvoice/modules.py:296-309 with x_mask=None."""
    for j, d in enumerate(dilations):
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = F.conv1d(xt, _w(sd, f"{prefix}.convs1.{j}"), sd[f"{prefix}.convs1.{j}.bias"],
                      dilation=d, padding=d * (k - 1) // 2)
        xt = F.leaky_relu(xt, LRELU_SLOPE)
        xt = F.conv1d(xt, _w(sd, f"{prefix}.convs2.{j}"), sd[f"{prefix}.convs2.{j}.bias"],
                      padding=(k - 1) // 2)
        x = xt + x
    return x


def generator(sd: StateDict, z: torch.Tensor, g: torch.Tensor, hp: Optional[dict] = None,
              taps: Optional[dict] = None) -> torch.Tensor:
    """HiFi-GAN decoder (openvoice/models.py:272-291)."""
    m = (hp or DEFAULT_HPARAMS)["model"]
    ks, ds = m["resblock_kernel_sizes"], m["resblock_dilation_sizes"]
    x = F.conv1d(z, sd["dec.conv_pre.weight"], sd["dec.conv_pre.bias"], padding=3)
    x = x + F.conv1d(g, sd["dec.cond.weight"], sd["dec.cond.bias"])
    if taps is not None:
        taps["dec.pre"] = x
    for i, (u, k) in enumerate(zip(m["upsample_rates"], m["upsample_kernel_sizes"])):
        x = F.leaky_relu(x, LRELU_SLOPE)
        x = F.conv_transpose1d(x, _w(sd, f"dec.ups.{i}"), sd[f"dec.ups.{i}.bias"],
                               stride=u, padding=(k - u) // 2)
        if taps is not None:
            taps[f"dec.ups{i}"] = x
        xs = None
        for j in range(len(ks)):
            r = resblock1(sd, f"dec.resblocks.{i * len(ks) + j}", x, ks[j], ds[j])
            xs = r if xs is None else xs + r
        x = xs / len(ks)
        if taps is not None:
            taps[f"dec.stage{i}"] = x
    x = F.leaky_relu(x)  # default slope 0.01 -- openvoice/models.py:287
    x = F.conv1d(x, sd["dec.conv_post.weight"], None, padding=3)  # bias=False, models.py:266
    return torch.tanh(x)


def voice_conversion(sd: StateDict, spec: torch.Tensor, lengths: torch.Tensor,
                     g_src: torch.Tensor, g_tgt: torch.Tensor, noise: torch.Tensor,
                     tau: float = 0.3, zero_g: bool = False, hp: Optional[dict] = None,
                     taps: Optional[dict] = None):
    """openvoice/models.py:492-499.  Returns (o_hat, y_mask, (z, z_p, z_hat))."""
    dt = spec.dtype
    if any(v.dtype != dt for v in sd.values()):
        sd = {k: v.to(dt) for k, v in sd.items()}
    ge = torch.zeros_like(g_src) if zero_g else g_src
    z, m_q, logs_q, mask = posterior_encoder(sd, spec, lengths, ge, noise.to(dt), tau)
    if taps is not None:
        taps["enc.m"], taps["enc.logs"] = m_q, logs_q
    z_p = flow(sd, z, mask, g_src, reverse=False)
    z_hat = flow(sd, z_p, mask, g_tgt, reverse=True)
    gd = torch.zeros_like(g_tgt) if zero_g else g_tgt
    o_hat = generator(sd, z_hat * mask, gd, hp, taps)
    return o_hat, mask, (z, z_p, z_hat)


def voice_conversion_ragged(sd: StateDict, spec: torch.Tensor, lengths: torch.Tensor,
                            g_src: torch.Tensor, g_tgt: torch.Tensor, noise: torch.Tensor,
                            tau: float = 0.3, zero_g: bool = False):
    """What ``convert`` does for a list of utterances: each one alone at its exact length
    (openvoice/api.py:148-154 is batch 1).  Outputs are zero-padded to the batch maximum."""
    B, _, T = spec.shape
    o = torch.zeros(B, 1, 256 * T, dtype=spec.dtype)
    zs = [torch.zeros(B, noise.shape[1], T, dtype=spec.dtype) for _ in range(3)]
    for b in range(B):
        L = int(lengths[b])
        ob, _, lat = voice_conversion(sd, spec[b:b + 1, :, :L], lengths[b:b + 1], g_src[b:b + 1],
                                      g_tgt[b:b + 1], noise[b:b + 1, :, :L], tau, zero_g)
        o[b, :, : ob.shape[2]] = ob[0]
        for dst, src in zip(zs, lat):
            dst[b, :, :L] = src[0]
    return o, sequence_mask(lengths, T, spec.dtype), tuple(zs)


# --------------------------------------------------------------------------------------
# front end / speaker embedding (rows a2 and f2 of SURVEY.md section 8)
# --------------------------------------------------------------------------------------
def spectrogram(y: torch.Tensor, n_fft: int = 1024, hop: int = 256, win: int = 1024) -> torch.Tensor:
    """Linear magnitude spectrogram (openvoice/mel_processing.py:40-75): reflect pad
    (n_fft-hop)/2 both sides, periodic hann, centre=False, sqrt(re^2+im^2+1e-6)."""
    p = int((n_fft - hop) / 2)
    yp = F.pad(y.unsqueeze(1), (p, p), mode="reflect").squeeze(1)
    window = torch.hann_window(win, dtype=y.dtype, device=y.device)
    s = torch.stft(yp, n_fft, hop_length=hop, win_length=win, window=window, center=False,
                   normalized=False, onesided=True, return_complex=True)
    s = torch.view_as_real(s)
    return torch.sqrt(s.pow(2).sum(-1) + 1e-6)


def reference_encoder(sd: StateDict, spec_t: torch.Tensor) -> torch.Tensor:
    """Tone-colour embedding (openvoice/models.py:339-359): LayerNorm over frequency,
    6x(Conv2d 3x3 stride 2 + ReLU), GRU(->128) last hidden state, Linear(128->gin).
    ``spec_t`` is [N, T, spec_channels]."""
    N, T, Fq = spec_t.shape
    x = F.layer_norm(spec_t, (Fq,), sd["ref_enc.layernorm.weight"], sd["ref_enc.layernorm.bias"])
    x = x.view(N, 1, T, Fq)
    for i in range(6):
        x = F.relu(F.conv2d(x, _w(sd, f"ref_enc.convs.{i}"), sd[f"ref_enc.convs.{i}.bias"],
                            stride=2, padding=1))
    x = x.transpose(1, 2).contiguous().view(N, x.shape[2], -1)
    w_ih, w_hh = sd["ref_enc.gru.weight_ih_l0"], sd["ref_enc.gru.weight_hh_l0"]
    b_ih, b_hh = sd["ref_enc.gru.bias_ih_l0"], sd["ref_enc.gru.bias_hh_l0"]
    h = torch.zeros(N, 128, dtype=x.dtype)
    for t in range(x.shape[1]):
        gi = x[:, t] @ w_ih.T + b_ih
        gh = h @ w_hh.T + b_hh
        r = torch.sigmoid(gi[:, :128] + gh[:, :128])
        u = torch.sigmoid(gi[:, 128:256] + gh[:, 128:256])
        n = torch.tanh(gi[:, 256:] + r * gh[:, 256:])
        h = (1 - u) * n + u * h
    return h @ sd["ref_enc.proj.weight"].T + sd["ref_enc.proj.bias"]


def convert_waveform(sd: StateDict, audio: torch.Tensor, src_se: torch.Tensor, tgt_se: torch.Tensor,
                     noise: Optional[torch.Tensor], tau: float = 0.3, zero_g: bool = False,
                     hp: Optional[dict] = None) -> torch.Tensor:
    """The arithmetic of ``ToneColorConverter.convert`` (openvoice/api.py:147-155) for one
    waveform already at the model's sampling rate, watermark disabled."""
    d = (hp or DEFAULT_HPARAMS)["data"]
    spec = spectrogram(audio[None], d["filter_length"], d["hop_length"], d["win_length"])
    T = spec.shape[2]
    if noise is None:
        noise = torch.zeros(1, 192, T, dtype=spec.dtype)
    o, _, _ = voice_conversion(sd, spec, torch.tensor([T]), src_se, tgt_se, noise, tau, zero_g, hp)
    return o[0, 0]
