"""CPU oracle of time-varying speaking style: ``SynthesizerTrn.infer`` (models.py:467-490) with speaker vectors per
token.  The duration predictors read ``g_tok`` [B, gin, T] per token; the flow reverse and the generator read
``g_frames``, ``g_tok`` expanded along the alignment path exactly as m_p is (frame y takes the vector of the token
covering it, 0 past y_lengths).  A [B, gin, 1] ``g_tok`` is one vector per row and conditions every frame, as
emb_g(sid) does.  Built from ``tts_oracle``'s modules; ``make_golden_tts_style.py`` pins it on the reference's."""
from __future__ import annotations

from typing import Optional

import torch

import tts_oracle as T
import vc_oracle as V


def expand_g(g_tok: torch.Tensor, tok: torch.Tensor, y_mask: torch.Tensor) -> torch.Tensor:
    """[B, gin, Ty]: g_tok gathered at each frame's token, zero past y_lengths; a [B, gin, 1] g_tok stays as it is."""
    if g_tok.shape[-1] == 1:
        return g_tok
    return torch.gather(g_tok, 2, tok[:, None, :].expand(-1, g_tok.shape[1], -1)) * y_mask


def tts_infer_g(sd, tokens: torch.Tensor, lengths: torch.Tensor, g_tok: torch.Tensor, noise_w: torch.Tensor,
                noise: torch.Tensor, noise_scale: float = 0.667, length_scale: float = 1.0, noise_scale_w: float = 0.6,
                sdp_ratio: float = 0.2, hp: Optional[dict] = None, tts: Optional[dict] = None) -> dict:
    """``tts_oracle.tts_infer`` (padded decode) with ``g_tok`` in place of emb_g(sid)."""
    hp = hp or V.DEFAULT_HPARAMS
    tts = tts or T.TTS_HPARAMS
    x, m_p, logs_p, x_mask = T.text_encoder(sd, tokens, lengths, hp, tts)
    logw_s = T.sdp_reverse(sd, x, x_mask, g_tok, noise_w, noise_scale_w, tts)
    logw_d = T.duration_predictor(sd, x, x_mask, g_tok)
    logw = logw_s * sdp_ratio + logw_d * (1 - sdp_ratio)
    w_ceil = torch.ceil(torch.exp(logw) * x_mask * length_scale)
    y_lengths = torch.clamp_min(w_ceil.sum([1, 2]), 1).long()
    Ty = int(y_lengths.max())
    y_mask = V.sequence_mask(y_lengths, Ty, x.dtype)
    tok = T.generate_path(w_ceil, y_lengths)
    gi = tok[:, None, :].expand(-1, m_p.shape[1], -1)
    m_y = torch.gather(m_p, 2, gi) * y_mask
    logs_y = torch.gather(logs_p, 2, gi) * y_mask
    g_frames = expand_g(g_tok, tok, y_mask)
    z_p = m_y + noise[:, :, :Ty] * torch.exp(logs_y) * noise_scale
    z = V.flow(sd, z_p, y_mask, g_frames, reverse=True)
    o = V.generator(sd, z * y_mask, g_frames, hp)
    return {"logw_sdp": logw_s, "logw_dp": logw_d, "w_ceil": w_ceil[:, 0], "y_lengths": y_lengths, "z_p": z_p, "z": z,
            "o": o}
