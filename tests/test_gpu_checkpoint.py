"""-m gpu: ovc_finalize_weights checks every checkpoint tensor it reads against the shape the model gives it.

A mis-shaped tensor is refused with OVC_ERR_INVALID (ValueError) and a missing one with OVC_ERR_MISSING (OvcError),
and the message names the key (and, for a mis-shaped one, its shape and the expected shape).  A refused load keeps the
loaded tensors, so the caller can replace the bad one and finalize again.

One converter context (v1 hyper-parameters, with ref_enc) holds the synthetic checkpoint.  Each case replaces one
tensor with a mis-shaped one, expects finalize to refuse it, and puts the good tensor back.  The cases:
- first dim - 1 (when it is > 1) and last dim + 1 for the keys of state_dict_schema().  A refused finalize first packs
  everything before the bad key, so the sweep is limited to layer 0 and the last layer of each repeated stack (WN
  layers, couplings, upsamplers, ResBlocks and their convs, ReferenceEncoder convs): 211 of the 971 cases.  The file
  takes about 2.5 minutes on an H100 80 GB HBM3 (700 W power limit); the full sweep has 4.6 times as many cases;
- an extra trailing dim of size 2 for one key per place the library reads a tensor (SITES);
- the removal of one key per such place, in a fresh context.
The TTS members have one hand-picked case per place they are read: many of their dims are hyper-parameters read off
the shapes, so a blanket sweep would mutate valid checkpoints.  Last, the restored checkpoint must load and compute
exactly what a context that never saw a bad tensor computes.
"""
import re

import pytest
import torch

from oracle import tts_oracle as TO
from oracle import vc_oracle as O
from openvoice_b200._native import NativeConverter, OvcError
from openvoice_b200.utils import HParams

pytestmark = pytest.mark.gpu

SCHEMA = O.state_dict_schema()
TTS_SCHEMA = TO.tts_state_dict_schema()

# one key per place in ovc_lib.cu that reads a converter tensor
SITES = [
    "enc_q.pre.weight", "enc_q.pre.bias", "enc_q.proj.weight", "enc_q.proj.bias",
    "enc_q.enc.in_layers.0.weight_v", "enc_q.enc.in_layers.15.weight_g",
    "enc_q.enc.res_skip_layers.15.weight_v", "flow.flows.2.enc.res_skip_layers.1.bias",
    "flow.flows.2.pre.weight", "flow.flows.2.pre.bias", "flow.flows.6.post.weight", "flow.flows.6.post.bias",
    "dec.conv_pre.weight", "dec.ups.1.weight_v", "dec.ups.3.bias",
    "dec.resblocks.5.convs1.2.weight_v", "dec.resblocks.11.convs2.0.bias", "dec.conv_post.weight",
    "enc_q.enc.cond_layer.weight_v", "flow.flows.4.enc.cond_layer.bias", "flow.flows.0.enc.in_layers.3.bias",
    "dec.cond.weight", "dec.cond.bias", "dec.conv_pre.bias",
    "ref_enc.convs.5.weight_v", "ref_enc.convs.0.bias", "ref_enc.gru.weight_ih_l0", "ref_enc.gru.bias_hh_l0",
    "ref_enc.proj.weight", "ref_enc.layernorm.bias",
]

# one (key, mutation) per place pack_tts reads a tensor; None removes the key
TTS_CASES = [
    ("enc_p.emb.weight", "extra"), ("enc_p.encoder.attn_layers.0.emb_rel_k", "extra"),
    ("enc_p.encoder.ffn_layers.0.conv_1.weight", "extra"), ("dp.conv_1.weight", "last+1"), ("emb_g.weight", "last+1"),
    ("enc_p.encoder.attn_layers.1.conv_k.weight", "last+1"), ("enc_p.encoder.attn_layers.5.conv_v.bias", "first-1"),
    ("enc_p.encoder.attn_layers.2.conv_o.bias", "last+1"), ("enc_p.proj.weight", "first-1"),
    ("enc_p.encoder.ffn_layers.3.conv_2.weight", "first-1"), ("enc_p.encoder.norm_layers_2.5.beta", "extra"),
    ("enc_p.encoder.attn_layers.4.emb_rel_v", "last+1"), ("dp.proj.weight", "last+1"), ("sdp.flows.0.logs", "first-1"),
    ("sdp.flows.5.convs.convs_sep.2.weight", "last+1"), ("sdp.flows.7.proj.weight", "first-1"),
    ("sdp.cond.bias", None), ("dp.norm_2.gamma", None),
]


def mutate(shape, how):
    return {"first-1": (shape[0] - 1,) + shape[1:], "last+1": shape[:-1] + (shape[-1] + 1,), "extra": shape + (2,)}[how]


def end_layers(keys):
    """The keys whose every layer index is the first or the last of its stack."""
    idx = {}   # key prefix before a layer index -> the indices seen there
    for k in keys:
        parts = k.split(".")
        for j, p in enumerate(parts):
            if p.isdigit():
                idx.setdefault(tuple(parts[:j]), set()).add(int(p))

    def at_ends(k):
        parts = k.split(".")
        return all(int(p) in (min(idx[tuple(parts[:j])]), max(idx[tuple(parts[:j])]))
                   for j, p in enumerate(parts) if p.isdigit())
    return [k for k in keys if at_ends(k)]


def cases():
    out = []
    for k in end_layers(list(SCHEMA)):
        out += [(k, how) for how in ("first-1", "last+1") if how != "first-1" or SCHEMA[k][0] > 1]
    return out + [(k, "extra") for k in SITES if len(SCHEMA[k]) < 4]


def converter(sd, drop=None):
    nat = NativeConverter(HParams(**O.DEFAULT_HPARAMS), 0)
    nat.load_state_dict({k: v for k, v in sd.items() if k != drop})
    return nat


def refuse(nat, key, exc):
    with pytest.raises(exc, match=re.escape(f"'{key}'")) as e:
        nat.finalize()
    return str(e.value)


@pytest.fixture(scope="module")
def sd():
    return O.synthetic_state_dict(1234)


@pytest.fixture(scope="module")
def ctx(sd):
    nat = converter(sd)
    yield nat
    nat.close()


@pytest.mark.parametrize("key,how", cases())
def test_misshaped_tensor_is_refused(ctx, sd, key, how):
    shape = mutate(tuple(SCHEMA[key]), how)
    ctx.load_state_dict({key: torch.full(shape, 0.01)})
    try:
        msg = refuse(ctx, key, ValueError)
        assert str(list(shape)) in msg
        if not key.endswith(".weight_g"):   # weight_g only has to hold one value per output channel
            assert str(list(SCHEMA[key])) in msg
    finally:
        ctx.load_state_dict({key: sd[key]})


@pytest.mark.parametrize("key", [k for k in SITES if k != "ref_enc.proj.weight"])
def test_missing_tensor_is_refused(sd, key):
    nat = converter(sd, drop=key)
    try:
        refuse(nat, key, OvcError)
    finally:
        nat.close()


def test_converter_without_ref_enc_proj_loads(sd):
    """ref_enc.proj.weight marks a checkpoint with a ReferenceEncoder: without it the converter loads and only
    reference_encoder is refused."""
    nat = converter(sd, drop="ref_enc.proj.weight")
    try:
        nat.finalize()
        with pytest.raises(OvcError, match="ref_enc"):
            nat.reference_encoder(torch.zeros(1, SCHEMA["ref_enc.layernorm.weight"][0], 32, device="cuda"))
    finally:
        nat.close()


@pytest.fixture(scope="module")
def tts_sd():
    return TO.synthetic_tts_state_dict()


@pytest.fixture(scope="module")
def tts_ctx(tts_sd):
    nat = converter(tts_sd)
    yield nat
    nat.close()


@pytest.mark.parametrize("key,how", TTS_CASES)
def test_tts_tensor_is_refused(tts_ctx, tts_sd, key, how):
    if how is None:
        nat = converter(tts_sd, drop=key)
        try:
            refuse(nat, key, OvcError)
        finally:
            nat.close()
        return
    shape = mutate(tuple(TTS_SCHEMA[key]), how)
    tts_ctx.load_state_dict({key: torch.full(shape, 0.01)})
    try:
        assert str(list(shape)) in refuse(tts_ctx, key, ValueError)
    finally:
        tts_ctx.load_state_dict({key: tts_sd[key]})


def test_tts_checkpoint_loads_after_refusals(tts_ctx):
    tts_ctx.finalize()
    assert tts_ctx.tts_info()["has_tts"] == 1


def test_restored_checkpoint_computes_as_before(ctx, native):
    """finalize keeps the loaded tensors when it refuses one, so the context that refused every case above loads once
    each bad tensor is replaced, and then computes bit for bit what a context that only ever saw the good checkpoint
    computes."""
    if not ctx.finalized:
        ctx.finalize()
    ctx.set_precision(native.native.precision)
    spec, lengths, gs, gt, noise = O.synthetic_inputs(2, 40, 7, lengths=[40, 29])
    args = (spec.cuda(), lengths.cuda(), gs.cuda(), gt.cuda())
    o, lat = ctx.voice_conversion(*args, noise=noise.cuda(), tau=0.3)
    ro, _, rlat = native.voice_conversion(*args, noise=noise.cuda(), tau=0.3)
    assert torch.equal(o, ro)
    for a, b in zip(lat, rlat):
        assert torch.equal(a, b)
    assert torch.equal(ctx.reference_encoder(args[0]), native.native.reference_encoder(args[0]))
