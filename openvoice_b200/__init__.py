"""openvoice_b200 -- H100-native (sm_90a) tone-colour-converter hot path of OpenVoice.

Drop-in surface of the reference's ``openvoice.api`` / ``openvoice.se_extractor`` for the
``ToneColorConverter.convert -> SynthesizerTrn.voice_conversion`` path; the arithmetic runs in
``libovc_b200.so`` (hand-written CUDA, C ABI in ``include/ovc.h``).  Also the V1 base-speaker TTS front half
(``BaseSpeakerTTS`` -> ``SynthesizerTrn.infer``) and the multi-GPU replica driver (``distributed``).
There is no CPU fallback.
"""
__version__ = "0.1.0"

from . import utils  # noqa: F401


def __getattr__(name):  # lazy: importing the package must not require torch/CUDA
    import importlib
    if name in ("ToneColorConverter", "OpenVoiceBaseClass", "BaseSpeakerTTS", "NativeSynthesizer", "ToneTrack"):
        return getattr(importlib.import_module(".api", __name__), name)
    if name in ("api", "se_extractor", "schema", "ref_enc", "distributed"):
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
