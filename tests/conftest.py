import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def synthetic_sd():
    from oracle import vc_oracle as O
    return O.synthetic_state_dict(1234)


@pytest.fixture(scope="session")
def hps():
    from oracle import vc_oracle as O
    from openvoice_b200.utils import HParams
    return HParams(**O.DEFAULT_HPARAMS)


_native_cache = {}


def pytest_generate_tests(metafunc):
    # every GPU parity test that takes `native` runs in both arithmetic modes of the generator
    if "native" in metafunc.fixturenames:
        metafunc.parametrize("native", ["fp32", "f16x3"], indirect=True)


def get_native(zero_g=False):
    """One NativeSynthesizer per flavour for the whole session (weights: 128 MB)."""
    import copy
    from oracle import vc_oracle as O
    from openvoice_b200.api import NativeSynthesizer
    from openvoice_b200.utils import HParams
    if zero_g not in _native_cache:
        hp = copy.deepcopy(O.DEFAULT_HPARAMS)
        hp["model"]["zero_g"] = zero_g
        m = NativeSynthesizer(HParams(**hp), "cuda:0")
        missing, unexpected = m.load_state_dict(O.synthetic_state_dict(1234))
        assert not missing and not unexpected
        _native_cache[zero_g] = m
    return _native_cache[zero_g]


@pytest.fixture
def native(request):
    m = get_native(False)
    m.native.set_precision(getattr(request, "param", "fp32"))
    yield m
    m.native.set_precision(m.precision)


@pytest.fixture(scope="session")
def native_v2():
    return get_native(True)


_tts_cache = {}


def get_native_tts():
    """NativeSynthesizer on the synthetic V1 base-speaker checkpoint (enc_p / dp / sdp / emb_g + enc_q / flow / dec)."""
    import copy
    from oracle import tts_oracle as T
    from oracle import vc_oracle as O
    from openvoice_b200.api import NativeSynthesizer
    from openvoice_b200.utils import HParams
    if "m" not in _tts_cache:
        hp = copy.deepcopy(O.DEFAULT_HPARAMS)
        hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
        m = NativeSynthesizer(HParams(**hp), "cuda:0")
        missing, unexpected = m.load_state_dict(T.synthetic_tts_state_dict())
        assert not missing, missing
        assert all(k.startswith("sdp.flows.1.") for k in unexpected), unexpected   # never run in reverse (models.py:172)
        _tts_cache["m"] = m
    return _tts_cache["m"]
