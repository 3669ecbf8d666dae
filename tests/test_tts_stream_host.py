"""CPU tests of streaming base-speaker TTS: the window plan, and the argument checks that run before anything is
launched (include/ovc.h: ovc_tts_decode_windows)."""
import pytest
import torch


@pytest.mark.parametrize("first,window,halo", [(32, 256, 64), (1, 1, 0), (7, 3, 5), (256, 32, 64), (100, 100, 16)])
def test_plan_covers_every_frame_once_in_order(first, window, halo):
    from openvoice_b200.api import plan_tts_windows
    for frames in range(1, 2001):
        plan = plan_tts_windows(frames, first, window, halo)
        e_prev = 0
        for k, (lo, hi, e0, e1) in enumerate(plan):
            assert e0 == e_prev and e1 > e0
            assert e1 - e0 == (first if k == 0 else window) or e1 == frames
            assert lo == max(0, e0 - halo) and hi == min(frames, e1 + halo)
            assert 0 <= lo <= e0 and e1 <= hi <= frames
            e_prev = e1
        assert e_prev == frames
        assert plan[0][0] == 0 and plan[-1][1] == frames


def test_plan_refusals():
    from openvoice_b200.api import plan_tts_windows
    for args in ((0, 32, 256, 64), (10, 0, 256, 64), (10, 32, 0, 64), (10, 32, 256, -1)):
        with pytest.raises(ValueError):
            plan_tts_windows(*args)


def test_halo_covers_the_decode_receptive_field():
    """TTS_HALO_FRAMES >= flow reverse (4 couplings x 4 WaveNet layers, k = 5, dilation 1) + generator (+-13.3)."""
    from openvoice_b200.api import TTS_HALO_FRAMES, ToneColorConverter
    flow = 4 * 4 * (5 - 1) // 2
    assert TTS_HALO_FRAMES >= flow + 14 and TTS_HALO_FRAMES < ToneColorConverter.HALO_FRAMES


def _engine():
    """A BaseSpeakerTTS that never touched a device: every refusal below must happen before one is needed."""
    from oracle import tts_oracle as T
    from oracle import vc_oracle as O
    from openvoice_b200.api import BaseSpeakerTTS
    from openvoice_b200.utils import HParams
    import copy
    hp = copy.deepcopy(O.DEFAULT_HPARAMS)
    hp["data"]["n_speakers"] = T.TTS_HPARAMS["n_speakers"]
    hp["speakers"] = {"default": 1}
    eng = BaseSpeakerTTS.__new__(BaseSpeakerTTS)
    eng.hps = HParams(**hp)
    eng.device = "cuda:0"
    eng.text_frontend = None
    return eng


def test_stream_refusals_before_any_launch():
    eng = _engine()
    ok = dict(ids=[[1, 2, 3]], speaker="default", seed=1)
    cases = [
        lambda: eng.tts_stream_batch([dict(ok, speed=0.0)]),
        lambda: eng.tts_stream_batch([dict(ok, speed=-1.0)]),
        lambda: eng.tts_stream_batch([dict(ok, speed=float("nan"))]),
        lambda: eng.tts_stream_batch([ok, dict(ok, ids=[])]),                 # an empty request
        lambda: eng.tts_stream_batch([ok], window_frames=0),
        lambda: eng.tts_stream_batch([ok], first_window_frames=0),
        lambda: eng.tts_stream_batch([dict(ok, seed=-3)]),
        lambda: eng.tts_stream(ids=[[1, 2]], speaker="default", speed=0.0),
        lambda: eng.tts_stream(ids=[], speaker="default"),
        lambda: eng.tts_stream(ids=[[1, 2]], speaker="default", window_frames=-5),
    ]
    for i, case in enumerate(cases):
        with pytest.raises(ValueError):
            case()
        assert not hasattr(eng, "model"), i


def test_window_refusals_before_any_launch():
    from openvoice_b200.api import NativeSynthesizer, TtsState
    m = NativeSynthesizer.__new__(NativeSynthesizer)      # no native context: reaching it would raise AttributeError
    m.device = torch.device("cuda", 0)
    st = TtsState(None, None, None, None, [100, 7], [1, 2], [0, 1], [0.667, 0.667])
    for wins, w_max in (([], None), ([(2, 0, 5)], None), ([(-1, 0, 5)], None), ([(0, -1, 5)], None), ([(0, 0, 0)], None),
                        ([(0, 90, 11)], None), ([(1, 0, 8)], None), ([(0, 0, 50)], 49), ([(0, 0, 5), (1, 3, 5)], None)):
        with pytest.raises(ValueError):
            m.tts_decode_windows(st, wins, w_max=w_max)


def test_native_window_arrays_must_agree():
    from openvoice_b200._native import NativeConverter
    nc = NativeConverter.__new__(NativeConverter)
    with pytest.raises(ValueError):
        nc.tts_decode_windows(None, None, None, None, [0, 1], [0, 0], [5], [1, 1], [0, 0], [1.0, 1.0], 5)
    with pytest.raises(ValueError):
        nc.tts_decode_windows(None, None, None, None, [], [], [], [], [], [], 5)

