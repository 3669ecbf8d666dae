"""CPU-side tests: the C ABI library loads and exports what include/ovc.h declares, hparams
marshalling / validation, loud failure without a GPU, config + audio helpers, and the multi-GPU
driver logic under gloo (world_size 2)."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "ovc.h")).read()
    return sorted(set(re.findall(r"OVC_API\s+[\w\s\*]+?\b(ovc_\w+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from openvoice_b200 import _native
    lib = _native.load_library()
    declared = header_functions()
    assert len(declared) >= 13
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/ovc.h but not exported"
    assert sorted(_native.EXPORTS) == declared
    assert lib.ovc_abi_version() == _native.ABI_VERSION


def test_library_contains_sm90a_tma_code():
    """The shipped cubin is sm_90a and stages weights with TMA bulk copies (UBLKCP)."""
    lib = os.path.join(ROOT, "openvoice_b200", "libovc_b200.so")
    out = subprocess.run(["cuobjdump", "-lelf", lib], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    sass = subprocess.run(["bash", "-c", f"cuobjdump -sass -fun '_ZN3ovc10conv1d_f32INS_7ConvCfgILi1ELi1ELi2ELi2ELi8ELi2ELi1ELi16EEEEEvNS_8ConvArgsE' {lib} | grep -c -E 'UBLKCP|SYNCS'"],
                          capture_output=True, text=True).stdout.strip()
    assert int(sass or 0) > 0


def test_hparams_marshalling(hps):
    from openvoice_b200 import _native
    s = _native.hparams_struct(hps)
    assert (s.spec_channels, s.inter_channels, s.hidden_channels, s.gin_channels) == (513, 192, 192, 256)
    assert list(s.resblock_kernel_sizes)[:3] == [3, 7, 11] and list(s.upsample_rates) == [8, 8, 2, 2]
    assert [list(r) for r in s.resblock_dilations][:3] == [[1, 3, 5]] * 3
    assert s.zero_g == 0 and s.hop_length == 256 and s.resblock == 1


def test_create_fails_loudly_without_gpu_and_on_bad_hparams(hps):
    """No CPU fallback: without a device ovc_create errors; unsupported hparams are refused."""
    from openvoice_b200 import _native
    lib = _native.load_library()
    bad = _native.hparams_struct(hps)
    bad.hidden_channels = 128
    h = C.c_void_p()
    assert lib.ovc_create(C.byref(bad), 0, C.byref(h)) == -1
    assert b"192" in lib.ovc_last_error()
    bad = _native.hparams_struct(hps)
    bad.upsample_rates[0] = 4
    assert lib.ovc_create(C.byref(bad), 0, C.byref(h)) == -1
    if not torch.cuda.is_available():
        with pytest.raises(_native.OvcError, match="no CUDA device"):
            _native.NativeConverter(hps, 0)
        from openvoice_b200.api import NativeSynthesizer
        with pytest.raises(RuntimeError):
            NativeSynthesizer(hps, "cpu")
    assert lib.ovc_voice_conversion(None, None, None, None, None, None, 0, 0.3, 1, 1, 0, None, None, None, None, None) < 0


def test_missing_library_is_an_error(monkeypatch, tmp_path):
    from openvoice_b200 import _native
    monkeypatch.setattr(_native, "_lib", None)
    monkeypatch.setenv("OVC_B200_LIB", str(tmp_path / "nope.so"))
    with pytest.raises(_native.OvcError, match="no CPU"):
        _native.load_library()


def test_product_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "openvoice_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in txt.replace("vc_oracle", "oracle") or f == "x", f
    txt = open(os.path.join(ROOT, "openvoice_b200", "api.py")).read()
    assert "import oracle" not in txt and "from oracle" not in txt


def test_hparams_loader_and_bit_codec(tmp_path):
    from openvoice_b200 import utils
    from oracle import vc_oracle as O
    p = tmp_path / "config.json"
    hp = dict(O.DEFAULT_HPARAMS, _version_="v2")
    p.write_text(json.dumps(hp))
    h = utils.get_hparams_from_file(str(p))
    assert h.data.sampling_rate == 22050 and h["model"]["upsample_rates"] == [8, 8, 2, 2]
    assert "model" in h and len(h) == 3 and getattr(h, "_version_") == "v2"
    bits = utils.string_to_bits("@MyShell")
    assert bits.shape == (8, 8) and utils.bits_to_string(bits) == "@MyShell"
    assert utils.bits_to_string(utils.string_to_bits("ab")) == "ab" + " " * 6   # space padded (utils.py:57)


def test_audio_loader(tmp_path):
    from scipy.io import wavfile
    from openvoice_b200.api import _load_audio, _write_audio
    x = (0.3 * np.sin(np.arange(22050) * 0.05)).astype(np.float32)
    np.save(tmp_path / "a.npy", x)
    assert np.array_equal(_load_audio(str(tmp_path / "a.npy"), 22050), x)
    wavfile.write(tmp_path / "a.wav", 22050, (x * 32767).astype(np.int16))
    y = _load_audio(str(tmp_path / "a.wav"), 22050)
    assert y.dtype == np.float32 and np.abs(y - x).max() < 1e-4
    wavfile.write(tmp_path / "b.wav", 44100, np.repeat((x * 32767).astype(np.int16), 2))
    z = _load_audio(str(tmp_path / "b.wav"), 22050)
    assert abs(len(z) - len(x)) <= 1
    _write_audio(str(tmp_path / "o.npy"), x, 22050)
    assert np.array_equal(np.load(tmp_path / "o.npy"), x)


def test_watermark_chunking_roundtrip():
    """add_watermark / detect_watermark chunk walk (16000-sample chunks every 32000 samples, 32 bits each,
    "too short" handling -- openvoice/api.py:162-201) with a stand-in codec model."""
    from openvoice_b200 import utils
    from openvoice_b200.api import ToneColorConverter

    class FakeWM:                                   # hides the 32 bits in the first 32 samples of a chunk
        def encode(self, sig, bits):
            out = sig.clone()
            out[:, :32] = bits * 0.5 + 0.25
            return out

        def decode(self, sig):
            return (sig[:, :32] - 0.25) / 0.5

    conv = ToneColorConverter.__new__(ToneColorConverter)     # no GPU needed for this logic
    conv.device = "cpu"
    conv.watermark_model = FakeWM()
    audio = np.zeros(32000 * 1 + 16000, dtype=np.float32)     # room for chunks 0 and 1
    out = conv.add_watermark(audio.copy(), "@MyShell")
    assert conv.detect_watermark(out, 2) == "@MyShell"
    assert np.count_nonzero(out[16000:32000]) == 0            # only the chunk windows are touched
    short = np.zeros(20000, dtype=np.float32)
    out2 = conv.add_watermark(short.copy(), "@MyShell")       # second chunk does not fit: first is still written
    assert np.count_nonzero(out2[:32]) > 0
    assert conv.detect_watermark(out2, 2) == "Fail"
    conv.watermark_model = None
    assert conv.add_watermark(short, "x") is short
    assert utils.string_to_bits("@MyShell").shape == (8, 8)


def test_lpt_shard_balances_and_covers():
    from openvoice_b200.distributed import lpt_shard
    costs = [10, 1, 7, 3, 3, 9, 2, 8]
    for w in (1, 2, 3, 8, 11):
        sh = lpt_shard(costs, w)
        assert sorted(i for s in sh for i in s) == list(range(len(costs)))
        loads = [sum(costs[i] for i in s) for s in sh]
        assert max(loads) - min(l for l in loads if l or w <= len(costs)) <= max(costs)
    assert lpt_shard(costs, 2) == lpt_shard(costs, 2)


_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch, torch.distributed as dist
from openvoice_b200.distributed import broadcast_state_dict, convert_sharded, lpt_shard
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
sd = {"a.weight": torch.arange(12.).reshape(3, 4), "b.bias": torch.tensor([1.5, -2.0]), "c": torch.ones(2, 1, 3)} if rank == 0 else None
got = broadcast_state_dict(sd)
assert set(got) == {"a.weight", "b.bias", "c"} and got["a.weight"].shape == (3, 4) and float(got["a.weight"][2, 3]) == 11.0
assert torch.equal(got["b.bias"], torch.tensor([1.5, -2.0]))
rng = np.random.default_rng(0)
audios = [rng.standard_normal(n).astype(np.float32) for n in (700, 50, 300, 1200, 256, 999, 10)]
calls = []
def fake_convert(batch, src, tgt, tau=0.3):
    calls.append(len(batch))
    return [(-a[: 256 * (len(a) // 256)] * tau).astype(np.float32) for a in batch]
out = convert_sharded(fake_convert, audios, None, None, tau=0.5)
mine = lpt_shard([len(a) for a in audios], world)[rank]
assert calls == ([len(mine)] if mine else [])
if rank == 0:
    assert len(out) == len(audios)
    for a, o in zip(audios, out):
        assert np.array_equal(o, (-a[: 256 * (len(a) // 256)] * 0.5).astype(np.float32))
else:
    assert out is None
# the device-gather path (convert_sharded_async) with a stand-in converter that keeps its batch in a tensor
from openvoice_b200.distributed import convert_sharded_async
class FakeConverter:
    class hps:
        class data:
            hop_length = 256
    device = torch.device("cpu")
    def convert_batch_device(self, batch, src, tgt, tau=0.3, slot=0):
        n = [256 * (len(a) // 256) for a in batch]
        o = torch.zeros(len(batch), max(n))
        for j, a in enumerate(batch):
            o[j, : n[j]] = torch.from_numpy(-a[: n[j]] * tau)
        return o, n
fc = FakeConverter()
long = [a for a in audios if len(a) >= 256]
jobs = [convert_sharded_async(fc, long, None, None, tau=t) for t in (0.5, 0.25, 2.0)]     # three calls in flight
for t, job in ((0.25, jobs[1]), (2.0, jobs[2])):        # the two youngest are still intact (two buffer generations)
    res = job.result()
    if rank == 0:
        assert len(res) == len(long)
        for a, o in zip(long, res):
            assert np.array_equal(o, (-a[: 256 * (len(a) // 256)] * t).astype(np.float32))
    else:
        assert res is None
dist.barrier()
dist.destroy_process_group()
sys.stdout.write(f"worker-{rank}-ok\n"); sys.stdout.flush()
"""


def test_multi_gpu_driver_under_gloo_world2(tmp_path):
    """The N>1 path (checkpoint broadcast, LPT sharding, waveform gather) with 2 CPU processes."""
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    import socket
    with socket.socket() as sk:          # a free port: back-to-back runs must not collide on TIME_WAIT
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script), ROOT],
                       capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "worker-0-ok" in r.stdout and "worker-1-ok" in r.stdout


def test_tts_key_schema_matches_the_oracle_schema(hps):
    """openvoice_b200.schema.tts_keys (what load_state_dict reports against) = the reference constructors' names as the
    oracle lists them, minus sdp.flows.1 (never run in reverse, models.py:172)."""
    from oracle import tts_oracle as T
    from openvoice_b200.schema import hot_path_keys, tts_keys
    want = {k for k in T.tts_state_dict_schema() if not k.startswith("sdp.flows.1.")}
    assert set(tts_keys(hps)) == want
    sd = T.synthetic_tts_state_dict()
    assert set(hot_path_keys(hps)) | set(tts_keys(hps)) <= set(sd)


def test_base_speaker_host_helpers():
    """commons.intersperse (commons.py:22-25) and BaseSpeakerTTS.audio_numpy_concat (api.py:56-63)."""
    import numpy as np
    from openvoice_b200.api import BaseSpeakerTTS
    assert BaseSpeakerTTS.intersperse([5, 6, 7], 0) == [0, 5, 0, 6, 0, 7, 0]
    assert BaseSpeakerTTS.intersperse([], 0) == [0]
    a = BaseSpeakerTTS.audio_numpy_concat([np.ones(10), np.full((1, 4), 2.0)], sr=1000, speed=2.0)
    gap = int(1000 * 0.05 / 2.0)
    assert a.dtype == np.float32 and len(a) == 10 + 4 + 2 * gap
    assert a[:10].tolist() == [1.0] * 10 and a[10:10 + gap].tolist() == [0.0] * gap and a[10 + gap:14 + gap].tolist() == [2.0] * 4
    assert BaseSpeakerTTS.language_marks == {"english": "EN", "chinese": "ZH"}


def test_on_device_watermark_chunking_matches_the_reference_loop(capsys):
    """Row f4: watermark_device (strided chunk view, ONE batched encode, scatter) against the per-chunk loop of
    openvoice/api.py:162-184 restated here, with a stand-in for the third-party wavmark model; incl. the
    "Audio too short" early stop."""
    import numpy as np
    import torch
    from openvoice_b200 import utils
    from openvoice_b200.api import watermark_device

    class FakeWM:
        calls = []

        def encode(self, sig, bits):                # [m, 16000], [m, 32] -> [m, 16000]
            FakeWM.calls.append(tuple(sig.shape))
            w = (bits * torch.arange(1, 33, dtype=torch.float32)).sum(1, keepdim=True) * 1e-4
            return sig * (1.0 + w) + 1e-3 * torch.sin(torch.arange(sig.shape[1], dtype=torch.float32))[None] * w

    def reference_loop(audio, message, model):
        bits = utils.string_to_bits(message).reshape(-1)
        K, coeff = 16000, 2
        for n in range(len(bits) // 32):
            trunck = audio[(coeff * n) * K: (coeff * n + 1) * K]
            if len(trunck) != K:
                print("Audio too short, fail to add watermark")
                break
            sig = torch.FloatTensor(trunck)[None]
            msg = torch.FloatTensor(bits[n * 32: (n + 1) * 32])[None]
            audio[(coeff * n) * K: (coeff * n + 1) * K] = model.encode(sig, msg).squeeze().numpy()
        return audio

    rng = np.random.default_rng(0)
    message = "@MyShell"                             # 8 chars -> 64 bits -> 2 chunks
    n_chunks = len(utils.string_to_bits(message).reshape(-1)) // 32
    for L in (32000 * n_chunks + 5000, 32000 * (n_chunks - 1) + 16000, 32000 * (n_chunks - 1) + 15999, 15000):
        a = rng.standard_normal(L).astype(np.float32)
        want = reference_loop(a.copy(), message, FakeWM())
        FakeWM.calls.clear()
        t = torch.from_numpy(a.copy())
        watermark_device(t, utils.string_to_bits(message).reshape(-1), FakeWM())
        assert np.allclose(t.numpy(), want, rtol=1e-6, atol=1e-6), L    # batched vs per-chunk: same math, last-bit differences
        assert len(FakeWM.calls) <= 1               # one batched encode for all chunks of the utterance
        short = "too short" in capsys.readouterr().out
        assert short == (L < 32000 * (n_chunks - 1) + 16000)


def test_streaming_module_imports_without_gpu():
    import openvoice_b200.streaming as S
    assert hasattr(S, "StreamingConverter")


def test_streaming_state_machine_with_a_stand_in_converter():
    """Host logic of StreamingConverter on the CPU: spectrogram frames computed from audio segments (a frame is taken only
    when its STFT support is complete; reflect padding only at the true ends of the stream), noise / frame bookkeeping,
    window + halo scheduling, flush -- with the oracle's STFT and a stand-in 'voice conversion' whose output at frame t
    depends on frames t-100 .. t+100 and on that frame's noise, so a wrong frame, offset or halo shows up."""
    import numpy as np
    import torch
    import torch.nn.functional as F
    from oracle import vc_oracle as O
    from openvoice_b200.streaming import StreamingConverter

    kern = torch.linspace(0.2, 1.0, 201)[None, None]

    class FakeNative:
        def spectrogram(self, wav, wlen):
            T = wav.shape[1] // 256
            return O.spectrogram(wav)[:, :, :T], torch.tensor([T])

    class FakeModel:
        native = FakeNative()

        def voice_conversion(self, sp, lens, src, tgt, tau=0.3, noise=None, ragged=True, latents=False):
            f = sp[:, :8].mean(1, keepdim=True) + tau * noise[:, :1]           # [1, 1, T]
            g = F.conv1d(f, kern, padding=100)                                  # receptive field +-100 frames, zero padding
            o = (g.transpose(1, 2) * torch.linspace(1.0, 2.0, 256)[None, None]).reshape(1, 1, -1)
            return o, None, None

    class FakeConverter:
        class hps:
            class data:
                hop_length, filter_length = 256, 1024

            class model:
                inter_channels = 4
        HALO_FRAMES = 128
        device = "cpu"
        model = FakeModel()

        def _stack_se(self, se, n):
            return se.reshape(1, -1)

    rng = np.random.default_rng(5)
    L = 22050 * 7 + 131
    wav = rng.standard_normal(L).astype(np.float32)
    T = L // 256
    noise = torch.randn(4, T, generator=torch.Generator().manual_seed(2))
    se = torch.zeros(1, 8, 1)
    conv = FakeConverter()
    sp, _ = conv.model.native.spectrogram(torch.from_numpy(wav)[None], None)
    whole = conv.model.voice_conversion(sp, None, None, None, tau=0.3, noise=noise[None])[0][0, 0].numpy()
    for W, sizes in ((64, [1000, 37, 50000, 256, 8191]), (300, [22050]), (1, [4096])):
        sc = StreamingConverter(conv, se, se, tau=0.3, window_frames=W, noise_fn=lambda a, b: noise[:, a:b])
        outs, pos, i, peak = [], 0, 0, 0
        while pos < L:
            n = min(sizes[i % len(sizes)], L - pos)
            outs.append(sc.push(wav[pos: pos + n]))
            pos += n
            i += 1
            peak = max(peak, sc.state_frames)
            assert sum(len(o) for o in outs) % 256 == 0 and sum(len(o) for o in outs) // 256 <= max(0, (pos - 640) // 256 + 1)
        outs.append(sc.flush())
        got = np.concatenate(outs)
        assert got.shape == whole.shape == (256 * T,)
        assert np.allclose(got, whole, rtol=1e-5, atol=1e-5), (W, float(np.abs(got - whole).max()))
        assert peak <= W + 2 * 128 + max(sizes) // 256 + 8
    # a stream that ends before the first window is complete: everything comes out of flush
    sc = StreamingConverter(conv, se, se, tau=0.3, window_frames=200, noise_fn=lambda a, b: noise[:, a:b])
    assert len(sc.push(wav[:30000])) == 0
    tail = sc.flush()
    sp2, _ = conv.model.native.spectrogram(torch.from_numpy(wav[:30000])[None], None)
    ref2 = conv.model.voice_conversion(sp2, None, None, None, tau=0.3, noise=noise[None, :, : 30000 // 256])[0][0, 0].numpy()
    assert tail.shape == ref2.shape and np.allclose(tail, ref2, rtol=1e-5, atol=1e-5)


def test_reference_arm_line_has_the_contract_keys():
    """`bench.py --impl reference` (the CPU arm the driver runs beside the native arm): one JSON line with the native arm's
    metric / unit / config and the e2e / cpu_baseline objects the tier contract asks for."""
    import json
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--ref-clips", "1", "--secs", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "audio_seconds_per_second" and line["unit"] == "audio-s/s"
    assert line["higher_is_better"] is True and line["value"] > 0 and line["steps"] == 1
    assert line["config"]["batch_per_gpu"] == 32 and "workload" in line["config"]
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0 and line["e2e"]["value"] == line["value"]
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
