"""Audio loading on the GPU (csrc/audio.cu): the reference's loadAudio KATs on jfk.wav, the resampler against the float64 restatement in
oracle/audio_ref.py for every stored format, channel count and channel mode, convertToMono bit for bit, segmentation, host / device
pointers, concurrent sessions, and long-form transcription of audio files on a toy model.

Resampler error bound.  The GPU computes y[m] = sum_k x[i_k] * hf[k] with f32 taps hf = fl32(h) and an f32 FMA chain over the K taps of
the output's phase, in a fixed order; the mono input x is the oracle's own f32 signal bit for bit (checked separately).  With
u = 2^-24: |hf - h| <= u |h| and the K-term FMA chain adds at most K u sum |hf x| (first order), so
    |y_gpu - y| <= (K + 2) u * Hmax * max|x|,   Hmax = max over phases of sum_k |h_k|.
At 44.1 kHz (K = 56, Hmax ~ 1.8) that is about 6.3e-6 * max|x| (fir_bound computes the value enforced); the measured error is printed as a
fraction of the bound and of the first-guess bound 2e-6 * max|x|."""
import os
import threading
import wave

import numpy as np
import pytest

import whisperkit_b200 as wk
from oracle import audio_ref as A
from oracle import decode_ref as D
from whisperkit_b200 import _lib
from whisperkit_b200.audio import AudioProcessor

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
JFK = os.path.join(GOLDEN, "jfk.wav")
RATES = [8000, 11025, 22050, 32000, 44056, 44100, 48000, 96000, 384000]
U = 2.0 ** -24


def jfk_s16():
    with wave.open(JFK, "rb") as w:
        return np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").copy()


def bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def fir_bound(rate, xmax):
    up, down = A.ratio(rate)
    if up == down == 1:
        return 0.0
    h = A.filter_taps(rate)
    K = -(-len(h) // up)
    hp = np.zeros(up * K)
    hp[: len(h)] = np.abs(h)
    hmax = hp.reshape(K, up).sum(axis=0).max()
    return (K + 2) * U * hmax * xmax


def jfk_44k_stereo(tmp_path):
    """jfk at 44.1 kHz stereo s16 (scipy resample_poly up, the right channel at 0.6 x and inverted), as a WAV file."""
    from scipy.signal import resample_poly
    x = resample_poly(jfk_s16().astype(np.float64), 441, 160)
    st = np.stack([x, -0.6 * x], axis=1)
    s = np.clip(np.round(st), -32768, 32767).astype(np.int16)
    return A.write_wav(str(tmp_path / "jfk44k.wav"), s, 44100, "s16"), s


# ------------------------------------------------------------------------------------------------ reference KATs (UnitTests.swift:296-345)
def test_jfk_kats_bit_exact():
    ref = jfk_s16().astype(np.float32) / np.float32(32768)
    a = AudioProcessor.loadAudio(JFK)
    assert a.dtype == np.float32 and len(a) == 176000
    assert np.array_equal(bits(a), bits(ref))
    b = AudioProcessor.loadAudio(JFK, startTime=1.2)
    assert len(b) == 156800 and np.array_equal(bits(b), bits(ref[19200:]))
    c = AudioProcessor.loadAudio(JFK, startTime=1.2, endTime=3.4)
    assert len(c) == 35200 and np.array_equal(bits(c), bits(ref[19200:54400]))
    assert np.array_equal(bits(AudioProcessor.loadAudioAsFloatArray(JFK)), bits(ref))


def test_jfk_44k_stereo_kats(tmp_path):
    path, s = jfk_44k_stereo(tmp_path)
    for mrf in (None, 10024):
        assert len(AudioProcessor.loadAudio(path, maxReadFrameSize=mrf)) == 176000
        assert len(AudioProcessor.loadAudio(path, startTime=1.2, maxReadFrameSize=mrf)) == 156800
        y = AudioProcessor.loadAudio(path, startTime=1.2, endTime=3.4, maxReadFrameSize=mrf)
        assert len(y) == 35200
        f = A.to_float(s, "s16")
        ref = A.load_reference(f, 44100, startTime=1.2, endTime=3.4, maxReadFrameSize=mrf)
        assert np.abs(y - ref).max() <= fir_bound(44100, np.abs(A.mono_signal(f, 44100, maxReadFrameSize=mrf)).max())


# ------------------------------------------------------------------------------------------------ resampler vs the float64 restatement
def _frames(rng, n, ch, fmt):
    if fmt == "u8":
        v = rng.integers(0, 256, (n, ch))
    elif fmt == "s16":
        v = rng.integers(-32768, 32768, (n, ch))
    elif fmt == "s24":
        v = rng.integers(-2 ** 23, 2 ** 23, (n, ch))
    elif fmt == "s32":
        v = rng.integers(-2 ** 31, 2 ** 31, (n, ch))
    else:
        v = rng.uniform(-1.5, 1.5, (n, ch)).astype(np.float32)
    return v, A.to_float(v, fmt)


def _as_input(v, fmt):
    """Interleaved frames as wk_audio_convert takes them."""
    if fmt == "s24":
        return np.frombuffer(A.encode_samples(v.reshape(-1), "s24"), np.uint8).reshape(len(v), -1).copy()
    return v.astype({"u8": np.uint8, "s16": np.int16, "s32": np.int32, "f32": np.float32}[fmt])


MODES = [("sum", None), ("sum", [1, 0, 1, 9]), ("sum", [7]), ("channel", 1), ("channel", 5)]


@pytest.mark.parametrize("rate", RATES)
def test_resampler_matches_oracle(rate, tmp_path):
    rng = np.random.default_rng(rate)
    worst = 0.0
    for fmt in A.FORMATS:
        for ch in (1, 2, 6):
            n = int(rate * 0.23) + 3 + ch
            v, f = _frames(rng, n, ch, fmt)
            f = f.reshape(n, ch)
            for mode in (MODES if ch > 1 else MODES[:1]):
                mrf = n // 3 + 1
                y = AudioProcessor.resampleAudio(_as_input(v, fmt), rate, mode, sampleFormat=fmt, channels=ch, maxReadFrameSize=mrf)
                mono = A.mono_signal(f, rate, mode, maxReadFrameSize=mrf)
                ref = A.resample(mono, rate)
                assert y.shape == ref.shape == (-(-n * A.ratio(rate)[0] // A.ratio(rate)[1]),)
                xmax = float(np.abs(mono).max())
                err = float(np.abs(y - ref).max())
                bound = fir_bound(rate, xmax)
                assert err <= bound, (fmt, ch, mode, err, bound)
                worst = max(worst, err / max(xmax, 1e-30))
        # the same frames through a WAV file give the same bits
        p = A.write_wav(str(tmp_path / f"{fmt}.wav"), v, rate, fmt)
        assert np.array_equal(bits(AudioProcessor.loadAudio(p, MODES[1], maxReadFrameSize=mrf)),
                              bits(AudioProcessor.resampleAudio(_as_input(v, fmt), rate, MODES[1], sampleFormat=fmt, channels=ch,
                                                                maxReadFrameSize=mrf)))
    b = fir_bound(rate, 1.0)
    print(f"[{rate} Hz] worst |err| / max|x| = {worst:.2e}: {worst / b if b else 0:.3f} of the derived bound {b:.2e}, "
          f"{worst / 2e-6:.3f} of 2e-6")


@pytest.mark.parametrize("ch", [2, 3, 6])
def test_mono_mix_is_bit_exact(ch):
    """16 kHz (no resampling): the output is convertToMono's f32 result per read chunk, bit for bit."""
    rng = np.random.default_rng(ch)
    n = 50_000
    v = rng.integers(-32768, 32768, (n, ch))
    v[1000:21000] //= 64                 # a quiet stretch: its read chunk gets its own scale
    v[30000:40000] = 0                   # an all-zero read chunk: scale 0
    f = A.to_float(v, "s16")
    for mode in MODES + [("sum", [ch - 1, ch - 1]), ("sum", [])]:
        y = AudioProcessor.resampleAudio(v.astype(np.int16), 16000, mode, maxReadFrameSize=10_000)
        ref = A.mono_signal(f, 16000, mode, maxReadFrameSize=10_000)
        assert np.array_equal(bits(y), bits(ref)), mode


def test_16k_mono_f32_returns_itself():
    x = np.random.default_rng(1).standard_normal(100_003).astype(np.float32)
    x[[5, 17]] = -0.0
    x[9] = np.float32(1e-40)             # a subnormal
    y = AudioProcessor.resampleAudio(x, 16000)
    assert np.array_equal(bits(y), bits(x))


# ------------------------------------------------------------------------------------------------ segmentation, pointers, sessions
def test_segmented_equals_single_shot(tmp_path):
    """Several device segments, with read chunks and 600 s pieces straddling segment edges: bit-identical to one segment."""
    rng = np.random.default_rng(5)
    v = (rng.standard_normal((1000 * 650 + 17, 2)) * 6000).astype(np.int16)   # 650 s at 1 kHz: two 600 s pieces
    p = A.write_wav(str(tmp_path / "long.wav"), v, 1000, "s16")
    for kw in (dict(maxReadFrameSize=77_777), dict()):
        one = AudioProcessor.loadAudioAsFloatArray(p, segmentSamples=1 << 26, **kw)
        assert len(one) == 16 * len(v)
        for seg in (1_000_448, 262_144, 1024):
            many = AudioProcessor.loadAudioAsFloatArray(p, segmentSamples=seg, **kw)
            assert np.array_equal(bits(many), bits(one)), (seg, kw)
    # 44.1 kHz stereo, downsampling
    w = (rng.standard_normal((44100 * 31 + 5, 2)) * 3000).astype(np.int16)
    q = A.write_wav(str(tmp_path / "s44.wav"), w, 44100, "s16")
    one = AudioProcessor.loadAudio(q, maxReadFrameSize=100_003, segmentSamples=1 << 24)
    many = AudioProcessor.loadAudio(q, maxReadFrameSize=100_003, segmentSamples=65_536)
    assert np.array_equal(bits(many), bits(one))
    ref = A.load_reference(A.to_float(w, "s16"), 44100, maxReadFrameSize=100_003)
    assert np.abs(one - ref).max() <= fir_bound(44100, 1.0)


def test_host_and_device_pointers_give_identical_bits():
    import torch
    rng = np.random.default_rng(2)
    v = rng.integers(-2 ** 23, 2 ** 23, (48000 * 3 + 7, 6))
    raw = _as_input(v, "s24")
    mode = ("sum", [0, 2, 2, 5])
    host = AudioProcessor.resampleAudio(raw, 48000, mode, sampleFormat="s24", maxReadFrameSize=50_000)
    dev_in = AudioProcessor.resampleAudio(torch.from_numpy(raw).cuda(), 48000, mode, sampleFormat="s24", maxReadFrameSize=50_000)
    out = torch.full((len(host) + 10,), float("nan"), device="cuda")
    dev_out = AudioProcessor.resampleAudio(raw, 48000, mode, sampleFormat="s24", maxReadFrameSize=50_000, out=out)
    both = AudioProcessor.resampleAudio(torch.from_numpy(raw).cuda(), 48000, mode, sampleFormat="s24", maxReadFrameSize=50_000,
                                        out=torch.empty(len(host), device="cuda"), segmentSamples=4096)
    assert dev_out.is_cuda and torch.isnan(out[len(host):]).all()
    for y in (dev_in, dev_out, both):
        assert np.array_equal(bits(y), bits(host))


def test_workspace_follows_the_call_size(tmp_path):
    """A short file allocates a small workspace: the segment never exceeds the call's output (a 1 s, 1 kHz u8 file once sized its
    output staging by the input-byte budget alone: 2 GiB of device memory)."""
    import torch
    p = A.write_wav(str(tmp_path / "short.wav"), np.random.default_rng(4).integers(0, 256, (1000, 1)), 1000, "u8")
    model = wk.Model("toy", max_batch=1, dtype="bf16")
    model.init_random(1)
    session = wk.TextDecoder(model, 1)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    y = AudioProcessor.loadAudio(p, session=session)
    used = free0 - torch.cuda.mem_get_info()[0]
    assert len(y) == 16000
    assert used < 64 << 20, f"{used / 2**20:.1f} MiB of device memory for a 1 s file"
    ref = A.load_reference(A.to_float(np.frombuffer(open(p, "rb").read()[44:], np.uint8)[:, None], "u8"), 1000)
    assert np.abs(y - ref).max() <= fir_bound(1000, 1.0)


def test_two_sessions_on_two_threads(tmp_path):
    path, _ = jfk_44k_stereo(tmp_path)
    q = A.write_wav(str(tmp_path / "m48.wav"), (np.random.default_rng(3).standard_normal(48000 * 20) * 5000).astype(np.int16), 48000, "s16")
    model = wk.Model("toy", max_batch=1, dtype="bf16")
    model.init_random(1)
    sessions = [wk.TextDecoder(model, 1), wk.TextDecoder(model, 1)]
    solo = {p: AudioProcessor.loadAudio(p, maxReadFrameSize=30_000) for p in (path, q)}
    got = {}

    def work(i, p):
        got[i] = [AudioProcessor.loadAudio(p, maxReadFrameSize=30_000, session=sessions[i], segmentSamples=8192) for _ in range(3)]

    th = [threading.Thread(target=work, args=(i, p)) for i, p in enumerate((path, q))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i, p in enumerate((path, q)):
        for y in got[i]:
            assert np.array_equal(bits(y), bits(solo[p]))


# ------------------------------------------------------------------------------------------------ pipeline
def _toy_kit():
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(1024))
    return wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=9, specialTokens=st))


def test_transcribe_audio_paths_equals_load_then_transcribe(tmp_path):
    from whisperkit_b200 import longform as L
    path, _ = jfk_44k_stereo(tmp_path)
    kit = _toy_kit()
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0)
    got = kit.transcribe(audioPaths=[path], decodeOptions=o)
    ref = L.transcribe_audio(kit, [AudioProcessor.loadAudio(path)], o)
    assert len(got) == 1
    assert [g.tokens for g in got[0].segments] == [g.tokens for g in ref[0].segments]
    assert [(g.seek, g.start, g.end, g.tokenLogProbs) for g in got[0].segments] == [(g.seek, g.start, g.end, g.tokenLogProbs) for g in ref[0].segments]
    assert got[0].windows == ref[0].windows
    one = kit.transcribe(audioPath=path, decodeOptions=o)
    assert [g.tokens for g in one.segments] == [g.tokens for g in ref[0].segments]


def test_invalid_files_fail_only_their_own_slot(tmp_path):
    path, _ = jfk_44k_stereo(tmp_path)
    bad_fmt = A.write_wav(str(tmp_path / "adpcm.wav"), np.zeros((1000, 1), np.int16), 16000, "s16", format_tag=2)
    bad_rate = A.write_wav(str(tmp_path / "slow.wav"), np.zeros((1000, 1), np.int16), 400, "s16")
    missing = str(tmp_path / "nope.wav")
    kit = _toy_kit()
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12, temperatureFallbackCount=0)
    res = kit.transcribe(audioPaths=[missing, path, bad_fmt, bad_rate], decodeOptions=o)
    assert isinstance(res[0], wk.WhisperError) and res[0].status == _lib.WK_ERR_LOAD_AUDIO_FAILED
    assert isinstance(res[2], wk.WhisperError) and res[2].status == _lib.WK_ERR_LOAD_AUDIO_FAILED
    assert isinstance(res[3], wk.WhisperError) and res[3].status == _lib.WK_ERR_INVALID_ARGUMENT
    alone = kit.transcribe(audioPaths=[path], decodeOptions=o)[0]
    assert [g.tokens for g in res[1].segments] == [g.tokens for g in alone.segments]
    with pytest.raises(wk.WhisperError):
        kit.transcribe(audioPath=missing, decodeOptions=o)


def test_log_mel_of_the_loaded_44k_file(tmp_path):
    """Log-mel of jfk loaded from 44.1 kHz stereo on the GPU vs the log-mel of the oracle-resampled signal (the mel tolerance of the
    pipeline tests, 1e-3); the distance to the 16 kHz golden log-mel (resampling round trip) is printed."""
    path, s = jfk_44k_stereo(tmp_path)
    kit = _toy_kit()
    y = AudioProcessor.loadAudio(path, session=kit.textDecoder)
    ref = A.load_reference(A.to_float(s, "s16"), 44100).astype(np.float32)
    fe = kit.featureExtractor
    mel_gpu = fe.logMelSpectrogram(y[None], samples_per_window=[len(y)]).numpy()[0]
    mel_ref = fe.logMelSpectrogram(ref[None], samples_per_window=[len(ref)]).numpy()[0]
    d = float(np.abs(mel_gpu - mel_ref).max())
    assert d <= 1e-3, d
    z = np.load(os.path.join(GOLDEN, "jfk_logmel_hf.npz"))
    g = float(np.abs(mel_gpu[:, ::8] - z["mel80_sub8"]).max())
    print(f"[jfk 44.1 kHz stereo] log-mel vs oracle-resampled {d:.2e}; vs the 16 kHz golden {g:.2e}")
