"""Audio loading, host side (no GPU): the float64 resampler restatement against scipy.signal.resample_poly, the library's filter design
against scipy.signal.firwin, the WAV header parser on written files, convertToMono's rules, the reference's read plan, and the output
lengths wk_audio_load reports without a device."""
import ctypes as C
import os
import wave

import numpy as np
import pytest
from scipy.signal import firwin, resample_poly

import whisperkit_b200 as wk
from oracle import audio_ref as A
from whisperkit_b200 import _lib
from whisperkit_b200.audio import AudioProcessor, filter_taps

RATES = [8000, 11025, 22050, 32000, 44056, 44100, 48000, 96000, 384000]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
JFK = os.path.join(GOLDEN, "jfk.wav")


@pytest.mark.parametrize("rate", RATES)
def test_resample_restatement_matches_scipy(rate):
    rng = np.random.default_rng(rate)
    up, down = A.ratio(rate)
    half = 10 * max(up, down)
    for n in (1, 5, 2 * half // up + 3, 1001, 3 * rate + 7):
        x = rng.uniform(-1, 1, n)
        y = A.resample(x, rate)
        ref = resample_poly(x, up, down)
        assert y.shape == ref.shape == (-(-n * up // down),)
        assert np.abs(y - ref).max() <= 1e-12, (rate, n)
    assert A.resample(np.zeros(0), rate).shape == (0,)


def test_passthrough_is_an_exact_copy():
    x = np.random.default_rng(0).standard_normal(1000).astype(np.float32)
    x[3] = -0.0
    y = A.resample(x, 16000)
    assert np.array_equal(y.astype(np.float32).view(np.uint32), x.view(np.uint32))
    assert A.ratio(16000) == (1, 1)


@pytest.mark.parametrize("rate", RATES + [1000, 12345, 16000])
def test_filter_taps_match_firwin(rate):
    h, up, down = filter_taps(rate)
    g = np.gcd(16000, rate)
    assert (up, down) == (16000 // g, rate // g)
    if up == down == 1:
        assert h.size == 0
        return
    mr = max(up, down)
    ref = firwin(2 * 10 * mr + 1, 1.0 / mr, window=("kaiser", 5.0)) * up
    assert h.shape == ref.shape
    assert np.abs(h - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("rate", [999, 384001, 0, -16000])
def test_filter_taps_reject_rates_outside_the_range(rate):
    with pytest.raises(wk.WhisperError) as e:
        filter_taps(rate)
    assert e.value.status == _lib.WK_ERR_INVALID_ARGUMENT


def _python_wave(path, samples, rate, width):
    with wave.open(path, "wb") as w:
        w.setnchannels(samples.shape[1])
        w.setsampwidth(width)
        w.setframerate(rate)
        w.writeframes(A.encode_samples(samples.reshape(-1), {1: "u8", 2: "s16", 3: "s24", 4: "s32"}[width]))


@pytest.mark.parametrize("width,fmt", [(1, "u8"), (2, "s16"), (3, "s24"), (4, "s32")])
def test_info_of_python_wave_files(tmp_path, width, fmt):
    rng = np.random.default_rng(width)
    lim = {1: (0, 256), 2: (-2**15, 2**15), 3: (-2**23, 2**23), 4: (-2**31, 2**31)}[width]
    s = rng.integers(*lim, size=(1234, 3))
    p = str(tmp_path / f"{fmt}.wav")
    _python_wave(p, s, 22050, width)
    info = AudioProcessor.audioInfo(p)
    assert info["sampleRate"] == 22050 and info["channels"] == 3 and info["sampleFormat"] == fmt
    assert info["frames"] == 1234 and info["blockAlign"] == 3 * width and info["dataOffset"] == 44


def test_info_of_hand_built_headers(tmp_path):
    s = np.zeros((100, 2), np.float32)
    p = A.write_wav(str(tmp_path / "f32.wav"), s, 48000, "f32")
    assert AudioProcessor.audioInfo(p)["sampleFormat"] == "f32"
    for fmt in ("s16", "f32", "s24"):
        p = A.write_wav(str(tmp_path / f"ext_{fmt}.wav"), np.zeros((10, 6), np.int32 if fmt != "f32" else np.float32), 44100, fmt,
                        extensible=True)
        info = AudioProcessor.audioInfo(p)
        assert (info["sampleFormat"], info["channels"], info["frames"], info["dataOffset"]) == (fmt, 6, 10, 68)
    # a LIST chunk and an odd-sized chunk (with its pad byte) before data
    p = A.write_wav(str(tmp_path / "list.wav"), np.zeros((7, 1), np.int16), 8000, "s16",
                    chunks_before=[(b"LIST", b"INFOISFT\x05\x00\x00\x00abcd\x00"), (b"odd ", b"xyz"), (b"fact", b"\x07\x00\x00\x00")])
    info = AudioProcessor.audioInfo(p)
    assert info["frames"] == 7 and info["dataOffset"] == 36 + 8 + 18 + 8 + 4 + 8 + 4 + 8
    # a data chunk shorter than its header says: the frames present
    p = A.write_wav(str(tmp_path / "trunc.wav"), np.zeros((50, 2), np.int16), 16000, "s16", data_size=10 ** 6)
    assert AudioProcessor.audioInfo(p)["frames"] == 50
    with open(p, "ab") as f:   # a partial trailing frame does not count
        f.write(b"\x01\x02")
    assert AudioProcessor.audioInfo(p)["frames"] == 50


@pytest.mark.parametrize("case,needle", [
    ("adpcm", "0x0002"), ("mp3", "0x0055"), ("rifx", "RIFX"), ("f64", "64-bit float"), ("s12", "12-bit"), ("text", "RIFF/WAVE"),
    ("missing", "does not exist")])
def test_unsupported_files_fail_with_load_audio_failed(tmp_path, case, needle):
    p = str(tmp_path / f"{case}.wav")
    s = np.zeros((16, 1), np.int16)
    if case == "adpcm":
        A.write_wav(p, s, 16000, "s16", format_tag=2)
    elif case == "mp3":
        A.write_wav(p, s, 16000, "s16", format_tag=0x55)
    elif case == "rifx":
        A.write_wav(p, s, 16000, "s16", riff=b"RIFX")
    elif case == "f64":
        A.write_wav(p, np.zeros((16, 1), np.float32), 16000, "f32", bits=64)
    elif case == "s12":
        A.write_wav(p, s, 16000, "s16", bits=12)
    elif case == "text":
        open(p, "w").write("not audio at all")
    for call in (lambda: AudioProcessor.audioInfo(p), lambda: AudioProcessor.loadAudio(p)):
        with pytest.raises(wk.WhisperError) as e:
            call()
        assert e.value.status == _lib.WK_ERR_LOAD_AUDIO_FAILED and e.value.case == "loadAudioFailed"
        assert needle in str(e.value), str(e.value)


def test_load_rejects_rates_outside_the_range(tmp_path):
    p = A.write_wav(str(tmp_path / "r.wav"), np.zeros((16, 1), np.int16), 500, "s16")
    assert AudioProcessor.audioInfo(p)["sampleRate"] == 500
    with pytest.raises(wk.WhisperError) as e:
        AudioProcessor.loadAudio(p)
    assert e.value.status == _lib.WK_ERR_INVALID_ARGUMENT


def test_convert_to_mono_hand_cases():
    f32 = np.float32
    x = np.array([[0.5, -0.25, 0.1], [-1.0, 0.5, 0.2], [0.25, 0.25, -0.3]], f32)
    # specificChannel: in range, out of range -> channel 0
    assert np.array_equal(A.convert_to_mono(x, ("channel", 2)), x[:, 2])
    assert np.array_equal(A.convert_to_mono(x, ("channel", 7)), x[:, 0])
    assert np.array_equal(A.convert_to_mono(x, ("channel", -1)), x[:, 0])
    # all invalid indices: channel 0 copied, not normalised
    assert np.array_equal(A.convert_to_mono(x * f32(1e-6), ("sum", [5, -2])), (x * f32(1e-6))[:, 0])
    # a known peak normalisation: channels 0 + 1 -> [0.25, -0.5, 0.5], peak 0.5; originals' peak 1.0 -> scale 2
    assert np.array_equal(A.convert_to_mono(x, ("sum", [0, 1])), np.array([0.5, -1.0, 1.0], f32))
    # invalid indices dropped, duplicates summed twice: 2 * ch1 + ch2 = [-0.4, 1.2, 0.2], originals' peak 0.5 -> scale 0.5 / 1.2
    y = A.convert_to_mono(x, ("sum", [1, 9, 1, 2]))
    mono = (f32(0) + x[:, 1]) + x[:, 1] + x[:, 2]
    assert np.array_equal(y, mono * (f32(0.5) / np.abs(mono).max()))
    # nil and [] mean all channels
    assert np.array_equal(A.convert_to_mono(x, ("sum", None)), A.convert_to_mono(x, ("sum", [])))
    assert np.array_equal(A.convert_to_mono(x, ("sum", None)), A.convert_to_mono(x, ("sum", [0, 1, 2])))
    # an all-zero chunk: scale 0 / max(0, 1e-4) = 0
    z = np.zeros((4, 2), f32)
    assert np.array_equal(A.convert_to_mono(z), np.zeros(4, f32))
    # a quiet chunk whose mix peaks below 1e-4 is scaled by peak / 1e-4
    q = np.array([[2e-5, 1e-5], [-1e-5, 3e-5]], f32)
    mono = q[:, 0] + q[:, 1]
    assert np.array_equal(A.convert_to_mono(q), mono * (np.float32(3e-5) / np.float32(1e-4)))
    # one channel: unchanged
    assert np.array_equal(A.convert_to_mono(x[:, :1], ("sum", [3])), x[:, 0])


def test_read_plan_of_a_25_minute_48k_file():
    length = 25 * 60 * 48000
    plan = A.read_plan(length, 48000, pieceSeconds=600.0)
    expected = []
    for s, e in ((0, 28_800_000), (28_800_000, 57_600_000), (57_600_000, length)):
        for p in range(s, e, 1_323_000):
            expected.append((p, min(p + 1_323_000, e)))
    assert plan == expected
    assert plan[21] == (27_783_000, 28_800_000)          # the partial last read of the first 600 s piece
    assert sum(b - a for a, b in plan) == length
    # loadAudio reads the same file as one piece
    assert A.read_plan(length, 48000)[:22] == [(p, p + 1_323_000) for p in range(0, 22 * 1_323_000, 1_323_000)]
    # startTime / endTime are converted in double and truncated
    assert A.read_plan(176000, 16000, 1.2, 3.4) == [(19200, 54400)]


def test_lengths_without_a_device(tmp_path):
    """wk_audio_load / wk_audio_convert with out = NULL report the length on the host (UnitTests.swift:296-345 counts)."""
    assert len(AudioProcessor.audioInfo(JFK)) and AudioProcessor.audioInfo(JFK)["frames"] == 176000
    lib = _lib.load()

    def n_out(path, **kw):
        from whisperkit_b200.audio import _load_opts
        o, keep = _load_opts(("sum", None), kw.get("startTime", 0.0), kw.get("endTime"), kw.get("maxReadFrameSize"),
                             kw.get("pieceSeconds", 0.0), 0)
        n = C.c_int64()
        _lib.check(lib.wk_audio_load(None, path.encode(), C.byref(o), None, 0, C.byref(n)))
        return n.value

    assert n_out(JFK) == 176000
    assert n_out(JFK, startTime=1.2) == 156800
    assert n_out(JFK, startTime=1.2, endTime=3.4) == 35200
    assert n_out(JFK, pieceSeconds=600.0) == 176000
    p = A.write_wav(str(tmp_path / "s.wav"), np.zeros((44100 * 11, 2), np.int16), 44100, "s16")
    assert n_out(p) == 176000
    assert n_out(p, startTime=1.2, maxReadFrameSize=10024) == 156800
    assert n_out(p, startTime=1.2, endTime=3.4) == 35200


def _length(opts):
    n = C.c_int64()
    _lib.check(_lib.load().wk_audio_load(None, JFK.encode(), C.byref(opts) if opts is not None else None, None, 0, C.byref(n)))
    return n.value


def test_zeroed_options_mean_the_whole_file():
    """A zero-initialised wk_audio_load_opts (what a C or Swift host starts from) is sumChannels(nil), startTime 0, endTime nil."""
    assert _length(None) == 176000
    assert _length(_lib.wk_audio_load_opts()) == 176000
    o = _lib.wk_audio_load_opts()
    o.piece_seconds = 600.0          # loadAudioAsFloatArray from a zeroed struct
    assert _length(o) == 176000
    o.has_end_time, o.end_time = 1, 0.0
    assert _length(o) == 0           # endTime = 0 given explicitly
    o.piece_seconds = 0.0
    assert _length(o) == 0


@pytest.mark.parametrize("piece", [0.0, 600.0])
def test_out_of_range_times(piece):
    o = _lib.wk_audio_load_opts()
    o.piece_seconds = piece
    o.has_end_time, o.end_time = 1, float("inf")     # +inf reads to the end
    assert _length(o) == 176000
    o.end_time = 1e300
    assert _length(o) == 176000
    o.end_time = -5.0                                  # ends before it starts: nothing
    assert _length(o) == 0
    o.has_end_time, o.start_time = 0, 1e300            # starts past the end: nothing
    assert _length(o) == 0
    for start, end in ((float("inf"), None), (-1.0, None), (float("nan"), None), (0.0, float("nan"))):
        o.start_time = start
        o.has_end_time, o.end_time = (0, 0.0) if end is None else (1, end)
        with pytest.raises(wk.WhisperError) as e:
            _length(o)
        assert e.value.status == _lib.WK_ERR_INVALID_ARGUMENT
    o.start_time, o.has_end_time, o.piece_seconds = 0.0, 0, 1e-3   # pieces shorter than a second are refused
    with pytest.raises(wk.WhisperError):
        _length(o)


def test_load_without_a_device_is_an_error():
    if wk.load().wk_device_available():
        pytest.skip("a Hopper device is present")
    with pytest.raises(wk.WhisperError) as e:
        AudioProcessor.loadAudio(JFK)
    assert e.value.case == "modelsUnavailable"
