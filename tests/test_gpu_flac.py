"""FLAC loading on the GPU (csrc/flac.cu): a FLAC file loads bit for bit like a WAV file holding the same integers, across channel counts,
sample sizes, rates, channel modes, time ranges, read sizes, segment sizes, host and device outputs, with and without a session.  The
FLAC files come from tests/flac_ref.py and, where present, from an independent encoder (tests/golden/*.flac)."""
import glob
import os
import threading

import numpy as np
import pytest

import whisperkit_b200 as wk
from oracle import audio_ref as A
from oracle import decode_ref as D
from tests import flac_ref as F
from whisperkit_b200 import _lib
from whisperkit_b200.audio import AudioProcessor

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
JFK = os.path.join(GOLDEN, "jfk.wav")


def bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def twins(tmp_path, name, x, rate, bps, **kw):
    """(flac path, wav path) of the same integers."""
    fp = str(tmp_path / f"{name}.flac")
    with open(fp, "wb") as f:
        f.write(F.encode(x, rate, bps, **kw))
    wp = A.write_wav(str(tmp_path / f"{name}.wav"), F.left_justify(x, bps), rate, F.container(bps))
    return fp, wp


def same(fp, wp, **kw):
    a = AudioProcessor.loadAudio(fp, **kw)
    b = AudioProcessor.loadAudio(wp, **kw)
    assert len(a) == len(b) and np.array_equal(bits(a), bits(b)), kw
    return a


CASES = [  # channels, bits per sample, rate, stereo mode
    (1, 16, 16000, "auto"), (2, 16, 44100, "auto"), (2, 16, 44100, "left_side"), (2, 16, 48000, "side_right"),
    (2, 24, 44100, "mid_side"), (2, 8, 8000, "independent"), (1, 12, 8000, "auto"), (2, 20, 96000, "mid_side"),
    (6, 24, 48000, "auto"), (8, 16, 44100, "auto"), (8, 32, 16000, "auto"), (2, 32, 44100, "mid_side"), (2, 32, 48000, "left_side"),
    (1, 32, 96000, "auto"), (6, 8, 16000, "auto"), (8, 20, 8000, "auto"),
]


@pytest.mark.parametrize("ch,bps,rate,stereo", CASES)
def test_flac_equals_its_wav_twin(tmp_path, ch, bps, rate, stereo):
    x = F.test_signal(int(rate * 1.37) + 11, ch, bps, seed=ch * 100 + bps)
    spec = lambda fi, c, v, sb: [dict(), dict(kind="lpc", order=8, precision=14), dict(kind="fixed", order=fi % 5),
                                 dict(kind="verbatim")][fi % 4]
    fp, wp = twins(tmp_path, "t", x, rate, bps, block_size=1152, stereo=stereo, spec=spec)
    info = AudioProcessor.audioInfo(fp)
    assert (info["sampleRate"], info["channels"], info["frames"], info["sampleFormat"]) == (rate, ch, len(x), F.container(bps))
    modes = [("sum", None)] + ([("sum", [ch - 1, 0, 0]), ("channel", ch - 1)] if ch > 1 else [])
    for mode in modes:
        same(fp, wp, channelMode=mode)
    same(fp, wp, startTime=0.311, endTime=1.057)
    same(fp, wp, maxReadFrameSize=10024)
    same(fp, wp, segmentSamples=4096, maxReadFrameSize=10024)
    a = AudioProcessor.loadAudioAsFloatArray(fp)
    assert np.array_equal(bits(a), bits(AudioProcessor.loadAudioAsFloatArray(wp)))


def test_outputs_and_sessions(tmp_path):
    import torch
    x = F.test_signal(44100 * 3 + 5, 2, 16, seed=7)
    fp, wp = twins(tmp_path, "s", x, 44100, 16, block_size=4096)
    ref = AudioProcessor.loadAudio(wp, segmentSamples=8192)
    kit = _toy_kit()
    for session in (None, kit.textDecoder):
        host = AudioProcessor.loadAudio(fp, session=session, segmentSamples=8192)
        out = torch.full((len(ref) + 7,), float("nan"), device="cuda")
        dev = AudioProcessor.loadAudio(fp, session=session, out=out, segmentSamples=8192)
        assert dev.is_cuda and torch.isnan(out[len(ref):]).all()
        assert np.array_equal(bits(host), bits(ref)) and np.array_equal(bits(dev), bits(ref))


def test_small_segments_cut_through_frames(tmp_path):
    x = F.test_signal(48000 * 4 + 3, 2, 24, seed=3)
    fp, wp = twins(tmp_path, "seg", x, 48000, 24, block_size=4608, stereo="mid_side")
    for seg in (1024, 3000, 65536):
        same(fp, wp, segmentSamples=seg, maxReadFrameSize=17_000)
        same(fp, wp, segmentSamples=seg, channelMode=("channel", 1), startTime=0.5, endTime=3.3)


# ------------------------------------------------------------------------------------------------ jfk, false sync, variable blocking
def _jfk_flacs():
    return sorted(glob.glob(os.path.join(GOLDEN, "jfk_*.flac")))


def test_jfk_kats_bit_exact(tmp_path):
    import wave
    with wave.open(JFK, "rb") as w:
        s = np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").astype(np.int64)
    ref = s.astype(np.float32) / np.float32(32768)
    own = str(tmp_path / "jfk_ref.flac")
    with open(own, "wb") as f:
        f.write(F.encode(s[:, None], 16000, 16, spec=lambda fi, c, v, sb: dict(kind="lpc", order=12, precision=15)))
    paths = [own] + _jfk_flacs()
    for p in paths:
        a = AudioProcessor.loadAudio(p)
        assert a.dtype == np.float32 and len(a) == 176000 and np.array_equal(bits(a), bits(ref)), p
        b = AudioProcessor.loadAudio(p, startTime=1.2)
        assert len(b) == 156800 and np.array_equal(bits(b), bits(ref[19200:]))
        c = AudioProcessor.loadAudio(p, startTime=1.2, endTime=3.4)
        assert len(c) == 35200 and np.array_equal(bits(c), bits(ref[19200:54400]))
        assert np.array_equal(bits(AudioProcessor.loadAudioAsFloatArray(p)), bits(ref))


def test_independent_fixtures_equal_their_samples(tmp_path):
    """Each committed fixture decodes on the GPU like the WAV of the integers the host decoder finds in it (the host tests check those
    integers against the STREAMINFO MD5)."""
    from tests.test_flac_host import host_decode
    for p in sorted(glob.glob(os.path.join(GOLDEN, "*.flac"))):
        st, _, x, fmt = host_decode(open(p, "rb").read())
        assert st == 0, p
        wp = A.write_wav(str(tmp_path / (os.path.basename(p) + ".wav")), F.left_justify(x, fmt[2]), fmt[0], F.container(fmt[2]))
        for mode in (("sum", None), ("channel", x.shape[1] - 1)):
            same(p, wp, channelMode=mode)


def test_false_sync_and_variable_blocking(tmp_path):
    from tests.test_flac_host import false_sync_stream, variable_stream
    for name, (data, x, rate, bps) in (("fs", false_sync_stream()), ("var", variable_stream())):
        fp = str(tmp_path / f"{name}.flac")
        open(fp, "wb").write(data)
        wp = A.write_wav(str(tmp_path / f"{name}.wav"), F.left_justify(x, bps), rate, F.container(bps))
        same(fp, wp)
        same(fp, wp, segmentSamples=1024, startTime=0.01)


# ------------------------------------------------------------------------------------------------ errors
def test_crc_failure_names_the_offset_and_the_session_recovers(tmp_path):
    x = F.test_signal(16000 * 3, 1, 16, seed=9)
    frames = F.encode(x, 16000, 16, block_size=2048, frames_only=True)
    data = bytearray(F.encode(x, 16000, 16, block_size=2048))
    start = AudioProcessor.audioInfo(_write(tmp_path / "ok.flac", bytes(data)))["dataOffset"]
    k = 5
    off = start + sum(len(f) for f in frames[:k])
    data[off + len(frames[k]) // 2] ^= 0x10                   # a residual bit of frame k
    bad = _write(tmp_path / "bad.flac", bytes(data))
    good, wp = twins(tmp_path, "good", x, 16000, 16, block_size=2048)
    kit = _toy_kit()
    with pytest.raises(wk.WhisperError) as e:
        AudioProcessor.loadAudio(bad, session=kit.textDecoder)
    assert e.value.status == _lib.WK_ERR_LOAD_AUDIO_FAILED and e.value.case == "loadAudioFailed"
    assert f"byte {off}" in str(e.value) and "CRC-16" in str(e.value), str(e.value)
    a = AudioProcessor.loadAudio(good, session=kit.textDecoder)
    assert np.array_equal(bits(a), bits(AudioProcessor.loadAudio(wp)))


def _write(p, data):
    with open(p, "wb") as f:
        f.write(data)
    return str(p)


# ------------------------------------------------------------------------------------------------ pipeline and threads
def _toy_kit():
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(1024))
    return wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=9, specialTokens=st))


def test_transcribe_flac_wav_and_a_broken_flac(tmp_path):
    x = F.test_signal(44100 * 7, 2, 16, seed=11)
    fp, wp = twins(tmp_path, "a", x, 44100, 16)
    data = bytearray(open(fp, "rb").read())
    data[len(data) // 2] ^= 0x01
    broken = _write(tmp_path / "broken.flac", bytes(data))
    kit = _toy_kit()
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12, temperatureFallbackCount=0)
    res = kit.transcribe(audioPaths=[fp, wp, broken], decodeOptions=o)
    assert not isinstance(res[0], wk.WhisperError) and not isinstance(res[1], wk.WhisperError)
    assert [g.tokens for g in res[0].segments] == [g.tokens for g in res[1].segments]
    assert [(g.seek, g.start, g.end, g.tokenLogProbs) for g in res[0].segments] == \
        [(g.seek, g.start, g.end, g.tokenLogProbs) for g in res[1].segments]
    assert isinstance(res[2], wk.WhisperError) and res[2].status == _lib.WK_ERR_LOAD_AUDIO_FAILED


def test_malformed_subframes_fail_with_their_reason(tmp_path):
    from tests.test_flac_host import malformed_subframes
    for name, data, reason in malformed_subframes():
        p = _write(tmp_path / f"{name}.flac", data)
        with pytest.raises(wk.WhisperError) as e:
            AudioProcessor.loadAudio(p)
        assert e.value.status == _lib.WK_ERR_LOAD_AUDIO_FAILED and reason in str(e.value), (name, str(e.value))


def test_two_sessions_on_two_threads(tmp_path):
    p1, _ = twins(tmp_path, "t1", F.test_signal(44100 * 5, 2, 16, seed=1), 44100, 16)
    p2, _ = twins(tmp_path, "t2", F.test_signal(48000 * 4, 6, 24, seed=2), 48000, 24, block_size=1152)
    model = wk.Model("toy", max_batch=1, dtype="bf16")
    model.init_random(1)
    sessions = [wk.TextDecoder(model, 1), wk.TextDecoder(model, 1)]
    solo = {p: AudioProcessor.loadAudio(p, maxReadFrameSize=30_000) for p in (p1, p2)}
    got = {}

    def work(i, p):
        got[i] = [AudioProcessor.loadAudio(p, maxReadFrameSize=30_000, session=sessions[i], segmentSamples=8192) for _ in range(3)]

    th = [threading.Thread(target=work, args=(i, p)) for i, p in enumerate((p1, p2))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for i, p in enumerate((p1, p2)):
        for y in got[i]:
            assert np.array_equal(bits(y), bits(solo[p]))
