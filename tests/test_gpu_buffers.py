"""Every device and pinned buffer the library allocates has one owner that releases it: wk_debug_live_bytes (the bytes held through that
owner, process-wide) comes back to its earlier value exactly after

  * a session that ran a beam decode, a best-of call with fallbacks, a wordTimestamps decode, an alignTokens call, a decode with more than
    4096 suppress entries (the suppress-pool regrowth) and an audio conversion is freed - twice, the second cycle leaving what the first left;
  * wk_filter_sample rejects a suppress list longer than 4096 entries;
  * a model whose mel workspace exists is freed.

Long-form transcription is not called here: its pinned staging is kept for the life of the calling thread by design."""
import ctypes as C
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from whisperkit_b200.audio import AudioProcessor  # noqa: E402

FORCE = dict(logProbThreshold=0.0, compressionRatioThreshold=None)   # every window walks the fallback ladder


def live():
    gc.collect()   # handles earlier tests left in reference cycles are released now, not in the middle of a measurement
    dev, pinned = C.c_int64(), C.c_int64()
    assert _lib.load().wk_debug_live_bytes(C.byref(dev), C.byref(pinned)) == 0
    return dev.value, pinned.value


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=16)
    d.update(kw)
    return wk.DecodingOptions(**d)


def session_cycle(model, enc2, st):
    dec = wk.TextDecoder(model, 4)
    prompt = dec.prefillDecoderInputs(opts(), st)
    dec.decodeText(enc2, prompt, opts(beamSize=2, temperatureFallbackCount=0), st)
    dec.decodeText(enc2, prompt, opts(bestOf=2, temperatureFallbackCount=1, seed=3, **FORCE), st)
    words = dec.decodeText(enc2, prompt, opts(wordTimestamps=True), st)
    dec.alignTokens(None, [r.tokens for r in words], st)
    # repeats count: the pool does not deduplicate, so 5000 entries below specialTokenBegin make it regrow past its 4096 entries
    dec.decodeText(enc2, prompt, opts(suppressTokens=[1, 2, 3, 4, 5] * 1000), st)
    frames = (np.sin(np.arange(44100) * 0.05) * 8000).astype(np.int16)
    assert len(AudioProcessor.resampleAudio(frames, 44100, session=dec)) == 16000
    dec.close()


def test_session_round_trip_returns_every_byte():
    model = wk.Model("toy", max_batch=4, dtype="bf16")
    model.init_random(7)
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(1024))
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    enc2 = enc.encodeFeatures(fe.logMelSpectrogram(np.stack([mel_ref.synthetic_pcm(700 + i) for i in range(2)])))
    first = wk.TextDecoder(model, 4)
    before = live()
    session_cycle(model, enc2, st)
    after_one = live()
    assert after_one == before
    session_cycle(model, enc2, st)
    assert live() == after_one
    first.close()
    enc2.close()
    model.close()


def test_rejected_filter_input_frees_its_temporaries():
    model = wk.Model("toy", max_batch=2, dtype="bf16")
    model.init_random(2)
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(1024))
    logits = np.random.default_rng(0).standard_normal((2, 1024)).astype(np.float32)
    before = live()
    with pytest.raises(wk.WhisperError) as e:
        wk.filter_and_sample(model, logits, [[1, 2], [3]], st, opts(suppressTokens=[7] * 5000))
    assert e.value.status == _lib.WK_ERR_INVALID_ARGUMENT
    assert live() == before
    model.close()


def test_model_round_trip_returns_every_byte():
    before = live()
    model = wk.Model("toy", max_batch=2, dtype="bf16")
    model.init_random(1)
    assert live()[0] > before[0]
    mel = wk.FeatureExtractor(model).logMelSpectrogram(mel_ref.synthetic_pcm(5)[None])   # the model's mel / encoder workspace
    mel.close()
    model.close()
    assert live() == before
