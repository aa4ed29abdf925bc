"""Language detection inside the decode loop (DecodingOptions.detectLanguage, TranscribeTask.swift:340-365): the same language as the
stand-alone TextDecoder.detectLanguage step, the same decode as naming that language up front (with and without promptTokens, beam
search, word timestamps, the FP8 cross K/V cache), report-only without a prefill prompt, mixed batches, the temperature ladder,
validation, and the long-form stream language."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from tests import language_ref as L  # noqa: E402

V = 1024
ST = D.SpecialTokens.toy(V)
LANGS = [ST.englishToken] + list(range(200, 260))   # <|en|> (the placeholder the prompt carries) + 60 stand-in language ids


def make_kit(slots, seed=4, **kw):
    return wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=slots, seed=seed, specialTokens=wk.SpecialTokens.from_any(ST), **kw))


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=24, temperatureFallbackCount=0, detectLanguage=True, allLanguageTokens=LANGS)
    d.update(kw)
    return wk.DecodingOptions(**d)


def pcm_of(n, base=300):
    return np.stack([mel_ref.synthetic_pcm(base + i) for i in range(n)])


def explicit(o, token):
    return dataclasses.replace(o, detectLanguage=False, languageToken=int(token))


def assert_same(a, b, where):
    assert a.tokens == b.tokens, where
    assert a.steps == b.steps, where
    np.testing.assert_array_equal(np.float32(a.tokenLogProbs), np.float32(b.tokenLogProbs), err_msg=str(where))
    assert np.float32(a.avgLogProb) == np.float32(b.avgLogProb), where


def test_in_loop_detection_matches_the_stand_alone_step_and_the_oracle():
    kit = make_kit(4)
    fe, enc, dec = kit.featureExtractor, kit.audioEncoder, kit.textDecoder
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm_of(4)))
    tok_sa, lp_sa = dec.detectLanguage(enc_t, kit.specialTokens, LANGS)
    logits = dec.predictLogits([ST.startOfTranscriptToken] * 4, [0] * 4)
    res = dec.decodeText(None, None, opts(), kit.specialTokens)
    diff = max(abs(r.languageLogProb - lp) for r, lp in zip(res, lp_sa))
    print(f"in-loop vs stand-alone detection: max |log-prob difference| = {diff:.3e}")
    assert [r.languageToken for r in res] == tok_sa
    assert diff <= 1e-5
    for i, r in enumerate(res):
        t, _ = L.detect_language(lambda tok, idx: logits[i], ST, LANGS, D.GreedyTokenSampler(0.0, ST.endToken, D.DecodingOptions()))
        assert r.languageToken == t, i
        assert r.tokens[1] == t                                    # the prompt was rebuilt with it


@pytest.mark.parametrize("case", ["plain", "promptTokens", "beam", "words", "fp8"])
def test_detection_equals_naming_the_detected_language(case):
    kw = {"promptTokens": dict(promptTokens=[9, 8, 7, 6]), "beam": dict(beamSize=2), "words": dict(wordTimestamps=True)}.get(case, {})
    kit = make_kit(4, crossKVDtype="fp8" if case == "fp8" else None)
    n = 5
    pcm = pcm_of(n, 320)
    o = opts(**kw)
    got = kit.transcribe(pcm, o)
    align = [kit.textDecoder.alignmentWeights(i) for i in range(n)] if case == "words" else None
    langs = [r.languageToken for r in got]
    assert all(t in LANGS for t in langs), langs
    ref = kit.transcribe(pcm, [explicit(o, t) for t in langs])
    for i in range(n):
        assert ref[i].languageToken is None
        assert_same(got[i], ref[i], (case, i))
        if align is not None:
            np.testing.assert_array_equal(align[i], kit.textDecoder.alignmentWeights(i), err_msg=str(i))


def test_report_only_without_prefill_prompt():
    kit = make_kit(3)
    pcm = pcm_of(4, 340)
    o = opts(usePrefillPrompt=False)
    got = kit.transcribe(pcm, o)
    steps_detect = kit.textDecoder.stats()["steps"]
    plain = kit.transcribe(pcm, dataclasses.replace(o, detectLanguage=False))
    assert kit.textDecoder.stats()["steps"] == steps_detect        # detection rode on step 0: not one launch more
    for i in range(4):
        assert got[i].languageToken in LANGS and plain[i].languageToken is None
        assert_same(got[i], plain[i], i)
    assert wk.DecodingOptions(usePrefillPrompt=False).detectsLanguage   # and it is the default without a prefill prompt


def test_mixed_batch_gives_each_window_its_alone_result():
    kit = make_kit(3)
    pcm = pcm_of(6, 360)
    mix = [opts(), opts(languageToken=LANGS[20], detectLanguage=False), opts(languageToken=ST.englishToken, detectLanguage=False),
           opts(promptTokens=[4, 5]), opts(usePrefillPrompt=False), opts(detectLanguage=False)]
    got = kit.transcribe(pcm, mix)
    for i in range(6):
        alone = kit.transcribe(pcm[i], mix[i])[0]
        assert got[i].tokens == alone.tokens and got[i].steps == alone.steps, i
        assert got[i].languageToken == alone.languageToken, i
        np.testing.assert_allclose(got[i].tokenLogProbs, alone.tokenLogProbs, atol=1e-5)
    assert [got[i].languageToken is not None for i in range(6)] == [True, False, False, True, True, False]


def test_ladder_reports_the_language_of_the_returned_rung():
    kit = make_kit(1)
    pcm = pcm_of(1, 380)
    o = opts(temperatureFallbackCount=3, logProbThreshold=0.0, compressionRatioThreshold=None, seed=11)   # every rung falls back
    a = kit.transcribe(pcm, o)[0]
    b = kit.transcribe(pcm, o)[0]
    assert a.tokens == b.tokens and a.languageToken == b.languageToken and a.languageLogProb == b.languageLogProb
    assert kit.textDecoder.stats()["ladder"] == 3
    last = dataclasses.replace(o, temperature=L.rung_temperatures(D.DecodingOptions(temperatureFallbackCount=3))[-1],
                               temperatureFallbackCount=0, seed=11 + 3)
    c = kit.transcribe(pcm, last)[0]                               # rung 3 alone: same temperature, same seed
    assert c.languageToken == a.languageToken and c.tokens == a.tokens


def test_bad_language_lists_fail_their_window_alone():
    kit = make_kit(3)
    pcm = pcm_of(5, 400)
    items = [opts(), opts(allLanguageTokens=[]), opts(allLanguageTokens=[5, V]), opts(allLanguageTokens=LANGS[:10]),
             opts(allLanguageTokens=[], languageToken=LANGS[3])]   # (a set language: the list is not used)
    out = kit.transcribe(pcm, items, returnErrors=True)
    assert isinstance(out[0], wk.DecodingResult) and isinstance(out[4], wk.DecodingResult)
    for i in (1, 2, 3):
        assert isinstance(out[i], wk.WhisperError) and out[i].status == -1, i
    assert out[0].tokens == kit.transcribe(pcm[0], items[0])[0].tokens
    with pytest.raises(wk.WhisperError):
        kit.transcribe(pcm[:2], items[:2])


def test_english_only_model_never_detects():
    en = wk.SpecialTokens.from_any(D.SpecialTokens.english_only())
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="tiny.en", maxBatch=2, seed=3, specialTokens=en))
    pcm = pcm_of(2, 420)
    o = opts(sampleLength=8, allLanguageTokens=None)
    got = kit.transcribe(pcm, o)
    plain = kit.transcribe(pcm, dataclasses.replace(o, detectLanguage=False))
    for i in range(2):
        assert got[i].languageToken is None and got[i].tokens == plain[i].tokens


def test_long_form_streams_keep_their_window_language():
    from whisperkit_b200.longform import transcribe_streams
    kit = make_kit(4)
    arrs = [mel_ref.synthetic_pcm(440 + i)[:80000] for i in range(3)]   # 5 s each
    o = opts(sampleLength=30)
    # windowClipTime 4.99 s: a stream stays live while seek < 0.01 s, so each stream is exactly one window
    segs, windows, langs = transcribe_streams(kit, arrs, o, windowClipTime=4.99, returnLanguages=True)
    assert windows == 3
    for i, a in enumerate(arrs):
        win = kit.transcribe(a[None], o, samplesPerWindow=[len(a)])[0]
        assert langs[i][0] == win.languageToken and abs(langs[i][1] - win.languageLogProb) <= 1e-5, i
        seg_e, _, lang_e = transcribe_streams(kit, [a], explicit(o, langs[i][0]), windowClipTime=4.99, returnLanguages=True)
        assert lang_e == [(-1, 0.0)]
        assert [g.tokens for g in segs[i]] == [g.tokens for g in seg_e[0]], i
