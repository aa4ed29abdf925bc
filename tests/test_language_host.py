"""Language detection inside decoding (DecodingOptions.detectLanguage) on the host: the oracle's per-rung detection and prompt rebuild
(tests/language_ref.py), the library's rebuild rule against it, when detection is skipped, and how the Python options resolve."""
import numpy as np

import whisperkit_b200 as wk
from oracle import decode_ref as D
from tests import language_ref as L

V = 1024
ST = D.SpecialTokens.toy(V)
LANGS = [ST.englishToken] + list(range(200, 260))


def make_predict_factory(boost_token, boost=8.0):
    """A deterministic toy model: logits depend on (token, position); [SOT] at position 0 favours `boost_token`."""
    def make():
        def predict(token, index):
            x = np.random.default_rng(token * 1000 + index).standard_normal(V).astype(np.float32)
            if token == ST.startOfTranscriptToken and index == 0:
                x[boost_token] += boost
            return x
        return predict
    return make


OPTION_VARIANTS = [
    dict(),
    dict(promptTokens=[5, 6, 7]),
    dict(prefixTokens=[11, 12]),
    dict(promptTokens=[5, 6, 7], prefixTokens=[11, 12]),
    dict(withoutTimestamps=True, task="translate"),
]


def test_prompt_rebuild_equals_the_explicit_language_prompt():
    """With usePrefillPrompt the detected <|xx|> replaces the slot right after the first SOT - with and without promptTokens (SOT is not
    first) and prefixTokens - exactly as prefillDecoderInputs rebuilds the prompt with the detected language."""
    for kw in OPTION_VARIANTS:
        o = D.DecodingOptions(**kw)
        placeholder = D.prefill_prompt(o, ST, True)
        for lang in (LANGS[0], LANGS[7], LANGS[-1]):
            assert L.rewrite_language_slot(placeholder, ST, LANGS, lang) == D.prefill_prompt(o, ST, True, lang), kw


def test_decode_with_fallback_detects_per_rung_and_decodes_with_the_detected_language():
    for kw in OPTION_VARIANTS:
        o = D.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12, temperatureFallbackCount=0, **kw)
        make = make_predict_factory(LANGS[9])
        res, detected, prompt = L.decode_with_fallback(make, o, ST, True, LANGS, detectLanguage=True)
        assert detected == LANGS[9]
        assert prompt == D.prefill_prompt(o, ST, True, detected)
        explicit, none, _ = L.decode_with_fallback(make, o, ST, True, LANGS, languageToken=detected, detectLanguage=True)
        assert none is None
        assert res.tokens == explicit.tokens and res.steps == explicit.steps
        np.testing.assert_array_equal(res.tokenLogProbs, explicit.tokenLogProbs)


def test_ladder_rungs_detect_at_their_own_temperature():
    """Each rung detects with its own sampler: with a flat language distribution a T > 0 rung can pick another language than T = 0."""
    o = D.DecodingOptions(sampleLength=6, temperatureFallbackCount=3, logProbThreshold=100.0, compressionRatioThreshold=None)
    make = make_predict_factory(LANGS[3], boost=0.0)
    res, detected, prompt = L.decode_with_fallback(make, o, ST, True, LANGS, detectLanguage=True, rng=np.random.default_rng(3))
    assert res.temperature == round(L.rung_temperatures(o)[-1], 3)   # logProbThreshold 100: every rung asks for a fallback
    assert detected in LANGS
    assert prompt[1] == detected
    t0, _ = L.detect_language(make(), ST, LANGS, D.GreedyTokenSampler(0.0, ST.endToken, o))
    logits = make()(ST.startOfTranscriptToken, 0)
    assert t0 == LANGS[int(np.argmax(logits[LANGS]))]


def test_report_only_without_prefill_prompt():
    """usePrefillPrompt = false: the prompt is [SOT] alone, there is no <|xx|> slot, detection only reports."""
    o = D.DecodingOptions(usePrefillPrompt=False)
    assert L.resolves_detection(o, None)
    p = D.prefill_prompt(None, ST, True)
    assert L.rewrite_language_slot(p, ST, LANGS, LANGS[4]) == p


def test_detection_skipped_for_a_set_language_or_an_english_only_model():
    o = D.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=6, temperatureFallbackCount=0)
    make = make_predict_factory(LANGS[2])
    _, detected, _ = L.decode_with_fallback(make, o, ST, True, LANGS, languageToken=LANGS[5], detectLanguage=True)
    assert detected is None
    _, detected, _ = L.decode_with_fallback(make, o, ST, False, LANGS, detectLanguage=True)
    assert detected is None
    # the Python options: an English-only model gets no language list
    en = wk.SpecialTokens.from_any(D.SpecialTokens.english_only())
    assert wk.api.language_tokens(en, 51864) == []
    opts = wk.DecodingOptions(detectLanguage=True)
    assert wk.api.with_language_tokens(opts, en, 51864) is opts


def test_python_options_resolve_like_the_reference():
    assert wk.DecodingOptions().to_c()[0].detect_language == 0                        # usePrefillPrompt = true
    assert wk.DecodingOptions(usePrefillPrompt=False).to_c()[0].detect_language == 1  # detectLanguage ?? !usePrefillPrompt
    assert wk.DecodingOptions(usePrefillPrompt=False, detectLanguage=False).to_c()[0].detect_language == 0
    o, keep = wk.DecodingOptions(detectLanguage=True, allLanguageTokens=[7, 8, 9]).to_c()
    assert o.detect_language == 1 and o.n_language_tokens == 3 and [o.language_tokens[i] for i in range(3)] == [7, 8, 9]
    assert wk.DecodingOptions().to_c()[0].n_language_tokens == 0
    # without a tokenizer the list is the vocabulary's language block [englishToken, translateToken)
    v3 = wk.SpecialTokens.from_any(D.SpecialTokens.large_v3())
    assert wk.api.language_tokens(v3, 51866) == list(range(50259, 50359))            # the 100 large-v3 languages
    assert len(wk.api.language_tokens(wk.SpecialTokens(), 51865)) == 99
    assert len(wk.api.LANGUAGE_CODES) == 100 and wk.api.LANGUAGE_CODES[0] == "en" and wk.api.LANGUAGE_CODES[-1] == "yue"
    filled = wk.api.with_language_tokens(wk.DecodingOptions(usePrefillPrompt=False), v3, 51866)
    assert filled.allLanguageTokens == list(range(50259, 50359))
    assert wk.api.with_language_tokens(wk.DecodingOptions(), v3, 51866).allLanguageTokens is None   # detection off: untouched
