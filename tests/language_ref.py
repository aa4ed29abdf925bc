"""Language-detection oracle (test infrastructure, restated on top of oracle/decode_ref.py):
  * TextDecoder.detectLanguage                    Sources/WhisperKit/Core/TextDecoder.swift:420-539
  * TranscribeTask.decodeWithFallback             Sources/WhisperKit/Core/TranscribeTask.swift:316-411
  * DecodingOptions.detectLanguage default        Sources/WhisperKit/Core/Configurations.swift:222
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence, Tuple

import numpy as np

from oracle import decode_ref as D


def resolves_detection(options: D.DecodingOptions, detectLanguage: Optional[bool]) -> bool:
    """detectLanguage ?? !usePrefillPrompt (Configurations.swift:222)."""
    return bool(detectLanguage) if detectLanguage is not None else not options.usePrefillPrompt


def detect_language(predict_logits: Callable[[int, int], np.ndarray], st: D.SpecialTokens, allLanguageTokens: Sequence[int],
                    sampler: D.GreedyTokenSampler) -> Tuple[int, float]:
    """TextDecoder.detectLanguage: one forward of [SOT] at position 0, LanguageLogitsFilter(sampleBegin = 0), the rung's sampler.
    Returns (language token, its log-prob)."""
    currentTokens = [st.startOfTranscriptToken]
    logits = np.array(predict_logits(st.startOfTranscriptToken, 0), dtype=np.float32).reshape(-1)
    logits = D.LanguageLogitsFilter(allLanguageTokens, len(logits), sampleBegin=0).filterLogits(logits, currentTokens)
    res = sampler.update(currentTokens, logits, [0.0])
    return res.tokens[-1], res.logProbs[-1]


def rung_temperatures(options: D.DecodingOptions):
    """Float16(temperature) + Float16(i) * Float16(increment), i = 0 ... temperatureFallbackCount (TranscribeTask.swift:327)."""
    f16 = np.float16
    return [float(f16(f16(options.temperature) + f16(f16(i) * f16(options.temperatureIncrementOnFallback))))
            for i in range(options.temperatureFallbackCount + 1)]


def decode_with_fallback(make_predict: Callable[[], Callable[[int, int], np.ndarray]], options: D.DecodingOptions, st: D.SpecialTokens,
                         isModelMultilingual: bool, allLanguageTokens: Sequence[int], languageToken: Optional[int] = None,
                         detectLanguage: Optional[bool] = None, rng=None):
    """decodeWithFallback: every rung of the temperature ladder first detects the language (multilingual model, no language set,
    detectLanguage) with that rung's sampler and, with usePrefillPrompt, rebuilds the prompt with it (prefillDecoderInputs); then
    decodeText.  `make_predict()` returns a fresh model call (empty KV cache).  Returns (DecodingResult, detected token or None,
    the prompt the returned rung decoded with)."""
    detect = isModelMultilingual and languageToken is None and resolves_detection(options, detectLanguage)
    prompt = D.prefill_prompt(options if options.usePrefillPrompt else None, st, isModelMultilingual, languageToken)
    detected, result = None, None
    for temp in rung_temperatures(options):
        sampler = D.GreedyTokenSampler(temp, st.endToken, options, rng)
        if detect:
            detected, _ = detect_language(make_predict(), st, allLanguageTokens, sampler)
            if options.usePrefillPrompt:
                prompt = D.prefill_prompt(options, st, isModelMultilingual, detected)
        result = D.decode_text(make_predict(), prompt, options, st, isModelMultilingual, sampler)
        if not (result.fallback is not None and result.fallback.needsFallback):
            break
    return result, detected, prompt


def rewrite_language_slot(prompt: Sequence[int], st: D.SpecialTokens, allLanguageTokens: Sequence[int], detected: int):
    """The library's in-place rebuild: the token right after the prompt's first SOT becomes the detected language when it holds a
    language token; otherwise the prompt is left alone (the language is only reported)."""
    p = list(prompt)
    if st.startOfTranscriptToken in p:
        i = p.index(st.startOfTranscriptToken) + 1
        if i < len(p) and p[i] in set(allLanguageTokens):
            p[i] = detected
    return p
