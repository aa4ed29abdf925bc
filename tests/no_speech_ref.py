"""No-speech probability oracle (test infrastructure, restated on top of oracle/decode_ref.py and oracle/seek_ref.py).  The reference
leaves DecodingResult.noSpeechProb at 0 (TextDecoder.swift:802), so openai/whisper decoding.py is the specification:
  * the value          softmax of the raw logits (before any logits filter, no temperature) of the step whose input is the prompt's
                       first <|startoftranscript|>, at <|nospeech|>
  * DecodingFallback   Models.swift:357-381 with that value in the silence rule
  * the seek loop      TranscribeTask.swift:98-279, each window's noSpeechProb feeding SegmentSeeker's skip rule (SegmentSeeker.swift:57-63)
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import numpy as np

from oracle import decode_ref as D
from oracle import seek_ref as S


def no_speech_prob(logits: np.ndarray, st: D.SpecialTokens) -> float:
    """openai/whisper: probs_at_sot = logits[sot_index].float().softmax(-1); no_speech_prob = probs_at_sot[no_speech] (float64 here)."""
    x = np.asarray(logits, dtype=np.float64).reshape(-1)
    e = np.exp(x - x.max())
    return float(e[st.noSpeechToken] / e.sum())


def decode_with_no_speech(predict_logits: Callable[[int, int], np.ndarray], prompt: Sequence[int], options: D.DecodingOptions,
                          st: D.SpecialTokens, isModelMultilingual: bool, sampler: Optional[D.GreedyTokenSampler] = None):
    """decodeText that also evaluates the rule at sot_index = prompt.index(SOT).  Returns (DecodingResult with the silence rule applied,
    noSpeechProb or None when the loop ended before the SOT step)."""
    sot_index = list(prompt).index(st.startOfTranscriptToken)
    r = D.decode_text(predict_logits, prompt, options, st, isModelMultilingual, sampler, keep_logits=True)
    p = no_speech_prob(r.stepLogits[sot_index], st) if len(r.stepLogits) > sot_index else None
    r.fallback = D.DecodingFallback.make(options, r.isFirstTokenLogProbTooLow, 0.0 if p is None else p, r.compressionRatio, r.avgLogProb)
    return r, p


def seek_loop(contentFrames: int, decode_window, windowSamples: int = 480000, timeToken: int = 50364,
              noSpeechThreshold: Optional[float] = 0.6, logProbThreshold: Optional[float] = -1.0, windowClipTime: float = 1.0):
    """oracle/seek_ref.seek_loop without clip timestamps or word timestamps, with each window's noSpeechProb in place of 0.0.
    decode_window(seek, segmentSize) -> object with tokens, tokenLogProbs, avgLogProb, compressionRatio, temperature, noSpeechProb.
    Returns (segments, [(seek, segmentSize, skipped)] per window)."""
    allSegments, windows = [], []
    seek = 0
    windowPadding = int(np.float32(windowClipTime) * np.float32(S.SAMPLE_RATE))
    while seek < contentFrames - windowPadding:
        segmentSize = min(windowSamples, contentFrames - seek)
        r = decode_window(seek, segmentSize)
        previousSeek = seek
        newSeek, segs = S.find_seek_point_and_segments(r.tokens, r.tokenLogProbs, r.noSpeechProb, r.avgLogProb, r.compressionRatio,
                                                       r.temperature, noSpeechThreshold, logProbThreshold, len(allSegments), seek,
                                                       segmentSize, S.SAMPLE_RATE, timeToken)
        windows.append((seek, segmentSize, segs is None))
        seek = max(seek, newSeek)
        if seek <= previousSeek:   # termination guard shared with csrc/longform.cu
            seek = previousSeek + segmentSize
        if segs is not None:
            allSegments.extend(segs)
    return allSegments, windows
