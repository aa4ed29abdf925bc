"""Stream transcription oracle (test infrastructure; see oracle/__init__.py).

CPU restatement of AudioStreamTranscriber (Sources/WhisperKit/Core/Audio/AudioStreamTranscriber.swift) and the AudioProcessor helpers
it uses, with Swift `Float` arithmetic mirrored in numpy float32:
  * processBuffer's relative energy    AudioProcessor.swift:907-917, calculateRelativeEnergy :724-741, calculateAverageEnergy :698-702
  * isVoiceDetected                    AudioProcessor.swift:636-655
  * shouldStopEarly                    AudioStreamTranscriber.swift:208-227, at every appended token (TextDecoder.swift:668-686,732-751)
  * truncation + finalize              the history cut after the stopping token, then TextDecoder.swift:776-853
  * the per-stream state machine       transcribeCurrentBuffer, AudioStreamTranscriber.swift:126-193
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

from .decode_ref import compression_ratio

F = np.float32
SAMPLE_RATE = 16000
BLOCK = 1600          # AudioProcessor.minBufferLength (100 ms)


def swift_min(x, y):
    return y if y < x else x


def swift_max(x, y):
    return y if y >= x else x


def rms(x) -> np.float32:
    """vDSP_rmsqv."""
    x = np.asarray(x, np.float64)
    return F(np.sqrt(np.sum(x * x) / len(x))) if len(x) else F(0)


def log10f(x) -> np.float32:
    with np.errstate(divide="ignore"):
        return F(np.log10(np.float64(x)))


def calculate_relative_energy(signal_rms, reference) -> np.float32:
    """calculateRelativeEnergy(of:relativeTo:) on a precomputed RMS; reference None -> 1e-3 as in Swift."""
    ref = swift_max(F(1e-8), F(1e-3) if reference is None else F(reference))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        db = F(F(20) * log10f(signal_rms))
        ref_db = F(F(20) * log10f(ref))
        normalized = F(F(db - ref_db) / F(F(0) - ref_db))
    return swift_max(F(0), swift_min(normalized, F(1)))


def relative_energies(pcm) -> List[np.float32]:
    """processBuffer over 1600-sample blocks from the start of the stream: reference = min RMS of the previous <= 20 blocks (+inf)."""
    x = np.asarray(pcm, np.float32)
    out, rmss = [], []
    for b in range(len(x) // BLOCK):
        r = rms(x[b * BLOCK:(b + 1) * BLOCK])
        ref = F(np.inf)
        for v in rmss[-20:]:
            ref = swift_min(ref, v)
        out.append(calculate_relative_energy(r, ref))
        rmss.append(r)
    return out


def is_voice_detected(relativeEnergy: Sequence[float], nextBufferInSeconds: float, silenceThreshold: float) -> bool:
    q = F(F(nextBufferInSeconds) / F(0.1))
    k = max(0, int(q)) if q > 0 else 0
    e = list(relativeEnergy)
    nxt = e[len(e) - min(k, len(e)):] if k else []
    check = max(10, len(nxt) - 10)
    return any(F(v) > F(silenceThreshold) for v in nxt[:check])


def should_stop_early(currentTokens: Sequence[int], avgLogprob: float, compressionCheckWindow: int,
                      compressionRatioThreshold: Optional[float], logProbThreshold: Optional[float]) -> bool:
    """shouldStopEarly -> false (stop) as True."""
    if len(currentTokens) > compressionCheckWindow:
        if F(compression_ratio(list(currentTokens)[-compressionCheckWindow:])) > F(compressionRatioThreshold if compressionRatioThreshold is not None else 0.0):
            return True
    if logProbThreshold is not None and F(avgLogprob) < F(logProbThreshold):
        return True
    return False


def stop_index(currentTokens: Sequence[int], logProbs: Sequence[float], promptLength: int, compressionCheckWindow: int,
               compressionRatioThreshold: Optional[float], logProbThreshold: Optional[float]) -> int:
    """The first appended (non-prefill) history index t >= promptLength whose history [0..t] meets the rule, else -1.  The progress
    callbacks of prefill steps see the prompt only and cannot stop (TextDecoder.swift:745)."""
    s = F(0)
    for i, lp in enumerate(logProbs):
        s = F(s + F(lp))
        if i < promptLength:
            continue
        if should_stop_early(currentTokens[:i + 1], F(s / F(i + 1)), compressionCheckWindow, compressionRatioThreshold, logProbThreshold):
            return i
    return -1


@dataclass
class Finalized:
    tokens: List[int]
    tokenLogProbs: List[float]
    avgLogProb: float
    compressionRatio: float
    needsFallback: bool


def truncate_and_finalize(currentTokens: Sequence[int], logProbs: Sequence[float], t: int, sot: int, eot: int, specialTokenBegin: int,
                          compressionRatioThreshold: Optional[float], logProbThreshold: Optional[float]) -> Finalized:
    """History cut after index t (t < 0: uncut), finalize (append EOT), slice SOT..EOT, avgLogProb, compressionRatio, DecodingFallback
    (first-token and no-speech rules not involved)."""
    toks, lps = list(currentTokens), [float(v) for v in logProbs]
    if t >= 0:
        toks, lps = toks[:t + 1], lps[:t + 1]
    if not toks or toks[-1] != eot:
        toks.append(eot)
        lps.append(0.0)
    a = toks.index(sot) if sot in toks else 0
    b = toks.index(eot)
    toks, lps = toks[a:b + 1], lps[a:b + 1]
    s = F(0)
    for v in lps:
        s = F(s + F(v))
    avg = float(s / F(len(lps)))
    cr = compression_ratio([x for x in toks if x < specialTokenBegin])
    fb = (compressionRatioThreshold is not None and cr > compressionRatioThreshold) or (logProbThreshold is not None and avg < logProbThreshold)
    return Finalized(toks, lps, avg, cr, bool(fb))


def segments_equal(a, b) -> bool:
    return (a.seek == b.seek and F(a.start) == F(b.start) and F(a.end) == F(b.end) and list(a.tokens) == list(b.tokens)
            and [F(v) for v in a.tokenLogProbs] == [F(v) for v in b.tokenLogProbs])


@dataclass
class StreamState:
    lastBufferSize: int = 0
    lastConfirmedSegmentEndSeconds: float = 0.0
    confirmedSegments: list = field(default_factory=list)
    unconfirmedSegments: list = field(default_factory=list)


class StreamMachine:
    """transcribeCurrentBuffer for one stream.  transcribe(buffer, clipStartSeconds) -> segments of TranscribeTask.run on the whole
    buffer with clipTimestamps = [clipStartSeconds]."""

    def __init__(self, transcribe: Callable, requiredSegmentsForConfirmation: int = 2, silenceThreshold: float = 0.3, useVAD: bool = True):
        self.transcribe = transcribe
        self.R = requiredSegmentsForConfirmation
        self.silenceThreshold = silenceThreshold
        self.useVAD = useVAD
        self.state = StreamState()
        self.duplicates = 0
        self.skips = {"short": 0, "vad": 0}

    def round(self, buffer) -> bool:
        """One call of transcribeCurrentBuffer on the stream's whole buffer (samples 0..n); returns whether it transcribed."""
        buffer = np.asarray(buffer, np.float32)
        n = len(buffer)
        nextBufferSeconds = F(F(n - self.state.lastBufferSize) / F(SAMPLE_RATE))
        if not nextBufferSeconds > 1:
            self.skips["short"] += 1
            return False
        if self.useVAD and not is_voice_detected(relative_energies(buffer), nextBufferSeconds, self.silenceThreshold):
            self.skips["vad"] += 1
            return False
        self.state.lastBufferSize = n
        segs = self.transcribe(buffer, self.state.lastConfirmedSegmentEndSeconds)
        self.apply(segs)
        return True

    def apply(self, segs) -> None:
        """The confirmation logic (AudioStreamTranscriber.swift:164-192)."""
        st = self.state
        if len(segs) > self.R:
            k = len(segs) - self.R
            cand = segs[:k]
            if F(cand[-1].end) > F(st.lastConfirmedSegmentEndSeconds):
                st.lastConfirmedSegmentEndSeconds = float(F(cand[-1].end))
                contained = any(all(segments_equal(st.confirmedSegments[a + j], cand[j]) for j in range(k))
                                for a in range(len(st.confirmedSegments) - k + 1))
                if contained:
                    self.duplicates += 1
                else:
                    st.confirmedSegments += cand
            st.unconfirmedSegments = segs[k:]
        else:
            st.unconfirmedSegments = list(segs)
