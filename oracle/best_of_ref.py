"""Best-of-N ranking oracle (test infrastructure; see oracle/__init__.py).  PARITY: SELF-ORACLE ONLY.

The reference's `DecodingOptions` has no `bestOf`.  openai/whisper's `best_of` (whisper/decoding.py, external, restated here from its
published algorithm) decodes a window on a temperature > 0 rung as N independent samples - each an ordinary decodeText run with its own
draws - and keeps one with the same ranker beam search finalizes with (oracle/beam_ref.py): MaximumLikelihoodRanker with
length_penalty = None, i.e. the highest sum of the sample's token log-probs divided by its number of sampled tokens (at least 1: the
original divides by zero for an empty sequence).  The library records no log-prob for the EOT that ends a sample, so the sum covers the
tokens before it.  Equal scores keep the earlier sample.  The kept sample then goes through decodeText's own result assembly and
DecodingFallback like any single decode.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np


def best_of_score(logProbs: Sequence[float], promptLength: int) -> np.float32:
    """The ranker's score of one sample: `logProbs` are its recorded per-token log-probs, prompt slots (0) included, in order
    (DecodingResult.logProbs / currentTokens); the divisor is the number of sampled tokens, at least 1.  f32, summed in order."""
    s = np.float32(0.0)
    for v in logProbs:
        s = np.float32(s + np.float32(v))
    return np.float32(s / np.float32(max(len(logProbs) - promptLength, 1)))


def rank_best_of(samples: Sequence[Sequence[float]], promptLength: int) -> int:
    """Index of the sample best_of keeps: the highest best_of_score, the lowest index among equal scores."""
    best, best_score = 0, None
    for i, lps in enumerate(samples):
        sc = best_of_score(lps, promptLength)
        if best_score is None or sc > best_score:
            best, best_score = i, sc
    return best
