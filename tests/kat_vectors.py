"""Known-answer vectors transcribed from the reference's own unit tests
(`Tests/WhisperKitTests/UnitTests.swift:1982-2115` of the reference repository): toy logits, token
histories and the exact expected -inf patterns for the four LogitsFiltering impls.
Shared by the oracle tests (CPU) and the CUDA sampler tests (GPU)."""
import numpy as np

NI = -np.inf
L7 = [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7]
L9 = [1.1, 5.2, 0.3, 0.4, 0.2, 0.1, 0.2, 0.1, 0.1]

# (name, kind, params, logits, tokens, expected)
SUPPRESS_TOKENS = [
    ("st1", [], L7, [], L7),
    ("st2", [0], L7, [], [NI, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7]),
    ("st3", [0, 2, 5, 6], L7, [], [NI, 0.2, NI, 0.4, 0.5, NI, NI]),
]

# (name, endToken, whitespaceToken, sampleBegin, logits, tokens, expected)
SUPPRESS_BLANK = [
    ("sb2", 0, 0, 0, L7, [], [NI, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7]),
    ("sb3", 0, 2, 0, L7, [], [NI, 0.2, NI, 0.4, 0.5, 0.6, 0.7]),
    ("sb4", 0, 2, 3, L7, [1, 2, 3], [NI, 0.2, NI, 0.4, 0.5, 0.6, 0.7]),
    ("sb5", 0, 2, 5, L7, [1, 2, 3], L7),
]

# (name, languageTokens, logitsDim, sampleBegin, logits, tokens, expected)
LANGUAGE = [
    ("lg1", [2, 4, 6], 7, 0, L7, [], [NI, NI, 0.3, NI, 0.5, NI, 0.7]),
    ("lg2", [2, 4, 6], 7, 2, L7, [1], L7),
]

TS_SPECIAL = dict(endToken=3, noTimestampsToken=2, timeTokenBegin=6, transcribeToken=4, translateToken=5)

# (name, multilingual, sampleBegin, logits, tokens, expected)
TIMESTAMP_RULES = [
    ("ts1", False, 0, L9, [4], [1.1, 5.2, NI, 0.4, 0.2, 0.1, 0.2, 0.1, 0.1]),
    ("ts2", False, 0, L9, [0, 6, 7, 3], [1.1, 5.2, NI, 0.4, 0.2, 0.1, NI, NI, 0.1]),
    ("ts3", False, 0, L9, [0, 6, 7], [1.1, 5.2, NI, 0.4, 0.2, 0.1, NI, NI, NI]),
    ("ts4", False, 0, L9, [0, 4, 7], [NI, NI, NI, NI, NI, NI, NI, 0.1, 0.1]),
    ("tm1", True, 0, L9, [0, 1, 2], L9),
    ("tm2", True, 0, L9, [0, 4, 6, 7, 3], [1.1, 5.2, NI, 0.4, 0.2, 0.1, NI, NI, 0.1]),
    ("tm3", True, 0, L9, [0, 5, 6, 7], [1.1, 5.2, NI, 0.4, 0.2, 0.1, NI, NI, NI]),
    ("tm4", True, 0, L9, [0, 4, 0, 7], [NI, NI, NI, NI, NI, NI, NI, 0.1, 0.1]),
]
