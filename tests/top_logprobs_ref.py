"""DecodingOptions.topLogProbs, restated in float64 from the rule (C header, wk_session_set_top_logprobs).

At a position the decode loop sampled, the candidates are the tokens its choice was made from: the filtered row (the loop's filters in
their order, oracle/decode_ref.createLogitsFilters with prefilledIndex 0 and the prompt as the initial prompt), whose finite entries
are the range the draw uses - only the timestamp tokens when the timestamp rule wins, because that rule masks the text tokens.  The
k best come first by value, ties to the lower id (block_argmax_row).  Each carries the log-prob its token would be reported with:
the log-softmax of the filtered row at temperature 0, of the row divided by the temperature at temperature > 0 (the tempered
probability before the top-k cut).  A bias set changes neither: values and ranking are the model's own.  -inf entries never appear.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import numpy as np

from oracle import decode_ref as D


def filtered_row(logits: np.ndarray, tokens: Sequence[int], options: D.DecodingOptions, st: D.SpecialTokens, multilingual: bool,
                 prompt_len: int) -> np.ndarray:
    """The row the sampler chooses from at the position after `tokens` (the window's history: prompt, then sampled tokens)."""
    x = np.array(logits, dtype=np.float32)
    for f in D.createLogitsFilters(options, 0, prompt_len, st, multilingual):
        x = f.filterLogits(x, list(tokens))
    return x


def top_logprobs(row: np.ndarray, k: int, temperature: float = 0.0) -> List[Tuple[int, float]]:
    """The k best (token, log-prob) of a filtered row, best first; fewer when the row has fewer finite entries."""
    x = np.asarray(row, dtype=np.float64)
    finite = np.isfinite(x)
    if k <= 0 or not finite.any():
        return []
    y = x if temperature == 0.0 else x / float(np.float32(temperature))
    m = float(np.max(y[finite]))
    lse = m + math.log(float(np.sum(np.exp(y[finite] - m))))
    ids = np.nonzero(finite)[0]
    order = sorted(ids.tolist(), key=lambda i: (-x[i], i))[:k]
    return [(int(i), float(y[i] - lse)) for i in order]


def as_dict(pairs: Sequence[Tuple[int, float]]) -> Dict[int, float]:
    return {t: v for t, v in pairs}


def timestamp_rule_won(row: np.ndarray, st: D.SpecialTokens) -> bool:
    """Whether the row's finite entries are all timestamps (the timestamp rule masked the text tokens)."""
    finite = np.isfinite(np.asarray(row, dtype=np.float64))
    return bool(finite.any()) and not finite[: st.timeTokenBegin].any()


def sets_match(got: Sequence[int], ref: Sequence[int], row: np.ndarray, tol: float = 1e-6) -> bool:
    """Token sets equal, except that a token may stand in for another whose filtered logit is within `tol` of it (a near-tie that the
    GPU's f32 logits may order either way)."""
    a, b = set(got), set(ref)
    if a == b:
        return True
    x = np.asarray(row, dtype=np.float64)
    only_a, only_b = sorted(a - b), sorted(b - a)
    if len(only_a) != len(only_b):
        return False
    return all(any(abs(x[i] - x[j]) < tol for j in only_b) for i in only_a)
