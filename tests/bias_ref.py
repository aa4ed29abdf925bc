"""Contextual biasing oracle (DecodingOptions.biasPhrases, C: wk_bias_create / wk_session_set_bias), written from the rule alone.

A set is P phrases w_p of 1..16 text token ids and one boost λ >= 0.  Every decode row keeps, per phrase, its KMP match length
m_p in [0, L_p): 0 at the row's first sampled position; forced prompt tokens and language detection do not move it.

  δ_p(m, v): while m > 0 and w_p[m] != v, m = f_p(m); then m + 1 if w_p[m] == v, else 0.  A result of L_p completes the phrase, and the
             stored state becomes f_p(L_p).
  bonus:     G = max_p m_p, g(v) = max_p δ_p(m_p, v) (a completion counting as L_p), b(v) = λ·(g(v) - G), in float32 as the kernel adds it.

b joins the filtered logits after every built-in filter: the greedy choice is argmax(filtered + b), beam candidates rank by
sum + (filtered + b - lse), and the reported log-probs stay log_softmax(filtered).  The best-of pick adds λ·Σ(g - G) over each sample's
appended tokens.  `decode_text_biased` runs oracle/decode_ref.decode_text with a biased sampler; `decode_text_beam_biased` is
oracle/beam_ref.decode_text_beam with the bonus in its ranking and a match state per beam.
"""
from __future__ import annotations

from typing import Callable, List, Sequence

import numpy as np

from oracle.beam_ref import top_candidates  # noqa: F401  (re-exported for the tests)
from oracle.decode_ref import (MAX_TOKEN_CONTEXT, DecodingFallback, DecodingOptions, DecodingResult, GreedyTokenSampler, SamplingResult,
                               SpecialTokens, compression_ratio, createLogitsFilters, decode_text)


def failure(w: Sequence[int]) -> List[int]:
    """f[k - 1] = f(k), the longest proper border of w[0..k), for k = 1..L."""
    f = [0] * len(w)
    b = 0
    for k in range(1, len(w)):
        while b > 0 and w[k] != w[b]:
            b = f[b - 1]
        if w[k] == w[b]:
            b += 1
        f[k] = b
    return f


def delta(w: Sequence[int], f: Sequence[int], m: int, v: int) -> int:
    while m > 0 and w[m] != v:
        m = f[m - 1]
    return m + 1 if w[m] == v else 0


class BiasState:
    """One row's match lengths over a phrase set."""

    def __init__(self, phrases: Sequence[Sequence[int]], boost: float):
        self.w = [list(map(int, p)) for p in phrases]
        self.f = [failure(p) for p in self.w]
        self.boost = np.float32(boost)
        self.m = [0] * len(self.w)

    def copy(self) -> "BiasState":
        c = BiasState.__new__(BiasState)
        c.w, c.f, c.boost, c.m = self.w, self.f, self.boost, list(self.m)
        return c

    @property
    def G(self) -> int:
        return max(self.m) if self.m else 0

    def g(self, v: int) -> int:
        return max(delta(w, f, m, v) for w, f, m in zip(self.w, self.f, self.m))

    def bonus(self, V: int) -> np.ndarray:
        """b(v) for every token, float32."""
        G = self.G
        b = np.full(V, self.boost * np.float32(0 - G), np.float32)
        for w, f, m in zip(self.w, self.f, self.m):
            k = m
            while True:                         # the failure chain: w[k] leads to k + 1 (the first such k is δ)
                v = w[k]
                if v < V:
                    b[v] = max(b[v], self.boost * np.float32(k + 1 - G))
                if k == 0:
                    break
                k = f[k - 1]
        return b

    def advance(self, v: int):
        """Moves every match on by token v; returns (g(v), G before, phrases completed)."""
        G, g, done = self.G, 0, []
        for p, (w, f) in enumerate(zip(self.w, self.f)):
            k = delta(w, f, self.m[p], v)
            g = max(g, k)
            if k == len(w):
                done.append(p)
                k = f[-1]
            self.m[p] = k
        return g, G, done


def banked(phrases, boost, tokens: Sequence[int]) -> int:
    """Σ (g - G) over a sequence of appended tokens: the bonus it banked, in units of λ."""
    s = BiasState(phrases, boost)
    acc = 0
    for v in tokens:
        g, G, _ = s.advance(v)
        acc += g - G
    return acc


class BiasedGreedySampler(GreedyTokenSampler):
    """Temperature 0: argmax of filtered + b from the prompt's last position on; the log-prob reported is the unbiased one.  trace gets one
    dict per appended token: token, G, g, completed phrases, revoked (g < G: the token broke a partial match and its bonus
    was taken back)."""

    def __init__(self, eotToken: int, options: DecodingOptions, prompt_len: int, phrases, boost: float, trace: list = None):
        super().__init__(0.0, eotToken, options)
        self.P, self.calls = prompt_len, 0
        self.state = BiasState(phrases, boost)
        self.trace = trace if trace is not None else []

    def update(self, tokens, logits, logProbs) -> SamplingResult:
        step = self.calls
        self.calls += 1
        if step < self.P - 1:
            return super().update(tokens, logits, logProbs)
        x = np.asarray(logits, dtype=np.float32)
        biased = (x + self.state.bonus(len(x))).astype(np.float32)
        tok = int(np.argmax(biased))
        m = np.max(x)
        e = np.exp(x - m)
        probs = e / np.sum(e, dtype=np.float32)
        lp = float(np.log(probs[tok]))
        if tok != self.eotToken:                # EOT ends the window: nothing is appended
            g, G, done = self.state.advance(tok)
            self.trace.append(dict(token=tok, G=G, g=g, completed=done, revoked=g < G))
        return SamplingResult(list(tokens) + [tok], list(logProbs) + [lp], tok == self.eotToken)


def decode_text_biased(predict_logits: Callable[[int, int], np.ndarray], initialPrompt: Sequence[int], options: DecodingOptions,
                       st: SpecialTokens, isModelMultilingual: bool, phrases, boost: float, trace: list = None) -> DecodingResult:
    sampler = BiasedGreedySampler(st.endToken, options, len(initialPrompt), phrases, boost, trace)
    return decode_text(predict_logits, initialPrompt, options, st, isModelMultilingual, sampler=sampler)


def _lse(row: np.ndarray) -> np.float32:
    m = np.max(row)
    return np.float32(m + np.log(np.sum(np.exp((row - m).astype(np.float64)))).astype(np.float32))


def decode_text_beam_biased(predict_logits, initialPrompt: Sequence[int], options: DecodingOptions, st: SpecialTokens, isModelMultilingual: bool,
                            beamSize: int, patience: float, phrases, boost: float, trace: list = None) -> DecodingResult:
    """oracle/beam_ref.decode_text_beam with every candidate scored sum + (filtered + b - lse) and a match state per beam, which a surviving
    beam takes from its source and moves on by its token."""
    maxCandidates = int(np.float32(beamSize) * np.float32(patience))
    P = len(initialPrompt)
    beams = [list(initialPrompt) for _ in range(beamSize)]
    beam_lps = [[0.0] * P for _ in range(beamSize)]
    states = [BiasState(phrases, boost) for _ in range(beamSize)]
    sums = [np.float32(0.0)] * beamSize
    nextToken = initialPrompt[-1]
    filters = createLogitsFilters(options, 0, P, st, isModelMultilingual, None)
    loopCount = min(options.sampleLength, MAX_TOKEN_CONTEXT - 1)
    finished = []
    firstLow = False
    steps = 0
    for tokenIndex in range(0, loopCount):
        isPrefill = tokenIndex < P - 1
        if tokenIndex < P:
            cur = beams[0][tokenIndex]
            if tokenIndex == P - 1 and cur >= st.timeTokenBegin and nextToken >= st.timeTokenBegin:
                for b in beams:
                    b[tokenIndex] = nextToken
        logits = np.asarray(predict_logits([list(b) for b in beams], tokenIndex), dtype=np.float32)
        steps += 1
        considered = range(beamSize) if tokenIndex > P - 1 else range(1)
        cand = []
        greedy = None
        for j in considered:
            row = logits[j].copy()
            for f in filters:
                row = f.filterLogits(row, beams[j])
            row = row.astype(np.float32)
            if not np.isfinite(np.max(row)):
                tops = []
            else:
                lse = _lse(row)
                biased = row if isPrefill else (row + states[j].bonus(len(row))).astype(np.float32)
                idx = [int(i) for i in np.argsort(-biased, kind="stable")[:beamSize + 1] if np.isfinite(biased[i])]
                tops = [(i, np.float32(row[i] - lse), np.float32(biased[i] - lse)) for i in idx]
            if j == 0:
                greedy = tops[0][:2] if tops else (st.endToken, np.float32(-np.inf))
            for tok, v, sc in tops:
                cand.append((np.float32(sums[j] + sc), j, tok, v))
        firstLow = bool(tokenIndex == 0 and options.firstTokenLogProbThreshold is not None and greedy[1] < options.firstTokenLogProbThreshold)
        nextToken = greedy[0]
        if isPrefill:
            if greedy[0] == st.endToken or firstLow:
                break
            continue
        if len(beams[0]) >= MAX_TOKEN_CONTEXT - 1 or firstLow:
            break
        order = sorted(range(len(cand)), key=lambda i: -cand[i][0])
        new_beams, new_lps, new_sums, new_states = [], [], [], []
        for i in order:
            score, j, tok, v = cand[i]
            if tok == st.endToken:
                if len(finished) < maxCandidates:
                    finished.append((beams[j] + [tok], beam_lps[j] + [0.0], score))
            else:
                s = states[j].copy()
                g, G, done = s.advance(tok)
                if trace is not None:
                    trace.append(dict(token=tok, G=G, g=g, completed=done, revoked=g < G))
                new_beams.append(beams[j] + [tok])
                new_lps.append(beam_lps[j] + [float(v)])
                new_sums.append(score)
                new_states.append(s)
                if len(new_beams) == beamSize:
                    break
        beams, beam_lps, sums, states = new_beams, new_lps, new_sums, new_states
        while len(beams) < beamSize:
            beams.append(list(beams[-1])); beam_lps.append(list(beam_lps[-1])); sums.append(np.float32(-np.inf)); states.append(states[-1].copy())
        nextToken = beams[0][-1]
        if len(finished) >= maxCandidates:
            break
    if len(finished) < beamSize:
        for j in sorted(range(len(beams)), key=lambda i: -sums[i]):
            finished.append((beams[j] + [st.endToken], beam_lps[j] + [0.0], sums[j]))
            if len(finished) >= beamSize:
                break

    def rank(entry):
        toks, _, score = entry
        return np.float32(score) / np.float32(max(len(toks) - P - 1, 1))
    best = max(range(len(finished)), key=lambda i: (rank(finished[i]), -i))
    segmentTokens, segmentLogProbs, _ = finished[best]
    startIndex = segmentTokens.index(st.startOfTranscriptToken) if st.startOfTranscriptToken in segmentTokens else 0
    endIndex = segmentTokens.index(st.endToken) if st.endToken in segmentTokens else len(segmentTokens)
    filteredTokens = segmentTokens[startIndex:endIndex + 1]
    filteredLogProbs = segmentLogProbs[startIndex:endIndex + 1]
    s = np.float32(0.0)
    for v in filteredLogProbs:
        s = np.float32(s + np.float32(v))
    avg = float(s / np.float32(len(filteredLogProbs)))
    ratio = compression_ratio([t for t in filteredTokens if t < st.specialTokenBegin])
    fb = DecodingFallback.make(options, firstLow, 0.0, ratio, avg)
    return DecodingResult(filteredTokens, filteredLogProbs, avg, ratio, round(float(np.float16(options.temperature)), 3), fb,
                          currentTokens=segmentTokens[:-1], logProbs=segmentLogProbs[:-1], steps=steps, isFirstTokenLogProbTooLow=firstLow)
