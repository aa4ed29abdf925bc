"""DecodingOptions.computeNoSpeechProb on the host: the openai/whisper rule (tests/no_speech_ref.py) against torch.softmax, the silence
branch of DecodingFallback and its precedence, SegmentSeeker's skip rule through the library's wk_find_seek_point_and_segments with a
nonzero noSpeechProb, the restated seek loop, and the new wk_decode_opts field."""
import ctypes as C

import numpy as np
import pytest

import whisperkit_b200 as wk
from oracle import decode_ref as D
from oracle import seek_ref as S
from tests import no_speech_ref as N
from whisperkit_b200 import _lib
from whisperkit_b200.longform import SegmentSeeker

torch = pytest.importorskip("torch")

V = 1024
ST = D.SpecialTokens.toy(V)


def test_rule_matches_torch_softmax():
    rng = np.random.default_rng(0)
    for scale, boost in ((1.0, 0.0), (3.0, 0.0), (1.0, 9.0), (20.0, -5.0)):
        x = (rng.standard_normal(V) * scale).astype(np.float32)
        x[ST.noSpeechToken] += boost
        ref = float(torch.softmax(torch.from_numpy(x).double(), dim=-1)[ST.noSpeechToken])
        assert abs(N.no_speech_prob(x, ST) - ref) <= 1e-15
        ref32 = float(torch.softmax(torch.from_numpy(x), dim=-1)[ST.noSpeechToken])   # openai: logits.float().softmax(-1)
        assert abs(N.no_speech_prob(x, ST) - ref32) <= 1e-6


def test_silence_fallback_precedence_and_strict_threshold():
    o = D.DecodingOptions()   # noSpeechThreshold 0.6, compression 2.4, logprob -1.0
    mk = D.DecodingFallback.make
    assert mk(o, False, 0.61, 9.0, -9.0) == D.DecodingFallback(False, "silence")   # above: silence, no ladder, over both thresholds
    assert mk(o, False, 0.6, 9.0, -9.0) == D.DecodingFallback(True, "compressionRatioThreshold")   # equal: strict >
    assert mk(o, False, 0.59, 1.0, -9.0) == D.DecodingFallback(True, "logProbThreshold")
    assert mk(o, False, 0.59, 1.0, -0.5) is None
    assert mk(o, True, 0.99, 1.0, -0.5) == D.DecodingFallback(True, "firstTokenLogProbThreshold")   # the first-token rule comes first
    assert mk(D.DecodingOptions(noSpeechThreshold=None), False, 0.99, 1.0, -9.0).fallbackReason == "logProbThreshold"


def make_predict(boost):
    """A deterministic toy model: logits depend on (token, position); the step that feeds SOT gets <|nospeech|> += boost."""
    def predict(token, index):
        x = np.random.default_rng(token * 1000 + index).standard_normal(V).astype(np.float32)
        if token == ST.startOfTranscriptToken:
            x[ST.noSpeechToken] += boost
        return x
    return predict


@pytest.mark.parametrize("kw", [dict(), dict(promptTokens=[5, 6, 7]), dict(prefixTokens=[11, 12]), dict(withoutTimestamps=True)])
def test_reference_decode_takes_the_sot_step(kw):
    o = D.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=10, **kw)
    prompt = D.prefill_prompt(o, ST, True)
    sot = prompt.index(ST.startOfTranscriptToken)
    assert sot == (4 if "promptTokens" in kw else 0)
    for boost, silent in ((12.0, True), (0.0, False)):
        r, p = N.decode_with_no_speech(make_predict(boost), prompt, o, ST, True)
        assert p == N.no_speech_prob(make_predict(boost)(ST.startOfTranscriptToken, sot), ST)
        assert (p > 0.6) == silent
        plain = D.decode_text(make_predict(boost), prompt, o, ST, True)
        assert r.tokens == plain.tokens and r.steps == plain.steps        # the value changes no token
        if silent:
            assert r.fallback == D.DecodingFallback(False, "silence")
        else:
            assert r.fallback == plain.fallback


def test_reference_reports_none_when_the_loop_ends_before_the_sot_step():
    def predict(token, index):   # EOT wins every step, so the loop ends during the previous-text prefill
        x = np.zeros(V, np.float32)
        x[ST.endToken] = 50.0
        return x
    o = D.DecodingOptions(firstTokenLogProbThreshold=None, promptTokens=[5, 6, 7], sampleLength=10)
    r, p = N.decode_with_no_speech(predict, D.prefill_prompt(o, ST, True), o, ST, True)
    assert p is None and r.steps == 1


def c_seek(tokens, p, avg, o, seek=32000, size=480000):
    return SegmentSeeker().findSeekPointAndSegments(tokens, [-0.5] * len(tokens), avg, 1.7, 0.2, o, 3, seek, size, 16000, ST.timeTokenBegin,
                                                    noSpeechProb=p)


@pytest.mark.parametrize("nst,lpt", [(0.6, -1.0), (0.6, None), (None, -1.0), (None, None), (0.3, -2.0)])
def test_skip_rule_through_the_library(nst, lpt):
    o = wk.DecodingOptions(noSpeechThreshold=nst, logProbThreshold=lpt)
    tb = ST.timeTokenBegin
    tokens = [ST.startOfTranscriptToken, tb, 11, 12, tb + 40, tb + 40, 13, tb + 90]
    for p in (0.0, 0.25, 0.3, 0.6, 0.61, 0.97):
        for avg in (-3.0, -1.0, -0.4):
            seek, segs = c_seek(tokens, p, avg, o)
            ref_seek, ref = S.find_seek_point_and_segments(tokens, [-0.5] * len(tokens), p, avg, 1.7, 0.2, nst, lpt, 3, 32000, 480000, 16000, tb)
            assert seek == ref_seek, (p, avg)
            skip = nst is not None and p > nst and not (lpt is not None and avg > lpt)
            assert (segs is None) == (ref is None) == skip, (p, avg)
            if ref is not None:
                assert [g.tokens for g in segs] == [g.tokens for g in ref]
                assert [np.float32(g.noSpeechProb) for g in segs] == [np.float32(p)] * len(ref)   # wk_segment.no_speech_prob carries it
                np.testing.assert_array_equal(np.float32([g.start for g in segs]), np.float32([g.start for g in ref]))


def test_restated_seek_loop_equals_the_oracle_loop_at_zero():
    """tests/no_speech_ref.seek_loop fed noSpeechProb = 0 is oracle/seek_ref.seek_loop; fed 0.9 on some windows it skips exactly those."""
    tb = ST.timeTokenBegin
    rng = np.random.default_rng(1)

    class R:
        pass

    def window(seek, size, p=0.0):
        r = R()
        a = int(rng.integers(20, 600))
        r.tokens = [ST.startOfTranscriptToken, tb, 11, 12, tb + a // 2, tb + a // 2, 13, tb + a]
        r.tokenLogProbs = [-0.5] * len(r.tokens)
        r.avgLogProb, r.compressionRatio, r.temperature, r.noSpeechProb = -1.5, 1.2, 0.0, p
        return r
    n = 3_000_000
    rng = np.random.default_rng(1)
    ref, ref_w = S.seek_loop(n, window, timeToken=tb)
    rng = np.random.default_rng(1)
    got, got_w = N.seek_loop(n, window, timeToken=tb)
    assert [(g.seek, g.tokens, g.start, g.end) for g in got] == [(g.seek, g.tokens, g.start, g.end) for g in ref]
    assert [w[:2] for w in got_w] == ref_w and not any(w[2] for w in got_w)
    silent = {0, 2}
    calls = []

    def window_p(seek, size):
        calls.append(seek)
        return window(seek, size, 0.9 if len(calls) - 1 in silent else 0.1)
    rng = np.random.default_rng(1)
    got, got_w = N.seek_loop(n, window_p, timeToken=tb)
    assert [i for i, w in enumerate(got_w) if w[2]] == sorted(silent)
    assert got_w[1][0] == got_w[0][0] + got_w[0][1]                  # a skipped window moves the seek by its whole size
    assert all(g.seek not in (calls[0], calls[2]) for g in got)


def test_opts_field_is_appended_and_defaults_to_zero():
    f = _lib.wk_decode_opts
    names = [n for n, _ in f._fields_]
    assert names[-1] == "compute_no_speech_prob" and names[-2] == "n_language_tokens"
    assert f.compute_no_speech_prob.offset == f.n_language_tokens.offset + 4
    assert C.sizeof(f) == f.n_language_tokens.offset + 8                # the field sits in what was the struct's tail padding
    assert f().compute_no_speech_prob == 0
    assert wk.DecodingOptions().to_c()[0].compute_no_speech_prob == 0
    assert wk.DecodingOptions(computeNoSpeechProb=True).to_c()[0].compute_no_speech_prob == 1
    assert wk.DecodingResult([], [], 0.0, 0.0, 0.0, None).noSpeechProb == 0.0
