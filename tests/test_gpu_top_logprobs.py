"""DecodingOptions.topLogProbs on the GPU: the sampler's one-pass top-k against tests/top_logprobs_ref.py on the GPU decoder's own logits
(predictLogits on the window's history), self-consistency at temperature 0, long-form slices, large-v3 scale and the refusals.  Any
k > 0 must leave every other output byte-identical to k = 0."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from tests import top_logprobs_ref as TL  # noqa: E402
from whisperkit_b200 import longform as L  # noqa: E402
from whisperkit_b200._lib import check  # noqa: E402

NEVER = dict(logProbThreshold=None, compressionRatioThreshold=None)
FORCE = dict(logProbThreshold=0.0, compressionRatioThreshold=None)   # every rung falls back (avgLogProb < 0)
SUPPRESSED = [5, 6, 7]


def st_of(variant):
    return D.SpecialTokens.toy(1024 if variant == "toy" else 2048)


def make_kit(slots, variant="toy", policy="bf16", seed=5, **kw):
    return wk.WhisperKit(wk.WhisperKitConfig(model=variant, maxBatch=slots, seed=seed, dtype=policy,
                                             specialTokens=wk.SpecialTokens.from_any(st_of(variant)), **kw))


def pcm_of(n, base):
    return np.stack([mel_ref.synthetic_pcm(base + i) for i in range(n)])


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=24, temperatureFallbackCount=0, **NEVER)
    d.update(kw)
    return wk.DecodingOptions(**d)


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def same(a, b, where):
    assert a.tokens == b.tokens, where
    assert np.array_equal(bits(a.tokenLogProbs), bits(b.tokenLogProbs)), where
    assert bits([a.avgLogProb, a.compressionRatio, a.noSpeechProb]).tolist() == bits([b.avgLogProb, b.compressionRatio, b.noSpeechProb]).tolist(), where
    assert (a.temperature, a.steps, a.currentTokenCount, a.languageToken, a.language) == \
        (b.temperature, b.steps, b.currentTokenCount, b.languageToken, b.language), where
    assert bits([a.languageLogProb or 0.0]).tolist() == bits([b.languageLogProb or 0.0]).tolist(), where
    assert a.fallback == b.fallback, where


def raw_pairs(kit, window, n, k):
    tok = (C.c_int32 * max(1, n * k))()
    lp = (C.c_float * max(1, n * k))()
    check(kit.model.lib.wk_session_top_logprobs(kit.textDecoder.handle, window, n, tok, lp))
    return np.array(tok[:n * k], np.int32).reshape(n, k), np.array(lp[:n * k], np.float32).reshape(n, k)


def check_self_consistent(kit, window, r, k, P, greedy=True):
    """Sampled positions [P, n - 1) carry up to k finite pairs, best first and distinct; forced positions and the closing EOT carry
    none; at temperature 0 entry 0 is the token and its tokenLogProbs entry, bit for bit."""
    n = len(r.tokens)
    assert len(r.topLogProbs) == n
    tok, lp = raw_pairs(kit, window, n, k)
    for i in range(n):
        valid = tok[i] >= 0
        if i < P or i == n - 1:
            assert not valid.any() and np.all(lp[i] == -np.inf), (window, i)
            assert r.topLogProbs[i] == {}
            continue
        m = int(valid.sum())
        assert m >= 1 and valid[:m].all() and not valid[m:].any(), (window, i, tok[i])
        assert np.all(np.isfinite(lp[i][:m])) and np.all(lp[i][m:] == -np.inf)
        assert len(set(tok[i][:m].tolist())) == m, (window, i, tok[i])
        assert np.all(np.diff(lp[i][:m].astype(np.float64)) <= 0), (window, i, lp[i])
        assert not set(tok[i][:m].tolist()) & set(SUPPRESSED + [kit.specialTokens.noTimestampsToken])
        assert list(r.topLogProbs[i]) == tok[i][:m].tolist()
        if greedy:
            assert tok[i][0] == r.tokens[i] and bits([lp[i][0]]) == bits([r.tokenLogProbs[i]]), (window, i)


# ---------------------------------------------------------------------------------------------------------------- 1. no perturbation
CASES = ["greedy", "sampled", "best_of3_ladder", "bias", "detect", "more_windows_than_slots"]


@pytest.mark.parametrize("variant,policy,cross", [("toy", "bf16", None), ("toy128", "f16", None), ("toy", "bf16", "fp8")])
@pytest.mark.parametrize("case", CASES)
def test_outputs_are_byte_identical_to_k0(variant, policy, cross, case):
    cfg = dict(crossKVDtype=cross) if cross else {}
    slots, n = (3, 7) if case == "more_windows_than_slots" else (8, 4)
    kit = make_kit(slots, variant, policy, seed=21, **cfg)
    pcm = pcm_of(n, 70)
    kw = dict(computeNoSpeechProb=True, suppressTokens=SUPPRESSED)
    if case == "sampled":
        kw.update(temperature=0.7, seed=11)
    elif case == "best_of3_ladder":
        kw.update(bestOf=3, temperatureFallbackCount=2, seed=4, **FORCE)
    elif case == "bias":
        kw.update(biasPhrases=[[1, 2, 3], [40, 41], [9]], biasBoost=3.0)
    elif case == "detect":
        kw.update(detectLanguage=True, allLanguageTokens=[st_of(variant).englishToken] + list(range(200, 260)))
    elif case == "more_windows_than_slots":
        kw.update(temperature=0.5, seed=2)
    base = opts(**kw)
    ref = kit.transcribe(pcm, base)
    assert all(r.topLogProbs == [] for r in ref)
    if case == "best_of3_ladder":
        assert all(r.temperature > 0 for r in ref)
    if case == "detect":
        assert all(r.languageToken is not None for r in ref)
    for k in (1, 5, 20):
        got = kit.transcribe(pcm, dataclasses.replace(base, topLogProbs=k))
        for i in range(n):
            same(ref[i], got[i], (case, k, i))
            assert len(got[i].topLogProbs) == len(got[i].tokens)
            assert all(len(d) <= k for d in got[i].topLogProbs)
        assert any(d for r in got for d in r.topLogProbs), (case, k)
    again = kit.transcribe(pcm, base)                               # k = 0 after k > 0: no trace
    for i in range(n):
        same(ref[i], again[i], (case, "after", i))
        assert again[i].topLogProbs == []


# ---------------------------------------------------------------------------------------------------------------- 2. self-consistency
@pytest.mark.parametrize("variant,policy", [("toy", "bf16"), ("toy128", "f16")])
def test_temperature_0_entry_0_is_the_sampled_token(variant, policy):
    kit = make_kit(4, variant, policy, seed=23)
    pcm = pcm_of(6, 90)
    for k in (1, 5, 20):
        o = opts(topLogProbs=k, suppressTokens=SUPPRESSED, sampleLength=40)
        P = len(kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens))
        got = kit.transcribe(pcm, o)
        for w, r in enumerate(got):
            check_self_consistent(kit, w, r, k, P)
    # decodeText on bound windows takes the option as well
    fe, enc = wk.FeatureExtractor(kit.model), wk.AudioEncoder(kit.model)
    dec = wk.TextDecoder(kit.model, 3)
    o = opts(topLogProbs=5, suppressTokens=SUPPRESSED)
    prompt = dec.prefillDecoderInputs(o, kit.specialTokens)
    bound = dec.decodeText(enc.encodeFeatures(fe.logMelSpectrogram(pcm[:3])), prompt, o, kit.specialTokens)
    for w, r in enumerate(bound):
        assert len(r.topLogProbs) == len(r.tokens)
        for i in range(len(prompt), len(r.tokens) - 1):
            t0, v0 = next(iter(r.topLogProbs[i].items()))
            assert t0 == r.tokens[i] and bits([v0]) == bits([r.tokenLogProbs[i]]), (w, i)
    dec.close()


# ---------------------------------------------------------------------------------------------------------------- 3. against the rule
def _window_predictor(model, pcm_window):
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    dec = wk.TextDecoder(model, 1)
    dec.bindEncoderOutput(enc.encodeFeatures(fe.logMelSpectrogram(pcm_window[None])))
    return dec


@pytest.mark.parametrize("variant,policy,temperature", [("toy", "bf16", 0.0), ("toy128", "f16", 0.0), ("toy", "bf16", 0.8)])
def test_pairs_match_the_reference_rule_on_gpu_logits(variant, policy, temperature):
    st_o = st_of(variant)
    kit = make_kit(2, variant, policy, seed=29)
    pcm = pcm_of(3, 120)
    k = 20
    o = opts(topLogProbs=k, temperature=temperature, seed=3, suppressTokens=SUPPRESSED, sampleLength=32)
    ref_o = D.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=32, logProbThreshold=None, compressionRatioThreshold=None,
                              suppressTokens=SUPPRESSED, temperature=temperature)
    prompt = kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens)
    P = len(prompt)
    got = kit.transcribe(pcm, o)
    ts_positions = checked = 0
    worst = 0.0
    for b in range(3):
        r = got[b]
        assert r.tokens[:P - 1] == prompt[:P - 1]                   # (a predicted first timestamp may replace the prompt's <|0.00|>)
        dec = _window_predictor(kit.model, pcm[b])
        hist = list(r.tokens[:-1])                                  # the history the loop fed (the closing EOT never was)
        logits = None
        for pos in range(len(hist)):
            if pos >= P:                                            # the logits of position pos came from feeding hist[pos - 1]
                row = TL.filtered_row(logits, hist[:pos], ref_o, st_o, True, P)
                ref = TL.top_logprobs(row, k, temperature)
                cand = r.topLogProbs[pos]
                assert TL.sets_match(list(cand), [t for t, _ in ref], row), (b, pos, list(cand), ref)
                assert all(np.isfinite(row[t]) for t in cand), (b, pos)
                refd = TL.as_dict(ref)
                for t, v in cand.items():
                    if t in refd:
                        worst = max(worst, abs(v - refd[t]))
                        assert abs(v - refd[t]) <= 2e-5, (b, pos, t, v, refd[t])
                ts_positions += TL.timestamp_rule_won(row, st_o)
                checked += 1
            logits = dec.predictLogits([hist[pos]], [pos])[0]
        dec.close()
    print(f"[{variant}/{policy} T={temperature}] {checked} positions, {ts_positions} where the timestamp rule won, worst |dv| {worst:.2e}")
    assert checked >= 10 and ts_positions >= 1


# ---------------------------------------------------------------------------------------------------------------- 4. long-form
def test_long_form_segments_carry_pairs_sliced_like_their_log_probs():
    kit = make_kit(4, seed=31)
    streams = [np.concatenate([mel_ref.synthetic_pcm(300 + 10 * i + j) for j in range(3)])[:n].astype(np.float32)
               for i, n in enumerate([480000 + 200000, 1000000])]
    o = opts(sampleLength=24)
    plain, _ = L.transcribe_streams(kit, streams, o)
    got, _ = L.transcribe_streams(kit, streams, dataclasses.replace(o, topLogProbs=5))
    sampled = 0
    for i in range(2):
        assert [g.tokens for g in got[i]] == [g.tokens for g in plain[i]]
        assert bits([v for g in got[i] for v in g.tokenLogProbs]).tolist() == bits([v for g in plain[i] for v in g.tokenLogProbs]).tolist()
        assert all(g.topLogProbs == [] for g in plain[i])
        for g in got[i]:
            assert len(g.topLogProbs) == len(g.tokenLogProbs)
            for t, lp, d in zip(g.tokens, g.tokenLogProbs, g.topLogProbs):
                if d:
                    t0, v0 = next(iter(d.items()))
                    assert t0 == t and bits([v0]) == bits([lp])
                    sampled += 1
    assert sampled >= 10
    res = L.transcribe_audio(kit, streams, dataclasses.replace(o, topLogProbs=5))
    assert all(len(g.topLogProbs) == len(g.tokenLogProbs) for r in res for g in r.segments)


# ---------------------------------------------------------------------------------------------------------------- 5. large-v3 scale
def test_large_v3_64_windows():
    W = 64
    LV3 = D.SpecialTokens(endToken=50257, englishToken=50259, noSpeechToken=50363, noTimestampsToken=50364, specialTokenBegin=50257,
                          startOfPreviousToken=50362, startOfTranscriptToken=50258, timeTokenBegin=50365, transcribeToken=50360,
                          translateToken=50359)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="large-v3", maxBatch=W, dtype="bf16", seed=3, specialTokens=wk.SpecialTokens.from_any(LV3)))
    pcm = pcm_of(W, 800)
    o = opts(sampleLength=224, languageToken=50259, suppressTokens=SUPPRESSED)
    P = len(kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens))
    plain = kit.transcribe(pcm, o)
    got = kit.transcribe(pcm, dataclasses.replace(o, topLogProbs=5))
    for w in range(W):
        same(plain[w], got[w], w)
        check_self_consistent(kit, w, got[w], 5, P)


# ---------------------------------------------------------------------------------------------------------------- 6. refusals
def test_refusals_leave_the_session_working():
    kit = make_kit(8, seed=37)
    pcm = pcm_of(3, 140)
    before = kit.transcribe(pcm, opts(topLogProbs=3))
    for bad in (dict(beamSize=2), dict(topLogProbs=21), dict(topLogProbs=-1)):
        with pytest.raises(wk.WhisperError) as e:
            kit.transcribe(pcm, opts(**{"topLogProbs": 3, **bad}))
        assert e.value.case == "invalidArgument", bad
    lib, sess = kit.model.lib, kit.textDecoder.handle
    for bad in (21, -1):
        with pytest.raises(wk.WhisperError) as e:
            check(lib.wk_session_set_top_logprobs(sess, bad))
        assert e.value.case == "invalidArgument"
    with pytest.raises(wk.WhisperError) as e:
        wk.AudioStreamTranscriber(kit, opts(topLogProbs=5))
    assert e.value.case == "invalidArgument"
    check(lib.wk_session_set_top_logprobs(sess, 4))                 # the C streamer and the long-form beam path refuse it as well
    try:
        with pytest.raises(wk.WhisperError) as e:
            wk.AudioStreamTranscriber(kit, opts())
        assert e.value.case == "invalidArgument"
        with pytest.raises(wk.WhisperError) as e:
            L.transcribe_streams(kit, [pcm[0]], opts(beamSize=2))
        assert e.value.case == "invalidArgument"
    finally:
        check(lib.wk_session_set_top_logprobs(sess, 0))
    after = kit.transcribe(pcm, opts(topLogProbs=3))
    for i in range(3):
        same(before[i], after[i], i)
        assert before[i].topLogProbs == after[i].topLogProbs
    # draftTokens
    model = wk.Model("toy", max_batch=8, dtype="bf16")
    model.init_random(41)
    model.setDraftDecoder(1, seed=42)
    st = kit.specialTokens
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, 8)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm[:2]))
    prompt = dec.prefillDecoderInputs(opts(), st)
    first = dec.decodeText(enc_t, prompt, opts(draftTokens=3), st)
    with pytest.raises(wk.WhisperError) as e:
        dec.decodeText(enc_t, prompt, opts(draftTokens=3, topLogProbs=2), st)
    assert e.value.case == "invalidArgument"
    second = dec.decodeText(enc_t, prompt, opts(draftTokens=3), st)
    for i in range(2):
        same(first[i], second[i], i)
    dec.close()
