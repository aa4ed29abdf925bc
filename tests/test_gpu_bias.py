"""DecodingOptions.biasPhrases on the GPU: the phrase bonus inside the fused decode loop against tests/bias_ref.py, which consumes the GPU
decoder's own logits (predictLogits on explicit prefixes), so token ids must match bit for bit and log-probs agree to the tolerances
tests/test_gpu_beam.py explains (5e-4 f16, 2e-3 bf16).  λ = 0 must leave every output byte-identical to a call without a set."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from tests import bias_ref as B  # noqa: E402
from whisperkit_b200 import longform as L  # noqa: E402
from whisperkit_b200._lib import check  # noqa: E402

TOL = {"f16": 5e-4, "bf16": 2e-3}
NEVER = dict(logProbThreshold=None, compressionRatioThreshold=None)
FORCE = dict(logProbThreshold=0.0, compressionRatioThreshold=None)   # every rung falls back (avgLogProb < 0)


def st_of(variant):
    return D.SpecialTokens.toy(1024 if variant == "toy" else 2048)


def make_kit(slots, variant="toy", policy="bf16", seed=5, **kw):
    return wk.WhisperKit(wk.WhisperKitConfig(model=variant, maxBatch=slots, seed=seed, dtype=policy,
                                             specialTokens=wk.SpecialTokens.from_any(st_of(variant)), **kw))


def pcm_of(n, base):
    return np.stack([mel_ref.synthetic_pcm(base + i) for i in range(n)])


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=20, temperatureFallbackCount=0, **NEVER)
    d.update(kw)
    return wk.DecodingOptions(**d)


def random_phrases(n, length, text_tokens, seed):
    rng = np.random.default_rng(seed)
    return [[int(v) for v in rng.integers(0, text_tokens, length)] for _ in range(n)]


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def same(a, b, where):
    assert a.tokens == b.tokens, where
    assert np.array_equal(bits(a.tokenLogProbs), bits(b.tokenLogProbs)), where
    assert bits([a.avgLogProb, a.compressionRatio, a.noSpeechProb]).tolist() == bits([b.avgLogProb, b.compressionRatio, b.noSpeechProb]).tolist(), where
    assert (a.temperature, a.steps, a.currentTokenCount, a.languageToken) == (b.temperature, b.steps, b.currentTokenCount, b.languageToken), where
    assert a.fallback == b.fallback, where


def text_of(r, P):
    return list(r.tokens[P:r.currentTokenCount]) if r.currentTokenCount else []


# ---------------------------------------------------------------------------------------------------------------- 1. identity at λ = 0
@pytest.mark.parametrize("case", ["greedy", "beam3", "best_of3_ladder", "word_timestamps", "fp8_cross_kv"])
def test_zero_boost_is_byte_identical_to_no_set(case):
    st_o = st_of("toy")
    kw, cfg = {}, {}
    if case == "beam3":
        kw = dict(beamSize=3)
    elif case == "best_of3_ladder":
        kw = dict(bestOf=3, temperatureFallbackCount=3, **FORCE)
    elif case == "word_timestamps":
        kw = dict(wordTimestamps=True)
    elif case == "fp8_cross_kv":
        cfg = dict(crossKVDtype="fp8")
    kit = make_kit(12, **cfg)
    pcm = pcm_of(5, 40)
    phrases = random_phrases(256, 4, st_o.specialTokenBegin, 1)
    base = opts(computeNoSpeechProb=True, **kw)
    plain = kit.transcribe(pcm, base)
    w_plain = [kit.textDecoder.alignmentWeights(i) for i in range(5)] if case == "word_timestamps" else None
    zero = kit.transcribe(pcm, dataclasses.replace(base, biasPhrases=phrases, biasBoost=0.0))
    for i in range(5):
        same(plain[i], zero[i], (case, i))
    if w_plain is not None:
        for i in range(5):
            assert np.array_equal(bits(kit.textDecoder.alignmentWeights(i)), bits(w_plain[i])), i
    # a boost that matters changes the decode, so the zero boost ran the bias path
    hot = kit.transcribe(pcm, dataclasses.replace(base, biasPhrases=phrases, biasBoost=5.0))
    assert any(h.tokens != p.tokens for h, p in zip(hot, plain))


# ---------------------------------------------------------------------------------------------------------------- 2. oracle parity
def _window_predictor(model, pcm_window, rows=1):
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    dec = wk.TextDecoder(model, rows)
    dec.bindEncoderOutput(enc.encodeFeatures(fe.logMelSpectrogram(np.repeat(pcm_window[None], rows, axis=0))))
    return dec


def _phrases_from(unbiased_text, text_tokens, rng):
    """Prefixes of the unbiased output (they complete) plus the same starts with an unlikely continuation (their partial match breaks)."""
    runs, cur = [], []                      # the output's runs of text tokens (timestamps split them)
    for t in unbiased_text:
        if t < text_tokens:
            cur.append(t)
        else:
            runs, cur = runs + [cur], []
    runs.append(cur)
    out = [max(runs, key=len)[:3]]
    text = [t for t in unbiased_text if t < text_tokens]
    for k in range(1, min(len(text), 9), 2):
        out.append([text[k], int(rng.integers(0, text_tokens)), int(rng.integers(0, text_tokens))])
    return [ph for ph in out if ph] + random_phrases(6, 2, text_tokens, int(rng.integers(1 << 30)))


@pytest.mark.parametrize("variant,policy", [("toy128", "f16"), ("toy", "bf16")])
def test_greedy_matches_the_oracle_on_gpu_logits(variant, policy):
    st_o = st_of(variant)
    st = wk.SpecialTokens.from_any(st_o)
    kit = make_kit(2, variant, policy, seed=17)
    pcm = pcm_of(3, 610)
    o = opts(sampleLength=24)
    prompt = kit.textDecoder.prefillDecoderInputs(o, st)
    P = len(prompt)
    plain = kit.transcribe(pcm, o)
    rng = np.random.default_rng(2)
    revoked = completed = 0
    for b in range(3):
        phrases = _phrases_from(text_of(plain[b], P), st_o.specialTokenBegin, rng)
        got = kit.transcribe(pcm[b], dataclasses.replace(o, biasPhrases=phrases, biasBoost=0.7))[0]
        dec = _window_predictor(kit.model, pcm[b])
        trace = []
        ref = B.decode_text_biased(lambda tok, i: dec.predictLogits([tok], [i])[0], prompt, D.DecodingOptions(firstTokenLogProbThreshold=None,
                                   sampleLength=24, logProbThreshold=None, compressionRatioThreshold=None), st_o, True, phrases, 0.7, trace)
        dec.close()
        assert got.tokens == ref.tokens, (b, got.tokens, ref.tokens)
        np.testing.assert_allclose(got.tokenLogProbs, ref.tokenLogProbs, atol=TOL[policy])
        revoked += sum(t["revoked"] for t in trace)
        completed += sum(bool(t["completed"]) for t in trace)
    print(f"[{variant}/{policy} greedy] revoked partial matches {revoked}, completions {completed}")
    assert revoked >= 1 and completed >= 1


@pytest.mark.parametrize("variant,policy,beam,patience", [("toy128", "f16", 3, 1.0), ("toy", "bf16", 4, 2.0), ("toy", "bf16", 3, 2.0),
                                                          ("toy128", "f16", 5, 1.0)])   # (beam 5, patience 2: 10 candidates, above the 8 kept)
def test_beam_matches_the_oracle_on_gpu_logits(variant, policy, beam, patience):
    st_o = st_of(variant)
    st = wk.SpecialTokens.from_any(st_o)
    kit = make_kit(2 * beam, variant, policy, seed=19)
    pcm = pcm_of(3, 630)
    o = opts(sampleLength=22, beamSize=beam, beamPatience=patience)
    prompt = kit.textDecoder.prefillDecoderInputs(o, st)
    P = len(prompt)
    plain = kit.transcribe(pcm, o)
    rng = np.random.default_rng(3)
    sets = [_phrases_from(text_of(plain[b], P), st_o.specialTokenBegin, rng) for b in range(3)]
    got = kit.transcribe(pcm, [dataclasses.replace(o, biasPhrases=s, biasBoost=0.7) for s in sets])   # 3 windows, 2 beam groups
    revoked = completed = 0
    for b in range(3):
        dec = _window_predictor(kit.model, pcm[b], beam)

        def predict(prefixes, tokenIndex):
            lg = None
            for t in range(tokenIndex + 1):
                lg = dec.predictLogits([p[t] for p in prefixes], [t] * beam)
            return lg
        trace = []
        ref = B.decode_text_beam_biased(predict, prompt, D.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=22, logProbThreshold=None,
                                        compressionRatioThreshold=None), st_o, True, beam, patience, sets[b], 0.7, trace)
        dec.close()
        assert got[b].tokens == ref.tokens, (b, got[b].tokens, ref.tokens)
        np.testing.assert_allclose(got[b].tokenLogProbs, ref.tokenLogProbs, atol=TOL[policy])
        revoked += sum(t["revoked"] for t in trace)
        completed += sum(bool(t["completed"]) for t in trace)
    print(f"[{variant}/{policy} beam {beam} patience {patience}] revoked {revoked}, completions {completed}")
    assert revoked >= 1 and completed >= 1


# ---------------------------------------------------------------------------------------------------------------- 3. best-of at T > 0
def test_best_of_keeps_the_best_biased_score_of_independent_copies():
    G, variant, policy = 4, "toy", "bf16"
    st_o = st_of(variant)
    st = wk.SpecialTokens.from_any(st_o)
    model = wk.Model(variant, max_batch=G, dtype=policy)
    model.init_random(11)
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, G)
    pcm = mel_ref.synthetic_pcm(905)
    enc1 = enc.encodeFeatures(fe.logMelSpectrogram(pcm[None]))
    encG = enc.encodeFeatures(fe.logMelSpectrogram(np.repeat(pcm[None], G, axis=0)))
    phrases = random_phrases(40, 2, 64, 5)          # short phrases over frequent ids: the samples bank different bonuses
    boost = 1.5
    picks = set()
    for seed in (3, 4, 5):
        kw = dict(temperature=0.8, seed=seed, biasPhrases=phrases, biasBoost=boost)
        prompt = dec.prefillDecoderInputs(opts(**kw), st)
        P = len(prompt)
        got = dec.decodeText(enc1, prompt, opts(bestOf=G, **kw), st)
        copies = dec.decodeText(encG, prompt, opts(**kw), st)
        ranks = []
        for r in copies:
            s = np.float32(0.0)
            for v in r.tokenLogProbs[:r.currentTokenCount]:
                s = np.float32(s + np.float32(v))
            s = np.float32(s + np.float32(boost) * np.float32(B.banked(phrases, boost, text_of(r, P))))
            ranks.append(np.float32(s / np.float32(max(r.currentTokenCount - P, 1))))
        best = max(range(G), key=lambda j: (ranks[j], -j))
        picks.add(best)
        assert len({tuple(r.tokens) for r in copies}) > 1
        assert got[0].tokens == copies[best].tokens, seed
        np.testing.assert_allclose(got[0].tokenLogProbs, copies[best].tokenLogProbs, atol=TOL[policy])
    print(f"[best-of {G}, biased] kept samples {sorted(picks)}")


# ---------------------------------------------------------------------------------------------------------------- 4. effect
def test_a_strong_boost_puts_the_phrase_in_every_window_with_unbiased_log_probs():
    variant, policy = "toy128", "f16"
    st_o = st_of(variant)
    st = wk.SpecialTokens.from_any(st_o)
    kit = make_kit(4, variant, policy, seed=23)
    pcm = pcm_of(4, 700)
    o = opts(sampleLength=16, withoutTimestamps=True)
    prompt = kit.textDecoder.prefillDecoderInputs(o, st)
    P = len(prompt)
    plain = kit.transcribe(pcm, o)
    seen = {tuple(text_of(r, P)[i:i + 3]) for r in plain for i in range(len(text_of(r, P)))}
    phrase = next([a, a + 1, a + 2] for a in range(100, 900) if (a, a + 1, a + 2) not in seen)
    got = kit.transcribe(pcm, dataclasses.replace(o, biasPhrases=[phrase], biasBoost=30.0))
    for b, r in enumerate(got):
        t = text_of(r, P)
        at = next(i for i in range(len(t) - 2) if t[i:i + 3] == phrase)
        dec = _window_predictor(kit.model, pcm[b])
        hist = list(prompt) + t                             # r.tokens starts at the prompt's SOT: entry e of the history is r.tokens[e]
        for i in range(P + at + 2):
            lg = dec.predictLogits([hist[i]], [i])[0].astype(np.float32)
            e = i + 1                                       # the step at position i samples history entry i + 1
            if e >= P + at:
                assert abs(r.tokenLogProbs[e] - float(lg[hist[e]] - B._lse(lg))) <= TOL[policy], (b, e)
        dec.close()


# ---------------------------------------------------------------------------------------------------------------- 5. per-window sets
@pytest.mark.parametrize("beam", [1, 3])
def test_per_window_sets_equal_each_window_alone(beam):
    st_o = st_of("toy")
    kit = make_kit(2 * beam, seed=29)
    pcm = pcm_of(5, 720)
    sets = [random_phrases(8 + 4 * i, 3, st_o.specialTokenBegin, 50 + i) for i in range(5)]
    os_ = [opts(beamSize=beam, biasPhrases=s, biasBoost=1.0 + 0.5 * i) for i, s in enumerate(sets)]
    got = kit.transcribe(pcm, os_)
    for i in range(5):
        alone = kit.transcribe(pcm[i], os_[i])[0]
        assert got[i].tokens == alone.tokens, i
        np.testing.assert_allclose(got[i].tokenLogProbs, alone.tokenLogProbs, atol=TOL["bf16"])


# ---------------------------------------------------------------------------------------------------------------- 6. long-form
def _create_set(lib, phrases, boost, stb):
    flat = [t for p in phrases for t in p]
    h = C.c_void_p()
    check(lib.wk_bias_create((C.c_int32 * len(flat))(*flat), (C.c_int32 * len(phrases))(*[len(p) for p in phrases]), len(phrases), boost, stb,
                             C.byref(h)))
    return h


def test_long_form_streams_with_their_own_sets():
    st_o = st_of("toy")
    kit = make_kit(4, seed=9)
    lib, sess = kit.model.lib, kit.textDecoder.handle
    o = opts(sampleLength=24)
    lens = [480000 + 200000, 300000, 1000000]
    streams = [np.concatenate([mel_ref.synthetic_pcm(300 + 10 * i + k) for k in range(3)])[:n].astype(np.float32) for i, n in enumerate(lens)]
    sets = [random_phrases(12, 3, st_o.specialTokenBegin, 70 + i) for i in range(3)]
    hs = [_create_set(lib, s, 2.0, st_o.specialTokenBegin) for s in sets]
    try:
        check(lib.wk_session_set_bias(sess, (C.c_void_p * 3)(*[h.value for h in hs]), 3))
        together, _ = L.transcribe_streams(kit, streams, o)
        for i in range(3):
            check(lib.wk_session_set_bias(sess, (C.c_void_p * 1)(hs[i].value), 1))
            alone, _ = L.transcribe_streams(kit, [streams[i]], o)
            assert [g.tokens for g in together[i]] == [g.tokens for g in alone[0]], i
        check(lib.wk_session_set_bias(sess, None, 0))
    finally:
        lib.wk_session_set_bias(sess, None, 0)
        for h in hs:
            lib.wk_bias_free(h)
    plain, _ = L.transcribe_streams(kit, streams, o)
    zero, _ = L.transcribe_streams(kit, streams, dataclasses.replace(o, biasPhrases=sets[0], biasBoost=0.0))
    for i in range(3):
        assert [g.tokens for g in plain[i]] == [g.tokens for g in zero[i]]
        assert bits([v for g in plain[i] for v in g.tokenLogProbs]).tolist() == bits([v for g in zero[i] for v in g.tokenLogProbs]).tolist()
    assert any([g.tokens for g in together[i]] != [g.tokens for g in plain[i]] for i in range(3))


# ---------------------------------------------------------------------------------------------------------------- 7. large-v3 dimensions
def test_large_v3_64_windows_256_phrases_match_the_oracle():
    W, policy = 64, "bf16"
    LV3 = D.SpecialTokens(endToken=50257, englishToken=50259, noSpeechToken=50363, noTimestampsToken=50364, specialTokenBegin=50257,
                          startOfPreviousToken=50362, startOfTranscriptToken=50258, timeTokenBegin=50365, transcribeToken=50360,
                          translateToken=50359)
    st = wk.SpecialTokens.from_any(LV3)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="large-v3", maxBatch=W, dtype=policy, seed=3, specialTokens=st))
    pcm = pcm_of(W, 800)
    o = opts(sampleLength=12, languageToken=50259, withoutTimestamps=True)   # (with timestamps a random large-v3 only emits timestamps)
    prompt = kit.textDecoder.prefillDecoderInputs(o, st)
    P = len(prompt)
    plain = kit.transcribe(pcm, o)
    # 256 x 4-token phrases whose chains cover the model's own tokens: up to 1024 candidates per step, deduplicated across phrases
    rng = np.random.default_rng(4)
    pool = sorted({t for r in plain for t in text_of(r, P) if t < LV3.specialTokenBegin}) + [int(v) for v in rng.integers(0, 50257, 16)]
    phrases = [[int(rng.choice(pool)) for _ in range(4)] for _ in range(256)]
    got = kit.transcribe(pcm, dataclasses.replace(o, biasPhrases=phrases, biasBoost=8.0))
    assert sum(g.tokens != p.tokens for g, p in zip(got, plain)) >= 1
    for b in (0, W - 1):
        dec = _window_predictor(kit.model, pcm[b])
        ref = B.decode_text_biased(lambda tok, i: dec.predictLogits([tok], [i])[0], prompt, D.DecodingOptions(
            firstTokenLogProbThreshold=None, sampleLength=12, logProbThreshold=None, compressionRatioThreshold=None, withoutTimestamps=True),
            LV3, True, phrases, 8.0)
        dec.close()
        assert got[b].tokens == ref.tokens, (b, got[b].tokens, ref.tokens)
        np.testing.assert_allclose(got[b].tokenLogProbs, ref.tokenLogProbs, atol=TOL[policy])


# ---------------------------------------------------------------------------------------------------------------- 8. refusals
def test_refusals_and_a_cleared_set_leaves_no_trace():
    st_o = st_of("toy")
    st = wk.SpecialTokens.from_any(st_o)
    model = wk.Model("toy", max_batch=4, dtype="bf16")
    model.init_random(31)
    model.setDraftDecoder(1, seed=32)
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, 4)
    pcm = pcm_of(2, 760)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    prompt = dec.prefillDecoderInputs(opts(), st)
    dec.decodeText(enc_t, prompt, opts(draftTokens=1), st)                   # the draft call itself is fine
    with pytest.raises(wk.WhisperError) as e:
        dec.decodeText(enc_t, prompt, opts(draftTokens=1, biasPhrases=[[1, 2]]), st)
    assert e.value.case == "invalidArgument"
    # streamer + an attached set
    kit = make_kit(4, seed=33)
    lib, sess = kit.model.lib, kit.textDecoder.handle
    with pytest.raises(wk.WhisperError):
        wk.AudioStreamTranscriber(kit, opts(biasPhrases=[[1, 2]]))
    tr = wk.AudioStreamTranscriber(kit, opts())
    sid = tr.addStream()
    tr.processBuffer(sid, mel_ref.synthetic_pcm(770)[:160000])
    h = _create_set(lib, [[1, 2]], 2.0, st_o.specialTokenBegin)
    hs = (C.c_void_p * 2)(h.value, h.value)
    try:
        check(lib.wk_session_set_bias(sess, hs, 1))
        with pytest.raises(wk.WhisperError) as e:
            tr.transcribeCurrentBuffers()
        assert e.value.case == "invalidArgument"
        # n_sets must be 1 or one per window
        check(lib.wk_session_set_bias(sess, hs, 2))
        pcm3 = pcm_of(3, 780)
        with pytest.raises(wk.WhisperError) as e:
            kit.transcribe(pcm3, opts())
        assert e.value.case == "invalidArgument"
    finally:
        check(lib.wk_session_set_bias(sess, None, 0))
        lib.wk_bias_free(h)
    tr.close()
    after = kit.transcribe(pcm3, opts())
    fresh = make_kit(4, seed=33).transcribe(pcm3, opts())
    for i in range(3):
        same(after[i], fresh[i], i)
