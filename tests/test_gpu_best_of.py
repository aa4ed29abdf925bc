"""DecodingOptions.bestOf on the GPU: openai/whisper's decode_with_fallback rule inside the batched decode loop - beam search on the
temperature-0 rung, bestOf independent samples (the most likely kept, oracle/best_of_ref.py rank_best_of) on every hotter rung, and the
ladder for beam calls.  Best-of is checked against the best of independent single-row decodes of the same window (copy j on row j, so
the same Philox subsequence); the G rows of a best-of window share one cross K/V block and run the multi-query kernel, the copies the
single-query kernel, so log-probs agree to the same policy tolerance as tests/test_gpu_beam.py explains."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import best_of_ref as BR  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from tests import language_ref  # noqa: E402

TOL = {"f16": 5e-4, "bf16": 2e-3}
ROW_TOL = {"bf16": 2e-2, "f16": 4e-3}      # tests/test_gpu_align.py: alignment pass vs decode-loop export
FORCE = dict(logProbThreshold=0.0, compressionRatioThreshold=None)   # every window falls back (avgLogProb < 0)
NEVER = dict(logProbThreshold=None, compressionRatioThreshold=None)  # no window falls back


def st_of(variant):
    return D.SpecialTokens.toy(1024 if variant == "toy" else 2048)


def make_kit(slots, variant="toy", policy="bf16", seed=5, **kw):
    return wk.WhisperKit(wk.WhisperKitConfig(model=variant, maxBatch=slots, seed=seed, dtype=policy,
                                             specialTokens=wk.SpecialTokens.from_any(st_of(variant)), **kw))


def pcm_of(n, base):
    return np.stack([mel_ref.synthetic_pcm(base + i) for i in range(n)])


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=20)
    d.update(kw)
    return wk.DecodingOptions(**d)


def at(r, temperature):
    return abs(r.temperature - temperature) < 1e-6


def same(a, b, where):
    assert a.tokens == b.tokens, where
    assert np.array_equal(np.asarray(a.tokenLogProbs, np.float32).view(np.uint32), np.asarray(b.tokenLogProbs, np.float32).view(np.uint32)), where
    assert a.temperature == b.temperature and a.steps == b.steps, where


@pytest.mark.parametrize("variant,policy,fp8", [("toy128", "f16", False), ("toy", "bf16", False), ("toy", "bf16", True)])
def test_best_of_equals_the_best_of_independent_copies(variant, policy, fp8):
    G = 4
    st_o = st_of(variant)
    st = wk.SpecialTokens.from_any(st_o)
    model = wk.Model(variant, max_batch=G, dtype=policy, crossKVDtype="fp8" if fp8 else None)
    model.init_random(11)
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, G)
    pcm = mel_ref.synthetic_pcm(900)
    enc1 = enc.encodeFeatures(fe.logMelSpectrogram(pcm[None]))
    encG = enc.encodeFeatures(fe.logMelSpectrogram(np.repeat(pcm[None], G, axis=0)))
    kept = []
    for seed in (3, 4, 5):
        kw = dict(temperature=0.6, temperatureFallbackCount=0, seed=seed)
        prompt = dec.prefillDecoderInputs(opts(**kw), st)
        got = dec.decodeText(enc1, prompt, opts(bestOf=G, **kw), st)
        assert len(got) == 1
        copies = dec.decodeText(encG, prompt, opts(**kw), st)
        recorded = [list(r.tokenLogProbs[:r.currentTokenCount]) for r in copies]      # the prompt starts with SOT: slot i = recorded i
        best = BR.rank_best_of(recorded, len(prompt))
        kept.append(best)
        distinct = len({tuple(r.tokens) for r in copies})
        print(f"[{variant}/{policy}{'/fp8' if fp8 else ''} seed {seed}] {distinct} distinct samples of {G}, kept sample {best}")
        assert distinct > 1                               # the rows draw differently, or the ranking tests nothing
        assert got[0].tokens == copies[best].tokens, seed
        np.testing.assert_allclose(got[0].tokenLogProbs, copies[best].tokenLogProbs, atol=TOL[policy])
        assert abs(got[0].avgLogProb - copies[best].avgLogProb) < TOL[policy]
        assert got[0].temperature == copies[best].temperature and at(got[0], 0.6)
    dec.close()
    model.close()


def test_best_of_one_is_the_plain_ladder():
    kit = make_kit(3)
    pcm = pcm_of(5, 910)
    base = opts(temperatureFallbackCount=2, seed=8, **FORCE)
    plain = kit.transcribe(pcm, base)
    ladder = kit.textDecoder.stats()["ladder"]
    one = kit.transcribe(pcm, dataclasses.replace(base, bestOf=1))
    assert ladder == kit.textDecoder.stats()["ladder"] == 2 * len(pcm)
    for i in range(len(pcm)):
        same(one[i], plain[i], i)


def test_beam_without_best_of_skips_the_ladder():
    kit = make_kit(6)
    pcm = pcm_of(4, 920)
    o = opts(beamSize=3, **FORCE)                          # default temperatureFallbackCount = 5
    got = kit.transcribe(pcm, o)
    assert kit.textDecoder.stats()["ladder"] == 0
    ref = kit.transcribe(pcm, dataclasses.replace(o, temperatureFallbackCount=0))
    for i in range(len(pcm)):
        same(got[i], ref[i], i)
        assert got[i].temperature == 0.0


def test_best_of_without_fallback_is_the_plain_beam_call():
    kit = make_kit(6)
    pcm = pcm_of(4, 930)
    o = opts(beamSize=3, temperatureFallbackCount=2, **NEVER)
    ref = kit.transcribe(pcm, o)
    got = kit.transcribe(pcm, dataclasses.replace(o, bestOf=3))
    assert kit.textDecoder.stats()["ladder"] == 0
    for i in range(len(pcm)):
        same(got[i], ref[i], i)


@pytest.mark.parametrize("policy", ["bf16", "f16"])
def test_the_ladder_walks_from_beam_to_best_of(policy):
    kit = make_kit(9, policy=policy)                      # 3 slots of 3 rows
    pcm = pcm_of(3, 940)
    o = opts(beamSize=3, bestOf=3, temperatureFallbackCount=2, seed=21, **FORCE)
    got = kit.transcribe(pcm, o)
    assert kit.textDecoder.stats()["ladder"] == 2 * len(pcm)
    t_last = language_ref.rung_temperatures(D.DecodingOptions(temperature=0.0, temperatureFallbackCount=2))[-1]
    # the last rung alone: rung 0 at that (Float16) temperature with seed + 2, the same windows in the same slots
    alone = kit.transcribe(pcm, dataclasses.replace(o, temperature=t_last, seed=o.seed + 2, temperatureFallbackCount=0))
    for i in range(len(pcm)):
        assert at(got[i], 0.4) and round(t_last, 3) == 0.4
        same(got[i], alone[i], i)


def test_groups_at_different_rungs_share_one_step():
    kit = make_kit(6)                                     # 3 slots of 2 rows, 7 windows
    pcm = pcm_of(7, 950)
    base = opts(beamSize=2, bestOf=2, temperatureFallbackCount=2, seed=4)
    per = [dataclasses.replace(base, **(FORCE if i % 2 else NEVER)) for i in range(len(pcm))]
    got = kit.transcribe(pcm, per)
    assert kit.textDecoder.stats()["ladder"] == 2 * sum(i % 2 for i in range(len(pcm)))
    for i in range(len(pcm)):
        if i % 2:
            assert at(got[i], 0.4)
            continue
        alone = kit.transcribe(pcm[i], per[i])[0]         # beam search at temperature 0 does not depend on its slot
        assert got[i].temperature == 0.0
        assert got[i].tokens == alone.tokens, i
        np.testing.assert_allclose(got[i].tokenLogProbs, alone.tokenLogProbs, atol=TOL["bf16"])


@pytest.mark.parametrize("policy", ["f16", "bf16"])
def test_word_timestamps_follow_the_kept_sample(policy):
    kit = make_kit(8, variant="toy128", policy=policy)    # 2 slots of 4 rows, 3 windows
    pcm = pcm_of(3, 960)
    o = opts(bestOf=4, temperatureFallbackCount=1, wordTimestamps=True, sampleLength=14, seed=6, **FORCE)
    res = kit.transcribe(pcm, o)
    loop = [kit.textDecoder.alignmentWeights(b, 224) for b in range(len(pcm))]
    got = kit.align(pcm, [r.tokens for r in res])
    for b, r in enumerate(res):
        assert at(r, 0.2)
        steps = r.steps
        written = steps if loop[b][steps].any() else steps - 1
        assert written >= 3
        ref = got[b][0]
        worst = max(float(np.abs(ref[i] - loop[b][i]).max() / max(np.abs(loop[b][i]).max(), 1e-12)) for i in range(1, written + 1))
        print(f"[{policy}] window {b}: align pass vs the kept sample's decode-loop rows 1..{written}: rel err {worst:.2e}")
        assert worst <= ROW_TOL[policy], worst


def test_no_speech_prob_and_language_come_from_the_group():
    langs = [st_of("toy").englishToken] + list(range(200, 260))
    kit = make_kit(6)
    pcm = pcm_of(5, 970)
    base = opts(temperatureFallbackCount=0, computeNoSpeechProb=True, detectLanguage=True, allLanguageTokens=langs, **NEVER)
    for beam, best_of in ((2, 2), (1, 3)):
        ref = kit.transcribe(pcm, dataclasses.replace(base, beamSize=beam))
        got = kit.transcribe(pcm, dataclasses.replace(base, beamSize=beam, bestOf=best_of))
        for i in range(len(pcm)):
            assert got[i].languageToken == ref[i].languageToken and got[i].languageToken in langs, (beam, i)
            if beam == best_of:                       # the same rows and kernels: the same bits
                assert got[i].noSpeechProb == ref[i].noSpeechProb and got[i].languageLogProb == ref[i].languageLogProb
                same(got[i], ref[i], (beam, i))
            else:                                     # three rows share a cross K/V block: multi-query vs single-query kernel
                assert abs(got[i].noSpeechProb - ref[i].noSpeechProb) <= 1e-3, (got[i].noSpeechProb, ref[i].noSpeechProb)
                assert abs(got[i].languageLogProb - ref[i].languageLogProb) <= 1e-2


def test_invalid_settings_are_refused():
    kit = make_kit(4)
    pcm = pcm_of(2, 980)
    for o in (opts(bestOf=9), opts(bestOf=5), opts(beamSize=2, bestOf=5), opts(bestOf=-1),
              opts(beamSize=2, bestOf=2, wordTimestamps=True), opts(beamSize=2, wordTimestamps=True)):
        with pytest.raises(wk.WhisperError) as e:
            kit.transcribe(pcm, o)
        assert e.value.case == "invalidArgument", o
    with pytest.raises(wk.WhisperError):
        kit.transcribe(pcm, [opts(bestOf=2), opts(bestOf=3)])
    ok = kit.transcribe(pcm, opts(bestOf=4, temperature=0.5, temperatureFallbackCount=0))   # G = 4 = the session's rows
    assert len(ok) == 2 and all(at(r, 0.5) for r in ok)


def _toy_split(tokens, special_begin):
    words, groups = [], []
    for t in tokens:
        if t >= special_begin:
            words.append(f"<|{t}|>"); groups.append([t])
        elif t % 3 == 0 or not words or groups[-1][0] >= special_begin:
            words.append(" " + chr(97 + t % 26)); groups.append([t])
        else:
            words[-1] += chr(97 + t % 26); groups[-1].append(t)
    return words, groups


def test_long_form_with_best_of():
    from whisperkit_b200 import longform as LF
    st_o = st_of("toy")
    kit = make_kit(6)
    streams = [np.concatenate([mel_ref.synthetic_pcm(990 + 10 * i + k) for k in range(2)])[:n].astype(np.float32)
               for i, n in enumerate([480000 + 150000, 300000])]
    o = opts(beamSize=2, bestOf=2, temperatureFallbackCount=1, sampleLength=24, **FORCE)
    segs, windows = LF.transcribe_streams(kit, streams, o)
    assert windows >= 3 and all(len(s) >= 1 for s in segs)
    assert all(abs(g.temperature - 0.2) < 1e-6 for s in segs for g in s)
    ow = opts(bestOf=3, temperatureFallbackCount=1, sampleLength=24, wordTimestamps=True, **FORCE)
    SB = st_o.specialTokenBegin
    segs, windows = LF.transcribe_streams(kit, streams, ow, split_to_word_tokens=lambda t: _toy_split(t, SB),
                                          decode=lambda t: "".join(chr(97 + v % 26) for v in t))
    n_words = 0
    for s in segs:
        for g in s:
            assert g.words is not None
            for w in g.words:
                assert w.start <= w.end, w
            starts = [w.start for w in g.words]
            assert starts == sorted(starts)
            n_words += len(g.words)
    assert n_words > 0
