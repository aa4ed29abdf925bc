"""DecodingOptions.computeNoSpeechProb on the H100 (toy variants, f16 and bf16): the value computed inside the batched decode loop against
a float64 softmax of the raw logits predictLogits returns at the prompt's SOT step and against the CPU oracle model, byte-identical
decoding with the option on and off, the silence rule on a model whose <|nospeech|> row is edited so that some windows are silent,
mixed batches, in-loop language detection, beam search, the FP8 cross K/V cache, the temperature ladder, the long-form skip rule
(tests/no_speech_ref.py's seek loop fed the same GPU window results) and validation."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402
from oracle import seek_ref as S  # noqa: E402
from tests import no_speech_ref as N  # noqa: E402
from whisperkit_b200._lib import check, wk_decode_result  # noqa: E402
from whisperkit_b200.api import make_batch_opts, session_no_speech_probs  # noqa: E402

DIMS = M.VARIANTS["toy"]
V = DIMS.vocab
ST = D.SpecialTokens.toy(V)
SOT, NS = ST.startOfTranscriptToken, ST.noSpeechToken
EMB = "model.decoder.embed_tokens.weight"
LANGS = [ST.englishToken] + list(range(200, 260))
LOGIT_TOL = {"bf16": 4e-3, "f16": 1e-3}   # the logits tolerances of tests/test_gpu_pipeline.py
POLICIES = ["f16", "bf16"]
PROMPTS = {"plain": {}, "noPrefill": dict(usePrefillPrompt=False), "promptTokens": dict(promptTokens=[9, 8, 7, 6]),
           "prefixTokens": dict(prefixTokens=[11, 12])}


def make_kit(policy, slots=4, w=None, seed=7, **kw):
    w = w if w is not None else M.random_weights(DIMS, seed=seed, policy=policy)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=slots, dtype=policy, weights=w, specialTokens=wk.SpecialTokens.from_any(ST),
                                            **kw))
    return kit, w


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=24, temperatureFallbackCount=0, computeNoSpeechProb=True)
    d.update(kw)
    return wk.DecodingOptions(**d)


def pcm_of(n, base=600):
    return np.stack([mel_ref.synthetic_pcm(base + i) for i in range(n)])


def encode(kit, pcm):
    return kit.audioEncoder.encodeFeatures(kit.featureExtractor.logMelSpectrogram(pcm))


def sot_logits(dec, prompt, enc_t=None):
    """predictLogits over the prompt up to its first SOT, every bound window: the raw logits of the SOT step [B, V].  enc_t binds
    the windows again first (a batched decode leaves the session's row count at windows x beams)."""
    if enc_t is not None:
        dec.bindEncoderOutput(enc_t)
    dec.prepareDecoderInputs()
    sot = list(prompt).index(SOT)
    for i in range(sot + 1):
        lg = dec.predictLogits([prompt[i]] * dec.batch, [i] * dec.batch)
    return lg


def check_values(res, logits, where):
    err = max(abs(r.noSpeechProb - N.no_speech_prob(lg, ST)) for r, lg in zip(res, logits))
    print(f"[{where}] noSpeechProb vs float64 softmax of predictLogits: max |error| = {err:.3e}")
    assert err <= 1e-6, (where, err)
    return err


@pytest.mark.parametrize("case", list(PROMPTS))
@pytest.mark.parametrize("policy", POLICIES)
def test_value_matches_predict_logits_and_the_oracle(policy, case):
    B = 3
    kit, w = make_kit(policy)
    dec = kit.textDecoder
    o = opts(**PROMPTS[case])
    enc_t = encode(kit, pcm_of(B))
    prompt = dec.prefillDecoderInputs(o if o.usePrefillPrompt else None, kit.specialTokens)
    lg = sot_logits(dec, prompt, enc_t)
    res = dec.decodeText(None, None, o, kit.specialTokens)
    check_values(res, lg, f"{policy}/{case}")
    assert all(0.0 < r.noSpeechProb < 1.0 for r in res)
    # the CPU oracle model on the GPU's encoder output, teacher-forced over the same prefix
    orc = M.WhisperOracle(DIMS, w, policy)
    with torch.no_grad():
        cross = orc.cross_kv(torch.from_numpy(enc_t.numpy()).transpose(1, 2).contiguous())
        cache = orc.new_cache(B)
        for i in range(prompt.index(SOT) + 1):
            lg_ref = orc.decode_step(torch.tensor([prompt[i]] * B), i, cache, cross).numpy()
    scale = float(np.abs(lg_ref).max())
    rel = float(np.abs(lg.astype(np.float64) - lg_ref).max()) / scale
    dp = max(abs(r.noSpeechProb - N.no_speech_prob(x, ST)) for r, x in zip(res, lg_ref))
    print(f"[{policy}/{case}] SOT-step logits rel err vs oracle {rel:.2e}, noSpeechProb |difference| {dp:.2e}")
    assert rel <= LOGIT_TOL[policy], rel
    assert dp <= 2 * LOGIT_TOL[policy] * scale, dp          # |d softmax_k| <= 2 max|d logit|


@pytest.mark.parametrize("policy", POLICIES)
def test_option_on_and_off_decode_identically(policy):
    kit, _ = make_kit(policy)
    pcm = pcm_of(5, 620)
    base = dict(noSpeechThreshold=None, wordTimestamps=True)
    on = kit.transcribe(pcm, opts(**base))
    align_on = [kit.textDecoder.alignmentWeights(i) for i in range(5)]
    off = kit.transcribe(pcm, opts(computeNoSpeechProb=False, **base))
    nan = session_no_speech_probs(kit.model.lib, kit.textDecoder.handle, 5)
    assert all(math.isnan(v) for v in nan)                           # C: not computed
    for i in range(5):
        a, b = on[i], off[i]
        assert a.tokens == b.tokens and a.steps == b.steps, i
        assert np.float32(a.tokenLogProbs).tobytes() == np.float32(b.tokenLogProbs).tobytes(), i
        assert np.float32(a.avgLogProb) == np.float32(b.avgLogProb) and a.fallback == b.fallback, i
        assert align_on[i].tobytes() == kit.textDecoder.alignmentWeights(i).tobytes(), i
        assert 0.0 < a.noSpeechProb < 1.0 and b.noSpeechProb == 0.0, i   # Python: 0.0 when not computed


def forced_silence_weights(policy, speech, seed=7):
    """The toy weights with the <|nospeech|> row of the tied embedding rewritten so that an all-zero window has noSpeechProb ~0.9 and
    `speech` ~0.1: the final-LayerNorm outputs x of the two SOT steps are recovered from their logits (x = lstsq(E, logits)), and the
    row is the least-norm e with x . e = the logit that gives the target probability against the rest of the row."""
    kit, w = make_kit(policy, slots=2)
    dec = kit.textDecoder
    L = sot_logits(dec, [SOT], encode(kit, np.stack([np.zeros(480000, np.float32), speech]))).astype(np.float64)
    E = w[EMB].double().numpy()
    X = np.linalg.lstsq(E, L.T, rcond=None)[0].T
    rest = np.delete(L, NS, axis=1)
    lse = rest.max(1) + np.log(np.exp(rest - rest.max(1, keepdims=True)).sum(1))
    target = np.array([0.9, 0.1])
    e = np.linalg.lstsq(X, np.log(target / (1 - target)) + lse, rcond=None)[0]
    w2 = dict(w)
    w2[EMB] = w[EMB].clone()
    w2[EMB][NS] = M.round_to(torch.from_numpy(e).float(), policy)
    return w2


@pytest.fixture(scope="module", params=POLICIES)
def silence(request):
    speech = mel_ref.synthetic_pcm(640)
    return request.param, speech, forced_silence_weights(request.param, speech)


def window_set(speech):
    z = np.zeros(480000, np.float32)
    return np.stack([z, speech, mel_ref.synthetic_pcm(641), z, speech * 0.5, mel_ref.synthetic_pcm(642)])


def test_forced_silence_marks_silent_windows_and_skips_the_ladder(silence):
    policy, speech, w = silence
    kit, _ = make_kit(policy, slots=3, w=w)
    pcm = window_set(speech)
    # thresholds at their defaults (0.6 / -1.0 / 2.4); every ladder rung decodes at temperature 0, so that a window's tokens do not depend
    # on the slot it lands in (a draw at temperature > 0 is keyed by the decode row)
    o = opts(temperatureFallbackCount=2, temperatureIncrementOnFallback=0.0)
    on = kit.transcribe(pcm, o)
    ladder_on = kit.textDecoder.stats()["ladder"]
    off = kit.transcribe(pcm, dataclasses.replace(o, computeNoSpeechProb=False))
    p = [r.noSpeechProb for r in on]
    print(f"[{policy}] forced-silence noSpeechProb per window: {np.round(p, 4).tolist()}")
    assert p[0] > 0.6 and p[3] > 0.6 and p[1] < 0.6                 # the all-zero windows and the design's speech window
    silent = [i for i in range(len(p)) if p[i] > 0.6]
    assert 0 < len(silent) < len(p)
    for i, (a, b) in enumerate(zip(on, off)):
        if i in silent:
            assert a.fallback == wk.DecodingFallback(False, "silence") and a.temperature == 0.0, i
        else:
            assert a.tokens == b.tokens and a.steps == b.steps and a.temperature == b.temperature and a.fallback == b.fallback, i
            np.testing.assert_array_equal(np.float32(a.tokenLogProbs), np.float32(b.tokenLogProbs))
    assert all(off[i].fallback != on[i].fallback for i in silent)    # without the value no window is silent
    # only the windows that still ask for a fallback walk the ladder (each of its 2 rungs asks again at the same temperature)
    assert ladder_on == 2 * sum(r.fallback is not None and r.fallback.needsFallback for r in on) < 2 * len(pcm)
    # a mixed batch (opt-in on some windows only): every window equals that window decoded alone
    items = [o if i % 2 == 0 else dataclasses.replace(o, computeNoSpeechProb=False) for i in range(len(pcm))]
    mixed = kit.transcribe(pcm, items)
    for i in range(len(pcm)):
        alone = kit.transcribe(pcm[i], items[i])[0]
        assert mixed[i].tokens == alone.tokens and mixed[i].steps == alone.steps and mixed[i].fallback == alone.fallback, i
        assert mixed[i].temperature == alone.temperature and mixed[i].noSpeechProb == alone.noSpeechProb, i
        assert (mixed[i].noSpeechProb == 0.0) == (i % 2 == 1), i


@pytest.mark.parametrize("policy", POLICIES)
def test_with_in_loop_language_detection(policy):
    kit, _ = make_kit(policy)
    dec = kit.textDecoder
    enc_t = encode(kit, pcm_of(3, 660))
    # step-0 form: the prompt starts with SOT, detection and the value share step 0
    o = opts(detectLanguage=True, allLanguageTokens=LANGS)
    lg0 = sot_logits(dec, [SOT], enc_t)
    res = dec.decodeText(None, None, o, kit.specialTokens)
    assert all(r.languageToken in LANGS for r in res)
    check_values(res, lg0, f"{policy}/detect step 0")
    # leading-step form: <|startofprev|> first, so detection runs one leading step on [SOT] at position 0; the value still comes from
    # the real SOT step of the prompt
    o = opts(detectLanguage=True, allLanguageTokens=LANGS, promptTokens=[9, 8, 7, 6])
    prompt = dec.prefillDecoderInputs(o, kit.specialTokens)
    lg = sot_logits(dec, prompt, enc_t)
    res = dec.decodeText(None, None, o, kit.specialTokens)
    assert all(r.languageToken in LANGS for r in res)
    check_values(res, lg, f"{policy}/detect leading step")
    lead_gap = min(abs(N.no_speech_prob(a, ST) - N.no_speech_prob(b, ST)) for a, b in zip(lg, lg0))
    assert lead_gap > 1e-5, lead_gap                                 # the leading step's value would be told apart


@pytest.mark.parametrize("policy", POLICIES)
def test_with_beam_search(policy):
    kit, _ = make_kit(policy)
    dec = kit.textDecoder
    enc_t = encode(kit, pcm_of(2, 680))
    for case in ("plain", "promptTokens"):
        o = opts(beamSize=2, **PROMPTS[case])
        lg = sot_logits(dec, dec.prefillDecoderInputs(o, kit.specialTokens), enc_t)
        res = dec.decodeText(None, None, o, kit.specialTokens)
        check_values(res, lg, f"{policy}/beam/{case}")


@pytest.mark.parametrize("policy", POLICIES)
def test_with_the_fp8_cross_kv_cache(policy):
    kit, _ = make_kit(policy, crossKVDtype="fp8")
    dec = kit.textDecoder
    enc_t = encode(kit, pcm_of(3, 700))
    for case in ("plain", "promptTokens"):
        o = opts(**PROMPTS[case])
        lg = sot_logits(dec, dec.prefillDecoderInputs(o, kit.specialTokens), enc_t)
        check_values(dec.decodeText(None, None, o, kit.specialTokens), lg, f"{policy}/fp8/{case}")


def test_ladder_reports_the_returned_rungs_value():
    kit, _ = make_kit("bf16", slots=2)
    pcm = pcm_of(2, 720)
    o = opts(temperatureFallbackCount=2, logProbThreshold=0.0, compressionRatioThreshold=None, noSpeechThreshold=None, seed=5)
    got = kit.transcribe(pcm, o)                                     # every rung asks for a fallback: rung 2 is returned
    assert kit.textDecoder.stats()["ladder"] == 4
    assert all(np.float32(r.temperature) == np.float32(0.4) for r in got)
    rung0 = kit.transcribe(pcm, dataclasses.replace(o, temperatureFallbackCount=0))
    for a, b in zip(got, rung0):
        assert a.noSpeechProb == b.noSpeechProb and 0.0 < a.noSpeechProb < 1.0   # raw logits at the SOT step: the same at every rung


def _long_streams(speech):
    z = np.zeros(1_600_000, np.float32)
    return [np.concatenate([speech[:160000], z, speech[200000:360000]]), speech.copy()]


@pytest.mark.parametrize("chunking", [None, "vad"])
def test_long_form_skips_silent_windows_like_the_reference_loop(silence, chunking):
    from whisperkit_b200 import longform as LF
    policy, speech, w = silence
    kit, _ = make_kit(policy, slots=4, w=w)
    o = opts(logProbThreshold=None, compressionRatioThreshold=None)
    streams = _long_streams(speech)
    got, _ = LF.transcribe_streams(kit, streams, o, chunkingStrategy=chunking)
    n_skipped = n_kept = 0
    for i, x in enumerate(streams):
        chunks = S.vad_chunk_all(x, 480000) if chunking == "vad" else [(0, len(x))]
        ref = []
        for a, b in chunks:
            xc = x[a:b]

            def decode_window(seek, size, xc=xc):
                win = np.zeros(480000, np.float32)
                win[:size] = xc[seek:seek + size]
                return kit.transcribe(win[None], o, samplesPerWindow=[size])[0]
            segs, wins = N.seek_loop(len(xc), decode_window, timeToken=ST.timeTokenBegin, noSpeechThreshold=o.noSpeechThreshold,
                                     logProbThreshold=o.logProbThreshold)
            n_skipped += sum(s for _, _, s in wins)
            n_kept += sum(not s for _, _, s in wins)
            for g in segs:
                g.seek += a
                g.start = float(np.float32(g.start) + np.float32(a) / np.float32(16000))
                g.end = float(np.float32(g.end) + np.float32(a) / np.float32(16000))
            ref += segs
        assert [g.tokens for g in got[i]] == [r.tokens for r in ref], (chunking, i)
        assert [g.seek for g in got[i]] == [r.seek for r in ref], (chunking, i)
        np.testing.assert_allclose([g.start for g in got[i]], [r.start for r in ref], atol=1e-4)
        np.testing.assert_allclose([g.end for g in got[i]], [r.end for r in ref], atol=1e-4)
        assert [np.float32(g.noSpeechProb) for g in got[i]] == [np.float32(r.noSpeechProb) for r in ref], (chunking, i)
    print(f"[{policy}/{chunking}] reference windows: {n_skipped} skipped as silent, {n_kept} kept")
    assert n_skipped > 0 and n_kept > 0


def test_a_prompt_without_sot_fails_its_window_alone():
    kit, _ = make_kit("bf16", slots=3)
    dec, lib = kit.textDecoder, kit.model.lib
    dec.bindEncoderOutput(encode(kit, pcm_of(3, 740)))
    good = dec.prefillDecoderInputs(opts(), kit.specialTokens)
    bad = [ST.startOfPreviousToken, 5, 6, ST.transcribeToken]
    st = kit.specialTokens.to_c()
    items = [opts(), opts(), opts(computeNoSpeechProb=False)]
    status = (C.c_int32 * 3)()
    bo, keep = make_batch_opts(3, items, [bad, good, bad], status=status)
    res = (wk_decode_result * 3)()
    check(lib.wk_decode_text_ex(dec.handle, C.byref(st), C.byref(bo), res))
    assert list(status) == [-4, 0, 0]                                # WK_ERR_PREPARE_DECODER_INPUTS for the opt-in window alone
    alone = dec.decodeText(None, good, opts(), kit.specialTokens)[1]
    assert list(res[1].tokens[:res[1].n_tokens]) == alone.tokens
    assert res[2].n_tokens > 0
    bo, keep = make_batch_opts(3, opts(), [bad, good, good])
    with pytest.raises(wk.WhisperError) as e:
        check(lib.wk_decode_text_ex(dec.handle, C.byref(st), C.byref(bo), res))
    assert "startoftranscript" in str(e.value)
