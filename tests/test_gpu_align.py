"""Forced alignment of given token sequences (wk_align_tokens / wk_align_windows, TextDecoder.alignTokens / WhisperKit.align): one
teacher-forced decoder pass over every position, checked against

  * the oracle decoder teacher-forced over the same tokens (oracle/model_ref.py decode_step with align_heads): every alignment row at the
    tolerances of test_gpu_pipeline.test_alignment_heads_weights_parity (2e-2 bf16, 4e-3 f16, relative to the row's largest value), rows
    summing to 1 within 5e-3, and the token log-probs (log_softmax(logits[:eot])[next token]) at the end-to-end logit tolerances (4e-3 bf16,
    1e-3 f16) relative to the row's largest |logit|;
  * the decode loop's own wordTimestamps export for the tokens it decoded (different GEMM paths: same tolerances, not the same bits);
  * itself: ragged sequences in more windows than the session has slots give the bits of each window aligned alone;
  * the fp32 oracle at large-v3 dimensions (64 windows of 224 tokens, two of them checked, errors printed);
  * the FP8-cache oracle (tests/fp8_ref.py) on an FP8 session;
  * the host word-timing code: beam-search results aligned afterwards get word timings;
  * per-window validation: an empty sequence, 225 tokens and an id >= vocab fail only their own window."""
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402
from tests import fp8_ref  # noqa: E402
from whisperkit_b200.wordtiming import WordTimingSeeker  # noqa: E402

ROW_TOL = {"bf16": 2e-2, "f16": 4e-3}
LOGIT_TOL = {"bf16": 4e-3, "f16": 1e-3}


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def build(variant, policy, B, seed, fp8=False):
    dims = M.VARIANTS[variant]
    w = M.random_weights(dims, seed=seed, policy=policy)
    orc = fp8_ref.FP8CrossKVOracle(dims, w, policy) if fp8 else M.WhisperOracle(dims, w, policy)
    model = wk.Model(variant, max_batch=B, dtype=policy, crossKVDtype="fp8" if fp8 else None)
    model.load_state_dict(w)
    return dims, orc, model


def make_seq(rng, prompt, n_text, st_o, timestamps=True):
    """prompt + text tokens (a timestamp token in the middle when asked) + EOT."""
    text = [int(v) for v in rng.integers(0, st_o.specialTokenBegin, n_text)]
    if timestamps and n_text > 4:
        text[n_text // 2] = st_o.timeTokenBegin + 7
    return list(prompt) + text + [st_o.endToken]


def oracle_align(orc, enc_b, toks, heads, eot):
    """Teacher-forced oracle over toks: alignment rows [n][T] (Float16 means) and log-probs [n] (NaN at 0 and at special targets), plus
    the largest |logit| of each predicting row."""
    with torch.no_grad():
        cross = orc.cross_kv(torch.from_numpy(enc_b[None]).transpose(1, 2).contiguous())
        cache = orc.new_cache(1)
        rows, lp, scale = [], np.full(len(toks), np.nan), np.zeros(len(toks))
        for i, t in enumerate(toks):
            lg, al = orc.decode_step(torch.tensor([t]), i, cache, cross, align_heads=heads)
            rows.append(al[0].numpy())
            if i + 1 < len(toks):
                scale[i + 1] = float(lg[0, :eot].abs().max())
                if toks[i + 1] < eot:
                    lp[i + 1] = float(torch.log_softmax(lg[0, :eot].double(), -1)[toks[i + 1]])
    return np.stack(rows), lp, scale


def check_against_oracle(tag, policy, weights, logprobs, toks, ref_rows, ref_lp, ref_scale):
    n = len(toks)
    assert weights.shape[0] == n + 1 and np.all(weights[0] == 0)
    worst = max(rel_err(weights[i + 1], ref_rows[i]) for i in range(n))
    assert all(abs(float(weights[i + 1].sum()) - 1.0) < 5e-3 for i in range(n))
    special = np.isnan(ref_lp)
    assert np.array_equal(np.isnan(logprobs), special)
    lp_err = float((np.abs(logprobs[~special] - ref_lp[~special]) / np.maximum(ref_scale[~special], 1.0)).max()) if (~special).any() else 0.0
    print(f"[{tag}/{policy}] n={n}: alignment rows rel err {worst:.2e}, log-prob err / max|logit| {lp_err:.2e}")
    assert worst <= ROW_TOL[policy], worst
    assert lp_err <= LOGIT_TOL[policy], lp_err


@pytest.mark.parametrize("policy", ["f16", "bf16"])
def test_align_tokens_matches_teacher_forced_oracle(policy):
    B = 3
    dims, orc, model = build("toy128", policy, B, seed=31)
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    pcm = np.stack([mel_ref.synthetic_pcm(700 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    prompt = dec.prefillDecoderInputs(wk.DecodingOptions(), st)
    rng = np.random.default_rng(3)
    seqs = [make_seq(rng, prompt, n, st_o) for n in (6, 13, 21)]
    for heads in ([], [(0, 1), (1, 0), (1, 3)]):
        model.setAlignmentHeads(heads)
        ref_heads = heads or [(l, h) for l in range(dims.dec_layers // 2, dims.dec_layers) for h in range(dims.n_heads)]
        got = dec.alignTokens(enc_t, seqs, st)
        for b in range(B):
            ref = oracle_align(orc, enc_gpu[b], seqs[b], ref_heads, st_o.endToken)
            check_against_oracle(f"heads {len(ref_heads)} window {b}", policy, got[b][0], got[b][1], seqs[b], *ref)
            full = dec.alignmentWeights(b, 225)
            assert np.all(full[len(seqs[b]) + 1:] == 0)
    dec.close()
    model.close()


@pytest.mark.parametrize("policy", ["f16", "bf16"])
def test_align_tokens_matches_the_decode_loop_export(policy):
    B = 3
    dims, orc, model = build("toy128", policy, B, seed=21)
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(dims.vocab))
    pcm = np.stack([mel_ref.synthetic_pcm(300 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12, wordTimestamps=True)
    res = dec.decodeText(enc_t, dec.prefillDecoderInputs(o, st), o, st)
    loop = [dec.alignmentWeights(b, 224) for b in range(B)]
    got = dec.alignTokens(None, [r.tokens for r in res], st)
    for b in range(B):
        steps = res[b].steps
        written = steps if loop[b][steps].any() else steps - 1
        assert written >= 3
        worst = max(rel_err(got[b][0][i], loop[b][i]) for i in range(1, written + 1))
        print(f"[{policy}] window {b}: align pass vs decode loop rows 1..{written}: rel err {worst:.2e}")
        assert worst <= ROW_TOL[policy], worst
    dec.close()
    model.close()


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def test_ragged_windows_are_batch_independent():
    st_o = D.SpecialTokens.toy(2048)
    st = wk.SpecialTokens.from_any(st_o)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy128", maxBatch=2, seed=41, specialTokens=st))
    lens = [4, 57, 224, 130, 33]
    pcm = np.stack([mel_ref.synthetic_pcm(800 + i) for i in range(len(lens))])
    rng = np.random.default_rng(5)
    seqs = [make_seq(rng, [st_o.startOfTranscriptToken], n - 2, st_o) for n in lens]
    assert [len(s) for s in seqs] == lens
    allr = kit.align(pcm, seqs)                                   # 5 windows through 2 slots: three chunks
    full = [kit.textDecoder.alignmentWeights(b, 225) for b in range(len(lens))]
    for b, n in enumerate(lens):
        assert np.all(full[b][n + 1:] == 0) and np.all(full[b][0] == 0)
        assert np.all(np.abs(full[b][1:n + 1].sum(-1) - 1.0) < 5e-3)
        alone = kit.align(pcm[b:b + 1], [seqs[b]])[0]
        assert _same(alone[0], allr[b][0]), b
        assert _same(alone[1], allr[b][1]), b
        assert np.isnan(allr[b][1][0]) and np.all(np.isfinite(allr[b][1][1:][np.array(seqs[b][1:]) < st_o.endToken]))


def test_large_v3_dims_64_windows_against_fp32_oracle():
    policy, W = "f16", 64
    dims = M.VARIANTS["large-v3"]
    w = M.random_weights(dims, seed=77, policy=policy)
    model = wk.Model("large-v3", max_batch=W, dtype=policy)
    model.load_state_dict(w)
    LV3 = D.SpecialTokens(endToken=50257, englishToken=50259, noSpeechToken=50363, noTimestampsToken=50364, specialTokenBegin=50257,
                          startOfPreviousToken=50362, startOfTranscriptToken=50258, timeTokenBegin=50365, transcribeToken=50360,
                          translateToken=50359)
    st = wk.SpecialTokens.from_any(LV3)
    pcm = np.stack([mel_ref.synthetic_pcm(900 + (i % 8)) for i in range(W)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, W)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    rng = np.random.default_rng(11)
    seqs = [make_seq(rng, [50258, 50259, 50360, 50364], 219, LV3) for _ in range(W)]
    assert all(len(s) == 224 for s in seqs)
    got = dec.alignTokens(enc_t, seqs, st)
    enc_gpu = enc_t.numpy()
    orc = M.WhisperOracle(dims, w, "fp32")
    heads = [(l, h) for l in range(dims.dec_layers // 2, dims.dec_layers) for h in range(dims.n_heads)]
    for b in (0, W - 1):
        rows, lp, scale = oracle_align(orc, enc_gpu[b], seqs[b], heads, LV3.endToken)
        row_err = max(rel_err(got[b][0][i + 1], rows[i]) for i in range(224))
        live = ~np.isnan(lp)
        lp_err = float((np.abs(got[b][1][live] - lp[live]) / np.maximum(scale[live], 1.0)).max())
        print(f"[large-v3/{policy} vs fp32 oracle] window {b}: alignment rows rel err {row_err:.2e}, log-prob err / max|logit| {lp_err:.2e}")
        assert np.array_equal(np.isnan(got[b][1]), ~live)
        assert row_err <= 2e-2 and lp_err <= 2e-3      # the f16 policy's own rounding is part of the difference (test_gpu_large.py: 2e-3)
    dec.close()
    model.close()


@pytest.mark.parametrize("policy", ["f16", "bf16"])
def test_fp8_cache_against_fp8_oracle(policy):
    B = 2
    dims, orc, model = build("toy128", policy, B, seed=21, fp8=True)
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    pcm = np.stack([mel_ref.synthetic_pcm(310 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    rng = np.random.default_rng(9)
    seqs = [make_seq(rng, dec.prefillDecoderInputs(wk.DecodingOptions(), st), n, st_o) for n in (9, 18)]
    heads = [(l, h) for l in range(dims.dec_layers // 2, dims.dec_layers) for h in range(dims.n_heads)]
    got = dec.alignTokens(enc_t, seqs, st)
    for b in range(B):
        check_against_oracle(f"fp8 window {b}", policy, got[b][0], got[b][1], seqs[b], *oracle_align(orc, enc_gpu[b], seqs[b], heads, st_o.endToken))
    dec.close()
    model.close()


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


def test_beam_search_results_get_word_timings():
    st_o = D.SpecialTokens.toy(1024)
    st = wk.SpecialTokens.from_any(st_o)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=8, seed=23, specialTokens=st))
    pcm = np.stack([mel_ref.synthetic_pcm(650 + i) for i in range(3)])
    o = wk.DecodingOptions(beamSize=4, firstTokenLogProbThreshold=None, sampleLength=16, temperatureFallbackCount=0)
    res = kit.transcribe(pcm, o)
    aligned = kit.align(pcm, [r.tokens for r in res])
    seeker = WordTimingSeeker()
    SB = st_o.specialTokenBegin
    for r, (weights, lps) in zip(res, aligned):
        assert weights.shape == (len(r.tokens) + 1, 1500) and lps.shape == (len(r.tokens),)
        seg = types.SimpleNamespace(id=0, seek=0, start=0.0, end=30.0, tokens=r.tokens, tokenLogProbs=list(np.nan_to_num(lps)))
        out = seeker.addWordTimestamps([seg], weights, lambda t: _toy_split(t, SB), 0, 0.0, SB,
                                       decode=lambda t: "".join(chr(97 + v % 26) for v in t))
        words = [w for _, _, ws in out for w in ws]
        assert words, r.tokens
        starts, ends = np.array([w.start for w in words]), np.array([w.end for w in words])
        assert np.all(np.diff(starts) >= 0) and np.all(np.diff(ends) >= 0) and np.all(ends >= starts)
        assert starts.min() >= 0.0 and ends.max() <= 30.0 + 1e-3


def test_invalid_sequences_fail_only_their_own_window():
    st_o = D.SpecialTokens.toy(1024)
    st = wk.SpecialTokens.from_any(st_o)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=29, specialTokens=st))
    pcm = np.stack([mel_ref.synthetic_pcm(660 + i) for i in range(5)])
    good = [st_o.startOfTranscriptToken, 5, 6, 7, st_o.endToken]
    seqs = [[], [5] * 225, [st_o.startOfTranscriptToken, 1024, st_o.endToken], good, good]
    out = kit.align(pcm, seqs, returnErrors=True)
    for i in range(3):
        assert isinstance(out[i], wk.WhisperError), i
    assert not isinstance(out[3], wk.WhisperError) and not isinstance(out[4], wk.WhisperError)
    alone = kit.align(pcm[3:4], [good])[0]
    assert _same(alone[0], out[3][0]) and _same(alone[1], out[3][1])
    with pytest.raises(wk.WhisperError):
        kit.align(pcm, seqs)
