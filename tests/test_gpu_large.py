"""Parity at the shapes bench.py times: whisper-large-v3 / large-v3-turbo / distil-large-v3 (d 1280, 20 heads, 32 encoder layers,
32 / 4 / 2 decoder layers, vocabulary 51866, 128 mels) with seeded weights, and the B = 64 lane shape.

  * log-mel <= 1e-3 against the oracle (128 mel bins);
  * encoder output and >= 8 teacher-forced decoder steps of logits against oracle.model_ref - against the oracle run under the same
    16-bit storage policy (the twin), and ALSO against the fp32 oracle on the same weights (no activation rounding at all), both
    printed.  north_star's tolerance for logits is 1e-3 relative: the f16 policy (the reference's own FloatType,
    ArgmaxCore/FloatType.swift:9-13) is held to it; bf16 (8 mantissa bits) is measured and held to the bound written below;
  * 24-step greedy token parity against the pure-CPU oracle loop (oracle.decode_ref), margin-gated as in test_gpu_pipeline.py, with
    the number of steps that were compared unconditionally asserted to be most of them;
  * a max_batch = 64 run whose rows 0 and 63 equal the same windows run alone.

The CPU side costs a few minutes (1.5 G parameters in fp32); everything is seeded."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402

LV3 = dict(endToken=50257, englishToken=50259, noSpeechToken=50363, noTimestampsToken=50364, specialTokenBegin=50257,
           startOfPreviousToken=50362, startOfTranscriptToken=50258, timeTokenBegin=50365, transcribeToken=50360, translateToken=50359)
# logits tolerance (relative to the row's largest |logit|): f16 is held to north_star's 1e-3.  bf16 cannot be: the 8-bit mantissa of every
# stored activation puts its error against the same-policy twin and the fp32 oracle at a few 1e-3, so its bound is wider (the test prints
# the measured errors).
TOL_TWIN = {"f16": 1e-3, "bf16": 7e-3}
TOL_FP32 = {"f16": 2e-3, "bf16": 1.5e-2}    # against the fp32 oracle: the storage policy's own rounding is part of the difference


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


_CACHE = {}


def weights_for(variant, policy):
    """Seeded weights of `variant`, rounded to `policy`; the 32-layer encoder is generated once per policy and shared by the three
    decoders (same seed, same order: the encoder comes first)."""
    key = (variant, policy)
    if key not in _CACHE:
        dims = M.VARIANTS[variant]
        enc_key = ("enc", policy)
        if enc_key not in _CACHE:
            w = M.random_weights(M.VARIANTS["large-v3"], seed=77, policy=policy)
            _CACHE[enc_key] = {k: v for k, v in w.items() if k.startswith("model.encoder.")}
            _CACHE[("large-v3", policy)] = w
        if key not in _CACHE:
            full = _CACHE[("large-v3", policy)]
            w = dict(_CACHE[enc_key])
            for k, v in full.items():
                if k.startswith("model.decoder.layers."):
                    if int(k.split(".")[3]) < dims.dec_layers:
                        w[k] = v
                elif not k.startswith("model.encoder."):
                    w[k] = v
            _CACHE[key] = w
    return M.VARIANTS[variant], _CACHE[key]


@pytest.fixture(scope="module")
def encoded():
    """mel + encoder parity once per policy (the encoder is common to the three checkpoints); hands the GPU encoder output on."""
    out = {}
    B = 2
    pcm = np.stack([mel_ref.synthetic_pcm(900 + i) for i in range(B)])
    for policy in ("bf16", "f16"):
        dims, w = weights_for("large-v3", policy)
        model = wk.Model("large-v3", max_batch=B, dtype=policy)
        model.load_state_dict(w)
        fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
        mel_t = fe.logMelSpectrogram(pcm)
        mel_gpu = mel_t.numpy()
        mel_o = np.stack([mel_ref.log_mel(x, dims.n_mels) for x in pcm])
        e_mel = rel_err(mel_gpu, mel_o)
        assert mel_gpu.shape == (B, 128, 3000) and e_mel <= 1e-3, e_mel
        enc_gpu = enc.encodeFeatures(mel_t).numpy()
        with torch.no_grad():
            twin = M.WhisperOracle(dims, w, policy).encode(torch.from_numpy(mel_gpu))
            e_twin = rel_err(enc_gpu, M.round_to(twin, policy).transpose(1, 2).numpy())
            full = M.WhisperOracle(dims, w, "fp32").encode(torch.from_numpy(mel_gpu))
            e_fp32 = rel_err(enc_gpu, full.transpose(1, 2).numpy())
        print(f"[large-v3 encoder/{policy}] log-mel rel err {e_mel:.2e}; encoder output vs same-policy oracle {e_twin:.2e}, vs fp32 oracle {e_fp32:.2e}")
        assert e_twin <= (2e-2 if policy == "bf16" else 3e-3), e_twin
        assert e_fp32 <= (6e-2 if policy == "bf16" else 1e-2), e_fp32
        out[policy] = (pcm, enc_gpu)
        model.close()
    return out


@pytest.mark.parametrize("variant", ["large-v3", "large-v3-turbo", "distil-large-v3"])
@pytest.mark.parametrize("policy", ["bf16", "f16"])
def test_logits_and_tokens_at_benchmarked_dims(encoded, variant, policy):
    B = 2
    dims, w = weights_for(variant, policy)
    pcm, _ = encoded[policy]
    model = wk.Model(variant, max_batch=B, dtype=policy)
    model.load_state_dict(w)
    info = model.info
    assert (info.d_model, info.n_heads, info.vocab, info.dec_layers, info.n_mels) == (1280, 20, 51866, dims.dec_layers, 128)
    fe, enc, dec, dec2 = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    orc, orc32 = M.WhisperOracle(dims, w, policy), M.WhisperOracle(dims, w, "fp32")
    st_o = D.SpecialTokens(**LV3)
    st = wk.SpecialTokens(**LV3)
    with torch.no_grad():
        enc_for_dec = torch.from_numpy(enc_gpu).transpose(1, 2).contiguous()
        cross, cross32 = orc.cross_kv(enc_for_dec), orc32.cross_kv(enc_for_dec)
        cache, cache32 = orc.new_cache(B), orc32.new_cache(B)
        dec.bindEncoderOutput(enc_t)
        dec.prepareDecoderInputs()
        rng = np.random.default_rng(1)
        worst, worst32 = 0.0, 0.0
        for pos in range(9):
            toks = rng.integers(0, dims.vocab, size=B)
            lg = dec.predictLogits(toks, [pos] * B)
            worst = max(worst, rel_err(lg, orc.decode_step(torch.from_numpy(toks), pos, cache, cross).numpy()))
            worst32 = max(worst32, rel_err(lg, orc32.decode_step(torch.from_numpy(toks), pos, cache32, cross32).numpy()))
    print(f"[{variant}/{policy}] 9 teacher-forced steps, logits rel err: vs same-policy oracle {worst:.2e} (tolerance {TOL_TWIN[policy]:.0e}), "
          f"vs fp32 oracle {worst32:.2e} (tolerance {TOL_FP32[policy]:.1e}); north_star's 1e-3 is {'met' if worst <= 1e-3 else 'NOT met'} by {policy}")
    assert worst <= TOL_TWIN[policy], worst
    assert worst32 <= TOL_FP32[policy], worst32
    # ---- 24-step greedy decode: device loop == reference loop on identical logits (bit-exact), and vs the pure-CPU oracle (margin-gated)
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=24)
    o_ref, o_gpu = D.DecodingOptions(**kw), wk.DecodingOptions(**kw)
    prompt = dec.prefillDecoderInputs(o_gpu, st)
    assert prompt == D.prefill_prompt(o_ref, st_o, True)
    res = dec.decodeText(enc_t, prompt, o_gpu, st)
    dec2.bindEncoderOutput(enc_t)
    compared, total = 0, 0
    for b in range(B):
        def predict_gpu(tok, idx):
            return dec2.predictLogits([tok] * B, [idx] * B)[b]
        ref_g = D.decode_text(predict_gpu, prompt, o_ref, st_o, True, keep_logits=True)
        assert res[b].tokens == ref_g.tokens and res[b].steps == ref_g.steps
        np.testing.assert_allclose(res[b].tokenLogProbs, ref_g.tokenLogProbs, atol=2e-4)
        with torch.no_grad():
            cross_b = orc.cross_kv(torch.from_numpy(enc_gpu[b:b + 1]).transpose(1, 2).contiguous())
            cache_b = orc.new_cache(1)

            def predict_cpu(tok, idx):
                return orc.decode_step(torch.tensor([tok]), idx, cache_b, cross_b)[0].numpy()
            ref = D.decode_text(predict_cpu, prompt, o_ref, st_o, True, keep_logits=True)
        scale = max(float(np.abs(l).max()) for l in ref.stepLogits)
        bound = TOL_TWIN[policy] * scale
        first = next((i for i, (x, y) in enumerate(zip(res[b].tokens, ref.tokens)) if x != y), None)
        n_steps = len(ref.stepMargins)
        clear = sum(1 for mg in ref.stepMargins if mg > 2 * bound)     # steps whose top-1 margin is outside the logit error bound
        upto = n_steps if first is None else max(first - 1, 0)
        compared += min(upto, n_steps)
        total += n_steps
        print(f"[{variant}/{policy}] window {b}: {n_steps} oracle steps, {clear} with a margin above 2x the logit bound ({bound:.1e}); "
              f"first token divergence at {first}")
        if first is not None:
            step = max(first - 1, 0)
            assert ref.stepMargins[min(step, n_steps - 1)] <= 2 * bound, (b, first, ref.stepMargins[step], bound)
    print(f"[{variant}/{policy}] token parity vs the pure-CPU oracle held unconditionally on {compared} of {total} decoder steps")
    assert compared >= total // 2
    for d_ in (dec, dec2):
        d_.close()
    model.close()


@pytest.mark.parametrize("policy", ["bf16"])
def test_batch64_rows_equal_the_same_windows_alone(policy):
    """The bench's lane shape: 64 windows through one session (Bp = 64 columns in every swap-AB GEMM, 1280 (b, h) attention streams).
    Windows are independent units, so rows 0 and 63 must equal the same windows transcribed alone, token for token."""
    B = 64
    model = wk.Model("large-v3", max_batch=B, dtype=policy)
    model.init_random(seed=5)
    st = wk.SpecialTokens(**LV3)
    kit_dec = wk.TextDecoder(model, B)
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    pcm = np.stack([mel_ref.synthetic_pcm(1000 + i) for i in range(B)]).astype(np.float32)
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=20, temperatureFallbackCount=0)
    prompt = kit_dec.prefillDecoderInputs(o, st)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    res = kit_dec.decodeText(enc_t, prompt, o, st)
    lg = kit_dec.lastLogits()
    assert all(r.steps == 20 or r.tokens[-1] == st.endToken for r in res)
    assert len({tuple(r.tokens) for r in res}) > 1            # different windows decode differently
    one = wk.TextDecoder(model, 1)
    for b in (0, 63):
        e1 = enc.encodeFeatures(fe.logMelSpectrogram(pcm[b:b + 1]))
        r1 = one.decodeText(e1, prompt, o, st)[0]
        assert r1.tokens == res[b].tokens, (b, r1.tokens, res[b].tokens)
        np.testing.assert_allclose(r1.tokenLogProbs, res[b].tokenLogProbs, atol=1e-5)
        if r1.steps == res[b].steps == 20:
            err = rel_err(one.lastLogits()[0], lg[b])
            print(f"row {b}: last-step logits, batch of 64 vs alone: rel err {err:.1e}")
            assert err <= 1e-6
    one.close()
    kit_dec.close()
    model.close()
