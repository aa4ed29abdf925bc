"""The FP8 (E4M3 + per-row f32 scale) cross-attention K/V cache on the H100: the two cross-attention kernels against torch fp32 on the
dequantized K/V (exact inputs: the same tolerances as the 16-bit kernel tests), the projection epilogue against the oracle's FP8 rounding
(tests/fp8_ref.py), end-to-end parity against the FP8-policy oracle (toy variants and large-v3 dimensions, teacher-forced logits, greedy
tokens, alignment-head rows), beam search against oracle/beam_ref.py on the GPU's logits, batch independence, and the policy setter.
Logits are held to the tolerances of the 16-bit end-to-end tests (test_gpu_pipeline.py, test_gpu_large.py)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from oracle import beam_ref as BR  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402
from tests import fp8_ref  # noqa: E402

LOGITS_TOL = {"bf16": 4e-3, "f16": 1e-3}   # the 16-bit end-to-end tolerances (test_gpu_pipeline.py): the FP8 oracle has the same rounding points

TD = {"bf16": (torch.bfloat16, _lib.WK_DTYPE_BF16), "f16": (torch.float16, _lib.WK_DTYPE_F16)}


@pytest.fixture(scope="module")
def toy():
    m = wk.Model("toy", max_batch=4)
    m.init_random(seed=3)
    yield m
    m.close()


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def quantized_kv(g, lead, H, T, peak=None):
    k = torch.randn(*lead, H, T, 64, device="cuda", generator=g) * 0.7
    v = torch.randn(*lead, H, T, 64, device="cuda", generator=g)
    if peak is not None:
        idx, row = peak
        k[idx] = row
    kc, ks = fp8_ref.quantize_rows(k)
    vc, vs = fp8_ref.quantize_rows(v)
    return kc.contiguous(), ks.contiguous(), vc.contiguous(), vs.contiguous()


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("B,H", [(64, 20), (3, 6), (1, 2)])
def test_fp8_cross_attention_kernel_vs_torch(toy, dt, B, H):
    tdt, wdt = TD[dt]
    T, dm = 1500, H * 64
    g = torch.Generator(device="cuda").manual_seed(B * 7 + H)
    q = torch.randn(B, dm, device="cuda", generator=g)
    peak = ((1, 0, 777), q[1, :64] * 3) if B > 2 else None
    kc, ks, vc, vs = quantized_kv(g, (B,), H, T, peak)
    out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
    align = torch.full((H, B, T), -1.0, device="cuda")
    done = torch.zeros(B, dtype=torch.int32, device="cuda")
    if B > 2:
        done[2] = 1
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_cross_attention_fp8(toy.handle, p(q), p(kc), p(vc), p(ks), p(vs), p(out), B, H, T, wdt, p(done), 1, p(align)))
    torch.cuda.synchronize()
    k, v = fp8_ref.dequantize_rows(kc, ks), fp8_ref.dequantize_rows(vc, vs)
    pr = torch.softmax(q.view(B, H, 1, 64) @ k.transpose(-1, -2) * 0.125, dim=-1)   # [B, H, 1, T]
    ref = (pr @ v).reshape(B, dm)
    live = done == 0
    got = out.float()
    err = (got[live] - ref[live]).abs().max().item()
    assert err <= (8e-3 if dt == "bf16" else 1e-3) * max(1.0, ref.abs().max().item()), err
    # the alignment export is the normalised softmax row itself (not p * v_scale)
    aref = pr[:, :, 0].transpose(0, 1)   # [H, B, T]
    aerr = (align[:, live] - aref[:, live]).abs().max().item()
    assert aerr <= 1e-5 * max(1.0, aref.abs().max().item()), aerr
    if B > 2:
        assert torch.all(got[2] == 7.0) and torch.all(align[:, 2] == -1.0)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("W,NQ,H,T", [(32, 5, 20, 1500), (3, 2, 6, 1500), (2, 8, 2, 250), (1, 3, 1, 1500)])
def test_fp8_cross_attention_beam_vs_torch(toy, dt, W, NQ, H, T):
    tdt, wdt = TD[dt]
    B, dm = W * NQ, H * 64
    g = torch.Generator(device="cuda").manual_seed(W * 31 + NQ * 7 + H)
    q = torch.randn(B, dm, device="cuda", generator=g)
    kc, ks, vc, vs = quantized_kv(g, (W,), H, T, ((0, 0, T - 3), q[1, :64] * 3))
    out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
    done = torch.zeros(B, dtype=torch.int32, device="cuda")
    if W > 2:
        done[2 * NQ:3 * NQ] = 1
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_cross_attention_fp8(toy.handle, p(q), p(kc), p(vc), p(ks), p(vs), p(out), B, H, T, wdt, p(done), NQ, None))
    torch.cuda.synchronize()
    k, v = fp8_ref.dequantize_rows(kc, ks), fp8_ref.dequantize_rows(vc, vs)
    qh = q.view(W, NQ, H, 64).transpose(1, 2)
    ref = (torch.softmax(qh @ k.transpose(-1, -2) * 0.125, dim=-1) @ v).transpose(1, 2).reshape(B, dm)
    live = done == 0
    got = out.float()
    err = (got[live] - ref[live]).abs().max().item()
    assert err <= (8e-3 if dt == "bf16" else 1e-3) * max(1.0, ref.abs().max().item()), err
    if W > 2:
        assert torch.all(got[2 * NQ:3 * NQ] == 7.0)
    if T % 500 == 0:
        # with the alignment export the grouped rows go through the single-query kernel (kv_div > 1): same output, softmax rows exported
        out2 = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
        align = torch.full((H, B, T), -1.0, device="cuda")
        torch.cuda.synchronize()
        _lib.check(toy.lib.wk_test_cross_attention_fp8(toy.handle, p(q), p(kc), p(vc), p(ks), p(vs), p(out2), B, H, T, wdt, p(done), NQ, p(align)))
        torch.cuda.synchronize()
        err2 = (out2.float()[live] - ref[live]).abs().max().item()
        assert err2 <= (8e-3 if dt == "bf16" else 1e-3) * max(1.0, ref.abs().max().item()), err2
        pr = torch.softmax(qh @ k.transpose(-1, -2) * 0.125, dim=-1)          # [W, H, NQ, T]
        aref = pr.permute(1, 0, 2, 3).reshape(H, B, T)
        assert (align[:, live] - aref[:, live]).abs().max().item() <= 1e-5
        if W > 2:
            assert torch.all(align[:, 2 * NQ:3 * NQ] == -1.0)


def build(variant, policy, B, seed=5, crossKVDtype="fp8"):
    dims = M.VARIANTS[variant]
    w = M.random_weights(dims, seed=seed, policy=policy)
    orc = fp8_ref.FP8CrossKVOracle(dims, w, policy)
    model = wk.Model(variant, max_batch=B, dtype=policy, crossKVDtype=crossKVDtype)
    model.load_state_dict(w)
    return dims, orc, model


@pytest.mark.parametrize("variant,policy", [("toy", "bf16"), ("toy128", "f16"), ("toy128", "bf16")])
def test_fp8_projection_readback_matches_oracle(variant, policy):
    B = 3
    dims, orc, model = build(variant, policy, B)
    assert model.info.cross_kv_dtype == _lib.WK_DTYPE_FP8_E4M3
    pcm = np.stack([mel_ref.synthetic_pcm(30 + i) for i in range(B)])
    enc_t = wk.AudioEncoder(model).encodeFeatures(wk.FeatureExtractor(model).logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    dec = wk.TextDecoder(model, B)
    dec.bindEncoderOutput(enc_t)
    L, H, T = dims.dec_layers, dims.n_heads, dims.n_audio_ctx
    n = 2 * L * B * H * T * 64
    got = np.empty(n, np.float32)
    _lib.check(model.lib.wk_debug_read(model.handle, dec.handle, 15, 0, got.ctypes.data_as(C.c_void_p), n))
    got = got.reshape(L, 2, B, H, T, 64)
    enc_for_dec = torch.from_numpy(enc_gpu).transpose(1, 2).contiguous()
    worst_step, worst_scale = 0.0, 0.0
    with torch.no_grad():
        encr = orc.r(enc_for_dec)
        for i in range(L):
            for j, name in enumerate(("k_proj", "v_proj")):
                x = orc._heads(orc._lin(encr, f"model.decoder.layers.{i}.encoder_attn.{name}"))   # [B, H, T, 64] f32
                codes, s = fp8_ref.quantize_rows(x)
                ref = fp8_ref.dequantize_rows(codes, s).numpy()
                g = got[i, j]
                # one E4M3 step at the reference value: 2^-3 relative for normals, 2^-9 * s in the subnormal range
                step = np.maximum(np.abs(ref) * 2.0 ** -3, s.numpy()[..., None] * 2.0 ** -9)
                worst_step = max(worst_step, float((np.abs(g - ref) / step).max()))
                gs = np.abs(g).max(-1) / 448.0            # the scale the engine used, recovered from its largest code (448 * s)
                worst_scale = max(worst_scale, float((np.abs(gs - s.numpy()) / np.maximum(s.numpy(), 1e-30)).max()))
    print(f"[{variant}/{policy}] FP8 cross K/V: max |diff| / E4M3 step {worst_step:.3f}, scale rel diff {worst_scale:.2e}")
    assert worst_step <= 1.0 + 1e-3
    assert worst_scale <= 1e-5
    dec.close()
    model.close()


@pytest.mark.parametrize("variant,policy", [("toy", "bf16"), ("toy128", "f16"), ("toy128", "bf16")])
def test_fp8_logits_and_greedy_tokens_vs_fp8_oracle(variant, policy):
    B = 3
    dims, orc, model = build(variant, policy, B, seed=11)
    pcm = np.stack([mel_ref.synthetic_pcm(10 + i) for i in range(B)])
    fe, enc, dec, dec2 = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    with torch.no_grad():
        cross = orc.cross_kv(torch.from_numpy(enc_gpu).transpose(1, 2).contiguous())
        cache = orc.new_cache(B)
        dec.bindEncoderOutput(enc_t)
        dec.prepareDecoderInputs()
        rng = np.random.default_rng(0)
        worst = 0.0
        for pos in range(6):
            toks = rng.integers(0, dims.vocab, size=B)
            worst = max(worst, rel_err(dec.predictLogits(toks, [pos] * B), orc.decode_step(torch.from_numpy(toks), pos, cache, cross).numpy()))
    print(f"[{variant}/{policy}] FP8 logits rel err vs FP8 oracle {worst:.2e} (tolerance {LOGITS_TOL[policy]:.0e})")
    assert worst <= LOGITS_TOL[policy], worst
    # greedy decode: the device loop on the FP8 cache equals the reference loop semantics on the same decoder's logits, and the oracle's
    # own greedy tokens wherever its smallest top-1 margin exceeds 20x the measured logit error
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=40, suppressTokens=[1, 2], suppressBlank=True)
    o_ref, o_gpu = D.DecodingOptions(**kw), wk.DecodingOptions(**kw)
    prompt = dec.prefillDecoderInputs(o_gpu, st)
    res = dec.decodeText(enc_t, prompt, o_gpu, st)
    dec2.bindEncoderOutput(enc_t)
    for b in range(B):
        ref_g = D.decode_text(lambda tok, idx: dec2.predictLogits([tok] * B, [idx] * B)[b], prompt, o_ref, st_o, True, keep_logits=True)
        assert res[b].tokens == ref_g.tokens, (b, res[b].tokens, ref_g.tokens)
        with torch.no_grad():
            cr = orc.cross_kv(torch.from_numpy(enc_gpu[b:b + 1]).transpose(1, 2).contiguous())
            cc = orc.new_cache(1)
            ref_o = D.decode_text(lambda tok, idx: orc.decode_step(torch.tensor([tok]), idx, cc, cr)[0].numpy(), prompt, o_ref, st_o, True,
                                  keep_logits=True)
        # identical to the FP8-policy oracle until the first step whose top-1 margin is inside the measured logit error (the rule of
        # test_gpu_pipeline.test_decode_text_token_parity)
        bound = LOGITS_TOL[policy] * max(float(np.abs(lg).max()) for lg in ref_o.stepLogits)
        first = next((i for i, (x, y) in enumerate(zip(res[b].tokens, ref_o.tokens)) if x != y), None)
        if first is None and len(res[b].tokens) != len(ref_o.tokens):
            first = min(len(res[b].tokens), len(ref_o.tokens))
        print(f"[{variant}/{policy}] seq {b}: min top-1 margin {min(ref_o.stepMargins):.2e}, logit bound {bound:.1e}, first divergence {first}")
        if first is not None:
            step = max(first - 1, 0)
            assert ref_o.stepMargins[min(step, len(ref_o.stepMargins) - 1)] <= 2 * bound, (b, first, bound)
    dec.close(); dec2.close()
    model.close()


def test_fp8_batch_of_64_windows_equals_each_window_alone():
    dims = M.VARIANTS["toy"]
    w = M.random_weights(dims, seed=2, policy="bf16")
    model = wk.Model("toy", max_batch=64, dtype="bf16", crossKVDtype="fp8")
    model.load_state_dict(w)
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(dims.vocab))
    opts = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=24)
    pcm = np.stack([mel_ref.synthetic_pcm(100 + i) for i in range(64)])
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    dec = wk.TextDecoder(model, 64)
    prompt = dec.prefillDecoderInputs(opts, st)
    batch = dec.decodeText(enc_t, prompt, opts, st)
    one = wk.TextDecoder(model, 1)
    for b in range(64):
        e1 = enc.encodeFeatures(fe.logMelSpectrogram(pcm[b:b + 1]))
        r1 = one.decodeText(e1, prompt, opts, st)[0]
        assert r1.tokens == batch[b].tokens, b
    one.close(); dec.close()
    model.close()


def test_cross_kv_dtype_setter():
    m = wk.Model("toy", max_batch=2, dtype="bf16")
    m.init_random(seed=1)
    assert m.info.cross_kv_dtype == _lib.WK_DTYPE_BF16           # never set: the model's 16-bit dtype
    assert m.lib.wk_model_set_cross_kv_dtype(m.handle, _lib.WK_DTYPE_F32) == -1
    assert m.lib.wk_model_set_cross_kv_dtype(m.handle, 99) == -1
    assert m.lib.wk_model_set_cross_kv_dtype(m.handle, _lib.WK_DTYPE_FP8_E4M3) == 0
    assert m.info.cross_kv_dtype == _lib.WK_DTYPE_FP8_E4M3
    assert m.lib.wk_model_set_cross_kv_dtype(m.handle, _lib.WK_DTYPE_BF16) == 0   # its own dtype: back to the default
    assert m.info.cross_kv_dtype == _lib.WK_DTYPE_BF16
    dec = wk.TextDecoder(m, 2)
    assert m.lib.wk_model_set_cross_kv_dtype(m.handle, _lib.WK_DTYPE_FP8_E4M3) == -1   # a session exists
    dec.close()
    assert m.lib.wk_model_set_cross_kv_dtype(m.handle, _lib.WK_DTYPE_FP8_E4M3) == -1   # ... or existed
    assert m.info.cross_kv_dtype == _lib.WK_DTYPE_BF16
    m.close()
    with pytest.raises(ValueError):
        wk.Model("toy", max_batch=2, crossKVDtype="int8")


@pytest.mark.parametrize("policy", ["f16", "bf16"])
def test_fp8_alignment_heads_rows_vs_fp8_oracle(policy):
    """wordTimestamps on an FP8 session: the alignmentWeights rows (the FP8 kernel's softmax export, averaged) against the FP8-policy oracle
    teacher-forced on the GPU's tokens, with the tolerances of test_gpu_pipeline.test_alignment_heads_weights_parity."""
    B = 3
    dims, orc, model = build("toy128", policy, B, seed=21)
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    pcm = np.stack([mel_ref.synthetic_pcm(300 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    for heads in ([], [(0, 1), (1, 0), (1, 3)]):
        model.setAlignmentHeads(heads)
        ref_heads = heads or [(l, h) for l in range(dims.dec_layers // 2, dims.dec_layers) for h in range(dims.n_heads)]
        o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12, wordTimestamps=True)
        prompt = dec.prefillDecoderInputs(o, st)
        res = dec.decodeText(enc_t, prompt, o, st)
        with torch.no_grad():
            for b in range(B):
                toks, steps = res[b].tokens, res[b].steps
                a = dec.alignmentWeights(b, 224)
                assert np.all(a[0] == 0) and np.all(a[steps + 1:] == 0)
                written = steps if a[steps].any() else steps - 1
                assert written >= 3
                cross = orc.cross_kv(torch.from_numpy(enc_gpu[b:b + 1]).transpose(1, 2).contiguous())
                cache = orc.new_cache(1)
                worst = 0.0
                for i in range(written):
                    _, al = orc.decode_step(torch.tensor([toks[i]]), i, cache, cross, align_heads=ref_heads)
                    worst = max(worst, rel_err(a[i + 1], al[0].numpy()))
                    assert abs(float(a[i + 1].sum()) - 1.0) < 5e-3
                print(f"[fp8/{policy}] alignment rows rel err vs FP8 oracle {worst:.2e}")
                assert worst <= (2e-2 if policy == "bf16" else 4e-3), worst
    dec.close()
    model.close()


@pytest.mark.parametrize("variant,policy,beam,patience", [("toy128", "f16", 5, 1.0), ("toy", "bf16", 3, 2.0)])
def test_fp8_beam_search_matches_beam_oracle_on_gpu_logits(variant, policy, beam, patience):
    """Beam search on an FP8 session (the beam rows of a window read one FP8 K/V block through the beam kernel) against oracle/beam_ref.py
    fed the same FP8 model's logits for explicit prefixes (single-query kernel), as test_gpu_beam.py does for the 16-bit cache."""
    vocab = 1024 if variant == "toy" else 2048
    st_o = D.SpecialTokens.toy(vocab)
    st = wk.SpecialTokens.from_any(st_o)
    n_win = 3
    kit = wk.WhisperKit(wk.WhisperKitConfig(model=variant, maxBatch=2 * beam, seed=17, specialTokens=st, dtype=policy, crossKVDtype="fp8"))
    assert kit.model.info.cross_kv_dtype == _lib.WK_DTYPE_FP8_E4M3
    pcm = np.stack([mel_ref.synthetic_pcm(600 + i) for i in range(n_win)])
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=22, temperatureFallbackCount=0, logProbThreshold=None, compressionRatioThreshold=None)
    o_gpu = wk.DecodingOptions(beamSize=beam, beamPatience=patience, **kw)
    o_ref = D.DecodingOptions(**kw)
    res = kit.transcribe(pcm, o_gpu)
    prompt = kit.textDecoder.prefillDecoderInputs(o_gpu, st)
    fe, enc = wk.FeatureExtractor(kit.model), wk.AudioEncoder(kit.model)
    for b in range(n_win):
        dec = wk.TextDecoder(kit.model, beam)
        dec.bindEncoderOutput(enc.encodeFeatures(fe.logMelSpectrogram(np.repeat(pcm[b][None], beam, axis=0))))

        def predict(prefixes, tokenIndex):
            lg = None
            for t in range(tokenIndex + 1):
                lg = dec.predictLogits([pp[t] for pp in prefixes], [t] * beam)
            return lg
        ref = BR.decode_text_beam(predict, prompt, o_ref, st_o, True, beam, patience)
        dec.close()
        assert res[b].tokens == ref.tokens, (b, res[b].tokens, ref.tokens)
        atol = 2e-3 if policy == "bf16" else 5e-4
        np.testing.assert_allclose(res[b].tokenLogProbs, ref.tokenLogProbs, atol=atol)
        assert abs(res[b].avgLogProb - ref.avgLogProb) < atol and res[b].steps == ref.steps


def test_fp8_teacher_forced_logits_at_large_v3_dims():
    """large-v3 (d 1280, 20 heads, 32 decoder layers, vocabulary 51866) with seeded bf16 weights and the FP8 cache: 9 teacher-forced
    steps against the FP8-policy oracle fed the GPU's encoder output, held to test_gpu_large.py's same-policy bf16 tolerance."""
    B = 2
    dims = M.VARIANTS["large-v3"]
    w = M.random_weights(dims, seed=77, policy="bf16")
    model = wk.Model("large-v3", max_batch=B, dtype="bf16", crossKVDtype="fp8")
    model.load_state_dict(w)
    pcm = np.stack([mel_ref.synthetic_pcm(900 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    orc = fp8_ref.FP8CrossKVOracle(dims, w, "bf16")
    with torch.no_grad():
        cross = orc.cross_kv(torch.from_numpy(enc_gpu).transpose(1, 2).contiguous())
        cache = orc.new_cache(B)
        dec.bindEncoderOutput(enc_t)
        dec.prepareDecoderInputs()
        rng = np.random.default_rng(1)
        worst = 0.0
        for pos in range(9):
            toks = rng.integers(0, dims.vocab, size=B)
            worst = max(worst, rel_err(dec.predictLogits(toks, [pos] * B), orc.decode_step(torch.from_numpy(toks), pos, cache, cross).numpy()))
    print(f"[large-v3/bf16 + fp8 cross K/V] 9 teacher-forced steps, logits rel err vs FP8-policy oracle {worst:.2e} (tolerance 7e-3)")
    assert worst <= 7e-3, worst
    dec.close()
    model.close()
