"""The FP8 (E4M3) encoder policy on the H100 (wk_model_set_encoder_dtype): the three FP8 GEMM modes against an fp32 matmul of the
dequantized operands (exact inputs: the tolerance is the f32 accumulation's plus the output's own rounding), FC1's output codes and scales
against the oracle's quantization of its own f32 result, the encoder against the FP8-policy oracle (tests/encoder_fp8_ref.py) with the
distance to the 16-bit oracle printed as the cost of the policy, teacher-forced logits and greedy tokens, batch independence, the
composition with the FP8 cross-K/V cache, and the setter."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402
from tests import encoder_fp8_ref as E  # noqa: E402
from whisperkit_b200.longform import transcribe_audio  # noqa: E402

TD = {"bf16": (torch.bfloat16, _lib.WK_DTYPE_BF16), "f16": (torch.float16, _lib.WK_DTYPE_F16)}
# engine encoder output against the FP8-policy oracle (max |diff| / max |ref|): both round to E4M3 at the same points, but an f32 sum that
# differs in its last bits may land on the other side of an E4M3 rounding boundary (one step is 2^-3 relative), so the bound is wider than
# the 16-bit encoder's
ENC_TOL = 1.5e-2
LOGITS_TOL = 1.5e-2
# The tensor cores add the E4M3 products of a k-block at less than f32 precision before the promotion into the f32 accumulator (measured:
# 7-8e-4 of max |result| at K = 5120 against an fp32 matmul of the same operands); the FP8 GEMM tests allow for it
FP8_ACC_TOL = 2e-3


@pytest.fixture(scope="module")
def toy():
    m = wk.Model("toy", max_batch=2)
    m.init_random(seed=3)
    yield m
    m.close()


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def scale_layout(scales, M):
    """[M, K / 128] -> the kernel's k-block-major [K / 128][round_up(M, 128)] (padding rows zero)."""
    ld = (M + 127) // 128 * 128
    out = torch.zeros(scales.shape[1], ld, device=scales.device)
    out[:, :M] = scales.T
    return out.contiguous()


SHAPES = {   # (N, K) of each kind: QKV, FC1, FC2
    "large-v3": {0: (3840, 1280), 1: (5120, 1280), 2: (1280, 5120)},
    "tiny": {0: (1152, 384), 1: (1536, 384), 2: (384, 1536)},
}


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("dims,windows,dt", [("large-v3", 1, "bf16"), ("large-v3", 37, "bf16"), ("large-v3", 64, "bf16"),
                                             ("tiny", 2, "bf16"), ("tiny", 3, "f16")])
def test_fp8_gemm_vs_fp32_matmul(toy, kind, dims, windows, dt):
    tdt, wdt = TD[dt]
    N, K = SHAPES[dims][kind]
    Mr = windows * 1500
    g = torch.Generator(device="cuda").manual_seed(kind * 100 + windows)
    x = torch.randn(Mr, K, device="cuda", generator=g)
    x[5, :128] = 0.0                                          # an all-zero block: s = 0
    if Mr > 40:
        x[37, 3] = 200.0                                      # an outlier that pushes the rest of its block into E4M3 subnormals
    ac, asc = E.quantize_blocks(x)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).to(tdt).float()
    wc, ws = E.quantize_weight(w)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    ref = (ac.view(torch.float8_e4m3fn).float() * asc.repeat_interleave(128, 1)) @ (wc.view(torch.float8_e4m3fn).float() * ws[:, None]).T
    ref = ref + bias
    a_scale = scale_layout(asc, Mr)
    out_scale = torch.full((N // 128, a_scale.shape[1]), -1.0, device="cuda") if kind == 1 else None
    if kind == 0:
        out = torch.zeros(Mr, N, device="cuda", dtype=tdt)
    elif kind == 1:
        out = torch.zeros(Mr, N, device="cuda", dtype=torch.uint8)
    else:
        res = torch.randn(Mr, N, device="cuda", generator=g)
        out = res.clone()
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_gemm_fp8(toy.handle, kind, p(ac), p(a_scale), p(wc), p(ws), p(bias), p(out), p(out_scale), Mr, N, K, wdt))
    torch.cuda.synchronize()
    if kind == 0:
        err = rel_err(out.float().cpu(), ref.cpu())
        tol = 5e-3 if dt == "bf16" else 1e-3   # the 16-bit output's own rounding (8 / 11 mantissa bits) over the f32 accumulation's
    elif kind == 2:
        err = rel_err((out - res).cpu(), ref.cpu())
        tol = FP8_ACC_TOL
    else:
        h = torch.nn.functional.gelu(ref)
        rc, rs = E.quantize_blocks(h)
        gs = out_scale[:, :Mr].T
        sc_err = float(((gs - rs).abs() / rs.clamp_min(1e-30)).max())
        got = out.view(torch.float8_e4m3fn).float() * gs.repeat_interleave(128, 1)
        r = rc.view(torch.float8_e4m3fn).float() * rs.repeat_interleave(128, 1)
        # one E4M3 step at the reference value (2^-3 relative for normals, 2^-9 * s in the subnormal range), beyond the accumulation's
        # own error in the f32 value that was quantized
        step = torch.maximum(r.abs() * 2.0 ** -3, rs.repeat_interleave(128, 1) * 2.0 ** -9)
        acc = FP8_ACC_TOL * h.abs().amax(1, keepdim=True)
        err = float((((got - r).abs() - acc).clamp_min(0) / step).max())
        print(f"[FP8 GEMM kind 1 {dims} x{windows} {dt}] max |diff| / E4M3 step {err:.3f}, scale rel diff {sc_err:.2e}, "
              f"codes equal {(out == rc).float().mean().item():.5f}")
        assert sc_err <= 2 * FP8_ACC_TOL, sc_err
        assert torch.all(out_scale[:, Mr:] == -1.0)           # rows past M are not written
        tol = 1.0 + 1e-3
    print(f"[FP8 GEMM kind {kind} {dims} x{windows} {dt}] err {err:.3e} (tolerance {tol:.1e})")
    assert err <= tol, err


def build(variant, policy, B, seed=5, crossKVDtype=None):
    dims = M.VARIANTS[variant]
    w = M.random_weights(dims, seed=seed, policy=policy)
    orc = (E.FP8EncoderCrossKVOracle if crossKVDtype == "fp8" else E.FP8EncoderOracle)(dims, w, policy)
    model = wk.Model(variant, max_batch=B, dtype=policy, encoderDtype="fp8", crossKVDtype=crossKVDtype)
    model.load_state_dict(w)
    return dims, w, orc, model


def encode_both(model, pcm):
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    mel = fe.logMelSpectrogram(pcm)
    mel_np = mel.numpy()
    enc_t = enc.encodeFeatures(mel)
    return mel_np, enc_t


@pytest.mark.parametrize("variant,policy", [("toy", "bf16"), ("toy", "f16"), ("toy128", "bf16"), ("toy128", "f16")])
def test_fp8_encoder_vs_fp8_oracle(variant, policy):
    B = 2
    dims, w, orc, model = build(variant, policy, B)
    enc_dtype = C.c_int32()
    _lib.check(model.lib.wk_model_encoder_dtype(model.handle, C.byref(enc_dtype)))
    assert enc_dtype.value == _lib.WK_DTYPE_FP8_E4M3
    pcm = np.stack([mel_ref.synthetic_pcm(40 + i) for i in range(B)])
    mel_np, enc_t = encode_both(model, pcm)
    got = enc_t.numpy()                                   # [B, d, 1500]
    with torch.no_grad():
        mel = torch.from_numpy(mel_np)
        ref = orc.encode(mel).transpose(1, 2).numpy()
        ref16 = M.WhisperOracle(dims, w, policy).encode(mel).transpose(1, 2).numpy()
    err, cost = rel_err(got, ref), rel_err(got, ref16)
    print(f"[{variant}/{policy}] FP8 encoder output: rel err vs FP8 oracle {err:.2e} (tolerance {ENC_TOL:.1e}); "
          f"distance to the 16-bit oracle (cost of the policy) {cost:.2e}; FP8 oracle vs 16-bit oracle {rel_err(ref, ref16):.2e}")
    assert err <= ENC_TOL, err
    model.close()


def test_fp8_encoder_large_v3_dims_two_windows():
    dims = M.VARIANTS["large-v3"]
    w = M.random_weights(dims, seed=77, policy="bf16")
    model = wk.Model("large-v3", max_batch=2, dtype="bf16", encoderDtype="fp8")
    model.load_state_dict(w)
    pcm = np.stack([mel_ref.synthetic_pcm(3), mel_ref.synthetic_pcm(4)])
    mel_np, enc_t = encode_both(model, pcm)
    got = enc_t.numpy()
    model.close()
    wc = {k: v.cuda() for k, v in w.items()}   # the oracle runs on the device in f32 (32 layers x 3000 rows)
    with torch.no_grad():
        mel = torch.from_numpy(mel_np).cuda()
        ref = E.FP8EncoderOracle(dims, wc, "bf16").encode(mel).transpose(1, 2).cpu().numpy()
        ref16 = M.WhisperOracle(dims, wc, "bf16").encode(mel).transpose(1, 2).cpu().numpy()
    err, cost = rel_err(got, ref), rel_err(got, ref16)
    print(f"[large-v3 dims, 2 windows, bf16] FP8 encoder rel err vs FP8 oracle {err:.2e}; distance to the 16-bit oracle {cost:.2e}; "
          f"FP8 oracle vs 16-bit oracle {rel_err(ref, ref16):.2e}")
    # 32 layers amplify the E4M3 rounding-boundary flips (measured 6.3e-2 against a policy cost of 8.8e-2 on an H100); the engine must still
    # be nearer the FP8 oracle than the 16-bit one
    assert err <= 1e-1 and err < cost, (err, cost)


@pytest.mark.parametrize("variant,policy,ckv", [("toy", "bf16", None), ("toy128", "f16", None), ("toy128", "bf16", "fp8")])
def test_fp8_encoder_logits_and_greedy_tokens(variant, policy, ckv):
    B = 3
    dims, w, orc, model = build(variant, policy, B, seed=11, crossKVDtype=ckv)
    pcm = np.stack([mel_ref.synthetic_pcm(10 + i) for i in range(B)])
    mel_np, enc_t = encode_both(model, pcm)
    dec = wk.TextDecoder(model, B)
    with torch.no_grad():
        enc_ref = orc.encode(torch.from_numpy(mel_np))
        cross = orc.cross_kv(enc_ref)
        cache = orc.new_cache(B)
        dec.bindEncoderOutput(enc_t)
        dec.prepareDecoderInputs()
        rng = np.random.default_rng(0)
        worst = 0.0
        for pos in range(6):
            toks = rng.integers(0, dims.vocab, size=B)
            worst = max(worst, rel_err(dec.predictLogits(toks, [pos] * B), orc.decode_step(torch.from_numpy(toks), pos, cache, cross).numpy()))
    print(f"[{variant}/{policy}/ckv={ckv}] teacher-forced logits rel err vs the FP8-encoder oracle {worst:.2e} (tolerance {LOGITS_TOL:.1e})")
    assert worst <= LOGITS_TOL, worst
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=40, suppressTokens=[1, 2], suppressBlank=True)
    o_ref, o_gpu = D.DecodingOptions(**kw), wk.DecodingOptions(**kw)
    prompt = dec.prefillDecoderInputs(o_gpu, st)
    res = dec.decodeText(enc_t, prompt, o_gpu, st)
    for b in range(B):
        with torch.no_grad():
            cr = orc.cross_kv(enc_ref[b:b + 1])
            cc = orc.new_cache(1)
            ref_o = D.decode_text(lambda tok, idx: orc.decode_step(torch.tensor([tok]), idx, cc, cr)[0].numpy(), prompt, o_ref, st_o, True,
                                  keep_logits=True)
        # identical to the oracle until the first step whose top-1 margin is inside the measured logit error (test_gpu_pipeline's rule)
        bound = LOGITS_TOL * max(float(np.abs(lg).max()) for lg in ref_o.stepLogits)
        first = next((i for i, (x, y) in enumerate(zip(res[b].tokens, ref_o.tokens)) if x != y), None)
        if first is None and len(res[b].tokens) != len(ref_o.tokens):
            first = min(len(res[b].tokens), len(ref_o.tokens))
        print(f"[{variant}/{policy}/ckv={ckv}] seq {b}: min top-1 margin {min(ref_o.stepMargins):.2e}, bound {bound:.1e}, first divergence {first}")
        if first is not None:
            step = max(first - 1, 0)
            assert ref_o.stepMargins[min(step, len(ref_o.stepMargins) - 1)] <= 2 * bound, (b, first, bound)
    dec.close()
    model.close()


def test_fp8_encoder_64_windows_equal_each_window_alone():
    dims = M.VARIANTS["toy"]
    w = M.random_weights(dims, seed=2, policy="bf16")
    model = wk.Model("toy", max_batch=64, dtype="bf16", encoderDtype="fp8")
    model.load_state_dict(w)
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(dims.vocab))
    opts = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=24)
    pcm = np.stack([mel_ref.synthetic_pcm(100 + i) for i in range(64)])
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_all = enc_t.numpy()
    dec = wk.TextDecoder(model, 64)
    prompt = dec.prefillDecoderInputs(opts, st)
    batch = dec.decodeText(enc_t, prompt, opts, st)
    one = wk.TextDecoder(model, 1)
    for b in range(64):
        e1 = enc.encodeFeatures(fe.logMelSpectrogram(pcm[b:b + 1]))
        assert np.array_equal(e1.numpy()[0], enc_all[b]), b      # the same bits: every scale comes from its own row
        r1 = one.decodeText(e1, prompt, opts, st)[0]
        assert r1.tokens == batch[b].tokens, b
    one.close(); dec.close()
    model.close()


def test_fp8_encoder_transcribe_paths_use_the_policy():
    """The window scheduler (greedy, beam search, word timestamps), the alignment pass and a long-form run on an FP8-encoder model, alone
    and with the FP8 cross-K/V cache: every path runs with the policy in place."""
    dims = M.VARIANTS["toy"]
    w = M.random_weights(dims, seed=9, policy="bf16")
    st_o = D.SpecialTokens.toy(dims.vocab)
    pcm = np.stack([mel_ref.synthetic_pcm(200 + i) for i in range(3)])
    for ckv in (None, "fp8"):
        pipe = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, weights=w, crossKVDtype=ckv, encoderDtype="fp8",
                                                 specialTokens=wk.SpecialTokens.from_any(st_o)))
        enc_dtype = C.c_int32()
        _lib.check(pipe.model.lib.wk_model_encoder_dtype(pipe.model.handle, C.byref(enc_dtype)))
        assert enc_dtype.value == _lib.WK_DTYPE_FP8_E4M3
        for kw in (dict(), dict(beamSize=3), dict(wordTimestamps=True)):
            opts = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=16, temperatureFallbackCount=0, **kw)
            out = pipe.transcribe(pcm, opts)
            assert len(out) == 3
        pipe.align(pcm, [[st_o.startOfTranscriptToken, 5, 6, 7], [st_o.startOfTranscriptToken, 9]] + [[st_o.startOfTranscriptToken]])
        long_pcm = np.concatenate([pcm[0], pcm[1][:240000]])   # 45 s: two seek windows
        transcribe_audio(pipe, [long_pcm], wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=16, temperatureFallbackCount=0))
        pipe.model.close()


def test_encoder_dtype_setter_and_default_path():
    m = wk.Model("toy", max_batch=2, dtype="bf16")
    m.init_random(seed=1)
    d = C.c_int32()
    _lib.check(m.lib.wk_model_encoder_dtype(m.handle, C.byref(d)))
    assert d.value == _lib.WK_DTYPE_BF16                              # never set: the model's 16-bit dtype
    pcm = np.stack([mel_ref.synthetic_pcm(1)])
    fe, enc = wk.FeatureExtractor(m), wk.AudioEncoder(m)
    mel = fe.logMelSpectrogram(pcm)
    assert m.lib.wk_model_set_encoder_dtype(m.handle, _lib.WK_DTYPE_F32) == -1
    assert m.lib.wk_model_set_encoder_dtype(m.handle, _lib.WK_DTYPE_F16) == -1   # not the model's dtype
    assert m.lib.wk_model_set_encoder_dtype(m.handle, 99) == -1
    assert m.lib.wk_model_set_encoder_dtype(m.handle, _lib.WK_DTYPE_FP8_E4M3) == 0
    assert m.lib.wk_model_set_encoder_dtype(m.handle, _lib.WK_DTYPE_BF16) == 0   # back to the default before any encode
    # the default path runs the 16-bit encoder kernels: no FP8 GEMM, the same bits as a model that never touched the setter
    e_default = enc.encodeFeatures(mel).numpy()
    assert m.lib.wk_model_set_encoder_dtype(m.handle, _lib.WK_DTYPE_FP8_E4M3) == -1   # wk_encode has run
    m2 = wk.Model("toy", max_batch=2, dtype="bf16")
    m2.init_random(seed=1)
    e_never = wk.AudioEncoder(m2).encodeFeatures(wk.FeatureExtractor(m2).logMelSpectrogram(pcm)).numpy()
    assert np.array_equal(e_default, e_never)
    dec = wk.TextDecoder(m2, 1)
    assert m2.lib.wk_model_set_encoder_dtype(m2.handle, _lib.WK_DTYPE_FP8_E4M3) == -1   # a session exists
    dec.close()
    m2.close()
    m.close()
    # an FP8 model set before the weights: load_state_dict / init_random requantize, so the result equals setting it after
    w = M.random_weights(M.VARIANTS["toy"], seed=4, policy="bf16")
    a = wk.Model("toy", max_batch=1, dtype="bf16", encoderDtype="fp8")
    a.load_state_dict(w)
    b = wk.Model("toy", max_batch=1, dtype="bf16")
    b.load_state_dict(w)
    _lib.check(b.lib.wk_model_set_encoder_dtype(b.handle, _lib.WK_DTYPE_FP8_E4M3))
    ea = wk.AudioEncoder(a).encodeFeatures(wk.FeatureExtractor(a).logMelSpectrogram(pcm)).numpy()
    eb = wk.AudioEncoder(b).encodeFeatures(wk.FeatureExtractor(b).logMelSpectrogram(pcm)).numpy()
    assert np.array_equal(ea, eb)
    a.close(); b.close()
