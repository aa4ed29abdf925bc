"""Kernel-level parity tests on the H100 (through the C ABI test hooks of libwkb200.so).
References: torch fp32 on the same 16-bit-rounded inputs (floating-point kernels), the CPU oracle (mel),
the reference's own known-answer vectors (filters)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from tests import kat_vectors as K  # noqa: E402

TD = {"bf16": (torch.bfloat16, _lib.WK_DTYPE_BF16), "f16": (torch.float16, _lib.WK_DTYPE_F16)}


@pytest.fixture(scope="module")
def toy():
    m = wk.Model("toy", max_batch=4)
    m.init_random(seed=3)
    yield m
    m.close()


def _sync():
    torch.cuda.synchronize()


def p(t):
    return C.c_void_p(t.data_ptr())


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K,gelu,out32", [
    (128, 256, 64, 0, 1), (256, 256, 128, 0, 0), (1000, 384, 128, 1, 0), (3000, 1280, 1280, 1, 0),
    (4500, 3840, 1280, 0, 0), (777, 1280, 5120, 0, 1), (130, 128, 64, 0, 1), (4200, 1280, 256, 1, 0), (8200, 512, 1280, 0, 1),
])
def test_gemm_tcgen05_vs_torch(toy, dt, M, N, K, gelu, out32):
    tdt, wdt = TD[dt]
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(tdt)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(tdt)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32 if out32 else tdt)
    _sync()
    wk._lib.check(toy.lib.wk_test_gemm(toy.handle, p(a), p(w), p(bias), p(out), M, N, K, wdt,
                                       _lib.WK_DTYPE_F32 if out32 else wdt, gelu))
    torch.cuda.current_stream().synchronize()
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias
    if gelu:
        ref = torch.nn.functional.gelu(ref)
    got = out.float()
    assert torch.isfinite(got).all()
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    tol = 2e-5 * scale * max(1, K / 256) if out32 else (8e-3 if dt == "bf16" else 1e-3) * scale
    assert err <= tol, f"max err {err} (scale {scale})"


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K", [(3000, 1280, 1280), (4500, 1280, 1280), (4097, 1280, 5120), (6000, 384, 384), (9000, 1280, 256)])
def test_gemm_residual_update_in_place(toy, dt, M, N, K):
    """out += A W^T + bias in place (the f32 residual stream; encoder out-proj / FC2), small and encoder-sized row counts with ragged
    last row tiles; every element must be touched exactly once (the epilogue reads and writes the residual in place)."""
    tdt, wdt = TD[dt]
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(tdt)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(tdt)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    x0 = torch.randn(M, N, device="cuda", generator=g) * 3.0
    out = x0.clone()
    _sync()
    wk._lib.check(toy.lib.wk_test_gemm_residual(toy.handle, p(a), p(w), p(bias), p(out), M, N, K, wdt))
    torch.cuda.synchronize()
    ref = x0 + a.float() @ w.float().t() + bias
    assert torch.isfinite(out).all()
    err = (out - ref).abs().max().item()
    assert err <= 2e-5 * ref.abs().max().item() * max(1, K / 256), err


@pytest.mark.parametrize("N,rows,Kd,splits", [(1280, 64, 1280, 0), (1280, 16, 1280, 20), (3840, 64, 1280, 5),
                                              (1280, 48, 5120, 16), (51866, 32, 256, 1), (384, 16, 384, 0)])
def test_gemm_swap_ab_splitk(toy, N, rows, Kd, splits):
    g = torch.Generator(device="cuda").manual_seed(N + rows)
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    x = (torch.randn(rows, Kd, device="cuda", generator=g)).to(torch.bfloat16)
    out = torch.full((rows, N), float("nan"), device="cuda")
    _sync()
    wk._lib.check(toy.lib.wk_test_gemm_splitk(toy.handle, p(w), p(x), p(out), N, rows, Kd, _lib.WK_DTYPE_BF16, splits))
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t()
    err = (out - ref).abs().max().item()
    assert torch.isfinite(out).all()
    assert err <= 3e-5 * ref.abs().max().item() * max(1, Kd / 256), err


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("B,H", [(64, 20), (3, 6), (1, 2)])
def test_decoder_cross_attention_kernel_vs_torch(toy, dt, B, H):
    """decoder_cross_attention_kernel alone at the benchmarked lane shape (B = 64 windows, H = 20 heads, T = 1500 encoder positions)
    against torch fp32 on the same 16-bit K/V; rows flagged done must be left untouched (ended windows skip their K/V stream)."""
    tdt, wdt = TD[dt]
    T, dm = 1500, H * 64
    g = torch.Generator(device="cuda").manual_seed(B * 7 + H)
    q = torch.randn(B, dm, device="cuda", generator=g)
    k = (torch.randn(B, H, T, 64, device="cuda", generator=g) * 0.7).to(tdt)
    v = torch.randn(B, H, T, 64, device="cuda", generator=g).to(tdt)
    if B > 2:   # a peaked row: one key dominates (exercises the max subtraction)
        k[1, 0, 777] = (q[1, :64] * 3).to(tdt)
    out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
    done = torch.zeros(B, dtype=torch.int32, device="cuda")
    if B > 2:
        done[2] = 1
    _sync()
    wk._lib.check(toy.lib.wk_test_cross_attention(toy.handle, p(q), p(k), p(v), p(out), B, H, T, wdt, p(done)))
    torch.cuda.synchronize()
    qh = q.view(B, H, 1, 64)
    ref = (torch.softmax(qh @ k.float().transpose(-1, -2) * 0.125, dim=-1) @ v.float()).reshape(B, dm)
    got = out.float()
    live = done == 0
    err = (got[live] - ref[live]).abs().max().item()
    tol = (8e-3 if dt == "bf16" else 1e-3) * max(1.0, ref.abs().max().item())   # f32 math, 16-bit output rounding
    assert err <= tol, err
    if B > 2:
        assert torch.all(got[2] == 7.0)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("W,NQ,H,T", [(32, 5, 20, 1500), (3, 2, 6, 1500), (2, 8, 2, 250), (1, 3, 1, 1500)])
def test_decoder_cross_attention_shared_kv_vs_torch(toy, dt, W, NQ, H, T):
    """The beam-search form of cross-attention: NQ adjacent decode rows (the beams of one window) read ONE K/V block.  Checked against
    torch fp32 on the same 16-bit K/V at the benchmarked beam shape (32 windows x 5 beams, H = 20, T = 1500); a window flagged done (its
    beams end together) must be left untouched; one peaked row exercises the max subtraction."""
    tdt, wdt = TD[dt]
    B, dm = W * NQ, H * 64
    g = torch.Generator(device="cuda").manual_seed(W * 31 + NQ * 7 + H)
    q = torch.randn(B, dm, device="cuda", generator=g)
    k = (torch.randn(W, H, T, 64, device="cuda", generator=g) * 0.7).to(tdt)
    v = torch.randn(W, H, T, 64, device="cuda", generator=g).to(tdt)
    k[0, 0, T - 3] = (q[1, :64] * 3).to(tdt)
    out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
    done = torch.zeros(B, dtype=torch.int32, device="cuda")
    if W > 2:
        done[2 * NQ:3 * NQ] = 1
    _sync()
    wk._lib.check(toy.lib.wk_test_cross_attention_shared(toy.handle, p(q), p(k), p(v), p(out), B, H, T, wdt, p(done), NQ))
    torch.cuda.synchronize()
    qh = q.view(W, NQ, H, 64).transpose(1, 2)                       # [W, H, NQ, 64]
    ref = torch.softmax(qh @ k.float().transpose(-1, -2) * 0.125, dim=-1) @ v.float()   # [W, H, NQ, 64]
    ref = ref.transpose(1, 2).reshape(B, dm)
    got = out.float()
    live = done == 0
    err = (got[live] - ref[live]).abs().max().item()
    tol = (8e-3 if dt == "bf16" else 1e-3) * max(1.0, ref.abs().max().item())
    assert err <= tol, err
    if W > 2:
        assert torch.all(got[2 * NQ:3 * NQ] == 7.0)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("B,H", [(64, 20), (5, 6)])
def test_decoder_self_attention_kernel_vs_torch(toy, dt, B, H):
    """decoder_self_attention_kernel alone at B = 64, H = 20 with per-row positions 0 / 1 / 100 / 222 (and everything between): reduces
    the q|k|v row, appends K/V at pos[b] in the cache, attends over positions <= pos[b]; against torch fp32."""
    tdt, wdt = TD[dt]
    dm, L = H * 64, 224
    g = torch.Generator(device="cuda").manual_seed(B * 3 + H)
    qkv = torch.randn(B, 3 * dm, device="cuda", generator=g)
    kc = torch.randn(B, H, L, 64, device="cuda", generator=g).to(tdt)
    vc = torch.randn(B, H, L, 64, device="cuda", generator=g).to(tdt)
    pos_list = [0, 1, 100, 222] + [int(x) for x in torch.randint(0, 223, (max(0, B - 4),), generator=torch.Generator().manual_seed(B))]
    pos = torch.tensor(pos_list[:B], dtype=torch.int32, device="cuda")
    out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
    done = torch.zeros(B, dtype=torch.int32, device="cuda")
    done[B - 1] = 1
    kc0, vc0 = kc.clone(), vc.clone()
    _sync()
    wk._lib.check(toy.lib.wk_test_self_attention(toy.handle, p(qkv), p(kc), p(vc), p(pos), p(out), B, H, wdt, p(done)))
    torch.cuda.synchronize()
    q, kn, vn = [t.view(B, H, 64) for t in qkv.split(dm, dim=1)]
    worst = 0.0
    for b in range(B - 1):
        t = int(pos[b])
        kk = torch.cat([kc0[b, :, :t].float(), kn[b].to(tdt).float()[:, None]], dim=1)     # [H, t+1, 64]
        vv = torch.cat([vc0[b, :, :t].float(), vn[b].to(tdt).float()[:, None]], dim=1)
        ref = (torch.softmax(q[b][:, None] @ kk.transpose(-1, -2) * 0.125, dim=-1) @ vv).reshape(dm)
        worst = max(worst, (out[b].float() - ref).abs().max().item() / max(1.0, ref.abs().max().item()))
        # the new row landed in the cache, rounded to the storage type; older rows are untouched
        assert torch.equal(kc[b, :, t], kn[b].to(tdt)) and torch.equal(vc[b, :, t], vn[b].to(tdt))
        assert torch.equal(kc[b, :, :t], kc0[b, :, :t])
    assert worst <= (8e-3 if dt == "bf16" else 1e-3), worst
    assert torch.all(out[B - 1].float() == 7.0) and torch.equal(kc[B - 1], kc0[B - 1])   # done row: no cache traffic at all


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("B,T,H", [(1, 1500, 2), (2, 1500, 6), (1, 200, 1), (3, 77, 2), (2, 1500, 20)])
def test_encoder_attention_vs_torch(toy, dt, B, T, H):
    tdt, wdt = TD[dt]
    dm = H * 64
    g = torch.Generator(device="cuda").manual_seed(B * T + H)
    qkv = (torch.randn(B * T, 3 * dm, device="cuda", generator=g)).to(tdt)
    out = torch.zeros(B * T, dm, device="cuda", dtype=tdt)
    _sync()
    wk._lib.check(toy.lib.wk_test_attention(toy.handle, p(qkv), p(out), B, T, H, wdt))
    torch.cuda.synchronize()
    q, k, v = [t.float().view(B, T, H, 64).transpose(1, 2) for t in qkv.split(dm, dim=1)]
    ref = torch.softmax(q @ k.transpose(-1, -2) * 0.125, dim=-1) @ v
    ref = ref.transpose(1, 2).reshape(B * T, dm)
    err = (out.float() - ref).abs().max().item()
    tol = 2e-2 if dt == "bf16" else 3e-3  # P is rounded to 16 bits before P.V; outputs are 16-bit
    assert err <= tol * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("T", [1500, 300])
def test_encoder_attention_growing_scores(toy, dt, T):
    """Scores far from N(0, 1): queries 4x larger and key magnitudes that grow with the position, so that the running row maximum keeps
    moving from key tile to key tile by more than any lazy-rescale threshold (the online-softmax correction path), plus one window whose
    scores are all equal (uniform attention)."""
    tdt, wdt = TD[dt]
    B, H = 3, 2
    dm = H * 64
    g = torch.Generator(device="cuda").manual_seed(T)
    qkv = torch.randn(B, T, 3 * dm, device="cuda", generator=g)
    ramp = torch.linspace(0.25, 3.0, T, device="cuda").view(1, T, 1)
    qkv[0, :, :dm] *= 4.0
    qkv[0, :, dm:2 * dm] *= ramp[0]
    qkv[1, :, :dm] *= 2.0
    qkv[1, :, dm:2 * dm] *= ramp[0].flip(0)
    qkv[2, :, :dm] = 0.0
    qkv = qkv.reshape(B * T, 3 * dm).to(tdt)
    out = torch.zeros(B * T, dm, device="cuda", dtype=tdt)
    _sync()
    wk._lib.check(toy.lib.wk_test_attention(toy.handle, p(qkv), p(out), B, T, H, wdt))
    torch.cuda.synchronize()
    q, k, v = [t.float().view(B, T, H, 64).transpose(1, 2) for t in qkv.split(dm, dim=1)]
    ref = torch.softmax(q @ k.transpose(-1, -2) * 0.125, dim=-1) @ v
    ref = ref.transpose(1, 2).reshape(B * T, dm)
    assert torch.isfinite(out.float()).all()
    err = (out.float() - ref).abs().max().item()
    tol = 2e-2 if dt == "bf16" else 3e-3
    assert err <= tol * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("variant,n_mels", [("toy", 80), ("toy128", 128)])
def test_log_mel_vs_oracle(variant, n_mels):
    m = wk.Model(variant, max_batch=4)
    fe = wk.FeatureExtractor(m)
    assert fe.melCount == n_mels and fe.windowSamples == 480000
    pcm = np.stack([mel_ref.synthetic_pcm(0), mel_ref.synthetic_pcm(1), np.zeros(480000, np.float32),
                    mel_ref.synthetic_pcm(2)])
    nv = [480000, 480000, 480000, 176000]
    pcm[3, 176000:] = 0
    # host input with explicit valid lengths (padOrTrim folded into the kernel)
    got = fe.logMelSpectrogram(pcm, samples_per_window=nv).numpy()
    assert got.shape == (4, n_mels, 3000)
    for i in range(4):
        ref = mel_ref.log_mel(pcm[i], n_mels)
        err = np.abs(got[i] - ref).max()
        # north_star tolerance: log-mel within 1e-3 (relative to the tensor scale, which is O(1)); f16 output
        assert err <= 1e-3 * max(1.0, np.abs(ref).max()), (i, err)
    # device-resident input, no lengths
    dev = torch.from_numpy(pcm[:2]).cuda()
    got2 = fe.logMelSpectrogram(dev).numpy()
    np.testing.assert_array_equal(got2, got[:2])
    m.close()


def _f16(v):
    return np.array(v, dtype=np.float16).astype(np.float32)


def test_filters_reference_kats_on_device(toy):
    """UnitTests.swift:1982-2115 through the fused CUDA filter+sampler kernel."""
    for name, sup, logits, tokens, exp in K.SUPPRESS_TOKENS:
        st = wk.SpecialTokens(specialTokenBegin=100)
        _, _, f = wk.filter_and_sample(toy, _f16(logits), [tokens], st, wk.DecodingOptions(suppressTokens=sup))
        np.testing.assert_array_equal(f[0], _f16(exp), err_msg=name)
    for name, eot, ws, sb, logits, tokens, exp in K.SUPPRESS_BLANK:
        st = wk.SpecialTokens.from_any(D.SpecialTokens.test_default(endToken=eot, whitespaceToken=ws))
        _, _, f = wk.filter_and_sample(toy, _f16(logits), [tokens], st, blankSampleBegin=sb)
        np.testing.assert_array_equal(f[0], _f16(exp), err_msg=name)
    for name, langs, dim, sb, logits, tokens, exp in K.LANGUAGE:
        st = wk.SpecialTokens.from_any(D.SpecialTokens.test_default())
        _, _, f = wk.filter_and_sample(toy, _f16(logits), [tokens], st, languageTokens=langs, languageSampleBegin=sb)
        np.testing.assert_array_equal(f[0], _f16(exp), err_msg=name)
    for name, multi, sb, logits, tokens, exp in K.TIMESTAMP_RULES:
        st = wk.SpecialTokens.from_any(D.SpecialTokens.test_default(**K.TS_SPECIAL))
        tok, lp, f = wk.filter_and_sample(toy, _f16(logits), [tokens], st, isModelMultilingual=multi, timestampSampleBegin=sb)
        np.testing.assert_array_equal(f[0], _f16(exp), err_msg=name)
        # sampler on the filtered row == oracle GreedyTokenSampler
        s = D.GreedyTokenSampler(0.0, st.endToken, D.DecodingOptions())
        r = s.update([], _f16(exp), [])
        assert tok[0] == r.tokens[-1], name
        assert abs(lp[0] - r.logProbs[-1]) < 1e-5, name


def test_filter_sampler_random_rows_vs_oracle(toy):
    """Bit-exact token choice vs the oracle on random full-vocabulary rows with random token histories."""
    rng = np.random.default_rng(7)
    V = 51866
    st_o = D.SpecialTokens.large_v3()
    st = wk.SpecialTokens.from_any(st_o)
    B = 24
    logits = rng.standard_normal((B, V)).astype(np.float32) * 2
    toks = []
    for b in range(B):
        prompt = [st_o.startOfTranscriptToken, st_o.englishToken, st_o.transcribeToken, st_o.timeTokenBegin]
        n = int(rng.integers(0, 12))
        hist = []
        for _ in range(n):
            if rng.random() < 0.4:
                hist.append(int(st_o.timeTokenBegin + rng.integers(0, 1500)))
            else:
                hist.append(int(rng.integers(0, 50000)))
        if b % 3 == 0:
            logits[b, st_o.timeTokenBegin:] += 6.0  # make the timestamp mass win
        toks.append(prompt + hist)
    opts = D.DecodingOptions(suppressTokens=[5, 17, 300], suppressBlank=True)
    tok, lp, filt = wk.filter_and_sample(toy, logits, toks, st, wk.DecodingOptions(suppressTokens=[5, 17, 300]),
                                         timestampSampleBegin=4, blankSampleBegin=4)
    for b in range(B):
        fs = [D.SuppressBlankFilter(st_o, 4), D.SuppressTokensFilter([5, 17, 300]),
              D.TimestampRulesFilter(st_o, 4, None, True)]
        row = logits[b].copy()
        for f in fs:
            row = f.filterLogits(row, toks[b])
        np.testing.assert_array_equal(np.isneginf(filt[b]), np.isneginf(row), err_msg=f"row {b}")
        r = D.GreedyTokenSampler(0.0, st_o.endToken, opts).update([], row, [])
        assert tok[b] == r.tokens[-1], b
        assert abs(lp[b] - r.logProbs[-1]) < 2e-4, (b, lp[b], r.logProbs[-1])


def test_temperature_topk_sampling_vs_oracle(toy):
    """GreedyTokenSampler with temperature > 0 (TokenSampler.swift:57-73): softmax(logits / T), top-k, multinomial draw inside
    the top-k mass, logprob = log of the full-vocabulary softmax prob.  The draw itself is Philox-seeded here (Float.random in
    the reference), so parity is: token in the oracle's top-k set, exact logprob, k = 1 == argmax, frequencies ~ probabilities."""
    rng = np.random.default_rng(3)
    V, B, T, K = 4096, 64, 0.7, 5
    st_o = D.SpecialTokens.test_default(endToken=V - 1, timeTokenBegin=V, specialTokenBegin=V - 1)
    st = wk.SpecialTokens.from_any(st_o)
    base = rng.standard_normal(V).astype(np.float32) * 3
    logits = np.tile(base, (B, 1))
    x = base.astype(np.float64) / T
    probs = np.exp(x - x.max())
    probs /= probs.sum()
    top = np.argsort(-probs, kind="stable")[:K]
    counts = np.zeros(K)
    n_draws = 0
    for seed in range(20):
        tok, lp, _ = wk.filter_and_sample(toy, logits, [[1]] * B, st, wk.DecodingOptions(temperature=T, topK=K, seed=seed))
        for b in range(B):
            assert tok[b] in top
            j = int(np.where(top == tok[b])[0][0])
            assert abs(lp[b] - np.log(probs[tok[b]])) < 2e-4
            counts[j] += 1
            n_draws += 1
    expect = probs[top] / probs[top].sum()
    assert np.abs(counts / n_draws - expect).max() < 0.05, (counts / n_draws, expect)
    assert len(set(np.round(counts))) > 1
    tok1, lp1, _ = wk.filter_and_sample(toy, logits[:4], [[1]] * 4, st, wk.DecodingOptions(temperature=T, topK=1, seed=9))
    assert all(t == int(np.argmax(base)) for t in tok1)


def test_sampler_row_without_finite_logit_is_flagged(toy):
    """A row whose every logit is -inf (or NaN) has no argmax: the kernel reports token -1 / logprob -inf instead of an out-of-range id
    (in the decode loop the window ends there and the host reports WhisperError.decodingLogitsFailed)."""
    st = wk.SpecialTokens()
    logits = np.full((3, 64), -np.inf, np.float32)
    logits[1, 5] = 1.0
    logits[2, :] = np.nan
    tok, lp, _ = wk.filter_and_sample(toy, logits, [[1], [1], [1]], st)
    assert tok[0] == -1 and np.isneginf(lp[0])
    assert tok[1] == 5 and abs(lp[1]) < 1e-6
    assert tok[2] == -1
