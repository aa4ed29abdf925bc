"""The wgmma GEMM's TMA-store epilogues on the H100: 16-bit and f32 outputs and the f32 residual update bit for bit against torch's single
rounding of the exact product, over ragged row counts and every encoder width, and the 16-bit cross-attention K/V projection (head-major
boxes, tiles that straddle two windows) against the oracle."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402

TD = {"bf16": (torch.bfloat16, _lib.WK_DTYPE_BF16), "f16": (torch.float16, _lib.WK_DTYPE_F16)}


@pytest.fixture(scope="module")
def toy():
    m = wk.Model("toy", max_batch=4)
    m.init_random(seed=3)
    yield m
    m.close()


def p(t):
    return C.c_void_p(t.data_ptr())


def exact_operands(M_, N, K, tdt, seed):
    """A and W of small integers times a power of two: every partial sum is exact in f32, so the accumulation order cannot matter."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randint(-4, 5, (M_, K), device="cuda", generator=g).float() * 0.25).to(tdt)
    w = (torch.randint(-4, 5, (N, K), device="cuda", generator=g).float() * 0.125).to(tdt)
    bias = torch.randn(N, device="cuda", generator=g)
    acc = a.float() @ w.float().t()
    return g, a, w, bias, acc


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


SHAPES = [(4500, 1280, 1280), (4097, 3840, 1280), (130, 5120, 1280), (4500, 384, 256), (4097, 1280, 5120)]


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M_,N,K", SHAPES)
@pytest.mark.parametrize("out32", [0, 1])
def test_gemm_store_rounding_bit_exact(toy, dt, M_, N, K, out32):
    tdt, wdt = TD[dt]
    _, a, w, bias, acc = exact_operands(M_, N, K, tdt, M_ + N + K)
    out = torch.full((M_, N), float("nan"), device="cuda", dtype=torch.float32 if out32 else tdt)
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_gemm(toy.handle, p(a), p(w), p(bias), p(out), M_, N, K, wdt, _lib.WK_DTYPE_F32 if out32 else wdt, 0))
    torch.cuda.synchronize()
    ref = acc + bias                      # one f32 rounding of the exact product plus the bias
    if not out32:
        ref = ref.to(tdt)                 # then one 16-bit rounding
    assert torch.equal(bits(out), bits(ref)), f"{(bits(out) != bits(ref)).sum().item()} elements differ"


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M_,N,K", [(4500, 1280, 1280), (130, 3840, 1280), (4097, 384, 384)])
def test_gemm_store_gelu(toy, dt, M_, N, K):
    """GELU epilogue through the staging box: the tolerance of test_gpu_kernels.py (the erf is an approximation)."""
    tdt, wdt = TD[dt]
    _, a, w, bias, acc = exact_operands(M_, N, K, tdt, 7 * M_ + N)
    out = torch.full((M_, N), float("nan"), device="cuda", dtype=tdt)
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_gemm(toy.handle, p(a), p(w), p(bias), p(out), M_, N, K, wdt, wdt, 1))
    torch.cuda.synchronize()
    ref = torch.nn.functional.gelu(acc + bias)
    got = out.float()
    assert torch.isfinite(got).all()
    scale = ref.abs().max().item()
    assert (got - ref).abs().max().item() <= (8e-3 if dt == "bf16" else 1e-3) * scale


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M_,N,K", [(4500, 1280, 1280), (4097, 1280, 5120), (130, 384, 1280), (4500, 3840, 256)])
def test_gemm_residual_bit_exact(toy, dt, M_, N, K):
    """x += acc + bias in place: every element equals torch's x0 + (acc + bias), including subnormal, signed-zero and rounding-tie x0."""
    tdt, wdt = TD[dt]
    g, a, w, bias, acc = exact_operands(M_, N, K, tdt, 3 * M_ + N + K)
    v = acc + bias
    x0 = torch.randn(M_, N, device="cuda", generator=g) * 3.0
    x0[:, 0::7] = 1e-40                                         # subnormal
    x0[:, 1::7] = -1e-41
    x0[:, 2::7] = 0.0
    x0[:, 3::7] = -0.0
    ulp = torch.nextafter(v.abs(), torch.tensor(float("inf"), device="cuda")) - v.abs()
    x0[:, 4::7] = (ulp / 2)[:, 4::7]                            # v + x0 exactly halfway between two floats
    x0[:, 5::7] = (-ulp / 2)[:, 5::7]
    out = x0.clone()
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_gemm_residual(toy.handle, p(a), p(w), p(bias), p(out), M_, N, K, wdt))
    torch.cuda.synchronize()
    ref = x0 + v
    assert torch.equal(bits(out), bits(ref)), f"{(bits(out) != bits(ref)).sum().item()} elements differ"


@pytest.mark.parametrize("variant,policy", [("toy", "bf16"), ("toy128", "f16"), ("toy128", "bf16")])
def test_cross_kv_16bit_readback_matches_oracle(variant, policy):
    """The 16-bit cross K/V cache written through head-major TMA boxes, 3 windows of 1500 rows (128-row tiles straddle windows), against
    the oracle's cross_kv of the engine's own encoder output.  Allowed: one 16-bit ulp plus the worst-case difference of two f32 sums of
    the same K products in different orders (2 K 2^-24 sum |a w|), which only matters where the sum cancels to near zero."""
    B = 3
    dims = M.VARIANTS[variant]
    wts = M.random_weights(dims, seed=5, policy=policy)
    orc = M.WhisperOracle(dims, wts, policy)
    model = wk.Model(variant, max_batch=B, dtype=policy)
    model.load_state_dict(wts)
    pcm = np.stack([mel_ref.synthetic_pcm(30 + i) for i in range(B)])
    enc_t = wk.AudioEncoder(model).encodeFeatures(wk.FeatureExtractor(model).logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    dec = wk.TextDecoder(model, B)
    dec.bindEncoderOutput(enc_t)
    L, H, T, d = dims.dec_layers, dims.n_heads, dims.n_audio_ctx, dims.d_model
    n = 2 * L * B * H * T * 64
    got = np.empty(n, np.float32)
    _lib.check(model.lib.wk_debug_read(model.handle, dec.handle, 15, 0, got.ctypes.data_as(C.c_void_p), n))
    got = got.reshape(L, 2, B, H, T, 64)
    mant = 7 if policy == "bf16" else 10
    worst = 0.0
    with torch.no_grad():
        enc = torch.from_numpy(enc_gpu).transpose(1, 2).contiguous()
        cross = orc.cross_kv(enc)
        encr = orc.r(enc)
        for i, (k, v) in enumerate(cross):
            for j, (ref, name) in enumerate(((k, "k_proj"), (v, "v_proj"))):
                pre = f"model.decoder.layers.{i}.encoder_attn.{name}"
                mag_sum = encr.abs() @ orc.w[pre + ".weight"].abs().t()
                if pre + ".bias" in orc.w:
                    mag_sum = mag_sum + orc.w[pre + ".bias"].abs()
                f32_err = (2 * d * 2.0 ** -24 * orc._heads(mag_sum)).numpy()
                ref = ref.float().numpy()
                g = got[i, j]
                mag = np.maximum(np.abs(ref), np.abs(g))
                ulp = np.exp2(np.floor(np.log2(np.maximum(mag, 2.0 ** -126))) - mant)
                if policy == "f16":
                    ulp = np.maximum(ulp, 2.0 ** -24)
                worst = max(worst, float((np.abs(g - ref) / (ulp + f32_err)).max()))
    print(f"[{variant}/{policy}] 16-bit cross K/V: max |diff| / (ulp + f32 order bound) {worst:.3f}")
    assert worst <= 1.0
    dec.close()
    model.close()
