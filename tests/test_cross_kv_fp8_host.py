"""FP8 (E4M3) cross-attention K/V cache, host side: the quantizer the GPU epilogue runs (through its host entry) against the oracle's
float8_e4m3fn rounding, the new C ABI, and how far the FP8 policy moves the oracle's logits (the basis of the GPU tolerances)."""
import ctypes as C

import numpy as np
import pytest

import whisperkit_b200 as wk
from whisperkit_b200 import _lib

torch = pytest.importorskip("torch")

from oracle import model_ref as M  # noqa: E402
from tests import fp8_ref  # noqa: E402

# Max |logit difference| / max |logit| between the FP8-policy and the bf16-policy oracle over the steps below: how far the policy itself
# moves the logits (printed).  The FP8 end-to-end GPU tests (tests/test_gpu_cross_kv_fp8.py) compare the engine with the FP8-policy oracle
# at the 16-bit tests' tolerances, which sit below this distance.
FP8_LOGITS_REL_BOUND = 1e-2


def host_quantize(x: np.ndarray):
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, 64)
    codes = np.zeros(x.shape, np.uint8)
    scales = np.zeros(x.shape[0], np.float32)
    _lib.check(wk.load().wk_cross_kv_quantize_rows(x.ctypes.data_as(C.c_void_p), x.shape[0], codes.ctypes.data_as(C.c_void_p),
                                                    scales.ctypes.data_as(C.c_void_p)))
    return codes, scales


def edge_rows() -> np.ndarray:
    g = np.random.default_rng(11)
    rows = []
    rows.append(np.zeros(64, np.float32))                                   # all-zero row
    z = np.zeros(64, np.float32)
    z[::2] = -0.0                                                           # +-0 only: still an all-zero row
    rows.append(z)
    r = g.standard_normal(64).astype(np.float32) * 0.01
    r[17] = 300.0                                                           # one large outlier: the rest falls into E4M3 subnormals
    rows.append(r)
    r = g.standard_normal(64).astype(np.float32)
    r[5] = -1e4
    rows.append(r)
    # ties at half a step: with amax = 448 (s = 1) the values below sit exactly between two E4M3 neighbours
    t = np.array([448.0, 1.0625, 1.1875, 2.125, 2.375, 17.0, 19.0, 0.0029296875, 0.0048828125, -0.0029296875, 240.0, 272.0,
                  -1.0625, -0.0, 0.0, 3.0 * 2.0 ** -10], np.float32)
    rows.append(np.resize(t, 64))
    rows.append(np.resize(np.array([448.0, 2.0 ** -10, 3.0 * 2.0 ** -10, 2.0 ** -9, 2.0 ** -11, -2.0 ** -10, 1e-6, -1e-6], np.float32), 64))
    rows.append(np.full(64, 1e-30, np.float32))                             # tiny amax: s is an f32 subnormal
    rows.append(np.full(64, -3.5, np.float32))
    r = np.linspace(-1.0, 1.0, 64).astype(np.float32) * 7.3
    rows.append(r)
    return np.stack(rows)


def test_new_symbols_are_exported():
    lib = wk.load()
    for n in ("wk_model_set_cross_kv_dtype", "wk_cross_kv_quantize_rows", "wk_test_cross_attention_fp8"):
        assert hasattr(lib, n)
    assert _lib.WK_DTYPE_FP8_E4M3 == 4
    assert "cross_kv_dtype" in [f for f, _ in _lib.wk_model_info._fields_]


@pytest.mark.parametrize("case", ["edges", "gaussian", "heavy_tailed", "scaled"])
def test_host_quantizer_matches_oracle_bit_exactly(case):
    g = np.random.default_rng({"edges": 1, "gaussian": 2, "heavy_tailed": 3, "scaled": 4}[case])
    if case == "edges":
        x = edge_rows()
    elif case == "gaussian":
        x = g.standard_normal((4096, 64)).astype(np.float32)
    elif case == "heavy_tailed":
        x = (g.standard_t(2, (4096, 64)) * 0.3).astype(np.float32)
        x[g.random(x.shape) < 0.05] = 0.0
    else:
        x = (g.standard_normal((2048, 64)) * np.exp(g.uniform(-30, 30, (2048, 1)))).astype(np.float32)
    codes, scales = host_quantize(x)
    ref_codes, ref_scales = fp8_ref.quantize_rows(torch.from_numpy(x))
    np.testing.assert_array_equal(scales.view(np.uint32), ref_scales.numpy().view(np.uint32))
    np.testing.assert_array_equal(codes, ref_codes.numpy())
    if case == "edges":
        assert np.all(codes[:2] == 0) and np.all(scales[:2] == 0)             # amax 0: s = 0, zero codes
        assert np.any((codes[2] & 0x78) == 0) and np.any(codes[2] & 0x07)     # the outlier row reaches E4M3 subnormals


def test_dequantized_rows_are_within_half_an_e4m3_step():
    x = np.random.default_rng(5).standard_normal((1000, 64)).astype(np.float32)
    codes, scales = host_quantize(x)
    deq = fp8_ref.dequantize_rows(torch.from_numpy(codes), torch.from_numpy(scales)).numpy()
    # E4M3 has 3 mantissa bits: relative error <= 2^-4 for normals, absolute <= 2^-10 * s in the subnormal range
    err = np.abs(deq - x)
    assert np.all(err <= np.maximum(np.abs(x) * 2.0 ** -4, scales[:, None] * 2.0 ** -10) * (1 + 1e-6))


@pytest.mark.parametrize("variant", ["toy", "toy128"])
def test_oracle_fp8_policy_logits_bound(variant):
    """The FP8 policy against the bf16 policy of the same oracle, teacher-forced over 8 steps on a seeded encoder output."""
    dims = M.VARIANTS[variant]
    w = M.random_weights(dims, seed=4, policy="bf16")
    o16 = M.WhisperOracle(dims, w, "bf16")
    o8 = fp8_ref.FP8CrossKVOracle(dims, w, "bf16")
    g = torch.Generator().manual_seed(9)
    enc = torch.randn(2, dims.n_audio_ctx, dims.d_model, generator=g)
    toks = torch.randint(0, dims.vocab, (2, 8), generator=g)
    worst = 0.0
    with torch.no_grad():
        c16, c8 = o16.cross_kv(enc), o8.cross_kv(enc)
        k16, k8 = o16.new_cache(2), o8.new_cache(2)
        for t in range(toks.shape[1]):
            a = o16.decode_step(toks[:, t], t, k16, c16)
            b = o8.decode_step(toks[:, t], t, k8, c8)
            worst = max(worst, float((a - b).abs().max() / a.abs().max()))
    print(f"{variant}: FP8 vs bf16 cross-K/V policy, max |dlogit| / max |logit| = {worst:.3e} (bound {FP8_LOGITS_REL_BOUND})")
    assert 0.0 < worst <= FP8_LOGITS_REL_BOUND
