"""FP8 (E4M3) encoder policy, host side: the block quantizer the GPU LayerNorm, FC1 epilogue and weight quantizer run (through its host
entry wk_fp8_quantize_blocks) against torch.float8_e4m3fn, codes and scales bit for bit, and the new C ABI."""
import ctypes as C

import numpy as np
import pytest

import whisperkit_b200 as wk
from whisperkit_b200 import _lib

torch = pytest.importorskip("torch")

from tests import encoder_fp8_ref as E  # noqa: E402
from tests.test_cross_kv_fp8_host import edge_rows  # noqa: E402


def host_quantize(x: np.ndarray, block: int):
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, cols = x.shape
    codes = np.zeros(x.shape, np.uint8)
    scales = np.zeros((rows, cols // block), np.float32)
    _lib.check(wk.load().wk_fp8_quantize_blocks(x.ctypes.data_as(C.c_void_p), rows, cols, block, codes.ctypes.data_as(C.c_void_p),
                                                scales.ctypes.data_as(C.c_void_p)))
    return codes, scales


def edge_matrix() -> np.ndarray:
    """Rows of 256 columns (two activation blocks): the cross-K/V edge rows (zeros, +-0, outliers, E4M3 subnormals, half-step ties,
    f32-subnormal scales) paired so that every block kind meets every other in one row, plus random rows."""
    e = edge_rows()   # [n, 64]
    blocks = np.concatenate([e, e[::-1]], axis=1)   # [n, 128]
    rows = [np.concatenate([blocks[i], blocks[j]]) for i in range(len(blocks)) for j in range(len(blocks))]
    g = np.random.default_rng(5)
    rows += list(g.standard_normal((16, 256)).astype(np.float32) * np.float32(3.0))
    return np.stack(rows).astype(np.float32)


def test_new_symbols_are_exported():
    lib = wk.load()
    for n in ("wk_model_set_encoder_dtype", "wk_model_encoder_dtype", "wk_fp8_quantize_blocks", "wk_test_gemm_fp8"):
        assert hasattr(lib, n)


@pytest.mark.parametrize("block", [128, 256])
def test_block_quantizer_matches_torch_float8(block):
    """block = 128 is the activation rule (one scale per row and 128-column block), block = cols the weight rule (one per row)."""
    x = edge_matrix()
    codes, scales = host_quantize(x, block)
    rc, rs = E.quantize_blocks(torch.from_numpy(x), block)
    np.testing.assert_array_equal(codes, rc.numpy())
    np.testing.assert_array_equal(scales.view(np.uint32), rs.numpy().view(np.uint32))
    if block == x.shape[1]:
        wc, ws = E.quantize_weight(torch.from_numpy(x))
        np.testing.assert_array_equal(codes, wc.numpy())
        np.testing.assert_array_equal(scales[:, 0].view(np.uint32), ws.numpy().view(np.uint32))


def test_block_quantizer_edge_cases():
    x = np.zeros((2, 256), np.float32)
    x[1, :128] = -0.0
    x[1, 128] = 448.0
    x[1, 129] = 1.0625          # half-way between 1.0 and 1.125 with s = 1: ties to the even code (1.0)
    x[1, 130] = 2.0 ** -10      # an E4M3 subnormal (2^-9 is the smallest step): ties to even (0)
    x[1, 131] = 3.0 * 2.0 ** -10
    codes, scales = host_quantize(x, 128)
    assert np.all(codes[0] == 0) and np.all(scales[0] == 0)
    assert np.all(codes[1, :128] == 0) and scales[1, 0] == 0     # an all-(+-0) block: s = 0, zero codes
    assert scales[1, 1] == np.float32(1.0)
    dec = torch.from_numpy(codes[1, 128:132].copy()).view(torch.float8_e4m3fn).float().numpy()
    np.testing.assert_array_equal(dec, np.array([448.0, 1.0, 0.0, 2.0 ** -8], np.float32))


def test_block_quantizer_rejects_ragged_blocks():
    x = np.zeros((1, 200), np.float32)
    c = np.zeros(200, np.uint8)
    s = np.zeros(2, np.float32)
    assert wk.load().wk_fp8_quantize_blocks(x.ctypes.data_as(C.c_void_p), 1, 200, 128, c.ctypes.data_as(C.c_void_p),
                                            s.ctypes.data_as(C.c_void_p)) == _lib.WK_ERR_INVALID_ARGUMENT


def test_encoder_dtype_argument_is_checked_before_the_device():
    with pytest.raises(ValueError):
        wk.Model("toy", encoderDtype="int8")
    assert wk.WhisperKitConfig().encoderDtype is None
