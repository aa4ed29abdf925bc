"""The packed bf16 cross K/V cache on the H100: the projection's packed epilogue against the 16-bit heads epilogue of the same GEMM and
against the host reference (tests/packed_kv_ref.py), byte for byte, raw rows included; then the single-query, beam and word-timestamp
cross-attention kernels on a packed cache against the same kernels on the 16-bit cache of the same values, bit for bit."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from tests import packed_kv_ref as P  # noqa: E402

W, H, T = 3, 4, 1500
D = H * 64
HS = (T + 15) // 16 * 16


@pytest.fixture(scope="module")
def toy():
    m = wk.Model("toy", max_batch=4)
    m.init_random(seed=3)
    yield m
    m.close()


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def project(toy, x, w, bias):
    """both epilogues of the cross-K/V projection: (16-bit blocks [W][H][T][64], packed blocks [W][H][T * 128] u8, headers [W][H][HS])"""
    raw = torch.zeros(W, H, T, 64, dtype=torch.bfloat16, device="cuda")
    pk = torch.zeros(W, H, T * 128, dtype=torch.uint8, device="cuda")
    hdr = torch.zeros(W, H, HS, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_cross_kv_project(toy.handle, p(x), p(w), p(bias), W, T, H, 0, p(raw), None))
    _lib.check(toy.lib.wk_test_cross_kv_project(toy.handle, p(x), p(w), p(bias), W, T, H, 1, p(pk), p(hdr)))
    return raw, pk, hdr


def check_against_reference(raw, pk, hdr):
    bits = raw.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1, 64)
    blocks = pk.cpu().numpy().reshape(W * H, T * 128)
    prim = blocks[:, :T * 96].reshape(-1, 96)
    sec = blocks[:, T * 96:].reshape(-1, 32)
    h = hdr.cpu().numpy().reshape(W * H, HS)[:, :T].reshape(-1)
    rp, rs, rh = P.pack_rows(bits)
    assert np.array_equal(h, rh)
    assert np.array_equal(prim, rp)
    israw = rh == P.RAW
    assert np.array_equal(sec[israw], rs[israw])
    assert np.array_equal(P.unpack_rows(prim, sec, h), bits)
    return israw.mean()


def identity_cache(toy, kv):
    """kv [W][H][T][64] bf16 through the projection with an identity weight: the 16-bit and the packed cache of (essentially) these values"""
    x = kv.permute(0, 2, 1, 3).reshape(W * T, D).contiguous()
    eye = torch.eye(D, dtype=torch.bfloat16, device="cuda")
    return project(toy, x, eye, None)


def adversarial_kv(seed, finite=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kv = torch.randn(W, H, T, 64, device="cuda", generator=g)
    kv[0, 0, 5] = 0.0                                    # all zeros: coded
    kv[0, 1, 7, 3] = 0.0                                 # one zero among normals: raw
    kv[1, 2, 124, 10] *= 2.0 ** 30                       # a 30-binade span: raw (last row of a stage)
    kv[1, 2, 125, 60] *= 2.0 ** -30                      # raw, secondary half
    kv[2, 3, 1499, :] *= 2.0 ** torch.arange(-20, 44, device="cuda").float()   # the block's last row: raw
    kv[2, 0, 640:700, 0] *= 2.0 ** 20                    # a run of raw rows across stage and tile boundaries
    kv[0, 2, 900, 2] = 2.0 ** -128                       # a bf16 subnormal next to normals: raw
    kv[1, 1, 300] = 2.0 ** -130                          # subnormals only: coded
    kv[1, 1, 301, :8] = 2.0 ** -128                      # subnormals with +-0: coded
    kv[1, 1, 301, 8:] = 0.0
    if not finite:
        kv[0, 3, 11, 4] = float("inf")
        kv[0, 3, 12, 5] = float("nan")
        kv[2, 1, 13, :] = 3.0e38                         # exponent 254
    return kv.to(torch.bfloat16)


def test_projection_packed_epilogue_matches_16bit_epilogue_and_reference(toy):
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(W * T, D, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(D, D, device="cuda", generator=g) * 0.06).to(torch.bfloat16)
    bias = torch.randn(D, device="cuda", generator=g) * 0.1
    raw, pk, hdr = project(toy, x, w, bias)
    rate = check_against_reference(raw, pk, hdr)
    print(f"raw-row rate of a seeded random projection: {rate:.5f}")
    assert rate < 0.05


def test_projection_raw_rows_byte_exact(toy):
    raw, pk, hdr = identity_cache(toy, adversarial_kv(5, finite=False))
    rate = check_against_reference(raw, pk, hdr)
    print(f"raw-row rate of the adversarial cache: {rate:.5f}")
    h = hdr.cpu().numpy()
    assert h[0, 1, 7] == P.RAW and h[2, 3, 1499] == P.RAW and h[0, 3, 11] == P.RAW and h[0, 3, 12] == P.RAW
    assert h[0, 0, 5] != P.RAW and h[1, 1, 300] != P.RAW and h[1, 1, 301] != P.RAW and h[2, 1, 13] == 254


def test_single_query_and_beam_bit_identical_on_packed_and_raw(toy):
    kr, kp, kh = identity_cache(toy, adversarial_kv(21))
    vr, vp, vh = identity_cache(toy, adversarial_kv(22))
    g = torch.Generator(device="cuda").manual_seed(3)
    bf = _lib.WK_DTYPE_BF16
    # single query: one row per window (B = W), one window ended
    q = torch.randn(W, D, device="cuda", generator=g)
    done = torch.zeros(W, dtype=torch.int32, device="cuda")
    done[1] = 1
    o_raw = torch.full((W, D), 7.0, dtype=torch.bfloat16, device="cuda")
    o_pk = o_raw.clone()
    align = torch.zeros(H, W, T, device="cuda")
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_cross_attention(toy.handle, p(q), p(kr), p(vr), p(o_raw), W, H, T, bf, p(done)))
    _lib.check(toy.lib.wk_test_cross_attention_packed(toy.handle, p(q), p(kp), p(vp), p(kh), p(vh), p(o_pk), W, H, T, p(done), 1, p(align)))
    assert torch.equal(o_raw.view(torch.int16), o_pk.view(torch.int16))
    assert torch.all(o_pk[1] == 7.0)
    assert torch.isfinite(align[:, 0]).all() and torch.allclose(align[:, 0].sum(-1), torch.ones(H, device="cuda"), atol=1e-4)
    # beam: NQ rows share each window's K/V block
    for nq in (2, 5):
        qb = torch.randn(W * nq, D, device="cuda", generator=g)
        db = torch.zeros(W * nq, dtype=torch.int32, device="cuda")
        b_raw = torch.zeros(W * nq, D, dtype=torch.bfloat16, device="cuda")
        b_pk = torch.ones(W * nq, D, dtype=torch.bfloat16, device="cuda")
        torch.cuda.synchronize()
        _lib.check(toy.lib.wk_test_cross_attention_shared(toy.handle, p(qb), p(kr), p(vr), p(b_raw), W * nq, H, T, bf, p(db), nq))
        _lib.check(toy.lib.wk_test_cross_attention_packed(toy.handle, p(qb), p(kp), p(vp), p(kh), p(vh), p(b_pk), W * nq, H, T, p(db), nq, None))
        assert torch.equal(b_raw.view(torch.int16), b_pk.view(torch.int16)), nq


def test_alignment_pass_bit_identical_on_packed_and_raw(toy):
    kr, kp, kh = identity_cache(toy, adversarial_kv(31))
    vr, vp, vh = identity_cache(toy, adversarial_kv(32))
    g = torch.Generator(device="cuda").manual_seed(4)
    q = (torch.randn(W * 224, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    seq = torch.tensor([224, 37, 130], dtype=torch.int32, device="cuda")
    outs = []
    for hdrs in ((None, None), (kh, vh)):
        out = torch.zeros(W * 224, D, dtype=torch.bfloat16, device="cuda")
        acc = torch.zeros(W * 224, T, device="cuda")
        kc, vc = (kr, vr) if hdrs[0] is None else (kp, vp)
        torch.cuda.synchronize()
        _lib.check(toy.lib.wk_test_align_cross_attention(toy.handle, p(q), p(kc), p(vc), p(hdrs[0]), p(hdrs[1]), p(seq), W, H, T, 0b1011, p(out), p(acc)))
        outs.append((out, acc))
    assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16))
    assert torch.equal(outs[0][1].view(torch.int32), outs[1][1].view(torch.int32))
    assert outs[1][1][:224].abs().sum() > 0
