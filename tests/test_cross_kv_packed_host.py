"""The packed bf16 cross K/V row format round-trips every bf16 row bit for bit (host reference, tests/packed_kv_ref.py)."""
import numpy as np

from tests import packed_kv_ref as P


def _bits(exps, signs=None, mants=None):
    exps = np.asarray(exps, np.uint32)
    signs = np.zeros(64, np.uint32) if signs is None else np.asarray(signs, np.uint32)
    mants = (np.arange(64, dtype=np.uint32) * 37 % 128) if mants is None else np.asarray(mants, np.uint32)
    return ((signs << 15) | (exps << 7) | mants).astype(np.uint16)


def _adversarial():
    rng = np.random.default_rng(7)
    rows, coded = [], []
    zeros = _bits(np.zeros(64), signs=np.arange(64) % 2, mants=np.zeros(64))   # +-0 only
    rows.append(zeros); coded.append(True)
    sub = _bits(np.zeros(64))                                                   # subnormals
    rows.append(sub); coded.append(True)
    mixed = _bits(np.r_[np.full(32, 130), np.zeros(32)], mants=np.r_[np.arange(32), np.zeros(32)])   # normals with +0: 130 binades
    rows.append(mixed); coded.append(False)
    for special in (0x7F80, 0xFF80, 0x7FC1):                                    # +Inf, -Inf, NaN
        r = _bits(np.full(64, 127)); r[5] = special
        rows.append(r); coded.append(False)
    for span in (14, 15, 16):                                                   # largest minus smallest exponent field = span
        e = 120 + rng.integers(0, span + 1, 64)
        e[0], e[1] = 120, 120 + span
        rows.append(_bits(e)); coded.append(span <= 15)
    rows.append(np.full(64, 0x3F80, np.uint16)); coded.append(True)             # constant row
    rows.append(_bits(np.full(64, 254), signs=rng.integers(0, 2, 64))); coded.append(True)   # exponent 254
    r = _bits(np.r_[np.full(63, 254), [239]]); rows.append(r); coded.append(True)            # 254 down to 239: offset 15
    r = _bits(np.r_[np.full(63, 254), [238]]); rows.append(r); coded.append(False)           # offset 16
    return np.stack(rows), np.array(coded)


def test_round_trip_adversarial_rows():
    bits, coded = _adversarial()
    prim, sec, hdr = P.pack_rows(bits)
    assert np.array_equal(hdr != P.RAW, coded)
    assert np.array_equal(P.unpack_rows(prim, sec, hdr), bits)


def test_round_trip_random_rows():
    rng = np.random.default_rng(11)
    x = (rng.standard_normal((4096, 64)) * np.exp(rng.uniform(-20, 20, (4096, 1)))).astype(np.float32)
    bits = (x.view(np.uint32) >> 16).astype(np.uint16)
    bits[::97, 3] = rng.integers(0, 1 << 16, bits[::97, 3].shape)   # arbitrary bit patterns too
    prim, sec, hdr = P.pack_rows(bits)
    assert np.array_equal(P.unpack_rows(prim, sec, hdr), bits)
    assert (hdr == P.RAW).mean() < 0.05


def test_coded_row_layout():
    # value 8 g + j: sign|mantissa byte g * 8 + j, offset nibble at bit 16 (j & 1) + 4 (j >> 1) of word g
    bits = _bits(np.full(64, 130))
    bits[9] = _bits([127] * 64)[9] | 0x8000   # group 1, j = 1: offset 3, negative
    prim, _, hdr = P.pack_rows(bits[None])
    assert hdr[0] == 130
    assert prim[0, 9] == (0x80 | (bits[9] & 0x7F))
    word1 = int(prim[0, 64 + 4:64 + 8].view(np.uint32)[0])
    assert word1 == 3 << 16
