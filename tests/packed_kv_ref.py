"""Host reference of the packed bf16 cross K/V rows (layout in whisperkit_b200/csrc/common.cuh).

A row is 64 bf16 values given as their uint16 bits.  Coded row: 64 sign|mantissa bytes, then 8 words of exponent offsets
(base - exponent field, 0..15), value 8 g + j at bit 16 (j & 1) + 4 (j >> 1) of word g; header = base.  Raw row (a span of more than
16 binades, or Inf/NaN): header 255, bytes 0..95 in the primary slot and 96..127 in the secondary slot.
"""
import numpy as np

RAW = 255


def _nibble_shift():
    j = np.arange(64) % 8
    return (16 * (j & 1) + 4 * (j >> 1)).astype(np.uint32)


def pack_rows(bits: np.ndarray):
    """bits [n, 64] uint16 -> primary [n, 96] u8, secondary [n, 32] u8, header [n] u8"""
    bits = np.ascontiguousarray(bits, dtype=np.uint16)
    n = bits.shape[0]
    e = ((bits >> 7) & 0xFF).astype(np.int32)
    emax, emin = e.max(axis=1), e.min(axis=1)
    raw = (emax == 255) | (emax - emin > 15)
    prim = np.zeros((n, 96), np.uint8)
    sec = np.zeros((n, 32), np.uint8)
    rb = bits[raw].view(np.uint8).reshape(-1, 128)
    prim[raw] = rb[:, :96]
    sec[raw] = rb[:, 96:]
    c = ~raw
    cb = bits[c].astype(np.uint32)
    prim[c, :64] = (((cb >> 8) & 0x80) | (cb & 0x7F)).astype(np.uint8)
    off = (emax[c, None] - e[c]).astype(np.uint32) << _nibble_shift()[None, :]
    words = np.bitwise_or.reduce(off.reshape(-1, 8, 8), axis=2).astype(np.uint32)
    prim[c, 64:] = words.view(np.uint8).reshape(-1, 32)
    hdr = np.where(raw, RAW, emax).astype(np.uint8)
    return prim, sec, hdr


def unpack_rows(prim: np.ndarray, sec: np.ndarray, hdr: np.ndarray) -> np.ndarray:
    """the inverse of pack_rows: [n, 64] uint16 bits"""
    n = prim.shape[0]
    out = np.zeros((n, 64), np.uint16)
    raw = hdr == RAW
    out[raw] = np.concatenate([prim[raw], sec[raw]], axis=1).view(np.uint16)
    c = ~raw
    sm = prim[c, :64].astype(np.uint32)
    words = np.ascontiguousarray(prim[c, 64:]).view(np.uint32).reshape(-1, 8)
    nib = (np.repeat(words, 8, axis=1) >> _nibble_shift()[None, :]) & 0xF
    e = hdr[c, None].astype(np.uint32) - nib
    out[c] = (((sm & 0x80) << 8) | (e << 7) | (sm & 0x7F)).astype(np.uint16)
    return out
