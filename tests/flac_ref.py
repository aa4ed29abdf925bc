"""A plain numpy restatement of an RFC 9639 FLAC *encoder*, written for the tests: it can emit every construct the decoder has to read,
on demand.  Lossless round trip is the oracle: decode(encode(x)) == x, and STREAMINFO carries the MD5 of x.

encode(x, rate, bps, **options) -> bytes, x an int array [n, channels] of bps-bit signed samples.  Per-frame and per-subframe choices
go through `spec`, a function (frame index, channel, samples, subframe bps) -> dict:
    kind         "auto" | "constant" | "verbatim" | "fixed" | "lpc"
    order        predictor order (fixed 0-4, lpc 1-32); auto picks the best fixed order
    precision    LPC coefficient precision 1-15 (default 12)
    shift        LPC shift (default: from the precision)
    partition    partition order 0-15 (default: the cheapest up to 8 that divides the block)
    rice2        5-bit Rice parameters (default: only when a parameter needs them)
    escape       partition indices coded as escaped (verbatim) partitions; escape_bits their width (default: the smallest that fits)
    wasted       False, or "auto" (default): shift out the common zero low bits
Frame-level options: stereo ("independent", "left_side", "side_right", "mid_side", "auto", or a per-frame list), block sizes, variable
blocking, the header's block-size / sample-rate / sample-size forms, metadata blocks before the audio, an ID3v2 prefix."""
from __future__ import annotations

import hashlib
from typing import Callable, List, Optional, Sequence

import numpy as np

# ------------------------------------------------------------------------------------------------ CRCs
_CRC8 = np.zeros(256, np.uint8)
for _i in range(256):
    _c = _i
    for _ in range(8):
        _c = ((_c << 1) ^ 0x07) & 0xFF if _c & 0x80 else (_c << 1) & 0xFF
    _CRC8[_i] = _c


def crc8(data: bytes) -> int:
    c = 0
    for b in data:
        c = int(_CRC8[c ^ b])
    return c


def _mulx16(v: np.ndarray) -> np.ndarray:
    """v * x^16 mod P for 16-bit polynomials v (P = x^16 + x^15 + x^2 + 1)."""
    c = v.astype(np.uint32)
    for _ in range(16):
        c = np.where(c & 0x8000, ((c << 1) ^ 0x8005) & 0xFFFF, (c << 1) & 0xFFFF)
    return c.astype(np.uint16)


_LEVELS: List[np.ndarray] = []   # _LEVELS[l][v] = v * x^(16 * 2^l) mod P


def _level(l: int) -> np.ndarray:
    while len(_LEVELS) <= l:
        if not _LEVELS:
            _LEVELS.append(_mulx16(np.arange(65536, dtype=np.uint32)))
        else:
            t = _LEVELS[-1]
            _LEVELS.append(t[t])
    return _LEVELS[l]


def crc16(data: bytes) -> int:
    """FLAC's CRC-16 (initial 0, MSB first).  With a zero initial value the CRC is linear and leading zeros do not change it, so it is
    computed as a tree: 16-bit words, then pairs of blocks, crc(A || B) = crc(A) * x^(16 |B|) + crc(B)."""
    b = np.frombuffer(bytes(data), np.uint8)
    if b.size == 0:
        return 0
    if b.size % 2:
        b = np.concatenate([np.zeros(1, np.uint8), b])
    c = _level(0)[(b[0::2].astype(np.uint32) << 8) | b[1::2]]
    l = 0
    while c.size > 1:
        if c.size % 2:
            c = np.concatenate([np.zeros(1, np.uint16), c])
        c = _level(l)[c[0::2]] ^ c[1::2]
        l += 1
    return int(c[0])


# ------------------------------------------------------------------------------------------------ bit writer
class BitWriter:
    """Fields (value, width) appended in order; numpy arrays of fields are packed without a per-bit loop."""

    def __init__(self):
        self.vals: List[np.ndarray] = []
        self.widths: List[np.ndarray] = []
        self.nbits = 0

    def put(self, value: int, width: int):
        if width == 0:
            return
        assert width <= 64 and 0 <= value < (1 << width), (value, width)
        self.vals.append(np.array([value], np.uint64))
        self.widths.append(np.array([width], np.int64))
        self.nbits += width

    def put_signed(self, value: int, width: int):
        assert -(1 << (width - 1)) <= value < (1 << (width - 1)), (value, width)
        self.put(value & ((1 << width) - 1), width)

    def put_array(self, vals: np.ndarray, widths: np.ndarray):
        vals, widths = np.asarray(vals, np.uint64), np.asarray(widths, np.int64)
        self.vals.append(vals)
        self.widths.append(widths)
        self.nbits += int(widths.sum())

    def put_signed_array(self, v: np.ndarray, width: int):
        if width == 0 or len(v) == 0:
            return
        v = np.asarray(v, np.int64)
        assert v.min() >= -(1 << (width - 1)) and v.max() < (1 << (width - 1)), width
        self.put_array(v.astype(np.uint64) & np.uint64((1 << width) - 1), np.full(len(v), width, np.int64))

    def pad_to_byte(self):
        if self.nbits % 8:
            self.put(0, 8 - self.nbits % 8)

    def getvalue(self) -> bytes:
        assert self.nbits % 8 == 0
        if not self.vals:
            return b""
        v = np.concatenate(self.vals)
        w = np.concatenate(self.widths)
        keep = (w > 0) & (v != 0)            # zero fields only advance the position
        end = np.cumsum(w)[keep]             # bit position just after each field
        v, w = v[keep], w[keep]
        start = end - w
        nwords = (self.nbits + 63) // 64
        out = np.zeros(nwords + 1, np.uint64)
        # split every field at the 64-bit word boundary: head bits in word start >> 6, tail bits in the next word
        wi = start >> 6
        off = start & 63
        head_w = np.minimum(w, 64 - off)
        tail_w = w - head_w
        head = (v >> tail_w.astype(np.uint64)) << (64 - off - head_w).astype(np.uint64)
        tail_mask = np.where(tail_w > 0, (np.uint64(1) << tail_w.astype(np.uint64)) - np.uint64(1), np.uint64(0))
        tail = np.where(tail_w > 0, (v & tail_mask) << (64 - tail_w).astype(np.uint64) % np.uint64(64), np.uint64(0))
        np.bitwise_or.at(out, wi, head)      # fields never overlap: OR == sum
        np.bitwise_or.at(out, wi + 1, tail)
        return out[:nwords].astype(">u8").tobytes()[: self.nbits // 8]


# ------------------------------------------------------------------------------------------------ residual coding
def _zigzag(r: np.ndarray) -> np.ndarray:
    r = np.asarray(r, np.int64)
    return ((r << 1) ^ (r >> 63)).astype(np.uint64)


def _rice_cost(u: np.ndarray, k: int) -> int:
    return int((u >> np.uint64(k)).sum()) + len(u) * (k + 1)


def _best_k(u: np.ndarray, kmax: int) -> int:
    if len(u) == 0:
        return 0
    m = float(u.mean())
    k0 = max(0, min(kmax, int(np.log2(m)) if m >= 1 else 0))
    best = min(range(max(0, k0 - 1), min(kmax, k0 + 2) + 1), key=lambda k: _rice_cost(u, k))
    return best


def _signed_width(r: np.ndarray) -> int:
    if len(r) == 0:
        return 0
    lo, hi = int(r.min()), int(r.max())
    if lo == 0 and hi == 0:
        return 0
    w = 1
    while not (-(1 << (w - 1)) <= lo and hi < (1 << (w - 1))):
        w += 1
    return w


def write_residual(bw: BitWriter, res: np.ndarray, block: int, order: int, partition: Optional[int], rice2: Optional[bool],
                   escape: Sequence[int] = (), escape_bits: Optional[int] = None):
    res = np.asarray(res, np.int64)
    u_all = _zigzag(res)
    if partition is not None:   # the largest order up to the one asked for that divides the block (a short last block)
        while partition > 0 and (block % (1 << partition) or (block >> partition) < order):
            partition -= 1
    cands = [partition] if partition is not None else [p for p in range(0, 9) if block % (1 << p) == 0 and (block >> p) >= order]
    best = None
    for po in cands:
        ps = block >> po
        ks, cost = [], 0
        for i in range(1 << po):
            a = 0 if i == 0 else i * ps - order
            b = (i + 1) * ps - order
            k = _best_k(u_all[a:b], 30)
            ks.append(k)
            cost += _rice_cost(u_all[a:b], k)
        if best is None or cost < best[0]:
            best = (cost, po, ks)
    _, po, ks = best
    need2 = any(k > 14 for k in ks)
    use2 = need2 if rice2 is None else rice2
    assert use2 or not need2
    bw.put(1 if use2 else 0, 2)
    bw.put(po, 4)
    pbits, esc = (5, 31) if use2 else (4, 15)
    ps = block >> po
    for i in range(1 << po):
        a = 0 if i == 0 else i * ps - order
        b = (i + 1) * ps - order
        r, u = res[a:b], u_all[a:b]
        if i in escape:
            nb = _signed_width(r) if escape_bits is None else escape_bits
            bw.put(esc, pbits)
            bw.put(nb, 5)
            bw.put_signed_array(r, nb)
            continue
        k = min(ks[i], esc - 1)
        bw.put(k, pbits)
        if len(u) == 0:
            continue
        q = (u >> np.uint64(k)).astype(np.int64)
        low = u & np.uint64((1 << k) - 1)
        # per sample: q zero bits, then the stop bit and k low bits as one field
        vals = np.empty(2 * len(u), np.uint64)
        wid = np.empty(2 * len(u), np.int64)
        vals[0::2], wid[0::2] = 0, q
        vals[1::2], wid[1::2] = (np.uint64(1) << np.uint64(k)) | low, k + 1
        bw.put_array(vals, wid)


# ------------------------------------------------------------------------------------------------ predictors
FIXED = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


def fixed_residual(x: np.ndarray, order: int) -> np.ndarray:
    x = np.asarray(x, np.int64)
    r = x.copy()
    for _ in range(order):
        r = np.diff(r)
    return r


def lpc_coefs(x: np.ndarray, order: int, precision: int, shift: Optional[int]):
    """Least-squares predictor, quantised to `precision` bits with a non-negative shift."""
    xf = np.asarray(x, np.float64)
    n = len(xf)
    if n <= order + 1:
        a = np.zeros(order)
    else:
        A = np.stack([xf[order - 1 - j: n - 1 - j] for j in range(order)], axis=1)
        a = np.linalg.lstsq(A, xf[order:], rcond=None)[0]
    lim = (1 << (precision - 1)) - 1
    if shift is None:
        m = float(np.abs(a).max()) if order else 0.0
        shift = 15
        while shift > 0 and m * (1 << shift) > lim:
            shift -= 1
    q = np.clip(np.round(a * (1 << shift)), -lim - 1, lim).astype(np.int64)
    return q, shift


def lpc_residual(x: np.ndarray, q: np.ndarray, shift: int) -> np.ndarray:
    x = np.asarray(x, np.int64)
    order = len(q)
    n = len(x)
    pred = np.zeros(n - order, np.int64)
    for j in range(order):
        pred += q[j] * x[order - 1 - j: n - 1 - j]
    return x[order:] - (pred >> shift)


def write_subframe(bw: BitWriter, x: np.ndarray, sbps: int, spec: dict):
    x = np.asarray(x, np.int64)
    block = len(x)
    kind = spec.get("kind", "auto")
    wasted = spec.get("wasted", "auto")
    if wasted == "auto":
        wasted = 0
        nz = int(np.bitwise_or.reduce(x.astype(np.uint64))) if block else 0
        while nz and wasted < sbps - 1 and not (nz >> wasted) & 1:
            wasted += 1
    wasted = int(wasted or 0)
    if wasted:
        assert not np.any(x & ((1 << wasted) - 1))
        x = x >> wasted
        sbps -= wasted
    if kind == "auto":
        kind = "constant" if np.all(x == x[0]) else "fixed"

    def header(t):
        bw.put(0, 1)
        bw.put(t, 6)
        bw.put(1 if wasted else 0, 1)
        if wasted:
            bw.put(0, wasted - 1)
            bw.put(1, 1)

    if kind == "constant":
        header(0)
        bw.put_signed(int(x[0]), sbps)
    elif kind == "verbatim":
        header(1)
        bw.put_signed_array(x, sbps)
    elif kind == "fixed":
        order = spec.get("order")
        if order is None:
            order = min(range(0, min(4, block - 1) + 1), key=lambda o: int(np.abs(fixed_residual(x, o)).sum()) + o * sbps)
        header(8 + order)
        bw.put_signed_array(x[:order], sbps)
        write_residual(bw, fixed_residual(x, order), block, order, spec.get("partition"), spec.get("rice2"), spec.get("escape", ()),
                       spec.get("escape_bits"))
    elif kind == "lpc":
        order = spec.get("order", 8)
        prec = spec.get("precision", 12)
        q, shift = lpc_coefs(x, order, prec, spec.get("shift"))
        header(31 + order)
        bw.put_signed_array(x[:order], sbps)
        bw.put(prec - 1, 4)
        bw.put_signed(shift, 5)
        bw.put_signed_array(q, prec)
        write_residual(bw, lpc_residual(x, q, shift), block, order, spec.get("partition"), spec.get("rice2"), spec.get("escape", ()),
                       spec.get("escape_bits"))
    else:
        raise ValueError(kind)


# ------------------------------------------------------------------------------------------------ frames and the stream
STEREO = {"independent": None, "left_side": 8, "side_right": 9, "mid_side": 10}
_BS_CODES = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13, 16384: 14, 32768: 15}
_RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
_BPS_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}


def utf8_number(v: int) -> bytes:
    if v < 0x80:
        return bytes([v])
    for n in range(2, 8):
        if v < (1 << (5 * n + 1)) or n == 7:
            break
    out = []
    for _ in range(n - 1):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = (0xFF00 >> n) & 0xFF
    out.append(lead | v)
    return bytes(reversed(out))


def frame_header(block: int, rate: int, assign: int, bps: int, number: int, variable: bool, bs_form="auto", rate_form="auto",
                 bps_form="auto") -> bytes:
    if bs_form == "auto" and block in _BS_CODES:
        bs_code, bs_tail = _BS_CODES[block], b""
    elif (bs_form in ("auto", "8bit")) and block <= 256:
        bs_code, bs_tail = 6, bytes([block - 1])
    else:
        bs_code, bs_tail = 7, (block - 1).to_bytes(2, "big")
    if rate_form == "streaminfo":
        rc, rt = 0, b""
    elif rate_form == "auto" and rate in _RATE_CODES:
        rc, rt = _RATE_CODES[rate], b""
    elif rate_form in ("auto", "khz") and rate % 1000 == 0 and rate // 1000 < 256:
        rc, rt = 12, bytes([rate // 1000])
    elif rate_form in ("auto", "hz") and rate < 65536:
        rc, rt = 13, rate.to_bytes(2, "big")
    else:
        assert rate % 10 == 0
        rc, rt = 14, (rate // 10).to_bytes(2, "big")
    sc = 0 if bps_form == "streaminfo" or bps not in _BPS_CODES else _BPS_CODES[bps]
    h = bytes([0xFF, 0xF8 | int(variable), bs_code << 4 | rc, assign << 4 | sc << 1]) + utf8_number(number) + bs_tail + rt
    return h + bytes([crc8(h)])


def encode_frame(x: np.ndarray, bps: int, rate: int, number: int, variable: bool, stereo: str, spec: Callable, fi: int,
                 forms: dict) -> bytes:
    block, ch = x.shape
    x = x.astype(np.int64)
    if ch == 2 and stereo == "auto":
        cost = {}
        l, r = x[:, 0], x[:, 1]
        s, m = l - r, (l + r) >> 1
        e = lambda v: int(np.abs(fixed_residual(v, 2)).sum()) if block > 2 else 0
        cost["independent"], cost["left_side"], cost["side_right"], cost["mid_side"] = e(l) + e(r), e(l) + e(s), e(s) + e(r), e(m) + e(s)
        stereo = min(cost, key=cost.get)
    if ch != 2:
        stereo = "independent"
    assign = STEREO[stereo]
    if assign is None:
        subs, sbps, assign = [x[:, c] for c in range(ch)], [bps] * ch, ch - 1
    else:
        l, r = x[:, 0], x[:, 1]
        s = l - r
        if assign == 8:
            subs, sbps = [l, s], [bps, bps + 1]
        elif assign == 9:
            subs, sbps = [s, r], [bps + 1, bps]
        else:
            subs, sbps = [(l + r) >> 1, s], [bps, bps + 1]
    bw = BitWriter()
    hdr = frame_header(block, rate, assign, bps, number, variable, **forms)
    for c in range(ch):
        write_subframe(bw, subs[c], sbps[c], spec(fi, c, subs[c], sbps[c]))
    bw.pad_to_byte()
    body = hdr + bw.getvalue()
    return body + crc16(body).to_bytes(2, "big")


def md5_of(x: np.ndarray, bps: int) -> bytes:
    w = (bps + 7) // 8
    a = np.ascontiguousarray(np.asarray(x, np.int64).reshape(-1)).astype("<i8")
    return hashlib.md5(a.view(np.uint8).reshape(-1, 8)[:, :w].tobytes()).digest()


def streaminfo(min_block, max_block, min_frame, max_frame, rate, ch, bps, total, md5) -> bytes:
    v = min_block << 16 | max_block
    v = v << 24 | min_frame
    v = v << 24 | max_frame
    v = v << 20 | rate
    v = v << 3 | (ch - 1)
    v = v << 5 | (bps - 1)
    v = v << 36 | total
    return v.to_bytes(18, "big") + md5


def metadata_block(btype: int, body: bytes, last: bool) -> bytes:
    return bytes([(0x80 if last else 0) | btype]) + len(body).to_bytes(3, "big") + body


def id3v2(payload: bytes = b"TIT2\x00\x00\x00\x05\x00\x00\x03abcd") -> bytes:
    n = len(payload)
    size = bytes([(n >> 21) & 0x7F, (n >> 14) & 0x7F, (n >> 7) & 0x7F, n & 0x7F])
    return b"ID3\x04\x00\x00" + size + payload


ALL_METADATA = [  # one block of every type, each skipped by its length
    (3, bytes(18 * 2)),                                           # SEEKTABLE (two placeholder points)
    (4, b"\x04\x00\x00\x00test\x01\x00\x00\x00\x07\x00\x00\x00TITLE=x"),   # VORBIS_COMMENT
    (2, b"wkb2" + bytes(12)),                                     # APPLICATION
    (5, bytes(396 + 4)),                                          # CUESHEET-sized body
    (6, (3).to_bytes(4, "big") + (9).to_bytes(4, "big") + b"image/png" + bytes(4) + bytes(16) + (3).to_bytes(4, "big") + b"abc"),
    (1, bytes(1000)),                                             # PADDING
    (99, b"unknown type"),
]


def encode(x: np.ndarray, rate: int, bps: int, *, block_size: int = 4096, blocks: Optional[Sequence[int]] = None,
           variable: bool = False, stereo="auto", spec: Optional[Callable] = None, bs_form="auto", rate_form="auto",
           bps_form="auto", metadata: Sequence = (), id3: Optional[bytes] = None, streaminfo_total: Optional[int] = None,
           frames_only: bool = False):
    """FLAC file bytes of x [n, channels] (bps-bit signed).  blocks: the block sizes in order (variable blocking needs them or uses
    block_size); stereo a mode name or a per-frame list; spec(frame, channel, samples, sbps) -> subframe options."""
    x = np.asarray(x, np.int64)
    if x.ndim == 1:
        x = x[:, None]
    n, ch = x.shape
    assert 1 <= ch <= 8 and 4 <= bps <= 32
    assert x.min() >= -(1 << (bps - 1)) and x.max() < (1 << (bps - 1))
    if blocks is None:
        blocks = [block_size] * (n // block_size) + ([n % block_size] if n % block_size else [])
    assert sum(blocks) == n
    spec = spec or (lambda fi, c, v, sb: {})
    forms = dict(bs_form=bs_form, rate_form=rate_form, bps_form=bps_form)
    frames, pos = [], 0
    for fi, b in enumerate(blocks):
        st = stereo[fi] if isinstance(stereo, (list, tuple)) else stereo
        number = pos if variable else fi
        frames.append(encode_frame(x[pos: pos + b], bps, rate, number, variable, st, spec, fi, forms))
        pos += b
    if frames_only:
        return frames
    fixed_bs = max(blocks) if blocks else block_size
    min_bs = min(blocks[:-1]) if variable and len(blocks) > 1 else fixed_bs
    sizes = [len(f) for f in frames]
    si = streaminfo(max(16, min(min_bs, fixed_bs)), max(16, max(blocks) if blocks else 16), min(sizes) if sizes else 0,
                    max(sizes) if sizes else 0, rate, ch, bps, n if streaminfo_total is None else streaminfo_total, md5_of(x, bps))
    meta = [(0, si)] + list(metadata)
    out = bytearray(id3 or b"")
    out += b"fLaC"
    for i, (t, body) in enumerate(meta):
        out += metadata_block(t, body, i == len(meta) - 1)
    for f in frames:
        out += f
    return bytes(out)


def parse_streaminfo(data: bytes) -> dict:
    """STREAMINFO of a FLAC file (after an optional ID3v2 tag)."""
    pos = 0
    if data[:3] == b"ID3":
        pos = 10 + ((data[6] & 0x7F) << 21 | (data[7] & 0x7F) << 14 | (data[8] & 0x7F) << 7 | (data[9] & 0x7F))
    assert data[pos: pos + 4] == b"fLaC"
    b = data[pos + 8: pos + 8 + 34]
    v = int.from_bytes(b[:18], "big")
    total = v & ((1 << 36) - 1); v >>= 36
    bps = (v & 31) + 1; v >>= 5
    ch = (v & 7) + 1; v >>= 3
    rate = v & ((1 << 20) - 1)
    return dict(rate=rate, channels=ch, bps=bps, total=total, md5=bytes(b[18:34]))


def container(bps: int) -> str:
    """The WAV sample format a FLAC stream of this sample size loads as."""
    return "s16" if bps <= 16 else "s24" if bps <= 24 else "s32"


def left_justify(x: np.ndarray, bps: int) -> np.ndarray:
    width = {"s16": 16, "s24": 24, "s32": 32}[container(bps)]
    return np.asarray(x, np.int64) << (width - bps)


def test_signal(n: int, ch: int, bps: int, seed: int = 0) -> np.ndarray:
    """A seeded signal that compresses like audio: a few tones per channel, correlated across channels, plus noise, at bps bits."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)[:, None]
    f = rng.uniform(0.002, 0.05, (3, ch))
    base = sum(np.sin(t * f[k] + rng.uniform(0, 6)) * rng.uniform(0.1, 0.3) for k in range(3))
    common = np.sin(t[:, 0] * 0.013)[:, None] * 0.2
    x = base + common + rng.standard_normal((n, ch)) * 0.02
    lim = (1 << (bps - 1)) - 1
    return np.clip(np.round(x * lim), -lim - 1, lim).astype(np.int64)
