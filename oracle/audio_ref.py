"""Reference restatement of audio loading (AudioProcessor.swift:229-625) in numpy: the sample conversions, the reference's read plan,
convertToMono, and the 16 kHz resampler as a float64 closed form of scipy.signal.resample_poly.  Also a WAV writer for test files.

Resampler (scipy.signal.resample_poly(x, up, down), default window ('kaiser', 5.0), zero padding), up / down = 16000 / rate reduced:
  half = 10 * max(up, down);  h = firwin(2 * half + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up
  p = down - half % down;     r = (half + p) // down
  y[m] = sum_i x[i] * h[(m + r) * down - p - i * up]   (terms whose h index is outside [0, 2 * half] are zero)
  n_out = ceil(n * up / down);  up == down == 1 is an exact copy."""
from __future__ import annotations

import math
import struct
from typing import List, Optional, Sequence, Tuple

import numpy as np

OUT_RATE = 16000
DEFAULT_READ_FRAME_SIZE = 1_323_000
FORMATS = ("u8", "s16", "s24", "s32", "f32")


def ratio(rate: int) -> Tuple[int, int]:
    g = math.gcd(OUT_RATE, int(rate))
    return OUT_RATE // g, int(rate) // g


def filter_taps(rate: int) -> np.ndarray:
    """resample_poly's filter for `rate` (float64, gain `up`); empty for 16 kHz."""
    from scipy.signal import firwin
    up, down = ratio(rate)
    if up == down == 1:
        return np.zeros(0)
    mr = max(up, down)
    return firwin(2 * 10 * mr + 1, 1.0 / mr, window=("kaiser", 5.0)) * up


def resample(x: np.ndarray, rate: int, h: Optional[np.ndarray] = None) -> np.ndarray:
    """The closed form above in float64 (x is taken as float64)."""
    x = np.asarray(x, dtype=np.float64)
    up, down = ratio(rate)
    if up == down == 1:
        return x.copy()
    h = filter_taps(rate) if h is None else h
    half = 10 * max(up, down)
    p = down - half % down
    r = (half + p) // down
    n = len(x)
    n_out = -(-n * up // down)
    m = np.arange(n_out, dtype=np.int64)
    t = (m + r) * down - p
    im = t // up
    phi = t - im * up
    y = np.zeros(n_out)
    taps = -(-(2 * half + 1) // up)
    for k in range(taps):
        j = phi + k * up
        i = im - k
        ok = (j <= 2 * half) & (i >= 0) & (i < n)
        y += np.where(ok, x[np.clip(i, 0, max(n - 1, 0))] if n else 0.0, 0.0) * np.where(ok, h[np.minimum(j, 2 * half)], 0.0)
    return y


def to_float(samples: np.ndarray, fmt: str) -> np.ndarray:
    """AVAudioFile's integer -> float32 convention on decoded sample values (u8 as stored, s24 as int32 values)."""
    s = np.asarray(samples)
    if fmt == "u8":
        return (s.astype(np.float32) - np.float32(128)) / np.float32(128)
    if fmt == "s16":
        return s.astype(np.float32) / np.float32(32768)
    if fmt == "s24":
        return s.astype(np.float32) / np.float32(8388608)
    if fmt == "s32":
        return s.astype(np.int32).astype(np.float32) / np.float32(2147483648)   # float32(x) rounds to nearest even
    return s.astype(np.float32)


def read_plan(length: int, rate: int, startTime: float = 0.0, endTime: Optional[float] = None, maxReadFrameSize: Optional[int] = None,
              pieceSeconds: float = 0.0) -> List[Tuple[int, int]]:
    """Absolute frame ranges the reference reads (and normalises) one at a time: loadAudio (pieceSeconds <= 0, one piece,
    AudioProcessor.swift:253-262) or loadAudioAsFloatArray (pieces of pieceSeconds, :318-347), each piece split into reads of
    maxReadFrameSize frames (resampleAudio(fromFile:), :408-447).  Int64(x) truncates, as Python's int() does."""
    sr = float(rate)
    R = maxReadFrameSize or DEFAULT_READ_FRAME_SIZE
    start = float(startTime or 0.0)
    pieces = []
    if pieceSeconds <= 0:
        s = int(start * sr)
        e = min(int(endTime * sr), length) if endTime is not None else length
        pieces.append((s, e))
    else:
        duration = length / sr
        end = min(endTime if endTime is not None else duration, duration)
        t = start
        while t < end:
            ce = min(t + pieceSeconds, end)
            pieces.append((int(t * sr), min(int(ce * sr), length)))
            t = ce
    out = []
    for s, e in pieces:
        p = s
        while p < e:
            out.append((p, min(p + R, e)))
            p = min(p + R, e)
    return out


def convert_to_mono(chunk: np.ndarray, mode=("sum", None)) -> np.ndarray:
    """convertToMono (AudioProcessor.swift:526-625) on one read chunk [frames, channels] float32: exact float32 operations."""
    chunk = np.asarray(chunk, dtype=np.float32)
    if chunk.ndim == 1:
        chunk = chunk[:, None]
    n, ch = chunk.shape
    if ch <= 1:
        return chunk[:, 0].copy()
    kind, arg = mode
    if kind == "channel":
        return chunk[:, arg if 0 <= arg < ch else 0].copy()
    if arg:
        idx = [i for i in arg if 0 <= i < ch]
        if not idx:
            return chunk[:, 0].copy()
    else:
        idx = list(range(ch))
    peak = np.float32(0)
    for i in idx:
        if n:
            peak = max(peak, np.abs(chunk[:, i]).max())
    mono = np.zeros(n, dtype=np.float32)
    for i in idx:
        mono += chunk[:, i]
    mono_peak = np.abs(mono).max() if n else np.float32(0)
    scale = np.float32(peak) / max(np.float32(mono_peak), np.float32(0.0001))
    return mono * np.float32(scale)


def mono_signal(frames: np.ndarray, rate: int, mode=("sum", None), **plan_kw) -> np.ndarray:
    """The mono signal the reference builds from float frames [n, channels]: convertToMono per read chunk, concatenated."""
    frames = np.asarray(frames, dtype=np.float32)
    if frames.ndim == 1:
        frames = frames[:, None]
    parts = [convert_to_mono(frames[a:b], mode) for a, b in read_plan(len(frames), rate, **plan_kw)]
    return np.concatenate(parts) if parts else np.zeros(0, np.float32)


def load_reference(frames: np.ndarray, rate: int, mode=("sum", None), **plan_kw) -> np.ndarray:
    """16 kHz output of loading these float frames: mono_signal, then the float64 resampler."""
    return resample(mono_signal(frames, rate, mode, **plan_kw), rate)


# ---------------------------------------------------------------------------------------------------------------- WAV files
_SUBFORMAT_TAIL = b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"


def encode_samples(samples: np.ndarray, fmt: str) -> bytes:
    """Interleaved sample values (u8 as stored, s24 as int32 values) -> little-endian bytes."""
    s = np.asarray(samples)
    if fmt == "u8":
        return s.astype(np.uint8).tobytes()
    if fmt == "s16":
        return s.astype("<i2").tobytes()
    if fmt == "s24":
        v = s.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)[:, :3]
        return np.ascontiguousarray(v).tobytes()
    if fmt == "s32":
        return s.astype("<i4").tobytes()
    return s.astype("<f4").tobytes()


def wav_bytes(samples: np.ndarray, rate: int, fmt: str, extensible: bool = False, chunks_before: Sequence[Tuple[bytes, bytes]] = (),
              data_size: Optional[int] = None, format_tag: Optional[int] = None, bits: Optional[int] = None, riff: bytes = b"RIFF") -> bytes:
    """A WAV file of samples [frames, channels] (or [frames]).  chunks_before: (id, payload) chunks written before `data` (odd
    payloads get their pad byte); data_size overrides the data chunk's header size (a truncated file); format_tag / bits override the
    fmt fields (unsupported formats)."""
    s = np.asarray(samples)
    ch = 1 if s.ndim == 1 else s.shape[1]
    bits = bits or {"u8": 8, "s16": 16, "s24": 24, "s32": 32, "f32": 32}[fmt]
    tag = format_tag if format_tag is not None else (3 if fmt == "f32" else 1)
    block = ch * bits // 8
    if extensible:
        fmt_payload = struct.pack("<HHIIHHHHI", 0xFFFE, ch, rate, rate * block, block, bits, 22, bits, 0) + struct.pack("<H", tag) + _SUBFORMAT_TAIL
    else:
        fmt_payload = struct.pack("<HHIIHH", tag, ch, rate, rate * block, block, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt_payload)) + fmt_payload
    for cid, payload in chunks_before:
        body += cid + struct.pack("<I", len(payload)) + payload + (b"\x00" if len(payload) & 1 else b"")
    data = encode_samples(s.reshape(-1), fmt)
    body += b"data" + struct.pack("<I", len(data) if data_size is None else data_size) + data
    return riff + struct.pack("<I", len(body)) + body


def write_wav(path: str, samples: np.ndarray, rate: int, fmt: str = "s16", **kw) -> str:
    with open(path, "wb") as f:
        f.write(wav_bytes(samples, rate, fmt, **kw))
    return path
