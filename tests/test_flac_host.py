"""FLAC, host side (no GPU): the CPU build of csrc/flac_core.cuh (tests/hostcheck/flac_hostcheck.cpp) against tests/flac_ref.py's
encoder for every construct RFC 9639 allows, the committed fixtures of an independent encoder against their STREAMINFO MD5, a malformed
corpus under AddressSanitizer and UndefinedBehaviorSanitizer, and wk_audio_info / the length query / the refusals without a device."""
import ctypes as C
import glob
import hashlib
import os
import subprocess
import wave

import numpy as np
import pytest

import whisperkit_b200 as wk
from tests import flac_ref as F
from whisperkit_b200 import _lib
from whisperkit_b200.audio import AudioProcessor
from whisperkit_b200.build import build_flac_hostcheck

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
JFK = os.path.join(GOLDEN, "jfk.wav")
_HC = None


def _lib_hc():
    global _HC
    if _HC is None:
        _HC = C.CDLL(build_flac_hostcheck())
        _HC.wk_flac_host_decode.argtypes = [C.c_char_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                            C.c_int64, C.POINTER(C.c_int64)]
    return _HC


def host_decode(data: bytes):
    """(status, byte offset, samples [n, channels] int64 or None, [rate, channels, bps, variable])"""
    lib = _lib_hc()
    fmt, tot, off = (C.c_int32 * 4)(), C.c_int64(), C.c_int64()
    st = lib.wk_flac_host_decode(data, len(data), fmt, C.byref(tot), None, 0, C.byref(off))
    if st:
        return st, off.value, None, list(fmt)
    out = np.zeros(tot.value * fmt[1], np.int32)
    st = lib.wk_flac_host_decode(data, len(data), fmt, C.byref(tot), out.ctypes.data_as(C.POINTER(C.c_int32)), out.size, C.byref(off))
    return st, off.value, (out.reshape(-1, fmt[1]).astype(np.int64) if st == 0 else None), list(fmt)


def jfk_s16():
    with wave.open(JFK, "rb") as w:
        return np.frombuffer(w.readframes(w.getnframes()), dtype="<i2").astype(np.int64)


# ------------------------------------------------------------------------------------------------ round trip of every construct
def _variants():
    v = []
    for bps in (4, 5, 8, 11, 12, 16, 17, 20, 23, 24, 25, 31, 32):
        v.append((f"bps{bps}", dict(ch=2, bps=bps), dict(bps_form="auto")))
    for ch in range(1, 9):
        v.append((f"ch{ch}", dict(ch=ch, bps=16), {}))
    for st in ("independent", "left_side", "side_right", "mid_side"):
        for bps in (16, 32):
            v.append((f"{st}{bps}", dict(ch=2, bps=bps), dict(stereo=st)))
    for o in range(5):
        v.append((f"fixed{o}", dict(ch=1, bps=16), dict(spec=lambda fi, c, x, sb, o=o: dict(kind="fixed", order=o, wasted=False))))
    for o, p in ((1, 1), (2, 5), (7, 12), (12, 15), (32, 15), (32, 3)):
        v.append((f"lpc{o}p{p}", dict(ch=2, bps=16), dict(spec=lambda fi, c, x, sb, o=o, p=p: dict(kind="lpc", order=o, precision=p))))
    v.append(("lpc_wide", dict(ch=2, bps=24), dict(stereo="mid_side", spec=lambda fi, c, x, sb: dict(kind="lpc", order=32, precision=15))))
    v.append(("lpc_wide32", dict(ch=2, bps=32), dict(stereo="left_side", spec=lambda fi, c, x, sb: dict(kind="lpc", order=4, precision=15))))
    v.append(("lpc_shift0", dict(ch=1, bps=16), dict(spec=lambda fi, c, x, sb: dict(kind="lpc", order=3, precision=8, shift=0))))
    v.append(("verbatim", dict(ch=2, bps=20), dict(spec=lambda fi, c, x, sb: dict(kind="verbatim"))))
    v.append(("constant", dict(ch=3, bps=16, const=True), {}))
    for po in (0, 1, 4, 8):
        v.append((f"part{po}", dict(ch=1, bps=16), dict(spec=lambda fi, c, x, sb, po=po: dict(kind="fixed", order=2, partition=po))))
    v.append(("part15", dict(ch=1, bps=16, n=32768 * 2), dict(block_size=32768, spec=lambda fi, c, x, sb: dict(kind="fixed", order=1,
                                                                                                              partition=15))))
    v.append(("rice2", dict(ch=1, bps=16), dict(spec=lambda fi, c, x, sb: dict(kind="fixed", order=1, rice2=True, partition=2))))
    v.append(("rice2_big", dict(ch=1, bps=32), dict(spec=lambda fi, c, x, sb: dict(kind="verbatim") if fi == 0 else dict(kind="fixed", order=0))))
    v.append(("escape", dict(ch=2, bps=16), dict(spec=lambda fi, c, x, sb: dict(kind="fixed", order=2, partition=2, escape=(0, 3)))))
    v.append(("escape0", dict(ch=1, bps=16, flat=True), dict(spec=lambda fi, c, x, sb: dict(kind="fixed", order=1, partition=2, escape=(1,)))))
    v.append(("wasted", dict(ch=2, bps=16, wasted=3), {}))
    v.append(("wasted_side", dict(ch=2, bps=24, wasted=5), dict(stereo="mid_side")))
    v.append(("bs8", dict(ch=1, bps=16, n=200 * 7 + 5), dict(block_size=200, bs_form="8bit")))
    v.append(("bs16", dict(ch=1, bps=16), dict(block_size=1000, bs_form="16bit")))
    v.append(("bs_codes", dict(ch=1, bps=16, n=192 * 3 + 1), dict(block_size=192)))
    for bs in (576, 1152, 2304, 4608, 256, 512, 2048, 8192, 16384):
        v.append((f"bs{bs}", dict(ch=1, bps=8, n=bs * 2 + 3), dict(block_size=bs)))
    for rate, form in ((44100, "auto"), (8000, "auto"), (88200, "auto"), (176400, "auto"), (192000, "auto"), (22050, "auto"),
                       (24000, "auto"), (32000, "auto"), (96000, "auto"), (11000, "khz"), (12345, "hz"), (44110, "tens"),
                       (16000, "streaminfo"), (384000, "tens")):
        v.append((f"rate{rate}{form}", dict(ch=1, bps=16, rate=rate), dict(rate_form=form)))
    v.append(("bps_si", dict(ch=2, bps=16), dict(bps_form="streaminfo")))
    v.append(("variable", dict(ch=2, bps=16, n=1000 + 517 + 4096 + 33 + 2000), dict(variable=True, blocks=[1000, 517, 4096, 33, 2000])))
    v.append(("variable_big", dict(ch=1, bps=16, n=70000), dict(variable=True, blocks=[4096] * 16 + [70000 - 4096 * 16])))
    v.append(("stereo_mix", dict(ch=2, bps=16, n=4096 * 4), dict(stereo=["independent", "left_side", "side_right", "mid_side"])))
    v.append(("metadata", dict(ch=2, bps=16), dict(metadata=F.ALL_METADATA)))
    v.append(("id3", dict(ch=1, bps=16), dict(id3=F.id3v2(), metadata=F.ALL_METADATA[:2])))
    v.append(("long_number", dict(ch=1, bps=8, n=16 * 300), dict(block_size=16, bs_form="8bit")))
    return v


def _signal(ch, bps, n=9000, const=False, flat=False, wasted=0, rate=16000, seed=0):
    if const:
        return np.tile(np.array([[5, -7, 0][:ch]]), (n, 1)).astype(np.int64)
    x = F.test_signal(n, ch, bps, seed=seed + ch * 31 + bps)
    if flat:
        x[1024:2048] = 100
        x[:] = np.where(np.arange(n)[:, None] % 4096 < 2048, 100, x)
    if wasted:
        x = (x >> wasted) << wasted
    return x


VARIANTS = _variants()


@pytest.mark.parametrize("name,sig,opts", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_round_trip(name, sig, opts):
    sig = dict(sig)
    rate = sig.pop("rate", 44100)
    x = _signal(**sig, rate=rate)
    bps = sig["bps"]
    data = F.encode(x, rate, bps, **opts)
    st, off, y, fmt = host_decode(data)
    assert st == 0, (name, st, off)
    assert fmt[:3] == [rate, x.shape[1], bps]
    assert np.array_equal(y, x), name
    si = F.parse_streaminfo(data)
    assert si["md5"] == F.md5_of(y, bps)


def test_crc16_matches_a_bitwise_restatement():
    rng = np.random.default_rng(0)
    for n in (0, 1, 2, 3, 17, 1000, 4097):
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        c = 0
        for b in d:
            c ^= b << 8
            for _ in range(8):
                c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        assert F.crc16(d) == c


# ------------------------------------------------------------------------------------------------ streams the GPU tests share
def false_sync_stream():
    """A VERBATIM subframe whose 16-bit samples spell a complete frame header, with a valid CRC-8, of the frame that really follows."""
    rate, bps, bs = 16000, 16, 1024
    x = F.test_signal(bs * 5, 1, bps, seed=5)
    fake = F.frame_header(bs, rate, 0, bps, 3, False)     # frame 3's header, placed inside frame 2
    fake = fake + b"\x00" * (len(fake) % 2)
    words = np.frombuffer(fake, ">i2").astype(np.int64)
    x[2 * bs + 100: 2 * bs + 100 + len(words), 0] = words
    fake7 = F.frame_header(bs, rate, 0, bps, 7, False)    # and a header with a sample number that continues nothing
    fake7 = fake7 + b"\x00" * (len(fake7) % 2)
    w7 = np.frombuffer(fake7, ">i2").astype(np.int64)
    x[2 * bs + 400: 2 * bs + 400 + len(w7), 0] = w7
    spec = lambda fi, c, v, sb: dict(kind="verbatim") if fi == 2 else {}
    data = F.encode(x, rate, bps, block_size=bs, spec=spec)
    assert fake[:len(fake) - len(fake) % 2] in data
    return data, x, rate, bps


def variable_stream():
    rate, bps = 44100, 16
    blocks = [1000, 517, 4096, 33, 2000, 4608, 1]
    x = F.test_signal(sum(blocks), 2, bps, seed=6)
    return F.encode(x, rate, bps, variable=True, blocks=blocks, bs_form="16bit", rate_form="hz"), x, rate, bps


def test_false_sync_decodes_to_the_input():
    data, x, _, _ = false_sync_stream()
    st, _, y, _ = host_decode(data)
    assert st == 0 and np.array_equal(y, x)
    data, x, _, _ = variable_stream()
    st, _, y, fmt = host_decode(data)
    assert st == 0 and np.array_equal(y, x) and fmt[3] == 1


# ------------------------------------------------------------------------------------------------ independent fixtures
def test_fixtures_match_their_streaminfo_md5():
    paths = sorted(glob.glob(os.path.join(GOLDEN, "*.flac")))
    assert paths, "tests/golden has no FLAC fixtures"
    jfk = jfk_s16()
    for p in paths:
        data = open(p, "rb").read()
        st, off, y, fmt = host_decode(data)
        assert st == 0, (p, st, off)
        si = F.parse_streaminfo(data)
        assert si["md5"] == F.md5_of(y, fmt[2]), p
        if os.path.basename(p).startswith("jfk_"):
            assert fmt[:3] == [16000, 1, 16] and np.array_equal(y[:, 0], jfk), p


# ------------------------------------------------------------------------------------------------ malformed corpus
def _frames(x, rate, bps, **kw):
    frames = F.encode(x, rate, bps, frames_only=True, **kw)
    head = F.encode(x, rate, bps, **kw)
    head = head[: len(head) - sum(len(f) for f in frames)]
    return head, [bytearray(f) for f in frames]


def _refresh(frame: bytearray, hlen: int):
    frame[hlen - 1] = F.crc8(bytes(frame[: hlen - 1]))
    frame[-2:] = F.crc16(bytes(frame[:-2])).to_bytes(2, "big")


def _set_bits(buf: bytearray, pos: int, width: int, value: int):
    for i in range(width):
        bit = (value >> (width - 1 - i)) & 1
        byte, off = divmod(pos + i, 8)
        buf[byte] = (buf[byte] & ~(0x80 >> off)) | (bit << (7 - off))


def _join(head, frames):
    return bytes(head) + b"".join(bytes(f) for f in frames)


HLEN = 6   # header bytes of the short stream's frames: 1024 samples (code), 16 kHz (code), frame number < 128


def _short(spec=None, **kw):
    x = F.test_signal(4096, 1, 16, seed=8)
    head, frames = _frames(x, 16000, 16, block_size=1024, spec=spec, **kw)
    return x, head, frames


def malformed_subframes():
    """(name, file, reason): frames with valid CRCs whose subframes break a rule; shared with the GPU tests."""
    out = []
    lpc = lambda fi, c, v, sb: dict(kind="lpc", order=4, precision=12, wasted=False)
    x, head, frames = _short(lpc)
    f = bytearray(frames[1]); _set_bits(f, HLEN * 8 + 8 + 4 * 16, 4, 15); _refresh(f, HLEN)
    out.append(("precision15", _join(head, frames[:1] + [f] + frames[2:]), "precision code 15"))
    f = bytearray(frames[1]); _set_bits(f, HLEN * 8 + 8 + 4 * 16 + 4, 5, 0b10011); _refresh(f, HLEN)
    out.append(("negative_shift", _join(head, frames[:1] + [f] + frames[2:]), "negative LPC shift"))
    fx = lambda fi, c, v, sb: dict(kind="fixed", order=4, partition=0, wasted=False)
    x, head, frames = _short(fx)
    f = bytearray(frames[2]); _set_bits(f, HLEN * 8 + 8 + 4 * 16 + 2, 4, 9); _refresh(f, HLEN)   # 1024 >> 9 = 2 < order 4
    out.append(("small_partition", _join(head, frames[:2] + [f] + frames[3:]), "partition smaller"))
    f = bytearray(frames[2]); f[HLEN] = 2 << 1; _refresh(f, HLEN)
    out.append(("subframe_type2", _join(head, frames[:2] + [f] + frames[3:]), "reserved subframe type"))
    f = bytearray(frames[2]); _set_bits(f, HLEN * 8 + 8 + 4 * 16, 2, 2); _refresh(f, HLEN)
    out.append(("residual_method2", _join(head, frames[:2] + [f] + frames[3:]), "reserved residual coding"))
    return out


def malformed_corpus():
    """(name, file): each must fail or decode to the input of the well-formed stream it came from."""
    x, head, frames = _short()
    good = _join(head, frames)
    out = [(n, d) for n, d, _ in malformed_subframes()]
    pos = len(head)
    for k, f in enumerate(frames):   # truncated at and inside every frame
        for cut in (0, 1, 5, len(f) // 2, len(f) - 1):
            out.append((f"trunc{k}_{cut}", good[: pos + cut]))
        pos += len(f)
    for name, byte, mask, value in (("bs_code0", 2, 0xF0, 0x00), ("bps_code3", 3, 0x0E, 0x06), ("reserved_bit", 3, 0x01, 0x01),
                                    ("stereo_in_mono", 3, 0xF0, 0x10), ("ch_code8", 3, 0xF0, 0x80)):
        f = bytearray(frames[1]); f[byte] = (f[byte] & ~mask) | value; _refresh(f, HLEN)
        out.append((name, _join(head, frames[:1] + [f] + frames[2:])))
    for code in range(11, 16):
        f = bytearray(frames[1]); f[3] = (f[3] & 0x0F) | code << 4; _refresh(f, HLEN)
        out.append((f"ch_code{code}", _join(head, frames[:1] + [f] + frames[2:])))
    f = bytearray(frames[1]); f[2] = (f[2] & 0xF0) | 15; _refresh(f, HLEN)
    out.append(("rate_code15", _join(head, frames[:1] + [f] + frames[2:])))
    f = bytearray(frames[2]); f[4] = 3; _refresh(f, HLEN)              # frame 2 claims to be frame 3: a gap, then an overlap
    out.append(("gap", _join(head, frames[:2] + [f] + frames[3:])))
    for name, k, byte in (("flip_header", 1, 2), ("flip_residual", 1, None), ("flip_crc", 1, -1)):
        f = bytearray(frames[k]); f[len(f) // 2 if byte is None else byte] ^= 0x04
        out.append((name, _join(head, frames[:k] + [f] + frames[k + 1:])))
    # an escape wider than the sample size: the partition's samples run past the frame
    esc = lambda fi, c, v, sb: dict(kind="fixed", order=0, partition=0, escape=(0,), wasted=False)
    _, h2, fr2 = _short(esc)
    f = bytearray(fr2[1]); _set_bits(f, HLEN * 8 + 8 + 2 + 4 + 4, 5, 31); _refresh(f, HLEN)
    out.append(("escape31", _join(h2, fr2[:1] + [f] + fr2[2:])))
    # STREAMINFO damage
    si = bytearray(good); si[8 + 10] ^= 0xFF                           # sample rate / channels / bps bits
    out.append(("streaminfo_fields", bytes(si)))
    out.append(("no_streaminfo", good[:4] + bytes([0x81, 0, 0, 4]) + b"abcd" + good[4 + 38:]))
    out.append(("metadata_past_end", good[:4] + bytes([0x80, 0, 0, 34]) + good[8:30]))
    return x, out


def test_malformed_corpus_under_sanitizers(tmp_path):
    exe = build_flac_hostcheck(sanitize=True, out_dir=str(tmp_path))
    x, corpus = malformed_corpus()
    paths = []
    for name, data in corpus:
        p = tmp_path / f"{name}.flac"
        p.write_bytes(data)
        paths.append(str(p))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    r = subprocess.run([exe] + paths, capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "Sanitizer" not in r.stderr, r.stderr[-4000:]
    lines = r.stdout.strip().splitlines()
    assert len(lines) == len(paths)
    failed = 0
    for (name, _), line in zip(corpus, lines):
        st, off, path = line.split(" ", 2)
        if int(st) == 0:
            y = np.fromfile(path + ".s32", "<i4").reshape(-1, 1).astype(np.int64)
            assert np.array_equal(y, x), f"{name} decoded to something else"
        else:
            failed += 1
    assert failed == len(corpus), "every malformed file is refused"


# ------------------------------------------------------------------------------------------------ the C ABI without a device
def _n_out(path, **kw):
    from whisperkit_b200.audio import _load_opts
    o, keep = _load_opts(("sum", None), kw.get("startTime", 0.0), kw.get("endTime"), kw.get("maxReadFrameSize"), 0.0, 0)
    n = C.c_int64()
    _lib.check(_lib.load().wk_audio_load(None, path.encode(), C.byref(o), None, 0, C.byref(n)))
    return n.value


def test_info_and_lengths_without_a_device(tmp_path):
    jfk = jfk_s16()
    p = tmp_path / "jfk.flac"
    p.write_bytes(F.encode(jfk[:, None], 16000, 16, id3=F.id3v2(), metadata=F.ALL_METADATA))
    info = AudioProcessor.audioInfo(str(p))
    data = p.read_bytes()
    assert info == dict(sampleRate=16000, channels=1, sampleFormat="s16", blockAlign=2, frames=176000,
                        dataOffset=data.index(b"\xff\xf8", len(F.id3v2()) + 4 + 38))
    assert _n_out(str(p)) == 176000
    assert _n_out(str(p), startTime=1.2, endTime=3.4) == 35200
    for bps, fmt, ch in ((8, "s16", 2), (12, "s16", 1), (17, "s24", 6), (24, "s24", 8), (25, "s32", 2), (32, "s32", 3)):
        q = tmp_path / f"b{bps}.flac"
        q.write_bytes(F.encode(F.test_signal(44100 * 11, ch, bps), 44100, bps, block_size=4608))
        info = AudioProcessor.audioInfo(str(q))
        assert (info["sampleFormat"], info["channels"], info["blockAlign"], info["frames"]) == (fmt, ch, ch * {"s16": 2, "s24": 3, "s32": 4}[fmt],
                                                                                              44100 * 11)
        assert _n_out(str(q)) == 176000 and _n_out(str(q), startTime=1.2, maxReadFrameSize=10024) == 156800


def test_refused_files(tmp_path):
    x = F.test_signal(5000, 2, 16)
    good = F.encode(x, 16000, 16)
    cases = {
        "ogg": (b"OggS\x00\x02" + bytes(20) + b"\x7fFLAC" + good, "Ogg"),
        "total0": (F.encode(x, 16000, 16, streaminfo_total=0), "unknown length"),
        "no_streaminfo": (good[:4] + bytes([0x81, 0, 0, 4]) + b"abcd" + good[4 + 38:], "missing STREAMINFO"),
        "bad_streaminfo": (good[:8] + b"\x00\x08" + good[10:], "malformed STREAMINFO"),
        "bs_code0": (None, "block-size code 0"),
        "bps_code3": (None, "sample-size code 3"),
        "ch_code12": (None, "reserved channel code"),
        "id3_not_flac": (F.id3v2() + b"RIFF" + bytes(40), "ID3v2"),
        "text": (b"not audio at all", "RIFF/WAVE"),
    }
    head, frames = _frames(x, 16000, 16)
    hl = len(F.frame_header(4096, 16000, 1, 16, 0, False))
    for name, byte, value in (("bs_code0", 2, lambda b: b & 0x0F), ("bps_code3", 3, lambda b: (b & 0xF1) | 0x06),
                              ("ch_code12", 3, lambda b: (b & 0x0F) | 0xC0)):
        f = bytearray(frames[0]); f[byte] = value(f[byte]); _refresh(f, hl)
        cases[name] = (_join(head, [f] + frames[1:]), cases[name][1])
    for name, (data, needle) in cases.items():
        p = tmp_path / f"{name}.flac"
        p.write_bytes(data)
        for call in (lambda: AudioProcessor.audioInfo(str(p)), lambda: _n_out(str(p))):
            with pytest.raises(wk.WhisperError) as e:
                call()
            assert e.value.status == _lib.WK_ERR_LOAD_AUDIO_FAILED and e.value.case == "loadAudioFailed", name
            assert needle in str(e.value) and str(p) in str(e.value), (name, str(e.value))
    slow = tmp_path / "slow.flac"
    slow.write_bytes(F.encode(x, 500, 16))
    assert AudioProcessor.audioInfo(str(slow))["sampleRate"] == 500
    with pytest.raises(wk.WhisperError) as e:
        _n_out(str(slow))
    assert e.value.status == _lib.WK_ERR_INVALID_ARGUMENT


def test_md5_is_over_the_input():
    x = F.test_signal(3000, 2, 24)
    data = F.encode(x, 48000, 24)
    w = np.asarray(x, "<i4").view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    assert F.parse_streaminfo(data)["md5"] == hashlib.md5(w).digest()
