"""Writes the FLAC fixtures of tests/golden with an encoder independent of this project: FFmpeg's libavcodec FLAC encoder, driven through
ctypes (run once by hand; the tests only read the files it wrote).

    python tests/golden/make_flac_golden.py /path/to/libs     # a directory holding libavcodec / libavformat / libavutil (FFmpeg 7 or 8)

Fixtures:
    jfk_fast.flac, jfk_max.flac    jfk.wav at compression levels 0 and 12 (fixed predictors vs. LPC up to order 32 with partition search)
    tone24_<mode>.flac             1.2 s of a seeded 44.1 kHz stereo 24-bit signal per stereo mode the encoder offers
Each file's STREAMINFO carries the encoder's MD5 of its input, which tests/test_flac_host.py compares with the decoded samples."""
import ctypes as C
import glob
import os
import sys
import tempfile
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
AVERROR_EOF = -0x20464F45
EAGAIN = -11


def _load(libdir):
    # the directory's libraries depend on each other (a wheel's bundled libs carry hashed names): load them until every one loads
    pending, loaded = sorted(glob.glob(os.path.join(libdir, "*.so*"))), {}
    while pending:
        left = []
        for p in pending:
            try:
                loaded[os.path.basename(p)] = C.CDLL(p, mode=C.RTLD_GLOBAL)
            except OSError:
                left.append(p)
        if len(left) == len(pending):
            raise OSError(f"cannot load {left}")
        pending = left

    def one(stem):
        return next(v for k, v in loaded.items() if k.startswith(stem))
    u, c, f = one("libavutil"), one("libavcodec"), one("libavformat")
    for fn in ("avcodec_find_encoder_by_name", "avcodec_find_decoder", "avcodec_alloc_context3", "av_frame_alloc", "av_packet_alloc",
               "av_packet_get_side_data"):
        getattr(c if hasattr(c, fn) else u, fn).restype = C.c_void_p
    c.avcodec_parameters_alloc.restype = C.c_void_p
    u.av_frame_alloc.restype = C.c_void_p
    c.av_packet_get_side_data.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_size_t)]
    return u, c, f


def _check(r, what):
    if r < 0:
        raise RuntimeError(f"{what} failed: {r}")
    return r


def _stream_par(ic):
    """codecpar of the only stream of an AVFormatContext (field offsets of FFmpeg 7 / 8, checked against the WAV's known values)"""
    assert C.cast(ic.value + 44, C.POINTER(C.c_uint32))[0] == 1                     # nb_streams
    streams = C.cast(ic.value + 48, C.POINTER(C.POINTER(C.c_void_p)))[0]          # streams
    par = C.cast(streams[0] + 16, C.POINTER(C.c_void_p))[0]                          # AVStream.codecpar
    assert C.cast(par, C.POINTER(C.c_int32))[0] == 1                                 # codec_type AVMEDIA_TYPE_AUDIO
    return par


def _configure(u, c, ctx, par_in, enc, ch, width, level, ch_mode, extra):
    """Encoder context from a copy of the WAV's parameters with the codec id and sample format of the FLAC encoder, then its options."""
    par = C.c_void_p(c.avcodec_parameters_alloc())
    _check(c.avcodec_parameters_copy(par, C.c_void_p(par_in)), "parameters_copy")
    assert C.cast(par.value + 56, C.POINTER(C.c_int32))[0] == 8 * width                # bits_per_coded_sample
    C.cast(par.value + 4, C.POINTER(C.c_int32))[0] = C.cast(enc + 20, C.POINTER(C.c_int32))[0]   # codec_id = AVCodec.id
    C.cast(par.value + 44, C.POINTER(C.c_int32))[0] = 1 if width == 2 else 2          # format: AV_SAMPLE_FMT_S16 / S32
    C.cast(par.value + 60, C.POINTER(C.c_int32))[0] = 8 * width                        # bits_per_raw_sample
    _check(c.avcodec_parameters_to_context(ctx, par), "parameters_to_context")
    S = 1
    _check(u.av_opt_set(ctx, b"ch_layout", {1: b"mono", 2: b"stereo"}[ch], S), "ch_layout")
    _check(u.av_opt_set_int(ctx, b"compression_level", level, S), "compression_level")
    _check(u.av_opt_set(ctx, b"ch_mode", ch_mode.encode(), S), "ch_mode")
    for k, v in extra:
        _check(u.av_opt_set(ctx, k.encode(), str(v).encode(), S), k)
    _check(c.avcodec_open2(ctx, C.c_void_p(enc), None), "avcodec_open2")


def encode(libs, wav_path, out_path, level, ch_mode="auto", extra=()):
    u, c, f = libs
    with wave.open(wav_path, "rb") as w:
        ch, width, rate = w.getnchannels(), w.getsampwidth(), w.getframerate()
    enc = c.avcodec_find_encoder_by_name(b"flac")
    S = 1   # AV_OPT_SEARCH_CHILDREN
    # the encoder's frame size first (it follows the compression level), so the demuxer can cut packets of exactly that many samples
    probe = C.c_void_p(c.avcodec_alloc_context3(C.c_void_p(enc)))
    ic = C.c_void_p()
    _check(f.avformat_open_input(C.byref(ic), wav_path.encode(), None, None), "avformat_open_input")
    par_in = _stream_par(ic)
    _configure(u, c, probe, par_in, enc, ch, width, level, ch_mode, extra)
    fs = C.c_int64()
    _check(u.av_opt_get_int(probe, b"frame_size", 0, C.byref(fs)), "frame_size")
    f.avformat_close_input(C.byref(ic))
    opts = C.c_void_p()
    u.av_dict_set(C.byref(opts), b"max_size", str(fs.value * ch * width).encode(), 0)
    _check(f.avformat_open_input(C.byref(ic), wav_path.encode(), None, C.byref(opts)), "avformat_open_input")
    par = _stream_par(ic)
    ectx = C.c_void_p(c.avcodec_alloc_context3(C.c_void_p(enc)))
    _configure(u, c, ectx, par, enc, ch, width, level, ch_mode, extra)
    dec = c.avcodec_find_decoder(C.cast(par + 4, C.POINTER(C.c_int32))[0])
    dctx = C.c_void_p(c.avcodec_alloc_context3(C.c_void_p(dec)))
    _check(c.avcodec_parameters_to_context(dctx, C.c_void_p(par)), "parameters_to_context")
    _check(c.avcodec_open2(dctx, C.c_void_p(dec), None), "decoder open")
    pkt, opkt, frame = C.c_void_p(c.av_packet_alloc()), C.c_void_p(c.av_packet_alloc()), C.c_void_p(u.av_frame_alloc())
    frames, streaminfo = [], None

    def drain():
        nonlocal streaminfo
        while True:
            r = c.avcodec_receive_packet(ectx, opkt)
            if r in (EAGAIN, AVERROR_EOF):
                return
            _check(r, "receive_packet")
            data = C.cast(opkt.value + 24, C.POINTER(C.c_void_p))[0]
            size = C.cast(opkt.value + 32, C.POINTER(C.c_int32))[0]
            if size:
                frames.append(C.string_at(data, size))
            n = C.c_size_t()
            sd = c.av_packet_get_side_data(opkt, 1, C.byref(n))   # AV_PKT_DATA_NEW_EXTRADATA: the final STREAMINFO
            if sd:
                streaminfo = C.string_at(sd, n.value)
            c.av_packet_unref(opkt)

    while f.av_read_frame(ic, pkt) >= 0:
        _check(c.avcodec_send_packet(dctx, pkt), "send_packet")
        c.av_packet_unref(pkt)
        while c.avcodec_receive_frame(dctx, frame) >= 0:
            _check(c.avcodec_send_frame(ectx, frame), "send_frame")
            u.av_frame_unref(frame)
            drain()
    _check(c.avcodec_send_frame(ectx, None), "flush")
    drain()
    assert streaminfo is not None and len(streaminfo) == 34, "the encoder returned no final STREAMINFO"
    with open(out_path, "wb") as o:
        o.write(b"fLaC" + bytes([0x80, 0, 0, 34]) + streaminfo + b"".join(frames))
    f.avformat_close_input(C.byref(ic))
    print(f"{os.path.basename(out_path)}: {len(frames)} frames, {os.path.getsize(out_path)} bytes")


def tone24(path):
    rng = np.random.default_rng(2024)
    n = 44100 * 6 // 5
    t = np.arange(n) / 44100
    l = 0.4 * np.sin(2 * np.pi * 440 * t) + 0.1 * np.sin(2 * np.pi * 3150 * t) + 0.01 * rng.standard_normal(n)
    r = 0.7 * l + 0.2 * np.sin(2 * np.pi * 660 * t + 0.3) + 0.01 * rng.standard_normal(n)
    s = np.clip(np.round(np.stack([l, r], 1) * (2 ** 23 - 1)), -2 ** 23, 2 ** 23 - 1).astype("<i4")
    with wave.open(path, "wb") as w:
        w.setnchannels(2)
        w.setsampwidth(3)
        w.setframerate(44100)
        w.writeframes(s.view(np.uint8).reshape(-1, 4)[:, :3].tobytes())


def main(libdir):
    libs = _load(libdir)
    jfk = os.path.join(HERE, "jfk.wav")
    encode(libs, jfk, os.path.join(HERE, "jfk_fast.flac"), 0)
    encode(libs, jfk, os.path.join(HERE, "jfk_max.flac"), 12)
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "tone24.wav")
        tone24(src)
        for mode in ("indep", "left_side", "right_side", "mid_side"):
            encode(libs, src, os.path.join(HERE, f"tone24_{mode}.flac"), 8, ch_mode=mode)


if __name__ == "__main__":
    main(sys.argv[1])
