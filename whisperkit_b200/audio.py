"""AudioProcessor: audio files and in-memory frames at any sample rate and channel layout -> 16 kHz mono float32 on the GPU.

Mirrors the loading half of Sources/WhisperKit/Core/Audio/AudioProcessor.swift over the C ABI (csrc/audio.cu, csrc/flac.cu):

  AudioProcessor.loadAudio(path, ...)          loadAudio(fromPath:channelMode:startTime:endTime:maxReadFrameSize:)  :229-305
  AudioProcessor.loadAudioAsFloatArray(path)   loadAudioAsFloatArray(fromPath:...)  (600 s pieces)                  :307-350
  AudioProcessor.loadAudio(at=paths)           loadAudio(at:channelMode:) -> [Result<[Float], Error>]               :352-371
  AudioProcessor.resampleAudio(frames, rate)   convertToMono + resampleAudio on interleaved frames in memory        :381-625

A channel mode is ("sum", None | [indices]) for ChannelMode.sumChannels or ("channel", i) for ChannelMode.specificChannel.  Files: WAV
(PCM u8/s16/s24/s32, IEEE float 32, plain or EXTENSIBLE) and native FLAC (1-8 channels, 4-32 bits, decoded on the GPU; it loads bit for
bit like a WAV file of the same integers); other files (lossy formats, Ogg) fail with WhisperError case "loadAudioFailed".  The resampler is
scipy.signal.resample_poly's Kaiser-windowed polyphase filter (include/wkb200.h has the exact contract)."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from ._lib import WhisperError, check, wk_audio_format, wk_audio_load_opts

DEFAULT_READ_FRAME_SIZE = 1_323_000   # Constants.defaultAudioReadFrameSize
PIECE_SECONDS = 600.0                 # loadAudioAsFloatArray reads 10 minutes at a time
SAMPLE_FORMATS = {"u8": _lib.WK_AUDIO_U8, "s16": _lib.WK_AUDIO_S16, "s24": _lib.WK_AUDIO_S24, "s32": _lib.WK_AUDIO_S32,
                  "f32": _lib.WK_AUDIO_F32}
_FORMAT_NAMES = {v: k for k, v in SAMPLE_FORMATS.items()}
_DTYPE_FORMATS = {"uint8": "u8", "int16": "s16", "int32": "s32", "float32": "f32"}

ChannelModeT = Tuple[str, Union[None, int, Sequence[int]]]


class ChannelMode:
    """AudioInputConfig.ChannelMode as plain tuples."""

    @staticmethod
    def sumChannels(indices: Optional[Sequence[int]] = None) -> ChannelModeT:
        return ("sum", None if indices is None else [int(i) for i in indices])

    @staticmethod
    def specificChannel(index: int) -> ChannelModeT:
        return ("channel", int(index))


DEFAULT_CHANNEL_MODE: ChannelModeT = ("sum", None)


def _session_handle(session):
    if session is None:
        return None
    return getattr(session, "handle", session)


def _load_opts(channelMode: ChannelModeT, startTime: Optional[float], endTime: Optional[float], maxReadFrameSize: Optional[int],
               pieceSeconds: float, segmentSamples: int):
    """wk_audio_load_opts and the int array it points into."""
    o = wk_audio_load_opts()
    keep = None
    kind, arg = channelMode
    if kind == "channel":
        o.channel_mode, o.channel = _lib.WK_CHANNELS_SPECIFIC, int(arg)
    elif kind == "sum":
        o.channel_mode = _lib.WK_CHANNELS_SUM
        if arg is not None and len(arg) > 0:
            keep = (C.c_int32 * len(arg))(*[int(i) for i in arg])
            o.channel_indices, o.n_channel_indices = C.cast(keep, C.POINTER(C.c_int32)), len(arg)
    else:
        raise ValueError(f"channel mode must be ('sum', indices) or ('channel', i), not {channelMode!r}")
    o.start_time = float(startTime or 0.0)
    o.has_end_time = 0 if endTime is None else 1
    o.end_time = 0.0 if endTime is None else float(endTime)
    o.max_read_frame_size = int(maxReadFrameSize or 0)
    o.piece_seconds = float(pieceSeconds)
    o.segment_samples = int(segmentSamples)
    return o, keep


def _run(fn, out):
    """Calls fn(out_ptr, cap, n_ptr) twice: for the length, then into `out` (or a new host array)."""
    n = C.c_int64()
    if out is None:
        check(fn(None, 0, C.byref(n)))
        out = np.empty(n.value, dtype=np.float32)
        if n.value == 0:
            return out
    cap = out.numel() if hasattr(out, "numel") else out.size
    ptr = C.c_void_p(out.data_ptr()) if hasattr(out, "data_ptr") else C.c_void_p(out.ctypes.data)
    check(fn(ptr, cap, C.byref(n)))
    return out[: n.value]


class AudioProcessor:
    @staticmethod
    def audioInfo(path: str) -> dict:
        """The WAV or FLAC header: sampleRate, channels, sampleFormat ("u8" ... "f32"; for FLAC the WAV container it loads as), blockAlign,
        frames, dataOffset (host only)."""
        f = wk_audio_format()
        check(_lib.load().wk_audio_info(path.encode(), C.byref(f)))
        return dict(sampleRate=f.sample_rate, channels=f.channels, sampleFormat=_FORMAT_NAMES[f.sample_format], blockAlign=f.block_align,
                    frames=f.frames, dataOffset=f.data_offset)

    @staticmethod
    def loadAudio(fromPath: Optional[str] = None, channelMode: ChannelModeT = DEFAULT_CHANNEL_MODE, startTime: Optional[float] = 0.0,
                  endTime: Optional[float] = None, maxReadFrameSize: Optional[int] = None, *, at: Optional[Sequence[str]] = None,
                  session=None, out=None, segmentSamples: int = 0, pieceSeconds: float = 0.0):
        """16 kHz mono float32 samples of a WAV or FLAC file (numpy, or `out` - a float32 host array or CUDA tensor - trimmed to the length).
        With at=paths: loadAudio(at:) - per path the loadAudioAsFloatArray samples, or the WhisperError that path raised.
        session: a TextDecoder (its CUDA stream and staging buffers) or None (a stream for this call)."""
        if at is not None:
            out_list: List[object] = []
            for p in at:
                try:
                    out_list.append(AudioProcessor.loadAudioAsFloatArray(p, channelMode, session=session))
                except WhisperError as e:
                    out_list.append(e)
            return out_list
        if fromPath is None:
            raise ValueError("loadAudio needs a path (or at=paths)")
        lib = _lib.load()
        o, keep = _load_opts(channelMode, startTime, endTime, maxReadFrameSize, pieceSeconds, segmentSamples)
        h, path = _session_handle(session), fromPath.encode()
        return _run(lambda ptr, cap, n: lib.wk_audio_load(h, path, C.byref(o), ptr, cap, n), out)

    @staticmethod
    def loadAudioAsFloatArray(fromPath: str, channelMode: ChannelModeT = DEFAULT_CHANNEL_MODE, startTime: Optional[float] = 0.0,
                              endTime: Optional[float] = None, *, maxReadFrameSize: Optional[int] = None, session=None, out=None,
                              segmentSamples: int = 0):
        """loadAudioAsFloatArray: loadAudio over 600 s pieces of the file (each piece's read chunks normalised on their own)."""
        return AudioProcessor.loadAudio(fromPath, channelMode, startTime, endTime, maxReadFrameSize, session=session, out=out,
                                        segmentSamples=segmentSamples, pieceSeconds=PIECE_SECONDS)

    @staticmethod
    def resampleAudio(frames, sampleRate: int, channelMode: ChannelModeT = DEFAULT_CHANNEL_MODE, *, sampleFormat: Optional[str] = None,
                      channels: Optional[int] = None, startTime: Optional[float] = 0.0, endTime: Optional[float] = None,
                      maxReadFrameSize: Optional[int] = None, session=None, out=None, segmentSamples: int = 0):
        """convertToMono + resampleAudio for interleaved frames in memory: a [frames, channels] (or [frames]) array of uint8 / int16 /
        int32 / float32, numpy or torch (host or CUDA).  24-bit samples are uint8 [frames, 3 * channels] with sampleFormat="s24".  The
        result equals loadAudio of a WAV file holding the same frames."""
        dt = str(frames.dtype).replace("torch.", "")
        fmt = sampleFormat or _DTYPE_FORMATS.get(dt)
        if fmt not in SAMPLE_FORMATS:
            raise ValueError(f"unsupported sample dtype {dt} / format {sampleFormat!r}")
        if hasattr(frames, "data_ptr"):
            frames = frames.contiguous()
            ptr = C.c_void_p(frames.data_ptr())
        else:
            frames = np.ascontiguousarray(frames)
            ptr = C.c_void_p(frames.ctypes.data)
        n = int(frames.shape[0])
        width = 1 if frames.ndim == 1 else int(frames.shape[1])
        if channels is None:
            channels = width // 3 if fmt == "s24" else width
        lib = _lib.load()
        o, keep = _load_opts(channelMode, startTime, endTime, maxReadFrameSize, 0.0, segmentSamples)
        h = _session_handle(session)
        return _run(lambda optr, cap, nout: lib.wk_audio_convert(h, ptr, SAMPLE_FORMATS[fmt], n, int(channels), int(sampleRate), C.byref(o),
                                                                 optr, cap, nout), out)


def filter_taps(sampleRate: int):
    """The resampler's filter design (host only): (taps float64 = firwin(...) * up, up, down)."""
    lib = _lib.load()
    up, down, n = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib.wk_audio_filter_taps(int(sampleRate), None, 0, C.byref(up), C.byref(down), C.byref(n)))
    taps = np.zeros(max(1, n.value), dtype=np.float64)
    check(lib.wk_audio_filter_taps(int(sampleRate), taps.ctypes.data_as(C.POINTER(C.c_double)), taps.size, C.byref(up), C.byref(down),
                                   C.byref(n)))
    return taps[: n.value], up.value, down.value
