"""AudioStreamTranscriber (Sources/WhisperKit/Core/Audio/AudioStreamTranscriber.swift) for many live streams at once.

The caller pushes 16 kHz mono float audio per stream (`processBuffer`, named after AudioProcessor.processBuffer; microphone capture is
the host's business).  Every `transcribeCurrentBuffers()` call is one round: each stream whose new audio passes the reference's gates
(more than 1 s; AudioProcessor.isVoiceDetected with useVAD) is transcribed from its last confirmed segment end on, all of them in one
batched pass of the seek loop, with shouldStopEarly applied inside the decode loop; then each stream confirms segments as the
reference does.  All logic lives in libwkb200.so (csrc/streaming.cu)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import WK_ERR_INVALID_ARGUMENT, WhisperError, check, wk_segment, wk_stream_config, wk_stream_state
from .api import DecodingOptions
from .longform import TranscriptionSegment, _segs


@dataclass
class StreamState:
    """AudioStreamTranscriber.State, the fields a server reads, plus what the stream holds."""
    lastBufferSize: int = 0
    lastConfirmedSegmentEndSeconds: float = 0.0
    confirmedSegments: List[TranscriptionSegment] = field(default_factory=list)
    unconfirmedSegments: List[TranscriptionSegment] = field(default_factory=list)
    transcribed: bool = False          # the last round transcribed this stream
    pushedSamples: int = 0
    heldSamples: int = 0               # audio held from the current clip start on
    duplicateConfirmations: int = 0    # rounds whose confirmation candidates were already confirmed (the reference's `contains`, :178)


def _same(a: StreamState, b: StreamState) -> bool:
    def key(g):
        return (g.id, g.seek, g.start, g.end, tuple(g.tokens), tuple(g.tokenLogProbs))
    return (a.lastBufferSize == b.lastBufferSize and a.lastConfirmedSegmentEndSeconds == b.lastConfirmedSegmentEndSeconds
            and [key(g) for g in a.confirmedSegments] == [key(g) for g in b.confirmedSegments]
            and [key(g) for g in a.unconfirmedSegments] == [key(g) for g in b.unconfirmedSegments])


class AudioStreamTranscriber:
    """One streamer per DecodingOptions.  Beam search, bestOf, draftTokens and topLogProbs are not supported in streams
    (WK_ERR_INVALID_ARGUMENT)."""

    def __init__(self, kit, decodingOptions: Optional[DecodingOptions] = None, requiredSegmentsForConfirmation: int = 2,
                 silenceThreshold: float = 0.3, compressionCheckWindow: int = 60, useVAD: bool = True,
                 stateChangeCallback: Optional[Callable[[StreamState, StreamState], None]] = None, split_to_word_tokens=None, decode=None):
        opts = kit.resolveLanguage(decodingOptions or DecodingOptions())
        if opts.bestOf:
            raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"bestOf={opts.bestOf} is not supported in streams")
        if opts.draftTokens:
            raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"draftTokens={opts.draftTokens} is not supported in streams")
        if opts.biasPhrases is not None:
            raise WhisperError(WK_ERR_INVALID_ARGUMENT, "biasPhrases is not supported in streams")
        if opts.topLogProbs:
            raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"topLogProbs={opts.topLogProbs} is not supported in streams")
        self.kit, self.options, self.lib = kit, opts, kit.model.lib
        self.stateChangeCallback = stateChangeCallback
        prompt = kit.textDecoder.prefillDecoderInputs(opts if opts.usePrefillPrompt else None, kit.specialTokens)
        st = kit.specialTokens.to_c()
        o, self._keep_opts = opts.to_c()
        p = (C.c_int32 * len(prompt))(*prompt)
        cfg = wk_stream_config(int(requiredSegmentsForConfirmation), float(silenceThreshold), int(compressionCheckWindow), 1 if useVAD else 0)
        hooks = None
        self._keep_hooks = None
        if opts.wordTimestamps:
            # as longform.transcribe_audio: explicit callables, else the tokenizer's native hooks, else its splitToWordTokens / decode
            from .wordtiming import make_hooks
            tok = getattr(kit, "tokenizer", None)
            if split_to_word_tokens is not None:
                hooks, self._keep_hooks = make_hooks(split_to_word_tokens, decode)
            elif tok is not None and hasattr(tok, "hooks"):
                hooks = tok.hooks()
            elif tok is not None:
                hooks, self._keep_hooks = make_hooks(tok.splitToWordTokens, tok.decode)
        self._hooks = hooks
        self.handle = C.c_void_p()
        check(self.lib.wk_streamer_create(kit.model.handle, kit.textDecoder.handle, C.byref(st), C.byref(o), p, len(prompt), C.byref(cfg),
                                          C.byref(hooks) if hooks is not None else None, C.byref(self.handle)))
        self._ids: List[int] = []

    # -------------------------------------------------------------------------------------------------------------- streams
    def addStream(self) -> int:
        i = C.c_int32()
        check(self.lib.wk_streamer_add_stream(self.handle, C.byref(i)))
        self._ids.append(int(i.value))
        return int(i.value)

    def removeStream(self, id: int) -> None:
        check(self.lib.wk_streamer_remove_stream(self.handle, int(id)))
        self._ids.remove(int(id))

    def processBuffer(self, id: int, samples) -> None:
        x = np.ascontiguousarray(samples, dtype=np.float32)
        check(self.lib.wk_streamer_push(self.handle, int(id), C.c_void_p(x.ctypes.data) if len(x) else None, len(x)))

    # -------------------------------------------------------------------------------------------------------------- rounds
    def transcribeCurrentBuffers(self) -> List[int]:
        """One round: returns the ids of the streams it transcribed; stateChangeCallback(old, new) for every stream whose state changed."""
        ids = list(self._ids)
        before = {i: self.state(i) for i in ids} if self.stateChangeCallback else {}
        cap = max(1, len(ids))
        out = (C.c_int32 * cap)()
        n = C.c_int32()
        check(self.lib.wk_streamer_round(self.handle, out, cap, C.byref(n)))
        done = [int(out[k]) for k in range(n.value)]
        if self.stateChangeCallback:
            for i in ids:
                new = self.state(i)
                if not _same(before[i], new):
                    self.stateChangeCallback(before[i], new)
        return done

    def state(self, id: int) -> StreamState:
        s = wk_stream_state()
        check(self.lib.wk_streamer_state(self.handle, int(id), C.byref(s)))
        segs = self._segments(id)
        nc = s.n_confirmed_segments
        return StreamState(int(s.last_buffer_size), float(s.last_confirmed_segment_end_seconds), segs[:nc], segs[nc:], bool(s.transcribed),
                           int(s.pushed_samples), int(s.held_samples), int(s.duplicate_confirmations))

    def _segments(self, id: int) -> List[TranscriptionSegment]:
        lib = self.lib
        h = C.c_void_p()
        check(lib.wk_streamer_result(self.handle, int(id), C.byref(h)))
        try:
            ns, nt = lib.wk_transcription_segment_count(h), lib.wk_transcription_token_count(h)
            raw = (wk_segment * max(1, ns))()
            check(lib.wk_transcription_segments(h, raw, max(1, ns)))
            tk = (C.c_int32 * max(1, nt))()
            lp = (C.c_float * max(1, nt))()
            check(lib.wk_transcription_tokens(h, tk, lp, max(1, nt)))
            segs = _segs(raw, ns, tk, lp)
            if self.options.wordTimestamps:
                from .wordtiming import WordTiming
                for g in segs:
                    g.words = []
                w = _lib.wk_word()
                for i in range(lib.wk_transcription_word_count(h)):
                    check(lib.wk_transcription_word(h, i, C.byref(w)))
                    segs[w.segment].words.append(WordTiming(w.word.decode("utf-8"), [int(w.tokens[k]) for k in range(w.n_tokens)],
                                                            float(w.start), float(w.end), float(w.probability), int(w.segment)))
        finally:
            lib.wk_transcription_free(h)
        tok = getattr(self.kit, "tokenizer", None)
        if tok is not None:
            sb = self.kit.specialTokens.specialTokenBegin
            for g in segs:
                g.text = tok.decode([t for t in g.tokens if t < sb] if self.options.skipSpecialTokens else g.tokens)
        return segs

    def close(self) -> None:
        if self.handle:
            self.lib.wk_streamer_free(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------------------------ host helpers
def relativeEnergy(samples) -> np.ndarray:
    """processBuffer's relative energies of the complete 1600-sample blocks of `samples` (AudioProcessor.swift:724-741,907-917)."""
    x = np.ascontiguousarray(samples, dtype=np.float32)
    cap = len(x) // 1600 + 1
    out = np.zeros(cap, np.float32)
    n = C.c_int64()
    check(_lib.load().wk_stream_relative_energy(C.c_void_p(x.ctypes.data) if len(x) else None, len(x), C.c_void_p(out.ctypes.data), cap, C.byref(n)))
    return out[: n.value].copy()


def isVoiceDetected(relativeEnergy: Sequence[float], nextBufferInSeconds: float, silenceThreshold: float) -> bool:
    """AudioProcessor.isVoiceDetected (AudioProcessor.swift:636-655)."""
    e = np.ascontiguousarray(relativeEnergy, dtype=np.float32)
    out = C.c_int32()
    check(_lib.load().wk_stream_voice_detected(C.c_void_p(e.ctypes.data) if len(e) else None, len(e), float(nextBufferInSeconds),
                                               float(silenceThreshold), C.byref(out)))
    return bool(out.value)
