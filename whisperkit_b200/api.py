"""Host-side mirror of the reference's protocol surface over the C ABI (ctypes).

Class / method names follow WhisperKit so parity tests read like the reference's own tests:

  FeatureExtractor.logMelSpectrogram      Sources/WhisperKit/Core/FeatureExtractor.swift:13-17,40-56
  AudioEncoder.encodeFeatures             Sources/WhisperKit/Core/AudioEncoder.swift:10-18,50-63
  TextDecoder.{prepareDecoderInputs,      Sources/WhisperKit/Core/TextDecoder.swift:60-105
     prefillDecoderInputs, predictLogits, decodeText}
  DecodingOptions                         Sources/WhisperKit/Core/Configurations.swift:155-247
  SpecialTokens                           Sources/WhisperKit/Core/Models.swift:1111-1149
  WhisperKit.transcribe(audioArrays:)     Sources/WhisperKit/Core/WhisperKit.swift:667-812

All arithmetic happens in libwkb200.so (sm_90a kernels); this module only marshals arguments.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Union

import numpy as np

from . import _lib
from ._lib import (PROGRESS_FN, WK_DTYPE_BF16, WK_DTYPE_F16, WK_DTYPE_F32, WK_ERR_INVALID_ARGUMENT, WhisperError, check, wk_batch_opts, wk_decode_opts,
                   wk_decode_result, wk_model_config, wk_model_info, wk_special_tokens)

MAX_TOKEN_CONTEXT = 224  # Constants.maxTokenContext (Models.swift:1334)
MAX_TOP_LOGPROBS = 20    # DecodingOptions.topLogProbs limit (OpenAI's top_logprobs)
WINDOW_SAMPLES = 480000  # Constants.defaultWindowSamples (Models.swift:1457)
FALLBACK_REASONS = {0: None, 1: "firstTokenLogProbThreshold", 2: "silence", 3: "compressionRatioThreshold",
                    4: "logProbThreshold"}
# Whisper's language codes in vocabulary order: <|en|> is englishToken, the rest follow it (Constants.languages, Models.swift)
LANGUAGE_CODES = (
    "en zh de es ru ko fr ja pt tr pl ca nl ar sv it id hi fi vi he uk el ms cs ro da hu ta no th ur hr bg lt la mi ml cy sk te fa lv bn "
    "sr az sl kn et mk br eu is hy ne mn bs kk sq sw gl mr pa si km sn yo so af oc ka be tg sd gu am yi lo uz fo ht ps tk nn mt sa lb "
    "my bo tl mg as tt haw ln ha ba jw su yue").split()


def language_tokens(specialTokens: "SpecialTokens", vocab: int, tokenizer=None) -> List[int]:
    """tokenizer.allLanguageTokens: the tokenizer's <|xx|> ids, or without one the vocabulary's language block
    [englishToken, translateToken) (100 ids on large-v3, 99 on the older multilingual vocabularies); [] for an English-only model."""
    if vocab == 51864:
        return []
    if tokenizer is not None:
        ids = [tokenizer.convertTokenToId(f"<|{c}|>") for c in LANGUAGE_CODES]
        return [int(i) for i in ids if i is not None and 0 <= i < vocab]
    return list(range(specialTokens.englishToken, specialTokens.translateToken))


def _ptr(x):
    """Raw address of a numpy array or torch tensor (host or device)."""
    if x is None:
        return None
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    return C.c_void_p(x.ctypes.data)


@dataclass
class SpecialTokens:
    endToken: int = 50257
    englishToken: int = 50259
    noSpeechToken: int = 50362
    noTimestampsToken: int = 50363
    specialTokenBegin: int = 50257
    startOfPreviousToken: int = 50361
    startOfTranscriptToken: int = 50258
    timeTokenBegin: int = 50364
    transcribeToken: int = 50359
    translateToken: int = 50358
    whitespaceToken: int = 220

    def to_c(self) -> wk_special_tokens:
        return wk_special_tokens(self.endToken, self.englishToken, self.noSpeechToken, self.noTimestampsToken,
                                 self.specialTokenBegin, self.startOfPreviousToken, self.startOfTranscriptToken,
                                 self.timeTokenBegin, self.transcribeToken, self.translateToken, self.whitespaceToken)

    @staticmethod
    def from_any(o) -> "SpecialTokens":
        return SpecialTokens(**{k: getattr(o, k) for k in SpecialTokens().__dict__})


@dataclass
class DecodingOptions:
    task: str = "transcribe"
    language: Optional[str] = None
    languageToken: Optional[int] = None  # id of "<|language|>" (tokenizer lookup is the host's job)
    temperature: float = 0.0
    temperatureIncrementOnFallback: float = 0.2
    temperatureFallbackCount: int = 5
    sampleLength: int = MAX_TOKEN_CONTEXT
    topK: int = 5
    usePrefillPrompt: bool = True
    skipSpecialTokens: bool = False
    withoutTimestamps: bool = False
    maxInitialTimestamp: Optional[float] = None
    promptTokens: Optional[List[int]] = None
    prefixTokens: Optional[List[int]] = None
    suppressBlank: bool = False
    suppressTokens: List[int] = field(default_factory=list)
    compressionRatioThreshold: Optional[float] = 2.4
    logProbThreshold: Optional[float] = -1.0
    firstTokenLogProbThreshold: Optional[float] = -1.5
    noSpeechThreshold: Optional[float] = 0.6
    concurrentWorkerCount: int = 16
    wordTimestamps: bool = False
    seed: int = 0
    beamSize: int = 1                 # extension: the reference's BeamSearchTokenSampler is an unimplemented stub (TokenSampler.swift:254-290)
    beamPatience: float = 1.0
    # detect each window's language inside the decode loop (multilingual model, no language set); None = !usePrefillPrompt, as the
    # reference resolves it (Configurations.swift:222)
    detectLanguage: Optional[bool] = None
    allLanguageTokens: Optional[List[int]] = None   # tokenizer.allLanguageTokens; WhisperKit.resolveLanguage fills it
    # compute DecodingResult.noSpeechProb in the decode loop (openai/whisper's rule; the reference leaves it 0), so that noSpeechThreshold
    # marks silent windows (fallback reason "silence") and the long-form loop skips them
    computeNoSpeechProb: bool = False
    # best-of-N sampling inside the temperature ladder (openai/whisper's best_of; the reference's DecodingOptions has none): None = off,
    # as before (a beam call skips the ladder); >= 1 = openai's decode_with_fallback - beam search at temperature 0 when beamSize > 1,
    # bestOf samples (the most likely kept) at temperature > 0, on every rung of the ladder, beam calls included.  One value per call
    # (C: wk_batch_opts.best_of, wk_transcribe_streams_ex)
    bestOf: Optional[int] = None
    # speculative greedy decoding with the model's draft decoder (Model.loadDraftDecoder / setDraftDecoder): 0 = off; k in 1..7 = the
    # draft proposes k tokens per round and the model checks them in one step.  Against draftTokens=0 on a session with as many decode
    # slots (maxBatch / (k + 1)), windows decoded at temperature 0 are byte-identical, and every window is when the call has no more
    # windows than slots; with more, a temperature > 0 draw follows the slot a window lands in, which the draft's timing changes (C
    # header, wk_transcribe_windows_draft).  A progress callback that stops
    # a window takes effect at a round boundary.  One value per call; refused with beamSize > 1, bestOf, wordTimestamps and streams
    # (C: wk_transcribe_windows_draft, wk_decode_text_draft, wk_transcribe_streams_draft)
    draftTokens: int = 0
    # contextual biasing inside the fused decode loop (C: wk_bias_create / wk_session_set_bias): phrases whose tokens earn biasBoost per
    # matched token while a partial match lasts, kept once the phrase completes.  A string is tokenized twice through the kit's tokenizer,
    # as encode(" " + s) and encode(s); a list of ints is taken as given.  Reported log-probs and thresholds stay the model's own.  The
    # 2.0 default is not tuned on a real checkpoint.  Refused with draftTokens and in AudioStreamTranscriber
    biasPhrases: Optional[List[Union[str, List[int]]]] = None
    biasBoost: float = 2.0
    # the k most likely tokens and their log-probs at every sampled position (DecodingResult.topLogProbs, TranscriptionSegment.topLogProbs):
    # k in 0..20, 0 = off.  Ranked on the filtered row the choice was made from, with the normaliser of tokenLogProbs (the tempered one
    # at temperature > 0; the model's own values under biasPhrases).  One value per call; refused with beamSize > 1, draftTokens and in
    # AudioStreamTranscriber (C: wk_session_set_top_logprobs)
    topLogProbs: int = 0

    @property
    def detectsLanguage(self) -> bool:
        return bool(self.detectLanguage) if self.detectLanguage is not None else not self.usePrefillPrompt

    def to_c(self):
        """Returns (struct, keepalive) - keepalive holds the int arrays the struct points into."""
        keep = []

        def arr(v):
            if v is None:
                return None, -1
            a = (C.c_int32 * max(1, len(v)))(*v)
            keep.append(a)
            return C.cast(a, C.POINTER(C.c_int32)), len(v)

        sup, nsup = arr(list(self.suppressTokens))
        pr, npr = arr(self.promptTokens)
        pf, npf = arr(self.prefixTokens)

        def opt(v):
            return (0, 0.0) if v is None else (1, float(v))

        o = wk_decode_opts()
        o.task_translate = 1 if self.task == "translate" else 0
        o.language_token = -1 if self.languageToken is None else int(self.languageToken)
        o.temperature = float(self.temperature)
        o.sample_length = int(self.sampleLength)
        o.top_k = int(self.topK)
        o.use_prefill_prompt = int(self.usePrefillPrompt)
        o.without_timestamps = int(self.withoutTimestamps)
        o.suppress_blank = int(self.suppressBlank)
        o.suppress_tokens, o.n_suppress_tokens = sup, max(nsup, 0)
        o.prompt_tokens, o.n_prompt_tokens = pr, npr
        o.prefix_tokens, o.n_prefix_tokens = pf, npf
        o.has_compression_ratio_threshold, o.compression_ratio_threshold = opt(self.compressionRatioThreshold)
        o.has_logprob_threshold, o.logprob_threshold = opt(self.logProbThreshold)
        o.has_first_token_logprob_threshold, o.first_token_logprob_threshold = opt(self.firstTokenLogProbThreshold)
        o.has_no_speech_threshold, o.no_speech_threshold = opt(self.noSpeechThreshold)
        o.seed = int(self.seed)
        o.temperature_fallback_count = int(self.temperatureFallbackCount)
        o.temperature_increment_on_fallback = float(self.temperatureIncrementOnFallback)
        o.word_timestamps = int(self.wordTimestamps)
        o.beam_size = int(self.beamSize)
        o.beam_patience = float(self.beamPatience)
        o.detect_language = int(self.detectsLanguage)
        lt, nlt = arr(self.allLanguageTokens)
        o.language_tokens, o.n_language_tokens = lt, max(nlt, 0)
        o.compute_no_speech_prob = int(self.computeNoSpeechProb)
        return o, keep


@dataclass
class DecodingFallback:
    needsFallback: bool
    fallbackReason: str


@dataclass
class DecodingResult:
    """Models.swift:383-439 (token-level fields; text needs the host tokenizer)."""
    tokens: List[int]
    tokenLogProbs: List[float]
    avgLogProb: float
    compressionRatio: float
    temperature: float
    fallback: Optional[DecodingFallback]
    currentTokenCount: int = 0
    steps: int = 0
    isFirstTokenLogProbTooLow: bool = False
    # the language detected in the decode loop (detectLanguage): <|xx|> id, its log-prob, and "xx" when a tokenizer is present
    languageToken: Optional[int] = None
    languageLogProb: Optional[float] = None
    language: Optional[str] = None
    noSpeechProb: float = 0.0   # DecodingOptions.computeNoSpeechProb; 0 where it was not computed, as in the reference
    # DecodingOptions.topLogProbs: one {token: logprob} per tokenLogProbs entry, best first; empty for forced prompt positions and the
    # closing EOT, and an empty list when the option is 0
    topLogProbs: List[Dict[int, float]] = field(default_factory=list)

    @staticmethod
    def from_c(r: wk_decode_result) -> "DecodingResult":
        n = r.n_tokens
        reason = FALLBACK_REASONS.get(r.fallback_reason)
        fb = DecodingFallback(bool(r.needs_fallback), reason) if reason else None
        return DecodingResult(list(r.tokens[:n]), list(r.token_logprobs[:n]), r.avg_logprob, r.compression_ratio,
                              r.temperature, fb, r.n_current_tokens, r.steps, bool(r.first_token_logprob_too_low))


def language_code(tokenizer, token: int) -> str:
    """DecodingResult.language of a detected <|xx|> token (TextDecoder.swift:516-523): its code, or "en" when the code is unknown."""
    code = tokenizer.decode([int(token)]).strip()
    if code.startswith("<|") and code.endswith("|>"):
        code = code[2:-2]
    return code if code in LANGUAGE_CODES else "en"


def session_languages(lib, session, n: int):
    """wk_session_languages for windows [0, n) of the session's last batched call: (tokens, logprobs), -1 / 0 = no detection."""
    tok = (C.c_int32 * max(1, n))()
    lp = (C.c_float * max(1, n))()
    check(lib.wk_session_languages(session, 0, n, tok, lp))
    return [int(v) for v in tok[:n]], [float(v) for v in lp[:n]]


def session_no_speech_probs(lib, session, n: int) -> List[float]:
    """wk_session_no_speech_probs for windows [0, n) of the session's last batched call; NaN = not computed."""
    out = (C.c_float * max(1, n))()
    check(lib.wk_session_no_speech_probs(session, 0, n, out))
    return [float(v) for v in out[:n]]


def attach_no_speech_probs(results: List["DecodingResult"], probs: Sequence[float]) -> None:
    for r, p in zip(results, probs):
        if isinstance(r, DecodingResult):
            r.noSpeechProb = 0.0 if math.isnan(p) else p


def top_logprob_dicts(tokens: Sequence[int], logprobs: Sequence[float], n: int, k: int) -> List[Dict[int, float]]:
    """The flat [n][k] pairs of wk_session_top_logprobs / wk_transcription_top_logprobs as one dict per position, best first; the -1
    padding is dropped."""
    out = []
    for i in range(n):
        d: Dict[int, float] = {}
        for j in range(i * k, i * k + k):
            if int(tokens[j]) >= 0:
                d[int(tokens[j])] = float(logprobs[j])
        out.append(d)
    return out


def attach_top_logprobs(lib, session, results: List["DecodingResult"], k: int) -> None:
    """DecodingResult.topLogProbs of every result of the session's last batched call that ran with topLogProbs = k."""
    if k == 0:
        return
    for w, r in enumerate(results):
        if not isinstance(r, DecodingResult):
            continue
        n = len(r.tokens)
        tok = (C.c_int32 * max(1, n * k))()
        lp = (C.c_float * max(1, n * k))()
        check(lib.wk_session_top_logprobs(session, w, n, tok, lp))
        r.topLogProbs = top_logprob_dicts(tok, lp, n, k)


def attach_languages(results: List["DecodingResult"], tokens: Sequence[int], logprobs: Sequence[float], tokenizer=None) -> None:
    for r, t, lp in zip(results, tokens, logprobs):
        if isinstance(r, DecodingResult) and t >= 0:
            r.languageToken, r.languageLogProb = int(t), float(lp)
            r.language = language_code(tokenizer, t) if tokenizer is not None else None


_DT = {"f32": WK_DTYPE_F32, "f16": WK_DTYPE_F16, "bf16": WK_DTYPE_BF16}
# cross-attention K/V cache storage (Model(crossKVDtype=...)): None keeps the model's dtype
_CKV_DT = {"fp8": _lib.WK_DTYPE_FP8_E4M3, "f16": WK_DTYPE_F16, "bf16": WK_DTYPE_BF16}


def _check_storage_dtypes(crossKVDtype: Optional[str], encoderDtype: Optional[str] = None) -> None:
    if crossKVDtype is not None and crossKVDtype not in _CKV_DT:
        raise ValueError(f"crossKVDtype must be one of {sorted(_CKV_DT)} or None, not {crossKVDtype!r}")
    if encoderDtype is not None and encoderDtype not in _CKV_DT:
        raise ValueError(f"encoderDtype must be one of {sorted(_CKV_DT)} or None, not {encoderDtype!r}")


class Model:
    """Owns a wk_model (weights + encoder workspaces on one GPU).

    crossKVDtype="fp8" stores the decoder's cross-attention K/V cache as E4M3 codes with one f32 scale per 64-value row
    (wk_model_set_cross_kv_dtype): about half the cache memory and the bytes the decode loop streams; None keeps `dtype`.

    encoderDtype="fp8" runs the encoder's QKV, FC1 and FC2 GEMMs on the FP8 tensor cores (wk_model_set_encoder_dtype): E4M3
    activations with one f32 scale per (row, 128-column block), E4M3 weight copies with one scale per output channel; the encoder output
    stays `dtype`.  None keeps `dtype`."""

    def __init__(self, variant: str = "large-v3", device: int = 0, max_batch: int = 16, dtype: str = "bf16",
                 config: Optional[dict] = None, crossKVDtype: Optional[str] = None, encoderDtype: Optional[str] = None):
        self.lib = _lib.load()
        _check_storage_dtypes(crossKVDtype, encoderDtype)
        cfg = wk_model_config()
        self.lib.wk_default_config(variant.encode(), C.byref(cfg))
        if config:
            for k, v in config.items():
                setattr(cfg, k, v)
        cfg.max_batch = max_batch
        cfg.dtype = _DT[dtype]
        self.cfg = cfg
        self.handle = C.c_void_p()
        check(self.lib.wk_model_create(C.byref(cfg), device, C.byref(self.handle)))
        self.variant = variant
        self.device = device
        self._set_storage_dtypes(crossKVDtype, encoderDtype)

    @classmethod
    def from_pretrained(cls, weights_dir: str, device: int = 0, max_batch: int = 16, dtype: str = "bf16",
                        crossKVDtype: Optional[str] = None, encoderDtype: Optional[str] = None) -> "Model":
        """HuggingFace checkpoint directory (config.json + *.safetensors)."""
        self = cls.__new__(cls)
        self.lib = _lib.load()
        _check_storage_dtypes(crossKVDtype, encoderDtype)
        self.handle = C.c_void_p()
        check(self.lib.wk_model_load(weights_dir.encode(), device, max_batch, _DT[dtype], C.byref(self.handle)))
        info = wk_model_info()
        check(self.lib.wk_model_info_get(self.handle, C.byref(info)))
        cfg = wk_model_config()
        for f in ("n_mels", "d_model", "n_heads", "enc_layers", "dec_layers", "vocab", "n_audio_ctx", "dtype", "max_batch"):
            setattr(cfg, f, getattr(info, f))
        self.cfg, self.variant, self.device = cfg, os.path.basename(weights_dir.rstrip("/")), device
        self._set_storage_dtypes(crossKVDtype, encoderDtype)
        return self

    def _set_storage_dtypes(self, crossKVDtype: Optional[str], encoderDtype: Optional[str] = None) -> None:
        try:
            if crossKVDtype is not None:
                check(self.lib.wk_model_set_cross_kv_dtype(self.handle, _CKV_DT[crossKVDtype]))
            if encoderDtype is not None:
                check(self.lib.wk_model_set_encoder_dtype(self.handle, _CKV_DT[encoderDtype]))
        except WhisperError:
            self.close()   # the model was created for this call: do not leak it
            raise

    def set_tensor(self, name: str, t) -> None:
        self._store(self.lib.wk_model_set_tensor, name, t)

    def _store(self, fn, name: str, t) -> None:
        if hasattr(t, "data_ptr"):
            import torch
            t = t.contiguous()
            dt = {torch.float32: WK_DTYPE_F32, torch.float16: WK_DTYPE_F16, torch.bfloat16: WK_DTYPE_BF16}[t.dtype]
            shape = list(t.shape)
        else:
            t = np.ascontiguousarray(t)
            dt = {np.dtype("float32"): WK_DTYPE_F32, np.dtype("float16"): WK_DTYPE_F16}[t.dtype]
            shape = list(t.shape)
        shp = (C.c_int64 * len(shape))(*shape)
        check(fn(self.handle, name.encode(), _ptr(t), dt, shp, len(shape)))

    def loadDraftDecoder(self, weights_dir: str) -> None:
        """The draft decoder for speculative decoding (DecodingOptions.draftTokens) from an HF Whisper checkpoint directory: its
        model.decoder.* tensors only (distil-large-v3 for large-v3).  Before the model's first session."""
        check(self.lib.wk_model_load_draft(self.handle, weights_dir.encode()))

    def setDraftDecoder(self, decLayers: int, weights: Optional[Dict[str, object]] = None, seed: Optional[int] = None,
                        std: float = 0.02) -> None:
        """A draft decoder of decLayers layers (the model's dimensions): seeded random weights when seed is given, then `weights` (HF
        decoder names -> tensors) on top.  Before the model's first session."""
        check(self.lib.wk_model_create_draft(self.handle, int(decLayers)))
        if seed is not None:
            check(self.lib.wk_model_init_draft_random(self.handle, int(seed), float(std)))
        for k, v in (weights or {}).items():
            self._store(self.lib.wk_model_set_draft_tensor, k, v)

    @property
    def draftLayers(self) -> int:
        n = C.c_int32()
        check(self.lib.wk_model_draft_layers(self.handle, C.byref(n)))
        return n.value

    def load_state_dict(self, weights: Dict[str, object]) -> None:
        for k, v in weights.items():
            self.set_tensor(k, v)
        check(self.lib.wk_model_finalize(self.handle))

    def setAlignmentHeads(self, pairs: Sequence[Sequence[int]]) -> None:
        """(layer, head) pairs averaged into `alignment_heads_weights`; [] restores the default (all heads of the last half of the layers)."""
        flat = [int(v) for p in pairs for v in p]
        arr = (C.c_int32 * max(1, len(flat)))(*flat)
        check(self.lib.wk_model_set_alignment_heads(self.handle, arr, len(flat) // 2))

    def init_random(self, seed: int = 0, std: float = 0.02) -> None:
        check(self.lib.wk_model_init_random(self.handle, seed, std))

    @property
    def info(self) -> wk_model_info:
        i = wk_model_info()
        check(self.lib.wk_model_info_get(self.handle, C.byref(i)))
        return i

    @property
    def stream(self) -> int:
        return int(self.lib.wk_model_stream(self.handle) or 0)

    def last_timings(self) -> dict:
        a = (C.c_float * 6)()
        check(self.lib.wk_last_timings(self.handle, a))
        return dict(zip(("logmels", "encoding", "crossKV", "decodingLoop", "h2d", "d2h"), [float(x) for x in a]))

    def close(self):
        if getattr(self, "handle", None) and self.handle.value:
            self.lib.wk_model_free(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceTensor:
    """Opaque device buffer handed between mel -> encoder -> decoder (the reference's marker protocols
    FeatureExtractorOutputType / AudioEncoderOutputType allow exactly this, FeatureExtractor.swift:10-11).  Owns its buffer, like the
    MLMultiArray the reference returns: released with the object."""

    def __init__(self, model: Model, handle):
        self.model, self.handle = model, handle

    def close(self):
        if getattr(self, "handle", None) and self.handle.value and getattr(self.model, "handle", None) and self.model.handle.value:
            self.model.lib.wk_tensor_free(self.handle)
        self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def shape(self):
        shp = (C.c_int64 * 4)()
        nd, dt = C.c_int32(), C.c_int32()
        check(self.model.lib.wk_tensor_shape(self.handle, shp, C.byref(nd), C.byref(dt)))
        return tuple(shp[: nd.value])

    def numpy(self, row_pad: int = 0) -> np.ndarray:
        """Reference layout, f32: mel [B, nMels, 3000]; encoder output [B, d, 1500].  row_pad > 0 reads back through explicit element
        strides into rows padded by that many elements (how an IOSurface-backed MLMultiArray lays its rows out)."""
        b, c, _, t = self.shape
        if row_pad:
            buf = np.zeros((b, c, t + row_pad), dtype=np.float32)
            check(self.model.lib.wk_tensor_to_host_strided(self.handle, _ptr(buf), c * (t + row_pad), t + row_pad, 1, buf.size))
            return buf[:, :, :t]
        out = np.empty((b, c, t), dtype=np.float32)
        check(self.model.lib.wk_tensor_to_host(self.handle, _ptr(out), out.size))
        return out


class FeatureExtractor:
    def __init__(self, model: Model):
        self.model = model

    @property
    def melCount(self) -> int:
        return self.model.info.n_mels

    @property
    def windowSamples(self) -> int:
        return self.model.info.window_samples

    def logMelSpectrogram(self, audio, samples_per_window: Optional[Sequence[int]] = None) -> DeviceTensor:
        """audio: [B, stride] (or [stride]) float32, numpy or torch (host or CUDA)."""
        if not hasattr(audio, "data_ptr"):
            audio = np.ascontiguousarray(audio, dtype=np.float32)
        if audio.ndim == 1:
            audio = audio[None]
        n, stride = int(audio.shape[0]), int(audio.shape[1])
        spw = None
        if samples_per_window is not None:
            spw = (C.c_int32 * n)(*[int(v) for v in samples_per_window])
        out = C.c_void_p()
        check(self.model.lib.wk_mel(self.model.handle, _ptr(audio), n, stride, spw, C.byref(out)))
        return DeviceTensor(self.model, out)


class AudioEncoder:
    def __init__(self, model: Model):
        self.model = model

    @property
    def embedSize(self) -> int:
        return self.model.info.d_model

    @property
    def sequenceLength(self) -> int:
        return self.model.info.n_audio_ctx

    def encodeFeatures(self, features: DeviceTensor) -> DeviceTensor:
        out = C.c_void_p()
        check(self.model.lib.wk_encode(self.model.handle, features.handle, C.byref(out)))
        return DeviceTensor(self.model, out)


class TextDecoder:
    """One decoding session (per-worker DecodingInputs + device KV caches)."""

    def __init__(self, model: Model, max_batch: Optional[int] = None):
        self.model = model
        self.lib = model.lib
        self.max_batch = max_batch or model.cfg.max_batch
        self.handle = C.c_void_p()
        check(self.lib.wk_session_create(model.handle, self.max_batch, C.byref(self.handle)))
        self.batch = 0

    # properties the reference reads off the CoreML model (TextDecoder.swift:313-331)
    @property
    def logitsSize(self) -> int:
        return self.model.info.vocab

    @property
    def kvCacheEmbedDim(self) -> int:
        return self.model.info.kv_embed_dim

    @property
    def kvCacheMaxSequenceLength(self) -> int:
        return self.model.info.kv_max_len

    @property
    def windowSize(self) -> int:
        return self.model.info.n_audio_ctx

    @property
    def embedSize(self) -> int:
        return self.model.info.d_model

    @property
    def isModelMultilingual(self) -> bool:
        return bool(self.model.info.is_multilingual)

    def prepareDecoderInputs(self) -> None:
        check(self.lib.wk_session_reset(self.handle))

    def prefillDecoderInputs(self, options: Optional[DecodingOptions], specialTokens: SpecialTokens) -> List[int]:
        st = specialTokens.to_c()
        o, keep = (options or DecodingOptions()).to_c()
        out = (C.c_int32 * MAX_TOKEN_CONTEXT)()
        n = C.c_int32()
        check(self.lib.wk_build_prompt(self.model.handle, C.byref(st), C.byref(o), 1 if options is not None else 0, out,
                                       MAX_TOKEN_CONTEXT, C.byref(n)))
        return list(out[: n.value])

    def bindEncoderOutput(self, enc: DeviceTensor) -> None:
        check(self.lib.wk_session_set_encoder_output(self.handle, enc.handle))
        self.batch = enc.shape[0]

    def predictLogits(self, inputIds: Sequence[int], cacheLength: Sequence[int]) -> np.ndarray:
        b = self.batch
        ids = (C.c_int32 * b)(*[int(v) for v in inputIds])
        cl = (C.c_int32 * b)(*[int(v) for v in cacheLength])
        out = np.empty((b, self.logitsSize), dtype=np.float32)
        check(self.lib.wk_decode_step(self.handle, ids, cl, _ptr(out)))
        return out

    def decodeText(self, encoderOutput: Optional[DeviceTensor], prompt, options, specialTokens: SpecialTokens,
                   callback=None, callbackEvery: int = 0) -> List[DecodingResult]:
        """decodeText for every bound window.  `prompt` / `options` may be one shared value or one per window;
        callback(window, tokens, avgLogprob) -> bool is the TranscriptionCallback (False = stop that window early)."""
        if encoderOutput is not None:
            self.bindEncoderOutput(encoderOutput)
        st = specialTokens.to_c()
        n = self.batch
        opts = [with_language_tokens(o, specialTokens, self.logitsSize) for o in options] if isinstance(options, (list, tuple)) \
            else with_language_tokens(options, specialTokens, self.logitsSize)
        bo, keep = make_batch_opts(n, opts, prompt, callback, callbackEvery, None)
        res = (wk_decode_result * n)()
        draft = draft_tokens_of(opts)
        top = top_logprobs_of(opts)
        with attached_bias(self.lib, self.handle, opts, specialTokens), top_logprobs_set(self.lib, self.handle, top):
            if draft:
                check(self.lib.wk_decode_text_draft(self.handle, C.byref(st), C.byref(bo), draft, res))
            else:
                check(self.lib.wk_decode_text_ex(self.handle, C.byref(st), C.byref(bo), res))
        out = [DecodingResult.from_c(r) for r in res]
        attach_languages(out, *session_languages(self.lib, self.handle, n))
        attach_no_speech_probs(out, session_no_speech_probs(self.lib, self.handle, n))
        attach_top_logprobs(self.lib, self.handle, out, top)
        return out

    def detectLanguage(self, encoderOutput: Optional[DeviceTensor], specialTokens: SpecialTokens, allLanguageTokens: Sequence[int],
                       temperature: float = 0.0):
        """TextDecoder.detectLanguage: returns (language_token[B], logprob[B])."""
        if encoderOutput is not None:
            self.bindEncoderOutput(encoderOutput)
        st = specialTokens.to_c()
        lang = (C.c_int32 * len(allLanguageTokens))(*[int(v) for v in allLanguageTokens])
        tok = (C.c_int32 * self.batch)()
        lp = (C.c_float * self.batch)()
        check(self.lib.wk_detect_language(self.handle, C.byref(st), lang, len(allLanguageTokens), float(temperature), tok, lp))
        return list(tok), list(lp)

    def alignmentWeights(self, window: int, rows: int = MAX_TOKEN_CONTEXT) -> np.ndarray:
        """DecodingResult.cache.alignmentWeights of one window of the last decodeText(wordTimestamps: true): [rows, 1500] (Float16 values)."""
        out = np.empty((rows, self.model.info.n_audio_ctx), dtype=np.float32)
        check(self.lib.wk_session_alignment_weights(self.handle, window, rows, _ptr(out)))
        return out

    def alignTokens(self, encoderOutput: Optional[DeviceTensor], tokenLists: Sequence[Sequence[int]], specialTokens: SpecialTokens,
                    returnErrors: bool = False):
        """Forced alignment of one token sequence per bound window (openai-whisper's find_alignment pass): each sequence is the full decoder
        input - prompt, text, EOT, e.g. DecodingResult.tokens.  Returns per window (alignmentWeights [n+1, 1500] f32, tokenLogProbs [n] f32),
        the weights in the decode loop's layout for WordTimingSeeker.findAlignment / addWordTimestamps.  With returnErrors a window whose
        sequence is invalid yields its WhisperError instead of failing the call."""
        if encoderOutput is not None:
            self.bindEncoderOutput(encoderOutput)
        st = specialTokens.to_c()
        flat, offsets = _flatten_token_lists(tokenLists)
        n = len(tokenLists)
        status = (C.c_int32 * n)()
        check(self.lib.wk_align_tokens(self.handle, C.byref(st), _ptr(flat), _ptr(offsets), n, status))
        return aligned_results(self.lib, self.handle, tokenLists, status, returnErrors, self.model.info.n_audio_ctx)

    def alignedLogProbs(self, window: int, n: int) -> np.ndarray:
        """tokenLogProbs of one window of the last alignTokens / WhisperKit.align call."""
        out = np.empty(n, dtype=np.float32)
        check(self.lib.wk_session_aligned_logprobs(self.handle, window, n, _ptr(out)))
        return out

    def stats(self) -> dict:
        """Scheduler counters of the last batched call (decode steps launched, live-row steps, admissions, ladder re-admissions)."""
        a = (C.c_int64 * 4)()
        check(self.lib.wk_session_stats(self.handle, a))
        return dict(zip(("steps", "row_steps", "admissions", "ladder"), [int(v) for v in a]))

    def draftStats(self) -> dict:
        """Speculative decoding counters of the last batched call (DecodingOptions.draftTokens): rounds that verified proposals, the
        proposals verified, the proposals accepted."""
        a = (C.c_int64 * 3)()
        check(self.lib.wk_session_draft_stats(self.handle, a))
        return dict(zip(("rounds", "proposed", "accepted"), [int(v) for v in a]))

    def lastLogits(self) -> np.ndarray:
        out = np.empty((self.batch, self.logitsSize), dtype=np.float32)
        check(self.lib.wk_session_last_logits(self.handle, _ptr(out)))
        return out

    def close(self):
        if getattr(self, "handle", None) and self.handle.value:
            self.lib.wk_session_free(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _flatten_token_lists(tokenLists: Sequence[Sequence[int]]):
    """Token sequences -> (flat int32 array, int32 offsets of n + 1 entries), the layout of wk_align_tokens / wk_align_windows."""
    lens = [len(t) for t in tokenLists]
    offsets = np.zeros(len(lens) + 1, dtype=np.int32)
    offsets[1:] = np.cumsum(lens)
    flat = np.zeros(max(1, int(offsets[-1])), dtype=np.int32)
    for i, t in enumerate(tokenLists):
        flat[offsets[i]:offsets[i + 1]] = np.asarray(list(t), dtype=np.int64)
    return flat, offsets


def aligned_results(lib, session, tokenLists, status, returnErrors: bool, n_audio_ctx: int):
    """Per-window (alignmentWeights [n+1, T], tokenLogProbs [n]) of the session's last align call; failed windows raise (or, with returnErrors,
    yield their WhisperError)."""
    out = []
    for i, t in enumerate(tokenLists):
        if status[i] != 0:
            err = WhisperError(int(status[i]), f"window {i}: " + lib.wk_last_error().decode("utf-8", "replace"))
            if not returnErrors:
                raise err
            out.append(err)
            continue
        n = len(t)
        w = np.empty((n + 1, n_audio_ctx), dtype=np.float32)
        check(lib.wk_session_alignment_weights(session, i, n + 1, _ptr(w)))
        lp = np.empty(n, dtype=np.float32)
        check(lib.wk_session_aligned_logprobs(session, i, n, _ptr(lp)))
        out.append((w, lp))
    return out


def with_language_tokens(opts: DecodingOptions, specialTokens: SpecialTokens, vocab: int, tokenizer=None) -> DecodingOptions:
    """Fills DecodingOptions.allLanguageTokens when the options detect the language and carry no list."""
    if opts.allLanguageTokens is not None or not opts.detectsLanguage or vocab == 51864:
        return opts
    import dataclasses
    return dataclasses.replace(opts, allLanguageTokens=language_tokens(specialTokens, vocab, tokenizer))


def draft_tokens_of(options) -> int:
    """The call's DecodingOptions.draftTokens: one value for every window (C: the draft_tokens argument of wk_transcribe_windows_draft)."""
    opt_list = list(options) if isinstance(options, (list, tuple)) else [options]
    draft = {int(o.draftTokens or 0) for o in opt_list}
    if len(draft) != 1:
        raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"draftTokens must be the same for every window of a call (got {sorted(draft)})")
    return draft.pop()


def top_logprobs_of(options) -> int:
    """The call's DecodingOptions.topLogProbs: one value in [0, 20] for every window."""
    opt_list = list(options) if isinstance(options, (list, tuple)) else [options]
    ks = {int(o.topLogProbs or 0) for o in opt_list}
    if len(ks) != 1:
        raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"topLogProbs must be the same for every window of a call (got {sorted(ks)})")
    k = ks.pop()
    if not 0 <= k <= MAX_TOP_LOGPROBS:
        raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"topLogProbs {k} outside [0, {MAX_TOP_LOGPROBS}]")
    return k


@contextlib.contextmanager
def top_logprobs_set(lib, session, k: int):
    """Sets the session's topLogProbs to k for one call and back to 0 after it."""
    if k == 0:
        yield
        return
    check(lib.wk_session_set_top_logprobs(session, k))
    try:
        yield
    finally:
        check(lib.wk_session_set_top_logprobs(session, 0))


def bias_phrase_tokens(phrases, tokenizer=None) -> List[List[int]]:
    """DecodingOptions.biasPhrases as token phrases: a string gives encode(" " + s) and encode(s) (distinct spellings once each), a list
    of ints is taken as given."""
    out: List[List[int]] = []
    for ph in phrases:
        if isinstance(ph, str):
            if tokenizer is None:
                raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"biasPhrases entry {ph!r} needs a tokenizer (or pass token ids)")
            for t in (tokenizer.encode(" " + ph), tokenizer.encode(ph)):
                if list(t) not in out:
                    out.append([int(v) for v in t])
        else:
            out.append([int(v) for v in ph])
    return out


@contextlib.contextmanager
def attached_bias(lib, session, options, specialTokens: "SpecialTokens", tokenizer=None):
    """Attaches the bias sets of `options` (one DecodingOptions, or one per window / stream) to the session for the duration of one call
    and detaches them after it.  Options with the same phrases and boost share one set; options without phrases leave their windows
    unbiased.  Does nothing when no option carries phrases."""
    opt_list = list(options) if isinstance(options, (list, tuple)) else [options]
    if all(o.biasPhrases is None for o in opt_list):
        yield
        return
    handles, by_key = [], {}
    try:
        for o in opt_list:
            if o.biasPhrases is None:
                handles.append(None)
                continue
            phrases = bias_phrase_tokens(o.biasPhrases, tokenizer)
            key = (tuple(tuple(p) for p in phrases), float(o.biasBoost))
            if key not in by_key:
                flat = [t for p in phrases for t in p]
                toks = (C.c_int32 * max(1, len(flat)))(*flat)
                lens = (C.c_int32 * max(1, len(phrases)))(*[len(p) for p in phrases])
                h = C.c_void_p()
                check(lib.wk_bias_create(toks, lens, len(phrases), float(o.biasBoost), int(specialTokens.specialTokenBegin), C.byref(h)))
                by_key[key] = h
            handles.append(by_key[key])
        arr = (C.c_void_p * len(handles))(*[h.value if h is not None else None for h in handles])
        check(lib.wk_session_set_bias(session, arr, len(handles)))
        try:
            yield
        finally:
            check(lib.wk_session_set_bias(session, None, 0))
    finally:
        for h in by_key.values():
            lib.wk_bias_free(h)


def make_batch_opts(n: int, options, prompt, callback=None, callbackEvery: int = 0, status=None, encoderChunk: int = 0):
    """wk_batch_opts for n windows.  options: DecodingOptions or a list of n; prompt: None (built per window from the options), one token
    list, or a list of n token lists.  Returns (struct, keepalive)."""
    keep = []
    bo = wk_batch_opts()
    opt_list = list(options) if isinstance(options, (list, tuple)) else [options]
    if len(opt_list) not in (1, n):
        raise ValueError(f"{len(opt_list)} DecodingOptions for {n} windows")
    arr = (wk_decode_opts * len(opt_list))()
    for i, o in enumerate(opt_list):
        c, k = o.to_c()
        arr[i] = c
        keep.append(k)
    keep.append(arr)
    bo.opts, bo.n_opts = arr, len(opt_list)
    best_of = {int(o.bestOf or 0) for o in opt_list}
    if len(best_of) != 1:
        raise WhisperError(WK_ERR_INVALID_ARGUMENT, f"bestOf must be the same for every window of a call (got {sorted(best_of)})")
    bo.best_of = best_of.pop()
    draft_tokens_of(opt_list)
    if prompt is not None and len(prompt) > 0 and isinstance(prompt[0], (list, tuple, np.ndarray)):
        if len(prompt) != n:
            raise ValueError(f"{len(prompt)} prompts for {n} windows")
        rows = [(C.c_int32 * max(1, len(p)))(*[int(v) for v in p]) for p in prompt]
        ptrs = (C.POINTER(C.c_int32) * n)(*[C.cast(r, C.POINTER(C.c_int32)) for r in rows])
        lens = (C.c_int32 * n)(*[len(p) for p in prompt])
        keep += [rows, ptrs, lens]
        bo.prompts, bo.prompt_lens = ptrs, lens
    elif prompt is not None:
        p = (C.c_int32 * max(1, len(prompt)))(*[int(v) for v in prompt])
        keep.append(p)
        bo.prompt, bo.n_prompt = p, len(prompt)
    if callback is not None:
        def tramp(user, window, tokens, n_tokens, avg):
            try:
                return 1 if callback(int(window), [int(tokens[i]) for i in range(n_tokens)], float(avg)) is not False else 0
            except Exception:
                return 0
        fn = PROGRESS_FN(tramp)
        keep.append(fn)
        bo.progress = fn
    bo.progress_every = int(callbackEvery)
    if status is not None:
        bo.status = status
    bo.encoder_chunk = int(encoderChunk)
    return bo, keep


def filter_and_sample(model: Model, logits: np.ndarray, tokens: Sequence[Sequence[int]], specialTokens: SpecialTokens,
                      options: Optional[DecodingOptions] = None, isModelMultilingual: bool = True,
                      timestampSampleBegin: Optional[int] = None, blankSampleBegin: Optional[int] = None,
                      languageTokens: Optional[Sequence[int]] = None, languageSampleBegin: int = 0):
    """LogitsFiltering chain (SuppressBlank, SuppressTokens, TimestampRules, Language) + GreedyTokenSampler.update on
    the device, stateless.  Returns (token[B], logprob[B], filtered_logits[B, V])."""
    lib = model.lib
    logits = np.ascontiguousarray(logits, dtype=np.float32)
    if logits.ndim == 1:
        logits = logits[None]
    b, v = logits.shape
    ld = max(1, max((len(t) for t in tokens), default=1))
    tk = np.zeros((b, ld), dtype=np.int32)
    nt = np.zeros(b, dtype=np.int32)
    for i, t in enumerate(tokens):
        tk[i, : len(t)] = t
        nt[i] = len(t)
    st = specialTokens.to_c()
    o, keep = (options or DecodingOptions()).to_c()
    tok = np.zeros(b, dtype=np.int32)
    lp = np.zeros(b, dtype=np.float32)
    filt = np.zeros((b, v), dtype=np.float32)
    lang = np.asarray(list(languageTokens), dtype=np.int32) if languageTokens is not None else None
    check(lib.wk_filter_sample(model.handle, C.byref(st), C.byref(o), int(isModelMultilingual), _ptr(logits), b, v,
                               _ptr(tk), ld, _ptr(nt), -1 if timestampSampleBegin is None else timestampSampleBegin,
                               -1 if blankSampleBegin is None else blankSampleBegin, _ptr(lang),
                               0 if lang is None else len(lang), languageSampleBegin, _ptr(tok), _ptr(lp), _ptr(filt)))
    return tok, lp, filt


@dataclass
class WhisperKitConfig:
    """Configurations.swift:7-121, fields meaningful on this backend."""
    model: str = "large-v3"
    device: int = 0
    maxBatch: int = 16
    dtype: str = "bf16"
    specialTokens: Optional[SpecialTokens] = None
    weights: Optional[Dict[str, object]] = None  # HF-named tensors; None -> seeded random weights
    seed: int = 0
    modelFolder: Optional[str] = None            # HuggingFace checkpoint directory: config.json + *.safetensors (+ tokenizer.json / vocab.json)
    crossKVDtype: Optional[str] = None           # "fp8": E4M3 cross-attention K/V cache (Model); None = dtype
    encoderDtype: Optional[str] = None           # "fp8": encoder QKV / FC1 / FC2 GEMMs on E4M3 operands (Model); None = dtype
    draftModelFolder: Optional[str] = None       # HF checkpoint whose decoder becomes the draft of DecodingOptions.draftTokens (Model.loadDraftDecoder)
    # audioInputConfig.channelMode: how transcribe(audioPath=...) mixes multi-channel files, ("sum", None | [indices]) or ("channel", i)
    channelMode: tuple = ("sum", None)


class WhisperKit:
    """Orchestrator: transcribe(audioArrays:) fans a batch of <=30 s windows through mel -> encoder -> decoder on the
    GPU (WhisperKit.swift:667-812 + the per-window body of TranscribeTask.run, TranscribeTask.swift:116-278)."""

    def __init__(self, config: WhisperKitConfig):
        self.config = config
        self.tokenizer = None
        if config.modelFolder is not None:
            # loadModels + loadTokenizer from a local folder (WhisperKit.swift:358-470): weights through the safetensors loader, the
            # decode-side tokenizer when the folder carries tokenizer.json or vocab.json
            self.model = Model.from_pretrained(config.modelFolder, config.device, config.maxBatch, config.dtype, config.crossKVDtype,
                                               config.encoderDtype)
            if any(os.path.exists(os.path.join(config.modelFolder, f)) for f in ("tokenizer.json", "vocab.json")):
                from .tokenizer import WhisperTokenizer
                self.tokenizer = WhisperTokenizer(config.modelFolder)
        else:
            self.model = Model(config.model, config.device, config.maxBatch, config.dtype, crossKVDtype=config.crossKVDtype,
                               encoderDtype=config.encoderDtype)
            if config.weights is not None:
                self.model.load_state_dict(config.weights)
            else:
                self.model.init_random(config.seed)
        if config.draftModelFolder is not None:
            self.model.loadDraftDecoder(config.draftModelFolder)
        self.featureExtractor = FeatureExtractor(self.model)
        self.audioEncoder = AudioEncoder(self.model)
        self.textDecoder = TextDecoder(self.model, config.maxBatch)
        info = self.model.info
        if config.specialTokens is not None:
            self.specialTokens = config.specialTokens
        elif self.tokenizer is not None:
            self.specialTokens = self.tokenizer.specialTokens
        elif info.vocab == 51866:
            self.specialTokens = SpecialTokens(endToken=50257, englishToken=50259, noSpeechToken=50363,
                                               noTimestampsToken=50364, specialTokenBegin=50257,
                                               startOfPreviousToken=50362, startOfTranscriptToken=50258,
                                               timeTokenBegin=50365, transcribeToken=50360, translateToken=50359)
        elif info.vocab == 51864:
            self.specialTokens = SpecialTokens(endToken=50256, englishToken=50258, noSpeechToken=50361,
                                               noTimestampsToken=50362, specialTokenBegin=50256,
                                               startOfPreviousToken=50360, startOfTranscriptToken=50257,
                                               timeTokenBegin=50363, transcribeToken=50358, translateToken=50357)
        else:
            self.specialTokens = SpecialTokens()

    def resolveLanguage(self, opts: DecodingOptions) -> DecodingOptions:
        """DecodingOptions.language -> the "<|xx|>" token id through the tokenizer, as prefillDecoderInputs does with
        tokenizer.convertTokenToId (TextDecoder.swift:181-186).  No tokenizer = an error, never a silent <|en|>.  Options that detect
        the language get allLanguageTokens (the tokenizer's <|xx|> ids, else the vocabulary's language block)."""
        if opts.language is None and opts.languageToken is None:
            return with_language_tokens(opts, self.specialTokens, self.model.info.vocab, self.tokenizer)
        if opts.language is None or opts.languageToken is not None or not self.textDecoder.isModelMultilingual:
            return opts
        if self.tokenizer is None:
            raise WhisperError(-4, f"DecodingOptions.language={opts.language!r} needs a tokenizer to resolve <|{opts.language}|> (or set languageToken)")
        tok = self.tokenizer.convertTokenToId(f"<|{opts.language}|>")
        if tok is None or tok < 0:
            raise WhisperError(-4, f"the tokenizer has no <|{opts.language}|> token")
        import dataclasses
        return dataclasses.replace(opts, languageToken=int(tok))

    def transcribe(self, audioArrays=None, decodeOptions=None, samplesPerWindow: Optional[Sequence[int]] = None, callback=None,
                   callbackEvery: int = 0, returnErrors: bool = False, encoderChunk: int = 0, *, audioPath: Optional[str] = None,
                   audioPaths: Optional[Sequence[str]] = None, chunkingStrategy: Optional[str] = None):
        """audioArrays: host float32 [N, stride<=480000-padded] (numpy, or pinned torch CPU tensor).  decodeOptions: one DecodingOptions
        or one per window (transcribeWithOptions' decodeOptionsArray, WhisperKit.swift:716-735).  One DecodingResult per window, in order;
        with returnErrors a window that failed yields its WhisperError instead of failing the call (the reference's Result<>, :775-790).

        audioPath= / audioPaths= (WhisperKit.swift:587-640, 823-860): audio files of any length, sample rate and channel layout, loaded
        with AudioProcessor.loadAudioAsFloatArray (config.channelMode) on this kit's session and transcribed together by
        longform.transcribe_audio (decodeOptions: one DecodingOptions).  audioPath returns its TranscriptionResult or raises; audioPaths
        returns one TranscriptionResult per path, or the WhisperError that path's load raised."""
        if audioPath is not None or audioPaths is not None:
            if audioArrays is not None or (audioPath is not None and audioPaths is not None):
                raise ValueError("pass one of audioArrays, audioPath, audioPaths")
            res = self._transcribe_paths([audioPath] if audioPath is not None else list(audioPaths), decodeOptions, chunkingStrategy)
            if audioPath is not None and isinstance(res[0], WhisperError):
                raise res[0]
            return res[0] if audioPath is not None else res
        a = audioArrays
        if not hasattr(a, "data_ptr"):
            a = np.ascontiguousarray(a, dtype=np.float32)
        if a.ndim == 1:
            a = a[None]
        n, stride = int(a.shape[0]), int(a.shape[1])
        if isinstance(decodeOptions, (list, tuple)):
            opts = [self.resolveLanguage(o or DecodingOptions()) for o in decodeOptions]
        else:
            opts = self.resolveLanguage(decodeOptions or DecodingOptions())
        st = self.specialTokens.to_c()
        status = (C.c_int32 * n)() if returnErrors else None
        bo, keep = make_batch_opts(n, opts, None, callback, callbackEvery, status, encoderChunk)
        spw = None
        if samplesPerWindow is not None:
            spw = (C.c_int32 * n)(*[int(v) for v in samplesPerWindow])
        res = (wk_decode_result * n)()
        # the prompt of every window is built inside the library from that window's options (prefillDecoderInputs); decodeWithFallback
        # (TranscribeTask.swift:316-411) runs there too: a window whose DecodingFallback asks for it is decoded again at the next temperature
        draft = draft_tokens_of(opts)
        top = top_logprobs_of(opts)
        with attached_bias(self.model.lib, self.textDecoder.handle, opts, self.specialTokens, self.tokenizer), \
                top_logprobs_set(self.model.lib, self.textDecoder.handle, top):
            if draft:
                check(self.model.lib.wk_transcribe_windows_draft(self.model.handle, self.textDecoder.handle, _ptr(a), n, stride, spw,
                                                                 C.byref(st), C.byref(bo), draft, res))
            else:
                check(self.model.lib.wk_transcribe_windows_ex(self.model.handle, self.textDecoder.handle, _ptr(a), n, stride, spw,
                                                              C.byref(st), C.byref(bo), res))
        self.textDecoder.batch = min(n, self.config.maxBatch)
        out = []
        for i, r in enumerate(res):
            if returnErrors and status[i] != 0:
                out.append(WhisperError(int(status[i]), f"window {i} failed"))
            else:
                out.append(DecodingResult.from_c(r))
        attach_languages(out, *session_languages(self.model.lib, self.textDecoder.handle, n), tokenizer=self.tokenizer)
        attach_no_speech_probs(out, session_no_speech_probs(self.model.lib, self.textDecoder.handle, n))
        attach_top_logprobs(self.model.lib, self.textDecoder.handle, out, top)
        return out

    def _transcribe_paths(self, paths: Sequence[str], decodeOptions, chunkingStrategy: Optional[str]):
        from . import longform
        from .audio import AudioProcessor
        loaded = AudioProcessor.loadAudio(at=paths, channelMode=self.config.channelMode, session=self.textDecoder)
        good = [a for a in loaded if not isinstance(a, WhisperError)]
        results = iter(longform.transcribe_audio(self, good, decodeOptions, tokenizer=self.tokenizer, chunkingStrategy=chunkingStrategy)
                       if good else [])
        return [a if isinstance(a, WhisperError) else next(results) for a in loaded]

    def align(self, audioArrays, tokenLists: Sequence[Sequence[int]], samplesPerWindow: Optional[Sequence[int]] = None,
              returnErrors: bool = False):
        """Forced alignment of one token sequence per <=30 s window (audioArrays as transcribe takes them; each sequence the full decoder
        input: prompt, text, EOT - e.g. a DecodingResult.tokens, beam search included).  Returns per window (alignmentWeights [n+1, 1500] f32,
        tokenLogProbs [n] f32); words then come from WordTimingSeeker.findAlignment / addWordTimestamps."""
        a = audioArrays
        if not hasattr(a, "data_ptr"):
            a = np.ascontiguousarray(a, dtype=np.float32)
        if a.ndim == 1:
            a = a[None]
        n, stride = int(a.shape[0]), int(a.shape[1])
        if len(tokenLists) != n:
            raise ValueError(f"{len(tokenLists)} token sequences for {n} windows")
        st = self.specialTokens.to_c()
        flat, offsets = _flatten_token_lists(tokenLists)
        spw = None if samplesPerWindow is None else (C.c_int32 * n)(*[int(v) for v in samplesPerWindow])
        status = (C.c_int32 * n)()
        lib = self.model.lib
        check(lib.wk_align_windows(self.model.handle, self.textDecoder.handle, _ptr(a), n, stride, spw, C.byref(st), _ptr(flat), _ptr(offsets),
                                   status))
        return aligned_results(lib, self.textDecoder.handle, tokenLists, status, returnErrors, self.model.info.n_audio_ctx)
