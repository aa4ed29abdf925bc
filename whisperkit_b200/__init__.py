"""whisperkit_b200 - Hopper (sm_90a) implementation of WhisperKit's hot path behind its protocol surface.

The compute lives in libwkb200.so (hand-written CUDA: wgmma/TMA GEMMs, fused log-mel, attention, fused
filter+sampler); this package is the thin host mirror of the reference interface over the C ABI
(include/wkb200.h).  Importing the package is cheap; the shared library is loaded on first use and its
absence is an error (there is no CPU / PyTorch fallback).
"""
from ._lib import WhisperError, load  # noqa: F401
from .api import (AudioEncoder, DecodingFallback, DecodingOptions, DecodingResult, DeviceTensor,  # noqa: F401
                  FeatureExtractor, Model, SpecialTokens, TextDecoder, WhisperKit, WhisperKitConfig,
                  filter_and_sample)
from .audio import AudioProcessor, ChannelMode  # noqa: F401
from .streaming import AudioStreamTranscriber  # noqa: F401

__all__ = ["WhisperKit", "WhisperKitConfig", "DecodingOptions", "DecodingResult", "DecodingFallback", "SpecialTokens",
           "FeatureExtractor", "AudioEncoder", "TextDecoder", "Model", "DeviceTensor", "filter_and_sample",
           "WhisperError", "load", "AudioProcessor", "ChannelMode", "AudioStreamTranscriber"]
