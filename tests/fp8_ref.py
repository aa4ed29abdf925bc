"""The FP8 (E4M3) cross-attention K/V storage policy as a rounding point of the oracle (oracle/model_ref.py).

Each 64-value row of a cross-attention K or V head ([..., T, 64]) is stored as 64 E4M3 codes plus one f32 scale:
s = amax(|row|) / 448, code = round-to-nearest-even, saturating, E4M3(x / s), value = code * s; a row whose amax is 0 gets s = 0 and
zero codes.  These are exactly the f32 operations of fp8_quantize_row (whisperkit_b200/csrc/common.cuh), which the engine's projection
epilogue runs on the GPU and wk_cross_kv_quantize_rows exposes on the host.  Everything else follows the oracle's 16-bit policy.
"""
from __future__ import annotations

import torch

from oracle import model_ref as M

FP8_MAX = 448.0


def quantize_rows(x: torch.Tensor):
    """x [..., 64] -> (codes uint8 [..., 64], scales f32 [...])."""
    x = x.float()
    s = x.abs().amax(-1) / FP8_MAX
    live = s > 0
    y = (x / torch.where(live, s, torch.ones_like(s))[..., None]).clamp(-FP8_MAX, FP8_MAX)   # clamp = the satfinite saturation
    codes = y.to(torch.float8_e4m3fn).view(torch.uint8)
    codes = torch.where(live[..., None], codes, torch.zeros_like(codes))
    return codes, torch.where(live, s, torch.zeros_like(s))


def dequantize_rows(codes: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    return codes.view(torch.float8_e4m3fn).float() * scales[..., None]


def fp8_round(x: torch.Tensor) -> torch.Tensor:
    return dequantize_rows(*quantize_rows(x))


class FP8CrossKVOracle(M.WhisperOracle):
    """WhisperOracle whose cross-attention K/V cache is stored in FP8: the projection's f32 result (bias included) is quantized per row
    instead of rounded to the 16-bit policy type."""

    def cross_kv(self, enc: torch.Tensor):
        encr = self.r(enc)
        out = []
        for i in range(self.dims.dec_layers):
            p = f"model.decoder.layers.{i}.encoder_attn."
            k = fp8_round(self._heads(self._lin(encr, p + "k_proj")))
            v = fp8_round(self._heads(self._lin(encr, p + "v_proj")))
            out.append((k, v))
        return out
