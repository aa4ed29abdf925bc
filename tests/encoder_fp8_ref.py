"""The FP8 (E4M3) encoder policy (wk_model_set_encoder_dtype) as a rounding point of the oracle (oracle/model_ref.py).

Only the QKV, FC1 and FC2 GEMMs of each encoder layer change:
  * activations (the LayerNorm outputs and FC1's GELU output, all f32) are quantized per (row, 128-column block): s = amax / 448,
    code = round-to-nearest-even, saturating E4M3(x / s), s = 0 and zero codes for an all-zero block;
  * weights (the model's 16-bit values) are quantized per output channel over the whole K row by the same rule;
  * the product is sum over k-blocks kb of (A_codes W_codes^T)[kb] * s_A[row][kb], times s_W[col] once, then the bias (and for FC1 the
    exact GELU before its quantization).
These are the f32 operations of fp8_row_scale / fp8_encode (whisperkit_b200/csrc/common.cuh), which the GPU kernels run and
wk_fp8_quantize_blocks exposes on the host.  Everything else follows the oracle's 16-bit policy.
"""
from __future__ import annotations

import torch

from oracle import model_ref as M
from tests import fp8_ref

BLOCK = 128


def quantize_blocks(x: torch.Tensor, block: int = BLOCK):
    """x [..., K] -> (codes uint8 [..., K], scales f32 [..., K / block])."""
    lead, k = x.shape[:-1], x.shape[-1]
    codes, scales = fp8_ref.quantize_rows(x.reshape(*lead, k // block, block))
    return codes.reshape(*lead, k), scales


def quantize_weight(w: torch.Tensor):
    """w [N, K] -> (codes [N, K], scales [N]): one scale per output channel."""
    return fp8_ref.quantize_rows(w)


def fp8_matmul(a_codes, a_scales, w_codes, w_scales):
    """sum_kb (a w^T)[kb] * a_scales[..., kb], times w_scales: [..., K] x [N, K] -> [..., N] f32."""
    a = a_codes.view(torch.float8_e4m3fn).float()
    w = w_codes.view(torch.float8_e4m3fn).float()
    acc = None
    for kb in range(a.shape[-1] // BLOCK):
        sl = slice(kb * BLOCK, (kb + 1) * BLOCK)
        t = (a[..., sl] @ w[:, sl].T) * a_scales[..., kb:kb + 1]
        acc = t if acc is None else acc + t
    return acc * w_scales


class FP8EncoderOracle(M.WhisperOracle):
    """WhisperOracle whose encoder QKV, FC1 and FC2 GEMMs take E4M3 operands."""

    def __init__(self, dims, weights, policy="bf16"):
        super().__init__(dims, weights, policy)
        self._wq = {}

    def _qw(self, name):
        if name not in self._wq:
            self._wq[name] = quantize_weight(self.w[name + ".weight"])
        return self._wq[name]

    def _fp8_lin(self, xq, name):
        y = fp8_matmul(*xq, *self._qw(name))
        b = self.w.get(name + ".bias")
        return y if b is None else y + b

    def encode(self, mel: torch.Tensor) -> torch.Tensor:
        d = self.dims
        x = conv_stem(self, mel)
        scale = (d.d_model // d.n_heads) ** -0.5
        for i in range(d.enc_layers):
            p = f"model.encoder.layers.{i}."
            xq = quantize_blocks(self._ln(x, p + "self_attn_layer_norm"))
            q = self._heads(self.r(self._fp8_lin(xq, p + "self_attn.q_proj")))
            k = self._heads(self.r(self._fp8_lin(xq, p + "self_attn.k_proj")))
            v = self._heads(self.r(self._fp8_lin(xq, p + "self_attn.v_proj")))
            s = (q @ k.transpose(-1, -2)) * scale
            a = torch.softmax(s, dim=-1) @ v
            a = self.r(a.transpose(1, 2).reshape(x.shape))
            x = x + self._lin(a, p + "self_attn.out_proj")
            xq = quantize_blocks(self._ln(x, p + "final_layer_norm"))
            hq = quantize_blocks(M.gelu(self._fp8_lin(xq, p + "fc1")))
            x = x + self._fp8_lin(hq, p + "fc2")
        return self._ln(x, "model.encoder.layer_norm")


def conv_stem(orc: M.WhisperOracle, mel: torch.Tensor) -> torch.Tensor:
    """The conv stem + positional embedding of WhisperOracle.encode (unchanged by the policy): [B, nMels, 3000] -> [B, 1500, d] f32."""
    import torch.nn.functional as F
    w = orc.w
    x = M.gelu(F.conv1d(mel, w["model.encoder.conv1.weight"], w["model.encoder.conv1.bias"], padding=1))
    if orc.policy != "fp32":
        x = M.round_to(x, "f16")
    x = F.conv1d(x, w["model.encoder.conv2.weight"], w["model.encoder.conv2.bias"], stride=2, padding=1)
    return M.gelu(x).transpose(1, 2) + w["model.encoder.embed_positions.weight"][None]


class FP8EncoderCrossKVOracle(FP8EncoderOracle, fp8_ref.FP8CrossKVOracle):
    """Both FP8 policies: the FP8 encoder and the FP8 cross-attention K/V cache."""
