"""Block-scaled fp8 (MX-style) codec for embedding rows: e4m3 values with one UE8M0 (power-of-two, 8-bit exponent) scale
per block of 32 values - the OCP microscaling (MX) fp8 layout and the storage
format BASELINE config #5 asks for (1 byte per value + 1 byte per 32 values = 1.03 B instead of 4 B).

This module is the *format definition* and its numerics (quantise / dequantise / fake-quantise, error bounds), in plain
PyTorch so that it runs on any backend. `models/deepfm.py` uses it for `table_precision="fp8_block"`: the model trains on
the values an fp8 table would deliver while the parameter manager keeps fp32 master rows (delta accumulation and AdaGrad
stay fp32, the "requantise at sync" scheme); a table that actually STORES one byte per value needs a 1-byte row type in
the store and is not implemented."""
from __future__ import annotations

import torch

BLOCK = 32
E4M3_MAX = 448.0


def _blocks(x: torch.Tensor):
    d = x.shape[-1]
    pad = (-d) % BLOCK
    if pad:
        x = torch.nn.functional.pad(x, (0, pad))
    return x.reshape(*x.shape[:-1], -1, BLOCK), d


def quantize_block_e4m3(x: torch.Tensor):
    """x [..., d] float -> (q [..., nb, 32] float8_e4m3fn, exp [..., nb] int8): value = q * 2**exp.
    The scale is the smallest power of two that brings the block's absolute maximum into e4m3's range (|v| <= 448);
    all-zero blocks get the smallest exponent."""
    xb, _ = _blocks(x.to(torch.float32))
    amax = xb.abs().amax(-1)
    exp = torch.ceil(torch.log2(amax.clamp(min=2.0 ** -120) / E4M3_MAX)).clamp(-127, 127)
    scale = torch.exp2(exp).unsqueeze(-1)
    q = (xb / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, exp.to(torch.int8)


def dequantize_block_e4m3(q: torch.Tensor, exp: torch.Tensor, d: int) -> torch.Tensor:
    """Inverse of :func:`quantize_block_e4m3`: fp32 [..., d]."""
    x = q.to(torch.float32) * torch.exp2(exp.to(torch.float32)).unsqueeze(-1)
    return x.reshape(*x.shape[:-2], -1)[..., :d]


def fake_quantize_block_e4m3(x: torch.Tensor) -> torch.Tensor:
    """The values a block-scaled e4m3 table would return for ``x`` (same shape and dtype as ``x``)."""
    q, e = quantize_block_e4m3(x)
    return dequantize_block_e4m3(q, e, x.shape[-1]).to(x.dtype)


def bytes_per_value() -> float:
    return 1.0 + 1.0 / BLOCK


class FakeQuantSTE(torch.autograd.Function):
    """Straight-through estimator: forward = fake quantisation, backward = identity (the gradient reaches the fp32
    master values)."""

    @staticmethod
    def forward(ctx, x):
        return fake_quantize_block_e4m3(x)

    @staticmethod
    def backward(ctx, g):
        return g
