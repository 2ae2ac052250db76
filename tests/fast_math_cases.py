"""The single-product FP16 math mode ('1xfp16', mask 31) for the per-launch checks of launch_cases.py.

The wgmma kernels contract x.w ~= x_hi.w_hi: the activation rounded to the nearest fp16 (no activation scale) times the
weight image, w * s rounded to the nearest fp16 with s the power of two that puts max|W| of the image into [4096, 8192),
accumulated in fp32 and multiplied by 1 / s in the epilogue.

* ``Arith1x`` is the worst-case error model of that contraction, put in place of the three tensor-core ``Arith`` objects of
  a float64 ``Restater`` by ``single_product``;
* ``RoundedRestater`` is the evaluation the statistical criterion compares against: the same launch in float64 on the
  operands rounded to fp16 exactly as the kernel rounds them (the launches without a tensor-core contraction keep the
  plain fp32 evaluation of ``Restater``).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import launch_cases as lc

MODE = 31


def weight_scale(W) -> float:
    """Scale of a weight image: the power of two that puts max|W| into [4096, 8192) (1 for an all-zero matrix)."""
    amax = float(W.abs().max())
    if not 0.0 < amax < 3.0e38:
        return 1.0
    return 2.0 ** (13 - math.frexp(amax)[1])


def f16_act(a):
    """An activation operand as the producer stores it: its fp32 value rounded to the nearest fp16."""
    return a.to(torch.float32).to(torch.float16).to(a.dtype)


def f16_weight(W):
    """A weight operand as the image holds it, undone: fp16(w * s) / s."""
    s = weight_scale(W)
    return (W.to(torch.float32) * s).to(torch.float16).to(W.dtype) / s


class Arith1x(lc.Arith):
    """Worst-case error of the single product x_hi.w_hi on wgmma (the FFMA model where the launch is not on wgmma).

    * operands: each is rounded once to fp16 (relative 2^-11 in the normal range), so a product is off by at most
      (1 + 2^-11)^2 - 1 = 2^-10 + 2^-22 relative;
    * subnormal floors: an activation below fp16's normal range is on the 2^-24 grid (2^-25 |w| per product), a weight
      below the normal range of the image costs 2^-25 / s |a|, as for 3xFP16 (``Arith.floor``);
    * accumulation: one wgmma per k-group of 16 adds 16 products to the fp32 accumulator; aligned to the largest exponent
      and truncated, each of the 17 addends loses < 1 ulp of the largest magnitude: 2 ceil(K / 16) 17 u * 1.01 M;
    * epilogue (x * inv_scale + b, one fma): one rounding."""

    def __init__(self, tc: bool):
        super().__init__(tc, True)

    def coef(self, K):
        if not self.tc:
            return super().coef(K)
        return 2.0 ** -10 + 2.0 ** -22 + 2 * math.ceil(K / 16) * 17 * lc.U * 1.01 + 2 * lc.U


def single_product(r: lc.Restater) -> lc.Restater:
    """r (a Restater of math mode 31) with the single-product model in place of its three tensor-core Arith objects."""
    r.ar_node, r.ar_gcl, r.ar_coord = (Arith1x(a.tc) for a in (r.ar_node, r.ar_gcl, r.ar_coord))
    return r


def contract(a, W, b):
    """a @ W^T (+ b) in float64 on the operands rounded as the single-product kernels round them."""
    y = f16_act(a).double() @ f16_weight(W).double().T
    return y + b.double() if b is not None else y


class RoundedRestater(lc.Restater):
    """fp32 restatement whose tensor-core contractions are evaluated in float64 on fp16-rounded operands."""

    def __init__(self, cfg, sd, inputs, mode=MODE, device='cpu'):
        super().__init__(cfg, sd, inputs, mode, torch.float32, device)

    def _node_gemm(self, a, ea, W, b, wmax=None):
        if not self.ar_node.tc:
            return super()._node_gemm(a, ea, W, b, wmax)
        return contract(a, W, b).to(self.dtype), None

    def _mlp2(self, u, eu, W2, b2, ar):
        if not ar.tc:
            return super()._mlp2(u, eu, W2, b2, ar)
        return F.silu(contract(F.silu(u), W2, b2).to(self.dtype)), None
