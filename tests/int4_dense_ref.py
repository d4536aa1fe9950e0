"""INT4 dense weights on the CPU -- test infrastructure only.

The format of `Transformer(..., dense_weights="int4")` (include/mistral_b200.h) restated with torch ops: the group quantiser, the
nibble packing, the dequantised weights W', the bf16x2 instruction pair the kernels dequantise with, and the checkpoint transform
that turns a bf16 checkpoint into the one whose bf16 model the INT4 model computes.
"""
import re
from typing import Dict, Tuple

import torch

GROUP = 128
SMALLEST_BF16 = torch.tensor([1], dtype=torch.int16).view(torch.bfloat16)[0]  # 2^-133, a subnormal

_DENSE_KEY = re.compile(r"^layers\.\d+\.(attention\.w[qkvo]|feed_forward\.w[123])\.weight$")


def group_scales(w: torch.Tensor) -> torch.Tensor:
    """bf16 [N, K/128]: s = 1 for an all-zero group, else bf16_rn(fp32(amax / 7)), raised to the smallest positive bf16 if 0."""
    N, K = w.shape
    a = w.to(torch.bfloat16).float().view(N, K // GROUP, GROUP).abs().amax(-1)
    s = (a / 7.0).to(torch.bfloat16)
    s = torch.where(s == 0, SMALLEST_BF16, s)
    return torch.where(a == 0, torch.ones_like(s), s)


def quantize_codes(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(q int8 [N, K] in -8..7, s bf16 [N, K/128]) of the bf16 weight w [N, K]: q = clamp(rint_even(fp32(w) / fp32(s)), -8, 7)."""
    N, K = w.shape
    s = group_scales(w)
    x = w.to(torch.bfloat16).float().view(N, K // GROUP, GROUP)
    q = torch.round(x / s.float()[..., None]).clamp_(-8, 7)  # torch.round rounds half to even
    return q.view(N, K).to(torch.int8), s


def pack(q: torch.Tensor) -> torch.Tensor:
    """uint8 [N, K/2]: byte j = (q[2j] + 8) | (q[2j + 1] + 8) << 4."""
    u = (q.to(torch.int16) + 8).to(torch.uint8)
    return u[:, 0::2] | (u[:, 1::2] << 4)


def unpack(codes: torch.Tensor) -> torch.Tensor:
    """int8 q [N, K] of the packed codes."""
    lo = (codes & 0xF).to(torch.int8) - 8
    hi = (codes >> 4).to(torch.int8) - 8
    return torch.stack((lo, hi), dim=-1).view(codes.shape[0], -1)


def quantize(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(codes uint8 [N, K/2], s bf16 [N, K/128]): what mb200_quantize_int4_groups writes."""
    q, s = quantize_codes(w)
    return pack(q), s


def dequantize(codes: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W' bf16 [N, K] = bf16_rn(fp32(q) * fp32(s)) (the fp32 product is exact: one rounding)."""
    q = unpack(codes).float()
    N, K = q.shape
    return (q.view(N, K // GROUP, GROUP) * s.float()[..., None]).view(N, K).to(torch.bfloat16)


def bf16x2_dequant(u: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """The kernels' two instructions on bf16 values: (bf16(128 + u) - bf16(136)) * s, each op one bf16 rounding of the exact
    result (sub.rn.bf16x2, mul.rn.bf16x2).  u are the stored nibbles 0..15 (int), s bf16; broadcasts."""
    biased = torch.tensor(0x4300, dtype=torch.int16).add(u.to(torch.int16)).view(torch.bfloat16)
    q = (biased.double() - 136.0).to(torch.bfloat16)
    return (q.double() * s.double()).to(torch.bfloat16)


def is_dense_key(k: str) -> bool:
    return _DENSE_KEY.match(k) is not None


def int4_dense_checkpoint(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """A reference-keyed checkpoint whose bf16 model is the INT4 model: every text-layer Linear weight replaced by W'; everything
    else (embedding, norms, lm head, vision tower) is the same tensor."""
    return {k: (dequantize(*quantize(v.to(torch.bfloat16))) if is_dense_key(k) else v) for k, v in state_dict.items()}
