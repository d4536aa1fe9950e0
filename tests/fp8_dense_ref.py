"""FP8 (e4m3) dense weights on the CPU -- test infrastructure only.

`Transformer(..., dense_weights="fp8")` (include/mistral_b200.h) restated with torch ops, on top of the storage format and
quantiser of oracle/fp8.py (`quantize_rows`, `dequantize_rows`).
"""
import re
from typing import Dict

import torch

from oracle.fp8 import dequantize_rows, quantize_rows

# `Transformer(..., dense_weights="fp8")` stores every text-layer Linear (wq, wk, wv, wo, w1, w2, w3) as (q, s) in that format, but
# computes differently from the experts' W' contract: the scale leaves the dot product (include/mistral_b200.h),
#     y[t, n] = bf16_rn(fp32(s[n] * acc[t, n])),   acc[t, n] = fp32 sum over k of x[t, k] * float(q[n, k])
# The FP8 dense model is the reference model with each of those Linears computed so (`fp8_dense_checkpoint`).
_DENSE_KEY = re.compile(r"^layers\.\d+\.(attention\.w[qkvo]|feed_forward\.w[123])\.weight$")


def dense_linear(x: torch.Tensor, q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """bf16(s * (x.float() @ float(q).T)) for bf16 x [..., K], uint8 (or float8_e4m3fn) q [N, K] and fp32 s [N]."""
    qf = (q.view(torch.float8_e4m3fn) if q.dtype == torch.uint8 else q).float()
    return ((x.float() @ qf.T) * s.float()).to(torch.bfloat16)


class DenseFp8Weight(torch.Tensor):
    """A Linear weight held as (q, s): a bf16 tensor of W's shape (its values are W', never read) that F.linear computes with
    `dense_linear`.  Lets the restatement model run unchanged with FP8 dense Linears."""

    q: torch.Tensor
    s: torch.Tensor

    @staticmethod
    def __new__(cls, q: torch.Tensor, s: torch.Tensor) -> "DenseFp8Weight":
        t = torch.Tensor._make_subclass(cls, dequantize_rows(q, s))
        t.q, t.s = q, s
        return t

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.nn.functional.linear and isinstance(args[1], DenseFp8Weight) and args[2:] in ((), (None,)) and not kwargs:
            return dense_linear(args[0], args[1].q, args[1].s)
        plain = lambda a: a.as_subclass(torch.Tensor) if isinstance(a, DenseFp8Weight) else a  # noqa: E731
        return func(*[plain(a) for a in args], **{k: plain(v) for k, v in kwargs.items()})


def is_dense_key(k: str) -> bool:
    return _DENSE_KEY.match(k) is not None


def fp8_dense_checkpoint(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """A reference-keyed checkpoint for the restatement model (oracle/restatement.py) with every text-layer Linear weight replaced
    by its DenseFp8Weight; everything else (embedding, norms, lm head, vision tower) is the same tensor."""
    return {k: (DenseFp8Weight(*quantize_rows(v.to(torch.bfloat16))) if is_dense_key(k) else v) for k, v in state_dict.items()}
