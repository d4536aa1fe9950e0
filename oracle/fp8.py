"""FP8 (e4m3) expert weights on the CPU -- test infrastructure only.

The storage format of `Transformer(..., expert_weights="fp8")` (include/mistral_b200.h) restated with torch ops.  Per row n of an
expert matrix W [N, K] (bf16):
    s[n]     = fp32(amax_k |W[n, k]| / 448)                  IEEE division; 1 for an all-zero row
    q[n, k]  = e4m3fn_rn(clamp(fp32(W[n, k] / s[n]), -448, 448))
    W'[n, k] = bf16_rn(fp32(float(q[n, k]) * s[n]))
`Tensor.to(torch.float8_e4m3fn)` rounds to nearest even and the clamp keeps it finite, which is the device's
cvt.rn.satfinite.e4m3x2.f32.  The FP8 model is the reference model run on the W' checkpoint (`fp8_checkpoint`).
"""
import re
from typing import Dict, Tuple

import torch

E4M3_MAX = 448.0
_EXPERT_KEY = re.compile(r"^layers\.\d+\.feed_forward\.experts\.\d+\.w[123]\.weight$")


def quantize_rows(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """q (uint8 bit patterns of e4m3fn [N, K]) and s (fp32 [N]) of a bf16 matrix."""
    assert w.dtype == torch.bfloat16 and w.dim() == 2, (w.dtype, w.shape)
    wf = w.float()
    amax = wf.abs().amax(dim=1)
    # a tensor divisor: for a Python-scalar divisor torch's CUDA kernel multiplies by the reciprocal, which is not the IEEE quotient
    s = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, E4M3_MAX))
    q = (wf / s[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8), s


def dequantize_rows(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W' = bf16(fp32(float(q) * s)) from uint8 (or float8_e4m3fn) q [N, K] and fp32 s [N]."""
    qf = (q.view(torch.float8_e4m3fn) if q.dtype == torch.uint8 else q).float()
    return (qf * s.float()[:, None]).to(torch.bfloat16)


def fp8_weights(w: torch.Tensor) -> torch.Tensor:
    """W' of one bf16 expert matrix."""
    return dequantize_rows(*quantize_rows(w))


def is_expert_key(k: str) -> bool:
    return _EXPERT_KEY.match(k) is not None


def fp8_checkpoint(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """A reference-keyed checkpoint with every expert matrix (w1, w2, w3 of every expert) replaced by its W'; everything else is
    the same tensor."""
    return {k: (fp8_weights(v.to(torch.bfloat16)) if is_expert_key(k) else v) for k, v in state_dict.items()}
