"""FP8 activations for FP8 dense weights on the CPU -- test infrastructure only.

`Transformer(..., dense_weights="fp8", prefill_compute="fp8")` (include/mistral_b200.h) restated with torch ops, on top of the FP8
dense restatement (tests/fp8_dense_ref.py).  A layer Linear call of T tokens with packed weight [N, K] takes FP8 activations when
T >= 128 and it does not take stream-K (T <= 128 with N % 128 == 0); for the model shapes here every packed N is a multiple of 128,
so the rule is T >= 129 (`A8_MIN_T`).  Then, for each token row v[t] of the Linear's bf16 input:
    a[t]     = max_k |v[t, k]|                                          (fp32)
    e[t]     = 0 if a[t] == 0, else the smallest integer with a[t] <= 448 * 2^e[t]
    xq[t, k] = e4m3fn_rn(v[t, k] * 2^-e[t])                             (the power of two is exact: one rounding)
    a row holding an inf or a NaN: e[t] = 0 and every xq[t, k] = NaN (0x7f)
    acc      = fp32 sum over k-blocks j (ascending) of block_j,  block_j = sum over the 128 k of block j of float(xq) * float(q)
    y[t, n]  = bf16(fp32(fp32(s[n] * acc[t, n]) * 2^e[t]))
The tensor cores' block sum keeps about 14 significant bits (measured on an H100 by tests/test_gpu_fp8_prefill.py): it is exact
for the exact designs of that file, and the model restatement (PrefillFp8Weight) approximates it on general data by truncating
the exact block sum to BLOCK_BITS bits.
"""
from typing import Dict, Tuple

import torch

from oracle.fp8 import quantize_rows

from .fp8_dense_ref import DenseFp8Weight, dense_linear, is_dense_key

E4M3_MAX = 448.0
E4M3_NAN = 0x7F
KBLOCK = 128
A8_MIN_T = 129
BLOCK_BITS = 14  # the restatement model's block sums: truncated to the measured width of the H100 tensor cores' sum


def act_exponent(a: torch.Tensor) -> torch.Tensor:
    """e for each entry of a (fp32, finite, >= 0): 0 where a == 0, else the smallest integer with a <= 448 * 2^e."""
    m, E = torch.frexp(a.double())  # a = m * 2^E, m in [0.5, 1): a <= 448 * 2^e  <=>  m * 2^(E - e) <= 448 = 0.875 * 2^9
    e = torch.where(m <= 0.875, E - 9, E - 8)
    return torch.where(a == 0, torch.zeros_like(e), e).to(torch.int32)


def quantize_act(v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(xq uint8 [T, K] e4m3 bit patterns, e int32 [T]) of a bf16 matrix v [T, K]."""
    assert v.dtype == torch.bfloat16 and v.dim() == 2, (v.dtype, v.shape)
    vf = v.float()
    bad = ~torch.isfinite(vf).all(dim=1)
    a = torch.where(bad, torch.zeros(()), vf.abs().nan_to_num(0.0).amax(dim=1))
    e = act_exponent(a)
    # v * 2^-e in float64 is exact; its fp32 rounding (only below 2^-126, where e4m3 has nothing but zero) and then the e4m3 one
    scaled = (v.double() * torch.pow(2.0, -e.double())[:, None]).float()
    q = scaled.to(torch.float8_e4m3fn).view(torch.uint8)
    q = torch.where(bad[:, None], torch.full_like(q, E4M3_NAN), q)
    return q.contiguous(), e


def dequantize_act(q: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """float(xq) * 2^e in float64 (exact)."""
    return q.view(torch.float8_e4m3fn).double() * torch.pow(2.0, e.double())[:, None]


def truncate_bits(b: torch.Tensor, bits: int) -> torch.Tensor:
    """b (float64) truncated toward zero to `bits` significant bits."""
    E = torch.floor(torch.log2(b.abs().clamp_min(1e-300)))
    ulp = torch.pow(2.0, E - (bits - 1))
    return torch.where(b == 0, b, torch.sign(b) * torch.floor(b.abs() / ulp) * ulp)


def a8_accumulate(xq: torch.Tensor, wq: torch.Tensor, block_bits: int = 24) -> torch.Tensor:
    """acc fp32 [T, N]: the k-block sums of float(xq) * float(wq), added in fp32 in block order.  Each block sum is exact and then
    rounded to fp32 (block_bits = 24), or truncated toward zero to block_bits significant bits: the tensor cores of an H100 keep
    about 14 (tests/test_gpu_fp8_prefill.py measures it), which block_bits = 14 approximates."""
    T, K = xq.shape
    assert K % KBLOCK == 0, K
    xf = xq.view(torch.float8_e4m3fn).double()
    wf = wq.view(torch.float8_e4m3fn).double()
    acc = torch.zeros(T, wq.shape[0], dtype=torch.float32, device=xq.device)
    for j in range(0, K, KBLOCK):
        b = xf[:, j:j + KBLOCK] @ wf[:, j:j + KBLOCK].T
        acc = acc + (b if block_bits >= 24 else truncate_bits(b, block_bits)).float()
    return acc


def a8_epilogue(acc: torch.Tensor, s: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """bf16(fp32(fp32(s * acc) * 2^e)); the second product rounds once (float64 holds it exactly)."""
    sa = acc.float() * s.float()[None, :]
    return (sa.double() * torch.pow(2.0, e.double())[:, None]).float().to(torch.bfloat16)


def a8_linear(v: torch.Tensor, q: torch.Tensor, s: torch.Tensor, block_bits: int = 24) -> torch.Tensor:
    """The FP8-activation Linear of bf16 v [T, K] with uint8 e4m3 q [N, K] and fp32 s [N]."""
    xq, e = quantize_act(v)
    return a8_epilogue(a8_accumulate(xq, q, block_bits), s, e)


class PrefillFp8Weight(DenseFp8Weight):
    """A DenseFp8Weight whose F.linear takes FP8 activations for calls of A8_MIN_T tokens or more (all leading dims flattened)."""

    @staticmethod
    def __new__(cls, q: torch.Tensor, s: torch.Tensor) -> "PrefillFp8Weight":
        return DenseFp8Weight.__new__(cls, q, s)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.nn.functional.linear and isinstance(args[1], PrefillFp8Weight) and args[2:] in ((), (None,)) and not kwargs:
            x, w = args[0], args[1]
            flat = x.reshape(-1, x.shape[-1])
            if flat.shape[0] < A8_MIN_T:
                return dense_linear(x, w.q, w.s)
            return a8_linear(flat.to(torch.bfloat16), w.q, w.s, BLOCK_BITS).reshape(*x.shape[:-1], w.q.shape[0])
        return super().__torch_function__(func, types, args, kwargs)


def fp8_prefill_checkpoint(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """fp8_dense_checkpoint with every text-layer Linear weight a PrefillFp8Weight."""
    return {k: (PrefillFp8Weight(*quantize_rows(v.to(torch.bfloat16))) if is_dense_key(k) else v) for k, v in state_dict.items()}



def edge_rows(K: int) -> torch.Tensor:
    """bf16 [R, K] rows at the quantiser's edges (K >= 16): a = 448 * 2^e exactly and the next bf16 above it, zero rows, a single
    nonzero, bf16 subnormals (down to the smallest, 2^-133), values that round to e4m3 subnormals (and the ties between them), -0,
    the largest bf16, and rows holding inf, -inf or NaN."""
    def row(vals, fill=0.0):
        r = torch.full((K,), fill, dtype=torch.float64)
        r[: len(vals)] = torch.tensor(vals, dtype=torch.float64)
        return r

    tiny = 2.0 ** -133
    rows = [
        row([448.0, -1.0, 0.5]),                                   # a = 448: e = 0
        row([-56.0, 3.0]),                                         # a = 448 * 2^-3
        row([450.0, 1.0]),                                         # the bf16 after 448: e = 1
        row([448.0 * 2.0 ** -40, 2.0 ** -50]),                     # a = 448 * 2^-40
        row([]),                                                   # all zeros
        row([0.0] * (K - 1) + [3.0]),                              # one nonzero, in the last column
        row([-0.0] * K),                                           # all -0
        row([-0.0, 5.0, -0.0]),                                    # -0 next to a value
        row([tiny, -tiny, 3 * tiny]),                              # bf16 subnormals, a = 3 * 2^-133
        row([tiny]),                                               # the smallest bf16: e = -141
        row([2.0 ** -127, 2.0 ** -130, 1.5 * 2.0 ** -126]),        # subnormal and the smallest normals
        row([448.0, 2.0 ** -9, 1.5 * 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -11, 7 * 2.0 ** -10, 2.0 ** -6 * 1.0625]),
        row([3.3895313892515355e38, -1.0]),                        # the largest bf16: e = 120
        row([1.0, float("inf"), 2.0]),
        row([float("-inf")]),
        row([1.0, float("nan")]),
    ]
    return torch.stack(rows).to(torch.bfloat16)
