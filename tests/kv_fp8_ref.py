"""FP8 (e4m3) KV cache on the CPU -- test infrastructure only.

The storage format of `BufferCache(..., kv_cache="fp8")` (include/mistral_b200.h, mb200_kv_quantize) restated with torch ops.
Per (slot, kv head) row x of hd bf16 values:
    e    = max(-124, smallest integer with amax|x| <= 448 * 2^e)     (all-zero row: -124)
    q[i] = e4m3fn_rn(fp32(x[i]) * 2^-e)
    x'   = q * 2^e                                                   (exact in bf16)
`Tensor.to(torch.float8_e4m3fn)` rounds to nearest even, which is the device's cvt.rn.satfinite.e4m3x2.f32 on values <= 448.

The FP8-cache model is the oracle restatement (oracle/restatement.py) with k <- k', v <- v' right after RoPE in every forward that
has a cache.  `attention_forward` below is the restatement's attention with that hook as an argument (identity by default), and
`fp8_kv_cache()` runs the restatement with the hook set to `kv_prime`.
"""
import contextlib
import functools
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import restatement as R
from oracle.attention_ref import attend_block, local_causal_allowed

E4M3_MAX = 448.0
EXP_MIN = -124


def quantize_kv_rows(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(q uint8 e4m3fn bit patterns [..., hd], e int8 [...]) of bf16 rows x [..., hd]."""
    assert x.dtype == torch.bfloat16, x.dtype
    xf = x.float()
    amax = xf.abs().amax(dim=-1)
    m, E = torch.frexp(amax)  # amax = m * 2^E, m in [0.5, 1): amax <= 1.75 * 2^(e + 8) <=> e >= E - 9 (+1 when 2m > 1.75)
    e = E - 9 + (m > 0.875).to(E.dtype)
    e = torch.where(amax == 0, torch.full_like(e, EXP_MIN), e).clamp_min(EXP_MIN)
    scale = torch.ldexp(torch.ones_like(amax), -e)  # 2^-e: a normal fp32 for every e the format produces
    q = (xf * scale[..., None]).to(torch.float8_e4m3fn)
    return q.view(torch.uint8), e.to(torch.int8)


def dequant(q: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """x' = q * 2^e in bf16 (exact) from uint8 (or float8_e4m3fn) q [..., hd] and int8 e [...]."""
    qf = (q.view(torch.float8_e4m3fn) if q.dtype == torch.uint8 else q).float()
    return (qf * torch.ldexp(torch.ones(e.shape), e.to(torch.int32))[..., None]).to(torch.bfloat16)


def kv_prime(x: torch.Tensor) -> torch.Tensor:
    """x' of bf16 rows x [..., hd]."""
    return dequant(*quantize_kv_rows(x))


def attention_forward(x: torch.Tensor, w: Dict[str, torch.Tensor], pre: str, args: R.OracleArgs, freqs_cis: torch.Tensor,
                      seqlens: List[int], seqpos: Optional[List[int]], cache: Optional[R.RingCache], layer: int,
                      kv_hook: Callable[[torch.Tensor], torch.Tensor] = lambda t: t) -> torch.Tensor:
    """oracle/restatement.py's attention_forward with `kv_hook` applied to k and v right after RoPE when there is a cache."""
    T = x.shape[0]
    H, KV, hd = args.n_heads, args.n_kv_heads, args.head_dim
    rep = H // KV
    xq = F.linear(x, w[pre + "wq.weight"]).view(T, H, hd)
    xk = F.linear(x, w[pre + "wk.weight"]).view(T, KV, hd)
    xv = F.linear(x, w[pre + "wv.weight"]).view(T, KV, hd)
    xq, xk = R.apply_rope(xq, xk, freqs_cis)

    if cache is None:
        out = attend_block(xq, xk.repeat_interleave(rep, dim=1), xv.repeat_interleave(rep, dim=1), None)
        return F.linear(out.view(T, H * hd), w[pre + "wo.weight"])

    xk, xv = kv_hook(xk), kv_hook(xv)
    assert seqpos is not None
    W = cache.sizes[layer]
    ck, cv = cache.k[layer], cache.v[layer]
    prefill = seqpos[0] == 0 or any(s > 1 for s in seqlens)
    outs = []
    o = 0
    for b, (s, p) in enumerate(zip(seqlens, seqpos)):
        q_b, k_b, v_b = xq[o:o + s], xk[o:o + s], xv[o:o + s]
        if prefill:
            old_k, old_v = R._unrotate(ck[b], p), R._unrotate(cv[b], p)
            keys, vals = torch.cat([old_k, k_b], 0), torch.cat([old_v, v_b], 0)
            allowed = local_causal_allowed(s, keys.shape[0], W)
        for t in range(max(0, s - W), s):
            slot = (p + t) % W
            ck[b, slot] = k_b[t]
            cv[b, slot] = v_b[t]
        if not prefill:
            n = min(p + 1, W)
            keys, vals = ck[b, :n], cv[b, :n]
            allowed = local_causal_allowed(s, n, None)
        outs.append(attend_block(q_b, keys.repeat_interleave(rep, dim=1), vals.repeat_interleave(rep, dim=1), allowed))
        o += s
    out = torch.cat(outs, 0)
    return F.linear(out.view(T, H * hd), w[pre + "wo.weight"])


@contextlib.contextmanager
def hooked_attention(kv_hook: Callable[[torch.Tensor], torch.Tensor]):
    """Inside the block, the restatement's blocks call `attention_forward` above with `kv_hook`."""
    orig = R.attention_forward
    R.attention_forward = functools.partial(attention_forward, kv_hook=kv_hook)
    try:
        yield
    finally:
        R.attention_forward = orig


def fp8_kv_cache():
    """Inside the block, the restatement is the FP8-cache model (its ring then holds x', which is what the e4m3 ring decodes to)."""
    return hooked_attention(kv_prime)
