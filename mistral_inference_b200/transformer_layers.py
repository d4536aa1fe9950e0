"""Attention / FeedForward / RMSNorm / TransformerBlock (API mirror of mistral_inference/transformer_layers.py).

The classes keep the reference's names and wiring, but every FLOP goes through libmb200 (C ABI in
include/mistral_b200.h); weights are stored pre-packed for the fused kernels:
  Attention.wqkv  [(H + 2*KV) * hd, dim] = wq ++ wk ++ wv        (one GEMM / one weight stream)
  FeedForward.w13 [2 * hidden, dim], row 2i = w1[i], row 2i+1 = w3[i]  (SiLU*mul in the epilogue)
`wq/wk/wv/w1/w3` are exposed as zero-copy views for state-dict compatibility.
With `lora` set (un-merged adapters) each fused call also owns a packed LoraAdapter and runs the `_lora` entry points.
With `fp8` (FP8 dense weights, include/mistral_b200.h) the packed matrices hold e4m3 bytes (uint8, same packing) next to one fp32
scale per row, and every call runs the `_fp8` entry points; with `a8` as well (prefill_compute="fp8") the `_fp8a8` ones, whose
prefill-sized calls quantise the activations per token to e4m3 and run the FP8 tensor cores.
With `int4` (INT4 dense weights, include/mistral_b200.h) they hold packed 4-bit codes (uint8 [N, K/2], same row packing) next to one
bf16 scale per group of 128 k of a row, and every call runs the `_int4` entry points.
"""
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _abi
from .args import LoraArgs, MoeArgs
from .cache import CacheView
from .moe import Fp8Expert, Int4Expert, MoeLayer, _Int4Rows, quantize_rows_


class _WeightView:
    """Stands in for an nn.Linear whose weight is a view into a packed parameter."""

    def __init__(self, getter):
        self._getter = getter

    @property
    def weight(self) -> torch.Tensor:
        return self._getter()


class LoraAdapter(nn.Module):
    """The un-merged LoRA adapters (lora.py:22-89) of one fused call, packed for the `_lora` entry points (include/mistral_b200.h):
      a [R, in]  rows s*r .. s*r + r - 1 = lora_A of segment s, R = S*r rounded up to 64, padding rows zero
      b [N, R]   row n = lora_B of n's segment in that segment's r columns, zeros elsewhere; `interleaved` (w13): segment s owns
                 rows 2i + s, like FeedForward.w13
    With `slots` > 1 the adapter is a bank of that many such adapters: slot j owns rows j*Rc .. of `a` and columns j*Rc .. of `b`,
    Rc = `rank_cols` (one slot's R), each laid out as above; a call given per-token slot ids runs each token through its own slot.
    `lora_A(s, slot)` / `lora_B(s, slot)` are zero-copy views under the reference's names.  Loads copy in place (captured decode
    graphs hold the pointers) and keep the zeros: every entry outside a segment's views stays zero."""

    def __init__(self, in_features: int, segments: List[int], lora: LoraArgs, interleaved: bool = False, slots: int = 1):
        super().__init__()
        assert not interleaved or (len(segments) == 2 and segments[0] == segments[1])
        assert slots >= 1, slots
        self.rank = lora.rank
        self.scaling = float(lora.scaling)  # fixed at construction, like LoRALinear.scaling
        self.segments = list(segments)
        self.interleaved = interleaved
        self.slots = slots
        self.rank_cols = -(-len(segments) * lora.rank // 64) * 64
        self.a = nn.Parameter(torch.zeros(slots * self.rank_cols, in_features), requires_grad=False)
        self.b = nn.Parameter(torch.zeros(sum(segments), slots * self.rank_cols), requires_grad=False)

    def _cols(self, s: int, slot: int) -> slice:
        assert 0 <= slot < self.slots, f"adapter slot {slot} outside [0, {self.slots})"
        o = slot * self.rank_cols
        return slice(o + s * self.rank, o + (s + 1) * self.rank)

    def _rows(self, s: int) -> torch.Tensor:
        if self.interleaved:
            return self.b.view(self.segments[0], 2, self.b.shape[1])[:, s]
        o = sum(self.segments[:s])
        return self.b[o: o + self.segments[s]]

    def lora_A(self, s: int, slot: int = 0) -> torch.Tensor:
        return self.a[self._cols(s, slot)]

    def lora_B(self, s: int, slot: int = 0) -> torch.Tensor:
        return self._rows(s)[:, self._cols(s, slot)]

    def put_A(self, s: int, v: torch.Tensor, slot: int = 0) -> None:
        want = self.lora_A(s, slot).shape
        assert v.shape == want, f"lora_A: shape {tuple(v.shape)} != {tuple(want)} (rank {self.rank})"
        self.lora_A(s, slot).copy_(v)

    def put_B(self, s: int, v: torch.Tensor, slot: int = 0) -> None:
        want = self.lora_B(s, slot).shape
        assert v.shape == want, f"lora_B: shape {tuple(v.shape)} != {tuple(want)} (rank {self.rank})"
        self.lora_B(s, slot).copy_(v)

    def zero(self, s: int, slot: int = 0) -> None:
        """A plain `X.weight` checkpoint entry: segment s gets a zero adapter (lora.py:76-89)."""
        self.lora_A(s, slot).zero_()
        self.lora_B(s, slot).zero_()

    def call(self, T: int, lora_rows: Optional[torch.Tensor] = None) -> "_abi.LoraStruct":
        """The adapter argument of one `_lora` call over T tokens, with its own scratch.  `lora_rows` (int32 [T] on the device): the
        slot of each token, -1 for none; None runs the whole packed adapter unmasked (one slot's adapter when `slots` is 1)."""
        R = self.a.shape[0]
        a_buf = torch.empty(T, R, dtype=self.a.dtype, device=self.a.device)
        l_buf = torch.empty(T, self.b.shape[0], dtype=self.a.dtype, device=self.a.device)
        st = _abi.lora_struct(self.a, self.b, self.scaling, a_buf, l_buf, lora_rows, self.rank_cols)
        st.keep = (a_buf, l_buf)  # alive until the call has been enqueued
        return st


class _Fp8Rows:
    """FP8 dense storage of a module's packed matrices: `<m>` is uint8 [N, K] (e4m3 bit patterns), `<m>_scale_bits` int32 [N] the
    bit patterns of the fp32 row scales (`Module.to(dtype)` casts every floating tensor; these must keep their bits).  `_slots`
    maps a reference Linear name to its (q rows, scale entries): zero-copy views, strided where rows interleave."""

    def _fp8_params(self, name: str, n: int, k: int) -> nn.Parameter:
        setattr(self, name + "_scale_bits", nn.Parameter(torch.empty(n, dtype=torch.int32), requires_grad=False))
        return nn.Parameter(torch.empty(n, k, dtype=torch.uint8), requires_grad=False)

    def _slots(self, name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        raise NotImplementedError

    def weight_e4m3(self, name: str) -> torch.Tensor:
        return self._slots(name)[0].view(torch.float8_e4m3fn)

    def weight_scale(self, name: str) -> torch.Tensor:
        return self._slots(name)[1]

    def quantize_(self, name: str, w: torch.Tensor) -> None:
        """Quantises the bf16 weight `w` of Linear `name` into place (one bf16 copy of `w` on the device while it runs)."""
        quantize_rows_(name, w, *self._slots(name))


class RMSNorm(nn.Module):
    """transformer_layers.py:109-120."""

    def __init__(self, dim: int, eps: float = 1e-6):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim), requires_grad=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _abi.rmsnorm(x, self.weight, self.eps)


class Attention(nn.Module, _Fp8Rows, _Int4Rows):
    """transformer_layers.py:31-93."""

    def __init__(self, dim: int, n_heads: int, head_dim: int, n_kv_heads: int, lora: Optional[LoraArgs] = None, fp8: bool = False,
                 int4: bool = False, lora_slots: int = 1, a8: bool = False):
        super().__init__()
        self.dim = dim
        self.n_heads = n_heads
        self.head_dim = head_dim
        self.n_kv_heads = n_kv_heads
        self.repeats = n_heads // n_kv_heads
        self.scale = head_dim ** -0.5
        self.q_dim = n_heads * head_dim
        self.kv_dim = n_kv_heads * head_dim
        self.fp8 = fp8
        self.int4 = int4
        self.a8 = a8
        assert not (fp8 and int4) and (fp8 or not a8)
        if fp8:
            self.wqkv = self._fp8_params("wqkv", self.q_dim + 2 * self.kv_dim, dim)
            self.wo_weight = self._fp8_params("wo", dim, self.q_dim)
        elif int4:
            self.wqkv = self._int4_params("wqkv", self.q_dim + 2 * self.kv_dim, dim)
            self.wo_weight = self._int4_params("wo", dim, self.q_dim)
        else:
            self.wqkv = nn.Parameter(torch.empty(self.q_dim + 2 * self.kv_dim, dim), requires_grad=False)
            self.wo_weight = nn.Parameter(torch.empty(dim, self.q_dim), requires_grad=False)
        self.lora = lora
        if lora is not None:
            self.wqkv_lora = LoraAdapter(dim, [self.q_dim, self.kv_dim, self.kv_dim], lora, slots=lora_slots)
            self.wo_lora = LoraAdapter(self.q_dim, [dim], lora, slots=lora_slots)

    # state-dict compatible views
    @property
    def wq(self) -> _WeightView:
        return _WeightView(lambda: self.wqkv[: self.q_dim])

    @property
    def wk(self) -> _WeightView:
        return _WeightView(lambda: self.wqkv[self.q_dim: self.q_dim + self.kv_dim])

    @property
    def wv(self) -> _WeightView:
        return _WeightView(lambda: self.wqkv[self.q_dim + self.kv_dim:])

    @property
    def wo(self) -> _WeightView:
        return _WeightView(lambda: self.wo_weight)

    @property
    def wqkv_scale(self) -> torch.Tensor:
        return self.wqkv_scale_bits.view(torch.float32)

    @property
    def wo_scale(self) -> torch.Tensor:
        return self.wo_scale_bits.view(torch.float32)

    @property
    def wqkv_gscale(self) -> torch.Tensor:
        return self.wqkv_gscale_bits.view(torch.bfloat16)

    @property
    def wo_gscale(self) -> torch.Tensor:
        return self.wo_gscale_bits.view(torch.bfloat16)

    def _slots(self, name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        rows = {"wq": slice(0, self.q_dim), "wk": slice(self.q_dim, self.q_dim + self.kv_dim), "wv": slice(self.q_dim + self.kv_dim, None)}
        scale, wo_scale = (self.wqkv_gscale, self.wo_gscale) if self.int4 else (self.wqkv_scale, self.wo_scale)
        if name in rows:
            return self.wqkv[rows[name]], scale[rows[name]]
        if name == "wo":
            return self.wo_weight, wo_scale
        raise ValueError(f"attention Linear {name!r}")

    def attend(self, x: torch.Tensor, norm_w: torch.Tensor, eps: float, rope: torch.Tensor, positions: torch.Tensor,
               cache: Optional[CacheView], ws: "_abi.Workspace", lora_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """RMSNorm + QKV + RoPE + cache phase + attention core.  Returns the pre-`wo` output [T, H*hd].  `lora_rows`: the adapter
        slot of each token (LoraAdapter.call)."""
        T = x.shape[0]
        q = torch.empty(T, self.q_dim, dtype=x.dtype, device=x.device)
        k = torch.empty(T, self.kv_dim, dtype=x.dtype, device=x.device)
        v = torch.empty(T, self.kv_dim, dtype=x.dtype, device=x.device)
        out = torch.empty(T, self.q_dim, dtype=x.dtype, device=x.device)
        H, KV, hd = self.n_heads, self.n_kv_heads, self.head_dim
        if cache is None:
            # cache-less forward: unmasked over the whole flattened batch (SURVEY.md Appendix E-2)
            self._qkv(x, norm_w, rope, positions, q, k, v, None, None, None, eps, ws, lora_rows)
            _abi.attn_prefill(q, k, v, None, None, None, None, out, 1, T, 0, H, KV, hd, causal=False)
            return out
        md = cache.metadata
        if cache.fp8:
            return self._attend_fp8(x, norm_w, eps, rope, positions, cache, ws, q, k, v, out, lora_rows)
        if md.prefill:
            # read the old ring, THEN write (transformer_layers.py:75-76)
            self._qkv(x, norm_w, rope, positions, q, k, v, None, None, None, eps, ws, lora_rows)
            _abi.attn_prefill(q, k, v, cache.cache_k, cache.cache_v, md.q_start, md.seqpos, out, len(md.seqlens), md.max_seqlen,
                              md.window, H, KV, hd, causal=True, first_prefill=md.first_prefill)
            _abi.kv_ring_write(k, v, cache.cache_k, cache.cache_v, md.cache_rows, KV, hd)
        else:
            # write, THEN read the ring (transformer_layers.py:78-81); the scatter is the QKV kernel's epilogue
            self._qkv(x, norm_w, rope, positions, q, k, v, cache.cache_k, cache.cache_v, md.cache_rows, eps, ws, lora_rows)
            B = len(md.seqlens)
            _abi.attn_decode(q, cache.cache_k, cache.cache_v, md.kv_len, out, H, KV, hd, decode_splits(B, KV, md.window), ws)
        return out

    def _attend_fp8(self, x, norm_w, eps, rope, positions, cache: CacheView, ws, q, k, v, out, lora_rows=None) -> torch.Tensor:
        """The FP8-cache model: k, v become k', v' (include/mistral_b200.h) right after RoPE, and attention sees only those."""
        H, KV, hd = self.n_heads, self.n_kv_heads, self.head_dim
        md = cache.metadata
        ring = (cache.cache_k, cache.cache_v, cache.cache_k_exp, cache.cache_v_exp)
        self._qkv(x, norm_w, rope, positions, q, k, v, None, None, None, eps, ws, lora_rows)
        if md.prefill:
            # k', v' in place; read the old ring, THEN write it from k', v' (transformer_layers.py:75-76)
            _abi.kv_quantize(k, v, True)
            _abi.attn_prefill_fp8(q, k, v, *ring, md.q_start, md.seqpos, out, len(md.seqlens), md.max_seqlen, md.window, H, KV, hd,
                                  first_prefill=md.first_prefill)
            _abi.kv_quantize(k, v, False, *ring, md.cache_rows)
        else:
            # write, THEN read the ring (transformer_layers.py:78-81)
            _abi.kv_quantize(k, v, False, *ring, md.cache_rows)
            B = len(md.seqlens)
            _abi.attn_decode_fp8(q, *ring, md.kv_len, out, H, KV, hd, decode_splits(B, KV, md.window), ws)
        return out

    def _qkv(self, x, norm_w, rope, positions, q, k, v, cache_k, cache_v, cache_rows, eps, ws, lora_rows=None) -> None:
        H, KV, hd = self.n_heads, self.n_kv_heads, self.head_dim
        if self.fp8:
            _abi.attn_qkv_fp8(x, norm_w, self.wqkv, self.wqkv_scale, rope, positions, q, k, v, cache_k, cache_v, cache_rows, H, KV, hd, eps, ws,
                              a8=self.a8)
        elif self.int4:
            _abi.attn_qkv_int4(x, norm_w, self.wqkv, self.wqkv_gscale, rope, positions, q, k, v, cache_k, cache_v, cache_rows, H, KV, hd, eps,
                               ws)
        elif self.lora is None:
            _abi.attn_qkv(x, norm_w, self.wqkv, rope, positions, q, k, v, cache_k, cache_v, cache_rows, H, KV, hd, eps, ws)
        else:
            _abi.attn_qkv_lora(x, norm_w, self.wqkv, rope, positions, q, k, v, cache_k, cache_v, cache_rows, H, KV, hd, eps, ws,
                               self.wqkv_lora.call(x.shape[0], lora_rows))

    def project_out(self, a: torch.Tensor, residual: torch.Tensor, out: torch.Tensor, ws: "_abi.Workspace",
                    lora_rows: Optional[torch.Tensor] = None) -> None:
        """out = residual + wo(a)."""
        if self.fp8:
            _abi.linear_residual_fp8(a, self.wo_weight, self.wo_scale, residual, out, ws, a8=self.a8)
        elif self.int4:
            _abi.linear_residual_int4(a, self.wo_weight, self.wo_gscale, residual, out, ws)
        elif self.lora is None:
            _abi.linear_residual(a, self.wo_weight, residual, out, ws)
        else:
            _abi.linear_residual_lora(a, self.wo_weight, residual, out, ws, self.wo_lora.call(a.shape[0], lora_rows))


def decode_splits(B: int, KV: int, W: int, n_sm: int = 132) -> int:
    """KV splits per (sequence, kv head): as many as fit ONE wave of two CTAs per SM (a second, partial wave costs more than the
    idle SMs of an incomplete first one; with B * KV >= 2 * n_sm / 2 there is no split and no combine step at all), at least 64
    keys per split."""
    s = max(1, (2 * n_sm) // (B * KV))
    return int(max(1, min(s, 64, (W + 63) // 64)))


class FeedForward(nn.Module, _Fp8Rows, _Int4Rows):
    """transformer_layers.py:96-106."""

    def __init__(self, dim: int, hidden_dim: int, lora: Optional[LoraArgs] = None, fp8: bool = False, int4: bool = False,
                 lora_slots: int = 1, a8: bool = False):
        super().__init__()
        self.dim = dim
        self.hidden_dim = hidden_dim
        self.fp8 = fp8
        self.int4 = int4
        self.a8 = a8
        assert not (fp8 and int4) and (fp8 or not a8)
        if fp8:
            self.w13 = self._fp8_params("w13", 2 * hidden_dim, dim)
            self.w2_weight = self._fp8_params("w2", dim, hidden_dim)
        elif int4:
            self.w13 = self._int4_params("w13", 2 * hidden_dim, dim)
            self.w2_weight = self._int4_params("w2", dim, hidden_dim)
        else:
            self.w13 = nn.Parameter(torch.empty(2 * hidden_dim, dim), requires_grad=False)
            self.w2_weight = nn.Parameter(torch.empty(dim, hidden_dim), requires_grad=False)
        self.lora = lora
        if lora is not None:
            self.w13_lora = LoraAdapter(dim, [hidden_dim, hidden_dim], lora, interleaved=True, slots=lora_slots)
            self.w2_lora = LoraAdapter(hidden_dim, [dim], lora, slots=lora_slots)

    @property
    def w1(self) -> _WeightView:
        return _WeightView(lambda: self.w13.view(self.hidden_dim, 2, self.dim)[:, 0])

    @property
    def w3(self) -> _WeightView:
        return _WeightView(lambda: self.w13.view(self.hidden_dim, 2, self.dim)[:, 1])

    @property
    def w2(self) -> _WeightView:
        return _WeightView(lambda: self.w2_weight)

    @property
    def w13_scale(self) -> torch.Tensor:
        return self.w13_scale_bits.view(torch.float32)

    @property
    def w2_scale(self) -> torch.Tensor:
        return self.w2_scale_bits.view(torch.float32)

    @property
    def w13_gscale(self) -> torch.Tensor:
        return self.w13_gscale_bits.view(torch.bfloat16)

    @property
    def w2_gscale(self) -> torch.Tensor:
        return self.w2_gscale_bits.view(torch.bfloat16)

    def _slots(self, name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        h, d = self.hidden_dim, self.dim
        if name in ("w1", "w3"):
            seg = 0 if name == "w1" else 1
            if self.int4:
                return self.w13.view(h, 2, d // 2)[:, seg], self.w13_gscale.view(h, 2, d // 128)[:, seg]
            return self.w13.view(h, 2, d)[:, seg], self.w13_scale.view(h, 2)[:, seg]
        if name == "w2":
            return (self.w2_weight, self.w2_gscale) if self.int4 else (self.w2_weight, self.w2_scale)
        raise ValueError(f"feed-forward Linear {name!r}")

    def run(self, x: torch.Tensor, norm_w: Optional[torch.Tensor], eps: float, residual: Optional[torch.Tensor],
            ws: "_abi.Workspace", lora_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[norm] -> gate/up -> silu*mul -> down [+ residual].  `lora_rows`: the adapter slot of each token (LoraAdapter.call)."""
        T = x.shape[0]
        g = torch.empty(T, self.hidden_dim, dtype=x.dtype, device=x.device)
        out = torch.empty(T, self.dim, dtype=x.dtype, device=x.device)
        if self.fp8:
            _abi.ffn_gateup_fp8(x, norm_w, self.w13, self.w13_scale, g, eps, ws, a8=self.a8)
            _abi.linear_residual_fp8(g, self.w2_weight, self.w2_scale, residual, out, ws, a8=self.a8)
        elif self.int4:
            _abi.ffn_gateup_int4(x, norm_w, self.w13, self.w13_gscale, g, eps, ws)
            _abi.linear_residual_int4(g, self.w2_weight, self.w2_gscale, residual, out, ws)
        elif self.lora is None:
            _abi.ffn_gateup(x, norm_w, self.w13, g, eps, ws)
            _abi.linear_residual(g, self.w2_weight, residual, out, ws)
        else:
            _abi.ffn_gateup_lora(x, norm_w, self.w13, g, eps, ws, self.w13_lora.call(T, lora_rows))
            _abi.linear_residual_lora(g, self.w2_weight, residual, out, ws, self.w2_lora.call(T, lora_rows))
        return out

    def forward(self, x: torch.Tensor, ws: Optional["_abi.Workspace"] = None) -> torch.Tensor:
        ws = ws or _abi.Workspace(_abi.workspace_bytes(x.shape[0], self.dim, 1, 1, 128, self.hidden_dim, 0, 1), x.device)
        return self.run(x, None, 0.0, None, ws)


def check_moe_lora(expert_weights: str, dense_weights: str) -> None:
    """Un-merged LoRA on a mixture-of-experts model is built for FP8 experts with bf16 attention Linears only."""
    if expert_weights == "int4":
        raise NotImplementedError("un-merged LoRA on INT4 experts is not built: the INT4 grouped expert GEMMs have no LoRA stage "
                                  "(expert_weights='fp8' runs the adapters)")
    if expert_weights != "fp8":
        raise NotImplementedError("un-merged LoRA on mixture-of-experts layers with bf16 experts is not built: the bf16 grouped expert "
                                  "GEMMs have no LoRA stage (merge the adapter instead: args.lora = None, then load_lora; or "
                                  "expert_weights='fp8')")
    if dense_weights != "bf16":
        raise NotImplementedError(f"un-merged LoRA on {dense_weights.upper()} dense weights is not built")


class TransformerBlock(nn.Module):
    """transformer_layers.py:123-169: pre-norm residual wiring; FeedForward or MoeLayer."""

    def __init__(self, dim: int, hidden_dim: int, n_heads: int, n_kv_heads: int, head_dim: int, norm_eps: float,
                 lora: Optional[LoraArgs] = None, moe: Optional[MoeArgs] = None, expert_shard: Tuple[int, int] = (0, 1), expert_group=None,
                 expert_weights: str = "bf16", dense_weights: str = "bf16", lora_slots: int = 1, prefill_compute: str = "bf16"):
        super().__init__()
        assert lora_slots == 1 or (lora is not None and moe is None), "a bank of adapter slots: dense layers with un-merged LoRA only"
        if lora is not None and moe is not None:
            check_moe_lora(expert_weights, dense_weights)
        self.n_heads = n_heads
        self.dim = dim
        self.norm_eps = norm_eps
        fp8, int4 = dense_weights == "fp8", dense_weights == "int4"
        assert not (fp8 or int4) or lora is None, "quantised dense weights: layers without un-merged LoRA only"
        assert not fp8 or moe is None, "FP8 dense weights: dense layers only"
        a8 = prefill_compute == "fp8"
        assert not a8 or fp8, "FP8 activations: FP8 dense weights only"
        # on a MoE block INT4 dense weights are the attention Linears only; the experts follow expert_weights
        self.attention = Attention(dim=dim, n_heads=n_heads, head_dim=head_dim, n_kv_heads=n_kv_heads, lora=lora, fp8=fp8, int4=int4,
                                   lora_slots=lora_slots, a8=a8)
        self.attention_norm = RMSNorm(dim, eps=norm_eps)
        self.ffn_norm = RMSNorm(dim, eps=norm_eps)
        self.feed_forward: nn.Module
        if moe is not None:
            g, G = expert_shard  # this rank allocates only the experts it owns (e % G == g): SURVEY.md 8(e)
            expert = {"fp8": lambda: Fp8Expert(dim, hidden_dim, lora), "int4": lambda: Int4Expert(dim, hidden_dim)}.get(
                expert_weights, lambda: FeedForward(dim=dim, hidden_dim=hidden_dim, lora=lora))
            self.feed_forward = MoeLayer(experts={e: expert() for e in range(moe.num_experts) if e % G == g},
                                         gate_weight=nn.Parameter(torch.empty(moe.num_experts, dim), requires_grad=False), moe_args=moe,
                                         expert_shard=expert_shard, expert_group=expert_group)
        else:
            self.feed_forward = FeedForward(dim=dim, hidden_dim=hidden_dim, lora=lora, fp8=fp8, int4=int4, lora_slots=lora_slots, a8=a8)

    def forward(self, x: torch.Tensor, rope: torch.Tensor, positions: torch.Tensor, cache: Optional[CacheView],
                ws: "_abi.Workspace", lora_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`lora_rows`: int32 [T] on the device, the adapter slot of each token (-1: none), or None for the unmasked adapter."""
        # r = attention(attention_norm(x)); h = x + r        (transformer_layers.py:165-166)
        a = self.attention.attend(x, self.attention_norm.weight, self.norm_eps, rope, positions, cache, ws, lora_rows)
        h = torch.empty_like(x)
        self.attention.project_out(a, x, h, ws, lora_rows)
        # r = feed_forward(ffn_norm(h)); out = h + r          (transformer_layers.py:167-168)
        if isinstance(self.feed_forward, MoeLayer):
            hn = _abi.rmsnorm(h, self.ffn_norm.weight, self.norm_eps)
            return self.feed_forward.run(hn, h, ws)  # router + grouped experts + ordered combine + residual, no host sync
        return self.feed_forward.run(h, self.ffn_norm.weight, self.norm_eps, h, ws, lora_rows)
