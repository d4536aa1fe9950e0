"""Transformer model shell (API mirror of mistral_inference/transformer.py).

`Transformer.from_folder / forward / forward_partial / load_state_dict` keep the reference's signatures and
on-disk contract (params.json + consolidated.safetensors | consolidated.00.pth, reference state-dict keys);
the layer loop calls the fused libmb200 kernels.  bf16 on CUDA only; there is no PyTorch/CPU fallback.
"""
import json
import logging
import math
import os
import re
from pathlib import Path
from typing import Any, Dict, List, Mapping, Optional, Tuple, Union

import torch
from torch import nn

from . import _abi
from .args import PATCH_MERGE, TransformerArgs
from .cache import KV_CACHE_FORMATS, BufferCache, CacheInputMetadata
from .rope import precompute_freqs_cis
from .moe import EXPERT_WEIGHTS, Fp8Expert, Int4Expert
from .transformer_layers import LoraAdapter, RMSNorm, TransformerBlock, check_moe_lora
from .vision_encoder import PatchMerger, VisionLanguageAdapter, VisionTransformer

ROPE_TABLE_LEN = 128_000  # transformer.py:116
# the LoRALinear modules of a text block (transformer_layers.py:50-54,100-103): name -> (adapter attribute path, segment)
_LORA_LINEARS = {"attention.wq": ("attention.wqkv_lora", 0), "attention.wk": ("attention.wqkv_lora", 1),
                 "attention.wv": ("attention.wqkv_lora", 2), "attention.wo": ("attention.wo_lora", 0),
                 "feed_forward.w1": ("feed_forward.w13_lora", 0), "feed_forward.w3": ("feed_forward.w13_lora", 1),
                 "feed_forward.w2": ("feed_forward.w2_lora", 0)}
_LORA_PARTS = (".linear.weight", ".lora_A.weight", ".lora_B.weight")
_EXPERT_LINEAR = re.compile(r"^feed_forward\.experts\.\d+\.w[123]$")  # the LoRALinears of a MoE block's experts (below `layers.{i}.`)
_VISION_PREFIXES = ("vision_encoder.", "vision_language_adapter.", "patch_merger.", "pre_mm_projector_norm.")  # transformer.py:279-291
_NVTX = os.environ.get("MB200_NVTX", "0") == "1"
MAX_LORA_SLOTS = 16  # every decode step reads every resident slot's adapters (DESIGN.md, "Multi-adapter LoRA")


def expand_lora_ids(lora_ids: List[int], seqlens: List[int]) -> torch.Tensor:
    """Per-sequence adapter slots -> the int32 slot of every token of the flattened batch (CPU)."""
    assert len(lora_ids) == len(seqlens), (len(lora_ids), len(seqlens))
    return torch.repeat_interleave(torch.tensor(lora_ids, dtype=torch.int32), torch.tensor(seqlens, dtype=torch.long))


class _nvtx:
    """NVTX range around a phase of the forward (MB200_NVTX=1; visible in nsys / ncu --nvtx): the layer loop, the decode step."""

    def __init__(self, name: str):
        self.name = name

    def __enter__(self):
        if _NVTX:
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if _NVTX:
            torch.cuda.nvtx.range_pop()


class _OutputView:
    def __init__(self, model: "Transformer"):
        self._m = model

    @property
    def weight(self) -> torch.Tensor:
        return self._m.output_weight


DENSE_WEIGHTS = ("bf16", "fp8", "int4")
PREFILL_COMPUTE = ("bf16", "fp8")


def _check_prefill_compute(args: TransformerArgs, prefill_compute: str, dense_weights: str) -> None:
    """The refusals of prefill_compute="fp8", before anything is allocated (after _check_dense_weights)."""
    if prefill_compute not in PREFILL_COMPUTE:
        raise ValueError(f"prefill_compute={prefill_compute!r}: expected one of {PREFILL_COMPUTE}")
    if prefill_compute == "bf16":
        return
    if dense_weights != "fp8":
        raise ValueError(f"prefill_compute='fp8' needs dense_weights='fp8' (got {dense_weights!r}): the FP8 tensor-core GEMM multiplies "
                         "e4m3 activations by e4m3 weights")
    # the e4m3 x e4m3 kernel reads 128-element k-blocks and 64- or 128-wide tiles (include/mistral_b200.h)
    q_dim, kv_dim = args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    for name, N, K in [("wqkv", q_dim + 2 * kv_dim, args.dim), ("wo", args.dim, q_dim), ("w13", 2 * args.hidden_dim, args.dim),
                       ("w2", args.dim, args.hidden_dim)]:
        if K % 128 != 0 or N % 64 != 0:
            raise ValueError(f"prefill_compute='fp8': {name} [{N}, {K}] does not fit the FP8 tensor-core GEMM (K must be a multiple of "
                             "128 and N of 64)")


def _check_dense_weights(args: TransformerArgs, dense_weights: str, expert_weights: str) -> None:
    """The refusals of dense_weights="fp8" / "int4", before anything is allocated."""
    if dense_weights not in DENSE_WEIGHTS:
        raise ValueError(f"dense_weights={dense_weights!r}: expected one of {DENSE_WEIGHTS}")
    if dense_weights == "bf16":
        return
    fmt = dense_weights.upper()
    if args.moe is not None and dense_weights == "fp8":
        raise ValueError("dense_weights='fp8' needs a dense model: FP8 attention Linears on mixture-of-experts models are not built "
                         "(dense_weights='int4' quantises their attention Linears, expert_weights='fp8' or 'int4' the experts)")
    if args.moe is not None and expert_weights == "bf16":
        # the attention Linears are a few per cent of a MoE model's bytes (Mixtral-8x22B: 9.9 of 281 GB): INT4 ones are only worth
        # their T <= 4 rounding differences next to quantised experts
        raise ValueError("dense_weights='int4' on a mixture-of-experts model quantises its attention Linears only and is built with "
                         "quantised experts: pass expert_weights='int4' (or 'fp8') as well")
    if args.lora is not None:
        raise NotImplementedError(f"un-merged LoRA on {fmt} dense weights is not built (merge the adapter into a bf16 model instead)")
    # every Linear must stay off the mma.sync GEMM at every token count: it has no e4m3 or int4 variant (include/mistral_b200.h);
    # INT4 scale groups are 128 k wide.  On a MoE model only the attention Linears are dense (the experts follow expert_weights).
    k_mult = 128 if dense_weights == "int4" else 64
    q_dim, kv_dim = args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    linears = [("wqkv", q_dim + 2 * kv_dim, args.dim), ("wo", args.dim, q_dim)]
    if args.moe is None:
        linears += [("w13", 2 * args.hidden_dim, args.dim), ("w2", args.dim, args.hidden_dim)]
    for name, N, K in linears:
        if K % k_mult != 0 or (N % 128 != 0 and N % 192 != 0):
            groups = " or would split a 128-wide scale group" if dense_weights == "int4" else ""
            raise ValueError(f"dense_weights={dense_weights!r}: {name} [{N}, {K}] would need the mma.sync GEMM, which has no {fmt} variant"
                             f"{groups} (K must be a multiple of {k_mult} and N of 128 or 192)")


class Transformer(nn.Module):
    def __init__(self, args: TransformerArgs, pipeline_rank: int = 0, num_pipeline_ranks: int = 1, softmax_fp32: bool = True,
                 expert_parallel: Optional[Tuple[int, int]] = None, expert_group: Any = None, expert_weights: str = "bf16", *,
                 kv_cache: str = "bf16", dense_weights: str = "bf16", lora_slots: int = 1, prefill_compute: str = "bf16"):
        """Same signature as the reference (transformer.py:34-40) plus `expert_parallel = (rank, world)`: MoE experts sharded
        `e % world == rank` over the ranks of `expert_group` (default process group), everything else replicated, one
        all-reduce of [T, dim] per MoE layer (SURVEY.md 8e); and `expert_weights`: "bf16", or "fp8" to store every MoE expert
        matrix as e4m3 with one fp32 scale per row (moe.Fp8Expert; the model then computes exactly what the bf16 model computes
        with the dequantised weights W', see include/mistral_b200.h), or "int4" to store them in the format of the INT4 dense
        Linears below (moe.Int4Expert; again exactly the bf16 model on W'); and `kv_cache`: "bf16", or "fp8" to keep the KV cache as e4m3
        with one power-of-two exponent per (slot, kv head) row (cache.BufferCache; the model is then the bf16 model with k, v
        replaced by their dequantised k', v' right after RoPE in every forward that has a cache, see include/mistral_b200.h); and
        `dense_weights`: "bf16", or "fp8" to store wq, wk, wv, wo, w1, w2 and w3 of every text layer of a dense model as e4m3 with
        one fp32 scale per row, applied after the dot product: y = bf16(s * sum_k x * q) (include/mistral_b200.h; the embedding,
        the lm head, the norms and the vision tower stay bf16).  That model is not bit-identical to any bf16 model.  "int4" stores the
        same Linears as symmetric 4-bit codes with one bf16 scale per group of 128 k of a row; that model computes exactly what the
        bf16 model computes with the dequantised weights W' (include/mistral_b200.h).  On a mixture-of-experts model "int4" stores
        wq, wk, wv and wo only, and needs quantised experts (`expert_weights` "int4" or "fp8").  `lora_slots` (with `args.lora`, dense
        models): every un-merged adapter is a bank of that many slots, loaded with `load_lora(slot=...)`, and each sequence of a batch
        runs through the slot its `lora_ids` entry names (`generate`, `forward`, ...); at most MAX_LORA_SLOTS.  `prefill_compute`
        (with dense_weights="fp8"): "bf16", or "fp8" to quantise the input of every layer Linear call of at least 128 tokens that does
        not take stream-K per token to e4m3 with a power-of-two scale and multiply it by the e4m3 weights on the FP8 tensor cores
        (include/mistral_b200.h); smaller calls, and so every decode step and chunks of at most 128 tokens, are unchanged.  The
        weights and the state dict are those of dense_weights="fp8"."""
        if not isinstance(lora_slots, int) or not 1 <= lora_slots <= MAX_LORA_SLOTS:
            raise ValueError(f"lora_slots={lora_slots!r}: expected an int in [1, {MAX_LORA_SLOTS}] (every decode step reads every slot)")
        if lora_slots > 1 and args.lora is None:
            raise ValueError(f"lora_slots={lora_slots} needs un-merged adapters: set args.lora (params.json `lora`)")
        if lora_slots > 1 and args.moe is not None:
            raise ValueError(f"lora_slots={lora_slots} on a mixture-of-experts model is not built: the grouped expert GEMMs have no "
                             "per-sequence adapter mask")
        super().__init__()
        self.lora_slots = lora_slots
        _check_dense_weights(args, dense_weights, expert_weights)
        _check_prefill_compute(args, prefill_compute, dense_weights)
        self.dense_weights = dense_weights
        self.prefill_compute = prefill_compute
        if kv_cache not in KV_CACHE_FORMATS:
            raise ValueError(f"kv_cache={kv_cache!r}: expected one of {KV_CACHE_FORMATS}")
        if kv_cache == "fp8" and args.head_dim != 128:
            raise ValueError(f"kv_cache='fp8' needs head_dim 128: the FP8 attention kernels read 128-byte rows (got {args.head_dim})")
        if kv_cache == "fp8" and args.n_heads // args.n_kv_heads not in (1, 2, 4, 6, 8):
            raise ValueError(f"kv_cache='fp8' supports 1, 2, 4, 6 or 8 query heads per kv head (got {args.n_heads // args.n_kv_heads}): "
                             "the FP8-cache attention kernels hold a group's query heads in MMA rows 0-7")
        self.kv_cache = kv_cache
        if expert_weights not in EXPERT_WEIGHTS:
            raise ValueError(f"expert_weights={expert_weights!r}: expected one of {EXPERT_WEIGHTS}")
        if expert_weights != "bf16" and args.moe is None:
            raise ValueError(f"expert_weights={expert_weights!r} needs a mixture-of-experts model: only the grouped expert GEMMs read "
                             f"{expert_weights.upper()} weights")
        if expert_weights == "int4" and (args.dim % 128 != 0 or args.hidden_dim % 128 != 0):
            raise ValueError(f"expert_weights='int4': dim={args.dim} and hidden_dim={args.hidden_dim} must be multiples of 128, the width "
                             "of the scale groups")
        self.expert_weights = expert_weights
        if args.lora is not None and args.moe is not None:
            check_moe_lora(expert_weights, dense_weights)
        self.args = args
        self.expert_parallel = expert_parallel or (0, 1)
        assert 0 <= self.expert_parallel[0] < self.expert_parallel[1], self.expert_parallel
        assert self.expert_parallel[1] == 1 or (args.moe is not None and num_pipeline_ranks == 1), \
            "expert sharding needs a MoE model and excludes pipeline ranks"
        self.vocab_size = args.vocab_size
        self.n_layers = args.n_layers
        self._rope_table: Optional[torch.Tensor] = None
        self._megakernel_refused: Optional[str] = None  # why the decode megakernel refuses this model's shapes ("" = it runs them)
        assert self.vocab_size > 0
        assert pipeline_rank < num_pipeline_ranks, (pipeline_rank, num_pipeline_ranks)
        self.pipeline_rank = pipeline_rank
        self.num_pipeline_ranks = num_pipeline_ranks
        self.softmax_fp32 = softmax_fp32

        self.tok_embeddings: Optional[nn.Embedding] = None
        self.norm: Optional[RMSNorm] = None
        self.output_weight: Optional[nn.Parameter] = None
        self.vision_encoder: Optional[VisionTransformer] = None
        self.vision_language_adapter: Optional[VisionLanguageAdapter] = None
        self.pre_mm_projector_norm: Optional[RMSNorm] = None
        self.patch_merger: Optional[PatchMerger] = None
        if pipeline_rank == 0:
            self.tok_embeddings = nn.Embedding(args.vocab_size, args.dim)
            self.tok_embeddings.weight.requires_grad_(False)
            ve = args.vision_encoder
            if ve is not None:  # transformer.py:59-75
                self.vision_encoder = VisionTransformer(ve)
                self.vision_language_adapter = VisionLanguageAdapter(ve.hidden_size, args.dim, ve.adapter_bias)
                if ve.add_pre_mm_projector_layer_norm:
                    self.pre_mm_projector_norm = RMSNorm(ve.hidden_size, eps=1e-5)
                if ve.mm_projector_id == PATCH_MERGE:
                    self.patch_merger = PatchMerger(vision_encoder_dim=ve.hidden_size, spatial_merge_size=ve.spatial_merge_size)
        if pipeline_rank == num_pipeline_ranks - 1:
            self.norm = RMSNorm(args.dim, eps=args.norm_eps)
            self.output_weight = nn.Parameter(torch.empty(args.vocab_size, args.dim), requires_grad=False)
        # contiguous layer ranges per pipeline rank, keyed by GLOBAL layer id (transformer.py:94-98)
        num_layers_per_rank = math.ceil(self.n_layers / self.num_pipeline_ranks)
        offset = self.pipeline_rank * num_layers_per_rank
        end = min(self.n_layers, offset + num_layers_per_rank)
        self.layers = nn.ModuleDict({
            str(i): TransformerBlock(dim=args.dim, hidden_dim=args.hidden_dim, n_heads=args.n_heads, n_kv_heads=args.n_kv_heads,
                                     head_dim=args.head_dim, norm_eps=args.norm_eps, lora=args.lora, moe=args.moe,
                                     expert_shard=self.expert_parallel, expert_group=expert_group, expert_weights=expert_weights,
                                     dense_weights=dense_weights, lora_slots=lora_slots, prefill_compute=prefill_compute)
            for i in range(offset, end)
        })
        self.n_local_layers = len(self.layers)
        for j, blk in enumerate(self.layers.values()):  # consecutive MoE layers alternate the expert-parallel exchange buffer
            if hasattr(blk.feed_forward, "layer_parity"):
                blk.feed_forward.layer_parity = j & 1
        self._ws: Optional[_abi.Workspace] = None
        self._ws_tokens = 0
        self.last_argmax: Optional[torch.Tensor] = None  # device token id(s) written by the last fused-argmax decode step
        self._last_static_logits = 0                     # data_ptr of the logits buffer that argmax belongs to

    # ------------------------------------------------------------------ properties
    @property
    def dtype(self) -> torch.dtype:
        return next(p.dtype for p in self.parameters() if p.is_floating_point())  # FP8 weights are stored as integers

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    @property
    def output(self) -> _OutputView:
        return _OutputView(self)

    @property
    def freqs_cis(self) -> torch.Tensor:
        """complex64 [128000, hd/2] on the model device (transformer.py:108-120)."""
        return torch.view_as_complex(self.rope_table)

    @property
    def rope_table(self) -> torch.Tensor:
        """fp32 [128000, hd/2, 2] (cos, sin): the same bits as the reference's table, built on the CPU."""
        if self._rope_table is None:
            theta = self.args.rope_theta or 1000000.0
            self._rope_table = torch.view_as_real(precompute_freqs_cis(self.args.head_dim, ROPE_TABLE_LEN, theta)).contiguous()
        if self._rope_table.device != self.device:
            self._rope_table = self._rope_table.to(device=self.device)
        return self._rope_table

    def workspace(self, num_tokens: int) -> _abi.Workspace:
        if self._ws is None or self._ws_tokens < num_tokens or self._ws.buf.device != self.device:
            a = self.args
            need = _abi.workspace_bytes(num_tokens, a.dim, a.n_heads, a.n_kv_heads, a.head_dim, a.hidden_dim, a.vocab_size,
                                        max(a.max_batch_size, 1))
            self._ws = _abi.Workspace(need, self.device)  # decode states remember the pointer they captured (see _decode_state)
            self._ws_tokens = num_tokens
        return self._ws

    # ------------------------------------------------------------------ forward
    def _check_runnable(self) -> None:
        if self.device.type != "cuda" or self.dtype != torch.bfloat16:
            raise _abi.Mb200Error(f"the libmb200 hot path runs bf16 on CUDA only (got {self.dtype} on {self.device}); no fallback exists")

    def _check_cache(self, cache: Optional[BufferCache]) -> None:
        assert cache is None or cache.kv_cache == self.kv_cache, (
            f"a {cache.kv_cache} KV cache passed to a model built with kv_cache={self.kv_cache!r}")

    def check_lora_ids(self, lora_ids: List[int], batch: int) -> None:
        """Raises ValueError unless `lora_ids` names one adapter slot in [0, lora_slots), or -1 for the base model, per sequence."""
        if self.args.lora is None:
            raise ValueError("lora_ids needs un-merged adapters: set args.lora (params.json `lora`)")
        if self.num_pipeline_ranks > 1:
            raise ValueError("lora_ids with pipeline ranks is not built: the stages would each need the per-token slots")
        if self.expert_parallel[1] > 1:
            raise ValueError("lora_ids with expert parallelism is not built: the grouped expert GEMMs have no per-sequence adapter mask")
        if self.args.moe is not None:
            raise ValueError("lora_ids on a mixture-of-experts model is not built: the grouped expert GEMMs have no per-sequence adapter mask")
        if len(lora_ids) != batch:
            raise ValueError(f"lora_ids has {len(lora_ids)} entries for {batch} sequences")
        bad = [i for i in lora_ids if not isinstance(i, int) or not -1 <= i < self.lora_slots]
        if bad:
            raise ValueError(f"lora_ids {bad}: expected adapter slots in [0, {self.lora_slots}) or -1 (no adapter)")

    def _lora_rows(self, lora_ids: Optional[List[int]], seqlens: List[int]) -> Optional[torch.Tensor]:
        """The device int32 slot of every token of one forward (uploaded once), or None: the caller's default (`_default_rows`)."""
        if lora_ids is None:
            return None
        self.check_lora_ids(lora_ids, len(seqlens))
        return expand_lora_ids(lora_ids, seqlens).to(self.device)

    def _default_rows(self, rows: Optional[torch.Tensor], num_toks: int) -> Optional[torch.Tensor]:
        """No ids: slot 0 for every token of a multi-slot model (the unmasked bank would sum every slot), the unmasked adapter of a
        single-slot one.  torch.zeros, not an upload, so that it can be captured in a graph."""
        if rows is None and self.lora_slots > 1:
            return torch.zeros(num_toks, dtype=torch.int32, device=self.device)
        return rows

    @torch.inference_mode()
    def forward_partial(self, input_ids: torch.Tensor, seqlens: List[int], cache: Optional[BufferCache] = None,
                        images: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        """Local forward pass (transformer.py:163-219): hidden states of this stage; the last stage returns
        the normalised final embeddings."""
        self._check_runnable()
        self._check_cache(cache)
        assert len(seqlens) <= self.args.max_batch_size, f"Max batch size is {self.args.max_batch_size}, got batch size of {len(seqlens)}"
        (num_toks,) = input_ids.shape
        assert sum(seqlens) == num_toks, (sum(seqlens), num_toks)
        ws = self.workspace(num_toks)

        input_metadata: Optional[List[CacheInputMetadata]] = None
        if cache is not None:
            self._check_positions(cache, seqlens)
            input_metadata = cache.get_input_metadata(seqlens)
            positions = input_metadata[0].positions
        else:
            positions = torch.cat([torch.arange(0, s, dtype=torch.int32) for s in seqlens]).to(self.device)

        if self.pipeline_rank == 0:
            assert self.tok_embeddings is not None
            h = self._embed(input_ids, images)
        else:
            h = torch.empty(num_toks, self.args.dim, device=self.device, dtype=self.dtype)
            torch.distributed.recv(h, src=self.pipeline_rank - 1)

        rope = self.rope_table
        rows = self._default_rows(None, num_toks)
        for local_layer_id, layer in enumerate(self.layers.values()):
            view = cache.get_view(local_layer_id, input_metadata[local_layer_id]) if cache is not None else None
            h = layer(h, rope, positions, view, ws, rows)

        if cache is not None:
            cache.update_seqlens(seqlens)
        if self.pipeline_rank < self.num_pipeline_ranks - 1:
            torch.distributed.send(h, dst=self.pipeline_rank + 1)
            return h
        assert self.norm is not None
        return self.norm(h)

    @torch.inference_mode()
    def forward(self, input_ids: torch.Tensor, seqlens: List[int], cache: Optional[BufferCache] = None,
                images: Optional[List[torch.Tensor]] = None, *, lora_ids: Optional[List[int]] = None) -> torch.Tensor:
        """transformer.py:221-242.  [T, vocab] logits, fp32 when softmax_fp32.  `lora_ids`: the adapter slot of each sequence (-1: no
        adapter); None is slot 0 for every sequence."""
        self._check_runnable()
        self._check_cache(cache)
        if lora_ids is not None:
            self.check_lora_ids(lora_ids, len(seqlens))
        last = self.pipeline_rank == self.num_pipeline_ranks - 1
        if last and self.num_pipeline_ranks == 1:
            if not self._uses_images(images) and self._graph_decode_ok(seqlens, cache):
                outs32 = self.decode_static(input_ids, cache, lora_ids=lora_ids).clone()
                return outs32 if self.softmax_fp32 else outs32.to(self.dtype)
            # single stage: final norm + lm head + .float() are one fused call (no [T, dim] normed round trip)
            h = self._hidden_no_norm(input_ids, seqlens, cache, images=images, lora_rows=self._lora_rows(lora_ids, seqlens))
            if cache is not None:
                cache.update_seqlens(seqlens)
            outs32 = torch.empty(h.shape[0], self.vocab_size, device=h.device, dtype=torch.float32)
            assert self.norm is not None and self.output_weight is not None
            _abi.lm_head(h, self.norm.weight, self.output_weight, outs32, self.args.norm_eps, self.workspace(h.shape[0]))
            return outs32 if self.softmax_fp32 else outs32.to(self.dtype)
        h = self.forward_partial(input_ids, seqlens, cache=cache, images=images)
        if not last:
            outs = torch.empty(h.shape[0], self.vocab_size, device=h.device, dtype=h.dtype)
        else:
            assert self.output_weight is not None
            outs = torch.empty(h.shape[0], self.vocab_size, device=h.device, dtype=h.dtype)
            _abi.linear_residual(h, self.output_weight, None, outs, self.workspace(h.shape[0]))
        if self.num_pipeline_ranks > 1:
            torch.distributed.broadcast(outs, src=self.num_pipeline_ranks - 1)
        return outs.float() if self.softmax_fp32 else outs

    def _hidden_no_norm(self, input_ids: torch.Tensor, seqlens: List[int], cache: Optional[BufferCache],
                        input_metadata: Optional[List[CacheInputMetadata]] = None,
                        images: Optional[List[torch.Tensor]] = None, lora_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        assert len(seqlens) <= self.args.max_batch_size, f"Max batch size is {self.args.max_batch_size}, got batch size of {len(seqlens)}"
        (num_toks,) = input_ids.shape
        assert sum(seqlens) == num_toks, (sum(seqlens), num_toks)
        ws = self.workspace(num_toks)
        if cache is not None:
            if input_metadata is None:
                self._check_positions(cache, seqlens)
                input_metadata = cache.get_input_metadata(seqlens)
            positions = input_metadata[0].positions
        else:
            positions = torch.cat([torch.arange(0, s, dtype=torch.int32) for s in seqlens]).to(self.device)
        assert self.tok_embeddings is not None
        h = self._embed(input_ids, images)
        rope = self.rope_table
        lora_rows = self._default_rows(lora_rows, num_toks)
        with _nvtx(f"mb200.layers[T={num_toks}]"):
            for local_layer_id, layer in enumerate(self.layers.values()):
                view = cache.get_view(local_layer_id, input_metadata[local_layer_id]) if cache is not None else None
                h = layer(h, rope, positions, view, ws, lora_rows)
        return h

    # ------------------------------------------------------------------ images (transformer.py:122-161,188-193)
    def _uses_images(self, images: Optional[List[torch.Tensor]]) -> bool:
        """A model without a vision encoder ignores `images`; an empty list takes the text path."""
        return self.vision_encoder is not None and bool(images)

    def _embed(self, input_ids: torch.Tensor, images: Optional[List[torch.Tensor]]) -> torch.Tensor:
        assert self.tok_embeddings is not None
        if self._uses_images(images):
            return self.embed_vision_language_features(input_ids, images)
        return self.tok_embeddings(input_ids)

    def embed_vision_language_features(self, input_ids: torch.Tensor, images: List[torch.Tensor]) -> torch.Tensor:
        """Encoder -> [pre_mm_projector_norm] -> [patch merger] -> adapter, then one kernel places the image features at the
        image-token positions (in order) and the text embeddings everywhere else."""
        ve = self.args.vision_encoder
        assert self.tok_embeddings is not None and self.vision_encoder is not None and self.vision_language_adapter is not None
        assert ve is not None
        with _nvtx(f"mb200.vision[{len(images)} images]"):
            feats = self.vision_encoder(images)
            ws = self.vision_encoder.workspace(feats.shape[0])
            if self.pre_mm_projector_norm is not None:
                feats = self.pre_mm_projector_norm(feats)
            if self.patch_merger is not None:
                p = ve.patch_size
                feats = self.patch_merger(feats, [(img.shape[1] // p, img.shape[2] // p) for img in images], ws)
            feats = self.vision_language_adapter(feats, ws)
        seq_len = input_ids.shape[0]
        out = torch.empty(seq_len, self.args.dim, dtype=self.tok_embeddings.weight.dtype, device=input_ids.device)
        n_img_tokens = _abi.embed_splice(input_ids, self.tok_embeddings.weight, feats, out, ve.image_token_id)
        assert n_img_tokens == feats.shape[0], (
            f"seq_len {seq_len} should be equal to N_txt + N_img {(seq_len - n_img_tokens, feats.shape[0], n_img_tokens)}")
        return out

    def _check_positions(self, cache: BufferCache, seqlens: List[int]) -> None:
        """The reference indexes freqs_cis[positions] and raises past the table (transformer.py:199); the kernels would read out of bounds."""
        host = cache._kv_seqlens_host or [0] * len(seqlens)
        last = max(p + s for p, s in zip(host, seqlens)) if seqlens else 0
        if last > ROPE_TABLE_LEN:
            raise IndexError(f"position {last - 1} is out of bounds for the rope table of {ROPE_TABLE_LEN} positions")

    # ------------------------------------------------------------------ CUDA-graph decode
    def _graph_decode_ok(self, seqlens: List[int], cache: Optional[BufferCache]) -> bool:
        if cache is None or self.num_pipeline_ranks != 1:
            return False
        if os.environ.get("MB200_DECODE_GRAPH", "1") == "0":
            return False
        host = cache._kv_seqlens_host
        return (host is not None and len(host) == len(seqlens) and host[0] != 0 and all(s == 1 for s in seqlens)
                and len(set(cache.cache_sizes)) <= 8)

    def _megakernel_ok(self, B: int) -> bool:
        # the megakernel has no LoRA stage and reads bf16 experts and a bf16 KV cache only: with un-merged adapters, FP8 experts or
        # an FP8 cache batch 1 takes the per-layer graph path (FP8 dense weights have a megakernel of their own: decode_step_fp8;
        # INT4 dense weights have none and take the graph path)
        # the shape limits (head ratio, K chunking, KV <= 8, MoE sizes, a shared-memory ring of >= 9 stages next to the
        # activations) are the library's, asked once per model: a model it refuses takes the per-layer path
        if not (B == 1 and self.num_pipeline_ranks == 1 and self.expert_parallel[1] == 1 and self.args.lora is None
                and self.expert_weights == "bf16" and self.kv_cache == "bf16" and self.dense_weights != "int4"
                and os.environ.get("MB200_MEGAKERNEL", "1") != "0"):
            return False
        if self._megakernel_refused is None:
            a, moe = self.args, self.args.moe
            if self.dense_weights == "fp8":
                self._megakernel_refused = _abi.decode_step_fp8_unsupported(a.dim, a.hidden_dim, a.n_heads, a.n_kv_heads, a.head_dim,
                                                                            self.vocab_size) or ""
            else:
                self._megakernel_refused = _abi.decode_step_unsupported(
                    a.dim, a.hidden_dim, a.n_heads, a.n_kv_heads, a.head_dim, self.vocab_size,
                    moe.num_experts if moe is not None else 0, moe.num_experts_per_tok if moe is not None else 0) or ""
        return self._megakernel_refused == ""

    def _decode_state(self, cache: BufferCache, key: Any) -> Dict[str, Any]:
        """Per-(cache, kind) decode state (descriptor tables, static buffers, captured graph).  It lives ON THE CACHE OBJECT, so
        it is freed with the cache (generate() allocates a cache per call); an entry is rebuilt when this model's workspace was
        reallocated since (a captured graph holds the old pointer)."""
        states = cache.__dict__.setdefault("_mb200_decode_states", {})
        ws_ptr = self._ws.ptr if self._ws is not None else 0
        st = states.get((id(self), key))
        if st is None or st["ws_ptr"] != ws_ptr or st["device"] != self.device:
            st = {"ws_ptr": ws_ptr, "device": self.device}
            states[(id(self), key)] = st
        return st

    @torch.inference_mode()
    def _decode_megakernel(self, tokens: torch.Tensor, cache: BufferCache) -> torch.Tensor:
        """Batch-1 decode step as ONE persistent cooperative kernel (csrc/decode_megakernel.cuh)."""
        import numpy as np

        a = self.args
        ws = self.workspace(1)
        st = self._decode_state(cache, "mk")
        fp8 = self.dense_weights == "fp8"
        if "layers" not in st:
            blocks = list(self.layers.values())
            desc = np.zeros((len(blocks), 12 if fp8 else 8), dtype=np.uint64)  # mb200_layer_desc(_fp8)
            moe = self.args.moe
            E = moe.num_experts if moe is not None else 0
            gate_tab, w13_tab, w2_tab = [], [], []
            for i, blk in enumerate(blocks):
                ff = blk.feed_forward
                if moe is None:
                    w13p, w2p = ff.w13.data_ptr(), ff.w2_weight.data_ptr()
                else:  # the kernel reads the expert tables instead
                    w13p = w2p = 0
                    gate_tab.append(ff.gate_weight.data_ptr())
                    w13_tab += [ff.experts[str(e)].w13.data_ptr() for e in range(E)]
                    w2_tab += [ff.experts[str(e)].w2_weight.data_ptr() for e in range(E)]
                desc[i, :8] = [blk.attention.wqkv.data_ptr(), blk.attention.wo_weight.data_ptr(), w13p, w2p,
                               blk.attention_norm.weight.data_ptr(), blk.ffn_norm.weight.data_ptr(), cache.cache_k[i].data_ptr(),
                               cache.cache_v[i].data_ptr()]
                if fp8:
                    desc[i, 8:] = [blk.attention.wqkv_scale.data_ptr(), blk.attention.wo_scale.data_ptr(), ff.w13_scale.data_ptr(),
                                   ff.w2_scale.data_ptr()]
            tab = lambda v: torch.tensor(v, dtype=torch.int64, device=self.device) if v else None  # noqa: E731
            st.update({"E": E, "k": moe.num_experts_per_tok if moe is not None else 0,
                       "moe_gate": tab(gate_tab), "moe_w13": tab(w13_tab), "moe_w2": tab(w2_tab),
                       "layers": torch.from_numpy(desc.view(np.int64)).to(self.device),
                       "windows": torch.tensor(cache.cache_sizes, dtype=torch.int32, device=self.device),
                       "token": torch.zeros(1, dtype=torch.long, device=self.device),
                       "next": torch.zeros(1, dtype=torch.long, device=self.device),
                       "logits": torch.empty(1, self.vocab_size, dtype=torch.float32, device=self.device)})
        if cache._kv_seqlens_host is None:
            cache.init_kvseqlens(1)
        pos = cache._kv_seqlens_host[0]
        if pos >= ROPE_TABLE_LEN:
            raise IndexError(f"position {pos} is out of bounds for the rope table of {ROPE_TABLE_LEN} positions")
        # `tokens` may be the previous step's fused argmax (st["next"]): then nothing is copied and the greedy loop is one
        # kernel launch per token
        tok = tokens.reshape(1)
        if tok.data_ptr() != st["next"].data_ptr():
            st["token"].copy_(tok, non_blocking=True)
            tok = st["token"]
        self.last_argmax = st["next"]
        with _nvtx("mb200.decode_megakernel"):
            if fp8:
                _abi.decode_step_fp8(st["layers"], st["windows"], self.n_local_layers, self.tok_embeddings.weight, self.norm.weight,
                                     self.output_weight, self.rope_table, tok, pos, 0, st["logits"], st["next"], a.dim, a.hidden_dim,
                                     a.n_heads, a.n_kv_heads, a.head_dim, self.vocab_size, a.norm_eps, ws)
            else:
                _abi.decode_step(st["layers"], st["windows"], self.n_local_layers, self.tok_embeddings.weight, self.norm.weight,
                                 self.output_weight, self.rope_table, tok, pos, 0, st["logits"], st["next"], a.dim, a.hidden_dim, a.n_heads,
                                 a.n_kv_heads, a.head_dim, self.vocab_size, a.norm_eps, ws, st["E"], st["k"], st["moe_gate"], st["moe_w13"],
                                 st["moe_w2"])
        cache.update_seqlens([1])
        self._last_static_logits = st["logits"].data_ptr()
        return st["logits"]

    @torch.inference_mode()
    def decode_static(self, tokens: torch.Tensor, cache: BufferCache, *, lora_ids: Optional[List[int]] = None) -> torch.Tensor:
        """One decode step for every sequence of `cache` (one new token each).  Batch 1: the persistent megakernel.  Batch > 1:
        the per-layer kernels replayed from a CUDA graph.  The step state lives on the DEVICE: `mb200_decode_meta` derives
        positions / ring rows / kv lengths from a device-side position vector and advances it inside the graph, so a replay
        needs no host write at all (a pinned staging buffer rewritten by the host while earlier copies are still queued was the
        round-1 design and a race).  Returns the STATIC fp32 logits buffer [B, V] (overwritten by the next step).  The first call
        per (cache, batch) runs eagerly (warm-up: loads modules, sets function attributes), the second captures.
        `lora_ids` (see forward) live in a static device vector of the step state, rewritten only when they change."""
        B = tokens.shape[0]
        self._check_cache(cache)
        if lora_ids is not None:
            self.check_lora_ids(lora_ids, B)
        if self._megakernel_ok(B):  # never with adapters
            return self._decode_megakernel(tokens, cache)
        seqlens = [1] * B
        self.workspace(B)
        masked = lora_ids is not None or self.lora_slots > 1
        st = self._decode_state(cache, ("graph", B, "lora_rows") if masked else ("graph", B))
        if masked:
            ids = list(lora_ids) if lora_ids is not None else [0] * B
            if "lora_rows" not in st:
                st.update({"lora_rows": torch.empty(B, dtype=torch.int32, device=self.device), "lora_ids": None})
            if st["lora_ids"] != ids:
                st["lora_rows"].copy_(torch.tensor(ids, dtype=torch.int32))  # pageable source: staged by the runtime, like seqpos
                st["lora_ids"] = ids
        host = cache._kv_seqlens_host
        assert host is not None and len(host) == B, "decode_static needs a prefilled cache of this batch size"
        if max(host) >= ROPE_TABLE_LEN:
            raise IndexError(f"position {max(host)} is out of bounds for the rope table of {ROPE_TABLE_LEN} positions")
        distinct = sorted(set(cache.cache_sizes))
        if "meta" not in st:
            st.update({"graph": None, "warmed": False, "expected": None,
                       "seqpos": torch.zeros(B, dtype=torch.int32, device=self.device),
                       "tokens": torch.zeros(B, dtype=torch.long, device=self.device),
                       "meta": torch.zeros(3 * B + 1 + 2 * B * len(distinct), dtype=torch.int32, device=self.device),
                       "logits": torch.empty(B, self.vocab_size, dtype=torch.float32, device=self.device),
                       "next": torch.zeros(B, dtype=torch.long, device=self.device)})
        if st["expected"] != host:  # another forward() advanced the cache since the last step (or this is the first one)
            st["seqpos"].copy_(torch.tensor(host, dtype=torch.int32))  # pageable source: staged by the runtime, no reuse hazard
        st["tokens"].copy_(tokens, non_blocking=True)  # device source (previous pick): D2D; host source: staged by the runtime
        layout = {"T": B, "B": B, "prefill": False, "first_prefill": False, "max_seqlen": 1, "windows": distinct}
        md = cache.metadata_from_block(st["meta"], layout, seqlens)

        def run() -> None:
            _abi.decode_meta(st["seqpos"], st["meta"], distinct)
            h = self._hidden_no_norm(st["tokens"], seqlens, cache, md, lora_rows=st.get("lora_rows"))
            _abi.lm_head(h, self.norm.weight, self.output_weight, st["logits"], self.args.norm_eps, self.workspace(B))
            _abi.argmax_rows(st["logits"], st["next"])  # greedy pick on the device (generate.py:156): feeds the next step

        if st["graph"] is None and not st["warmed"]:
            run()
            st["warmed"] = True
        elif st["graph"] is None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                run()
            st["graph"] = g
            g.replay()
        else:
            st["graph"].replay()
        cache.update_seqlens(seqlens)
        st["expected"] = list(cache._kv_seqlens_host)
        self.last_argmax = st["next"]
        self._last_static_logits = st["logits"].data_ptr()
        return st["logits"]

    # ------------------------------------------------------------------ speculative decoding: the verify step
    @torch.inference_mode()
    def verify_static(self, tokens: torch.Tensor, cache: BufferCache) -> Tuple[torch.Tensor, torch.Tensor]:
        """One forward of S = tokens.shape[1] tokens for every sequence of `cache` (the verify step of speculative decoding:
        [last, d_1 .. d_k]), on the chunked-prefill kernels at T = B * S.  Like decode_static, the step state lives on the
        device: `mb200_spec_meta` builds the metadata block from a device-side position vector, so from the second call per
        (cache, B, S) on the step is ONE CUDA-graph replay with no host write (the first call runs eagerly, the second captures).
        Unlike decode_static the positions are not advanced here: the acceptance kernel advances them by what the round keeps,
        and the caller reports that with `verify_accepted`.  Returns (the static fp32 logits [B * S, V], overwritten by the next
        step; the device positions [B] int32 the step read)."""
        B, S = tokens.shape
        self._check_runnable()
        self._check_cache(cache)
        assert self.num_pipeline_ranks == 1, "the verify step runs on a single pipeline stage"
        seqlens = [S] * B
        self.workspace(B * S)
        st = self._decode_state(cache, ("verify", B, S))
        host = cache._kv_seqlens_host
        assert host is not None and len(host) == B and min(host) > 0, "verify_static needs a prefilled cache of this batch size"
        if max(host) + S > ROPE_TABLE_LEN:
            raise IndexError(f"position {max(host) + S - 1} is out of bounds for the rope table of {ROPE_TABLE_LEN} positions")
        distinct = sorted(set(cache.cache_sizes))
        if "meta" not in st:
            st.update({"graph": None, "warmed": False, "expected": None,
                       "seqpos": torch.zeros(B, dtype=torch.int32, device=self.device),
                       "tokens": torch.zeros(B * S, dtype=torch.long, device=self.device),
                       "meta": torch.zeros(_abi.spec_meta_words(B, S, len(distinct)), dtype=torch.int32, device=self.device),
                       "logits": torch.empty(B * S, self.vocab_size, dtype=torch.float32, device=self.device)})
        if st["expected"] != host:  # the cache moved other than by the accepted lengths (or this is the first step)
            st["seqpos"].copy_(torch.tensor(host, dtype=torch.int32))
        st["tokens"].copy_(tokens.reshape(-1), non_blocking=True)
        layout = {"T": B * S, "B": B, "prefill": True, "first_prefill": False, "max_seqlen": S, "windows": distinct}
        md = cache.metadata_from_block(st["meta"], layout, seqlens)

        def run() -> None:
            _abi.spec_meta(st["seqpos"], st["meta"], S, distinct)
            h = self._hidden_no_norm(st["tokens"], seqlens, cache, md)
            _abi.lm_head(h, self.norm.weight, self.output_weight, st["logits"], self.args.norm_eps, self.workspace(B * S))

        if st["graph"] is None and not st["warmed"]:
            run()
            st["warmed"] = True
        elif st["graph"] is None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                run()
            st["graph"] = g
            g.replay()
        else:
            st["graph"].replay()
        st["expected"] = None  # valid again once verify_accepted reports what the device positions became
        self._last_static_logits = 0
        return st["logits"], st["seqpos"]

    def verify_accepted(self, cache: BufferCache, S: int, device_lens: List[int]) -> None:
        """After a verify step of S tokens per sequence: the acceptance kernel left `device_lens` in the step's device positions.
        The next step uploads the host lengths only where they differ (a rewound or frozen sequence)."""
        st = self._decode_state(cache, ("verify", len(device_lens), S))
        st["expected"] = list(device_lens)

    @torch.inference_mode()
    def last_token_logits(self, input_ids: torch.Tensor, seqlens: List[int], cache: BufferCache, *,
                          lora_ids: Optional[List[int]] = None) -> torch.Tensor:
        """fp32 logits [B, V] of each sequence's last token of a ragged forward that extends `cache` (the lm head runs on those
        rows only).  `lora_ids`: see forward."""
        self._check_runnable()
        self._check_cache(cache)
        self._last_static_logits = 0
        h = self._hidden_no_norm(input_ids, seqlens, cache, lora_rows=self._lora_rows(lora_ids, seqlens))
        cache.update_seqlens(seqlens)
        last_idx = torch.tensor(seqlens, device=input_ids.device).cumsum(0) - 1
        logits = torch.empty(len(seqlens), self.vocab_size, dtype=torch.float32, device=h.device)
        _abi.lm_head(h.index_select(0, last_idx), self.norm.weight, self.output_weight, logits, self.args.norm_eps,
                     self.workspace(h.shape[0]))
        return logits

    # ------------------------------------------------------------------ generate() support (SURVEY.md N1 / N2)
    def last_argmax_valid_for(self, logits: torch.Tensor) -> bool:
        """True when `last_argmax` is the decode kernel's own argmax of exactly this logits buffer."""
        return self.last_argmax is not None and logits.data_ptr() == self._last_static_logits

    @torch.inference_mode()
    def next_token_logits(self, tokens: torch.Tensor, cache: BufferCache, *, lora_ids: Optional[List[int]] = None) -> torch.Tensor:
        """fp32 logits [B, V] of one decode step for every sequence.  On the single-stage CUDA path this is the step's static
        buffer (no clone; valid until the next step), otherwise `forward`.  `lora_ids`: see forward."""
        B = tokens.shape[0]
        if self.pipeline_rank == self.num_pipeline_ranks - 1 == 0 and self._graph_decode_ok([1] * B, cache):
            self._check_runnable()
            return self.decode_static(tokens, cache, lora_ids=lora_ids)
        self._last_static_logits = 0
        out = self.forward(tokens, [1] * B, cache, lora_ids=lora_ids)
        return out if out.dtype == torch.float32 else out.float()

    @torch.inference_mode()
    def forward_logprobs(self, input_ids: torch.Tensor, seqlens: List[int], cache: Optional[BufferCache],
                         targets: torch.Tensor, images: Optional[List[torch.Tensor]] = None, *,
                         lora_ids: Optional[List[int]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """One prompt chunk for generate(): returns (lp [T] fp32 with lp[t] = log_softmax(logits[t])[targets[t]] where
        targets[t] >= 0, logits [B, V] fp32 of each sequence's last token).  Replaces forward + log_softmax over [T, V] +
        per-token gathers (generate.py:97-118): the lm head runs over blocks of rows, each followed by the fused
        log-softmax + gather kernel, so the full [T, V] logits never exist.  `lora_ids`: see forward."""
        self._last_static_logits = 0
        self._check_cache(cache)
        if lora_ids is not None:
            self.check_lora_ids(lora_ids, len(seqlens))
        T, V = input_ids.shape[0], self.vocab_size
        last_idx = torch.tensor(seqlens, device=input_ids.device).cumsum(0) - 1
        lp = torch.zeros(T, dtype=torch.float32, device=input_ids.device)
        if self.num_pipeline_ranks > 1:  # reference-compatible pipeline mode: logits arrive by broadcast (transformer.py:236-237)
            logits = self.forward(input_ids, seqlens, cache, images=images).float().contiguous()
            _abi.logprob_gather(logits, targets, out=lp)
            return lp, logits.index_select(0, last_idx)
        self._check_runnable()
        h = self._hidden_no_norm(input_ids, seqlens, cache, images=images, lora_rows=self._lora_rows(lora_ids, seqlens))
        if cache is not None:
            cache.update_seqlens(seqlens)
        assert self.norm is not None and self.output_weight is not None
        rows = max(128, (256 << 20) // (4 * V))
        ws = self.workspace(max(T, 1))
        block = torch.empty(min(rows, T), V, dtype=torch.float32, device=h.device)
        for r0 in range(0, T, rows):
            r1 = min(T, r0 + rows)
            _abi.lm_head(h[r0:r1], self.norm.weight, self.output_weight, block[: r1 - r0], self.args.norm_eps, ws)
            _abi.logprob_gather(block[: r1 - r0], targets[r0:r1], out=lp[r0:r1])
        last_logits = torch.empty(len(seqlens), V, dtype=torch.float32, device=h.device)
        _abi.lm_head(h.index_select(0, last_idx), self.norm.weight, self.output_weight, last_logits, self.args.norm_eps, ws)
        return lp, last_logits

    # ------------------------------------------------------------------ weights
    def _assign(self, k: str, v: torch.Tensor, lora_slot: int = 0) -> bool:
        """Copies reference-keyed tensor `v` into the packed parameters (LoRA keys: into adapter slot `lora_slot`).  Returns False
        when the key belongs to another pipeline rank."""
        def put(dst: torch.Tensor, setter=None, seg: int = 0) -> None:
            assert dst.shape == v.shape, f"{k}: shape {tuple(v.shape)} != expected {tuple(dst.shape)}"
            if setter is None:
                dst.copy_(v)
            else:
                setter(seg, v)

        if k == "tok_embeddings.weight":
            if self.tok_embeddings is None:
                return False
            put(self.tok_embeddings.weight)
        elif k == "norm.weight":
            if self.norm is None:
                return False
            put(self.norm.weight)
        elif k == "output.weight":
            if self.output_weight is None:
                return False
            put(self.output_weight)
        elif k.startswith(_VISION_PREFIXES):
            if self.pipeline_rank != 0:
                return False
            return self._assign_vision(k, v, put)
        elif k.startswith("layers."):
            _, lid, rest = k.split(".", 2)
            if lid not in self.layers:
                return False
            return self._assign_block(self.layers[lid], k, rest, put, lora_slot)
        else:
            raise ValueError(f"Unexpected key {k}")
        return True

    @staticmethod
    def _assign_block(blk: TransformerBlock, k: str, rest: str, put, lora_slot: int = 0) -> bool:
        """`rest` = the key below `layers.{i}.` of one TransformerBlock (text or vision)."""
        att = blk.attention
        if att.lora is not None:
            name, part = rest.rsplit(".", 1)[0], ""
            for suffix in _LORA_PARTS:
                if rest.endswith(suffix):
                    name, part = rest[: -len(suffix)], suffix
            slot = None
            if name in _LORA_LINEARS:
                path, seg = _LORA_LINEARS[name]
                slot = blk.get_submodule(path), seg
            elif _EXPERT_LINEAR.match(name) and (part or rest.endswith(".weight")) and hasattr(blk.feed_forward, "experts"):
                # the LoRALinears of FP8 experts
                e, lin = name.split(".")[2:]
                if e not in blk.feed_forward.experts:
                    return False  # an expert owned by another expert-parallel rank
                slot = blk.feed_forward.experts[e].adapter(lin)
            if slot is not None:
                adapter, seg = slot
                if part == ".lora_A.weight":
                    put(adapter.lora_A(seg, lora_slot), lambda s, w: adapter.put_A(s, w, lora_slot), seg)
                    return True
                if part == ".lora_B.weight":
                    put(adapter.lora_B(seg, lora_slot), lambda s, w: adapter.put_B(s, w, lora_slot), seg)
                    return True
                if part == "":  # a full checkpoint's plain weight: zero adapter (lora.py:76-89)
                    adapter.zero(seg, lora_slot)
                rest = name + ".weight"
        ff = blk.feed_forward
        if getattr(att, "fp8", False):  # FP8 dense weights: the reference's bf16 weight, quantised into place
            for mod, names in ((att, ("wq", "wk", "wv", "wo")), (ff, ("w1", "w2", "w3"))):
                for name in names:
                    if rest.startswith(f"{'attention' if mod is att else 'feed_forward'}.{name}."):
                        if rest.rsplit(".", 1)[1] != "weight":
                            raise ValueError(f"Unexpected key {k}")
                        put(mod.weight_e4m3(name), lambda _seg, w, mod=mod, name=name: mod.quantize_(name, w))
                        return True
        if getattr(att, "int4", False):  # INT4 dense weights: the reference's bf16 weight, quantised into place (the codes are [N, K/2])
            dense = ((att, ("wq", "wk", "wv", "wo")),) + (() if hasattr(ff, "experts") else ((ff, ("w1", "w2", "w3")),))
            for mod, names in dense:
                for name in names:
                    if rest.startswith(f"{'attention' if mod is att else 'feed_forward'}.{name}."):
                        if rest.rsplit(".", 1)[1] != "weight":
                            raise ValueError(f"Unexpected key {k}")
                        q = mod.weight_int4(name)
                        put(torch.empty(q.shape[0], 2 * q.shape[1], device="meta"),  # the bf16 shape, checked by put
                            lambda _seg, w, mod=mod, name=name: mod.quantize_int4_(name, w))
                        return True
        if rest == "attention.wq.weight":
            put(att.wqkv[: att.q_dim])
        elif rest == "attention.wk.weight":
            put(att.wqkv[att.q_dim: att.q_dim + att.kv_dim])
        elif rest == "attention.wv.weight":
            put(att.wqkv[att.q_dim + att.kv_dim:])
        elif rest == "attention.wo.weight":
            put(att.wo_weight)
        elif rest == "attention_norm.weight":
            put(blk.attention_norm.weight)
        elif rest == "ffn_norm.weight":
            put(blk.ffn_norm.weight)
        elif rest == "feed_forward.gate.weight":
            put(blk.feed_forward.gate_weight)
        else:
            parts = rest.split(".")
            if parts[0] != "feed_forward":
                raise ValueError(f"Unexpected key {k}")
            ff = blk.feed_forward
            if parts[1] == "experts":
                if parts[2] not in ff.experts:
                    return False  # an expert owned by another expert-parallel rank
                ff = ff.experts[parts[2]]
                parts = parts[2:]
                if isinstance(ff, Fp8Expert):  # the reference's bf16 weight, quantised into place
                    if parts[2:] != ["weight"] or parts[1] not in ("w1", "w2", "w3"):
                        raise ValueError(f"Unexpected key {k}")
                    name = parts[1]
                    put(ff.weight_e4m3(name), lambda _seg, w: ff.quantize_(name, w))
                    return True
                if isinstance(ff, Int4Expert):  # the reference's bf16 weight, quantised into place (the codes are [N, K/2])
                    if parts[2:] != ["weight"] or parts[1] not in ("w1", "w2", "w3"):
                        raise ValueError(f"Unexpected key {k}")
                    name = parts[1]
                    q = ff.weight_int4(name)
                    put(torch.empty(q.shape[0], 2 * q.shape[1], device="meta"), lambda _seg, w: ff.quantize_int4_(name, w))
                    return True
            elif hasattr(ff, "experts"):  # a MoE block has no dense feed_forward.w1/w2/w3
                raise ValueError(f"Unexpected key {k}")
            name = parts[1]
            if name == "w1":
                put(ff.w13.view(ff.hidden_dim, 2, ff.dim)[:, 0])
            elif name == "w3":
                put(ff.w13.view(ff.hidden_dim, 2, ff.dim)[:, 1])
            elif name == "w2":
                put(ff.w2_weight)
            else:
                raise ValueError(f"Unexpected key {k}")
        return True

    def _assign_vision(self, k: str, v: torch.Tensor, put) -> bool:
        ve, adapter = self.vision_encoder, self.vision_language_adapter
        if ve is None or adapter is None:
            raise ValueError(f"Unexpected key {k}")
        if k == "vision_encoder.patch_conv.weight":
            ve.patch_conv_weight[:, ve.k_conv:].zero_()  # the GEMM reads the padding columns
            put(ve.patch_conv.weight)
        elif k == "vision_encoder.ln_pre.weight":
            put(ve.ln_pre.weight)
        elif k.startswith("vision_encoder.transformer.layers."):
            _, _, _, lid, rest = k.split(".", 4)
            if not lid.isdigit() or int(lid) >= len(ve.transformer.layers):
                raise ValueError(f"Unexpected key {k}")
            return self._assign_block(ve.transformer.layers[int(lid)], k, rest, put)
        elif k in ("vision_language_adapter.w_in.weight", "vision_language_adapter.w_out.weight",
                   "vision_language_adapter.w_in.bias", "vision_language_adapter.w_out.bias"):
            dst = getattr(adapter, k.split(".", 1)[1].replace(".", "_"))
            if dst is None:
                raise ValueError(f"Unexpected key {k}")
            put(dst)
        elif k == "pre_mm_projector_norm.weight" and self.pre_mm_projector_norm is not None:
            put(self.pre_mm_projector_norm.weight)
        elif k == "patch_merger.merging_layer.weight" and self.patch_merger is not None:
            put(self.patch_merger.merging_layer_weight)
        else:
            raise ValueError(f"Unexpected key {k}")
        return True

    def _owns_key(self, k: str) -> bool:
        """False for checkpoint tensors that belong to another pipeline / expert-parallel rank (decided from the key alone, so a
        loader can skip reading them)."""
        if k.startswith(_VISION_PREFIXES):
            return self.pipeline_rank == 0
        if not k.startswith("layers."):
            return True
        _, lid, rest = k.split(".", 2)
        if lid not in self.layers:
            return False
        parts = rest.split(".")
        if len(parts) > 2 and parts[0] == "feed_forward" and parts[1] == "experts":
            return parts[2] in self.layers[lid].feed_forward.experts
        return True

    def load_state_dict(self, state_dict: Mapping[str, Any], strict: bool = True, assign: bool = False) -> None:  # type: ignore[override]
        """Takes a REFERENCE-keyed state dict (transformer.py:244-295), filters by pipeline rank and packs."""
        del assign  # tensors are copied into the packed buffers
        loaded = set()
        with torch.no_grad():
            for k, v in state_dict.items():
                if self._assign(k, v):
                    loaded.add(k)
                else:
                    logging.debug("Skipping parameter %s at pipeline rank %d", k, self.pipeline_rank)
        if strict:
            missing = self._missing_keys(loaded)
            assert not missing, f"missing keys: {sorted(missing)[:8]}"

    def reference_keys(self) -> List[str]:
        return list(self.state_dict().keys())

    def _missing_keys(self, loaded) -> set:
        """Keys of this rank that a load left unset.  With un-merged adapters a plain `X.weight` provides `X.linear.weight` and
        adapters may be absent (they stay zero); the reference's post-hook clears every missing key (lora.py:66-69), this keeps
        the base weights strict."""
        if self.args.lora is None:
            # an FP8 Linear's `X.weight_e4m3` and `X.weight_scale`, an INT4 one's `X.weight_int4` and `X.weight_gscale`, are set by the
            # reference's `X.weight`
            have = set(loaded) | {k[: -len(".weight")] + sfx for k in loaded
                                  for sfx in (".weight_e4m3", ".weight_scale", ".weight_int4", ".weight_gscale")}
            return set(self.reference_keys()) - have
        # an FP8 expert's `X.linear.weight_e4m3` and `X.linear.weight_scale` are set by `X.linear.weight` or a plain `X.weight`
        bases = {k[: -len(".linear.weight")] if k.endswith(".linear.weight") else k[: -len(".weight")] for k in loaded}
        have = set(loaded) | {b + sfx for b in bases for sfx in (".linear.weight", ".linear.weight_e4m3", ".linear.weight_scale")}
        return {k for k in self.reference_keys() if k not in have and not k.endswith((".lora_A.weight", ".lora_B.weight"))}

    def state_dict(self, *args: Any, **kwargs: Any) -> Dict[str, torch.Tensor]:  # type: ignore[override]
        """Reference-keyed views of the packed parameters."""
        out: Dict[str, torch.Tensor] = {}
        if self.tok_embeddings is not None:
            out["tok_embeddings.weight"] = self.tok_embeddings.weight
        if self.vision_encoder is not None and self.vision_language_adapter is not None:
            ve = self.vision_encoder
            out["vision_encoder.patch_conv.weight"] = ve.patch_conv.weight
            out["vision_encoder.ln_pre.weight"] = ve.ln_pre.weight
            for i, blk in enumerate(ve.transformer.layers):
                self._block_state(out, f"vision_encoder.transformer.layers.{i}.", blk)
            for n in ("w_in", "w_out"):
                lin = getattr(self.vision_language_adapter, n)
                out[f"vision_language_adapter.{n}.weight"] = lin.weight
                if lin.bias is not None:
                    out[f"vision_language_adapter.{n}.bias"] = lin.bias
            if self.pre_mm_projector_norm is not None:
                out["pre_mm_projector_norm.weight"] = self.pre_mm_projector_norm.weight
            if self.patch_merger is not None:
                out["patch_merger.merging_layer.weight"] = self.patch_merger.merging_layer_weight
        for lid, blk in self.layers.items():
            self._block_state(out, f"layers.{lid}.", blk)
        if self.norm is not None:
            out["norm.weight"] = self.norm.weight
            out["output.weight"] = self.output_weight
        return out

    @staticmethod
    def _block_state(out: Dict[str, torch.Tensor], p: str, blk: TransformerBlock) -> None:
        att = blk.attention
        fp8 = getattr(att, "fp8", False)
        int4 = getattr(att, "int4", False)
        if not (fp8 or int4):
            for n in ("wq", "wk", "wv", "wo"):
                Transformer._linear_state(out, p, blk, "attention." + n, getattr(att, n).weight)
        out[p + "attention_norm.weight"] = blk.attention_norm.weight
        out[p + "ffn_norm.weight"] = blk.ffn_norm.weight
        ff = blk.feed_forward
        if fp8:  # the stored format itself: no dequantised copies
            for mod, prefix, names in ((att, "attention.", ("wq", "wk", "wv", "wo")), (ff, "feed_forward.", ("w1", "w2", "w3"))):
                for n in names:
                    out[p + prefix + n + ".weight_e4m3"] = mod.weight_e4m3(n)
                    out[p + prefix + n + ".weight_scale"] = mod.weight_scale(n)
            return
        if int4:  # the stored format itself: no dequantised copies (on a MoE block the attention Linears only)
            moe = hasattr(ff, "experts")
            dense = ((att, "attention.", ("wq", "wk", "wv", "wo")),) + (() if moe else ((ff, "feed_forward.", ("w1", "w2", "w3")),))
            for mod, prefix, names in dense:
                for n in names:
                    out[p + prefix + n + ".weight_int4"] = mod.weight_int4(n)
                    out[p + prefix + n + ".weight_gscale"] = mod.weight_gscale(n)
            if not moe:
                return
        if hasattr(ff, "experts"):
            out[p + "feed_forward.gate.weight"] = ff.gate_weight
            for e, ex in ff.experts.items():  # keyed by the global expert id; the local ones only when sharded
                for n in ("w1", "w2", "w3"):
                    if isinstance(ex, Fp8Expert) and ex.lora is not None:  # LoRALinear's keys, the base in its stored format
                        adapter, seg = ex.adapter(n)
                        out[p + f"feed_forward.experts.{e}.{n}.lora_A.weight"] = adapter.lora_A(seg)
                        out[p + f"feed_forward.experts.{e}.{n}.lora_B.weight"] = adapter.lora_B(seg)
                        out[p + f"feed_forward.experts.{e}.{n}.linear.weight_e4m3"] = ex.weight_e4m3(n)
                        out[p + f"feed_forward.experts.{e}.{n}.linear.weight_scale"] = ex.weight_scale(n)
                    elif isinstance(ex, Fp8Expert):  # the stored format itself: no dequantised copies
                        out[p + f"feed_forward.experts.{e}.{n}.weight_e4m3"] = ex.weight_e4m3(n)
                        out[p + f"feed_forward.experts.{e}.{n}.weight_scale"] = ex.weight_scale(n)
                    elif isinstance(ex, Int4Expert):
                        out[p + f"feed_forward.experts.{e}.{n}.weight_int4"] = ex.weight_int4(n)
                        out[p + f"feed_forward.experts.{e}.{n}.weight_gscale"] = ex.weight_gscale(n)
                    else:
                        out[p + f"feed_forward.experts.{e}.{n}.weight"] = getattr(ex, n).weight
        else:
            for n in ("w1", "w2", "w3"):
                Transformer._linear_state(out, p, blk, "feed_forward." + n, getattr(ff, n).weight)

    @staticmethod
    def _linear_state(out: Dict[str, torch.Tensor], p: str, blk: TransformerBlock, name: str, weight: torch.Tensor) -> None:
        """`X.weight`, or with un-merged adapters LoRALinear's `X.lora_A.weight`, `X.lora_B.weight`, `X.linear.weight`."""
        if blk.attention.lora is None:
            out[p + name + ".weight"] = weight
            return
        path, seg = _LORA_LINEARS[name]
        adapter = blk.get_submodule(path)
        out[p + name + ".lora_A.weight"] = adapter.lora_A(seg)
        out[p + name + ".lora_B.weight"] = adapter.lora_B(seg)
        out[p + name + ".linear.weight"] = weight

    # ------------------------------------------------------------------ LoRA (lora.py:92-155)
    def load_lora(self, lora_path: Union[Path, str], scaling: float = 2.0, *, slot: int = 0) -> None:
        """Loads a LoRA checkpoint.  args.lora None: MERGES it into the packed weights (lora.py:120-139).  args.lora set: copies
        it into the un-merged adapters (lora.py:140-155) of adapter slot `slot` (in [0, lora_slots)), replacing that slot's
        previous adapter of every Linear it names."""
        import safetensors.torch

        lora_path = Path(lora_path)
        assert lora_path.is_file(), f"{lora_path} does not exist or is not a file"
        self._load_lora_state_dict(safetensors.torch.load_file(str(lora_path)), scaling=scaling, slot=slot)

    def _load_lora_state_dict(self, lora_state_dict: Dict[str, torch.Tensor], scaling: float = 2.0, slot: int = 0) -> None:
        """args.lora None: weight <- weight + (lora_B @ lora_A) * scaling for every Linear of this rank except the output layer,
        with the same torch ops and dtype as the reference (lora.py:129-137).
        args.lora set: each `X.lora_A/B.weight` is copied in place into this rank's adapter slots (captured decode graphs keep
        their pointers).  `scaling` is ignored, as in the reference: every adapter keeps args.lora.scaling.  Keys of layers that
        other pipeline ranks own are skipped (the reference's strict load_state_dict would raise on them)."""
        if not isinstance(slot, int) or not 0 <= slot < self.lora_slots:
            raise ValueError(f"adapter slot {slot!r} outside [0, {self.lora_slots})")
        lora_dtypes = set(p.dtype for p in lora_state_dict.values())
        assert len(lora_dtypes) == 1, f"LoRA weights have multiple different dtypes {lora_dtypes}. All weights need to have the same dtype"
        lora_dtype = lora_dtypes.pop()
        assert lora_dtype == self.dtype, f"LoRA weights dtype differs from model's dtype {lora_dtype} != {self.dtype}"
        assert all("lora" in key for key in lora_state_dict.keys())
        if self.dense_weights != "bf16" and any(key.startswith("layers.") for key in lora_state_dict):
            raise NotImplementedError(f"merging a LoRA adapter into {self.dense_weights.upper()} dense weights is not built: the layer "
                                      "Linears are stored quantised (load the adapter into a bf16 model)")
        if self.args.lora is None and self.expert_weights != "bf16" and any(".experts." in key for key in lora_state_dict):
            raise NotImplementedError(f"merging a LoRA adapter into {self.expert_weights.upper()} expert weights is not built: the experts "
                                      "are stored quantised (load the adapter into a bf16 model, or drop its expert Linears)")
        lora_state_dict = {k: v.to(self.device) for k, v in lora_state_dict.items()}
        if self.args.lora is not None:
            with torch.no_grad():
                for k, v in lora_state_dict.items():
                    if not k.endswith((".lora_A.weight", ".lora_B.weight")) or not k.startswith("layers."):
                        raise ValueError(f"Unexpected key {k}")
                    if not self._assign(k, v, slot):
                        logging.debug("Skipping parameter %s at pipeline rank %d", k, self.pipeline_rank)
            return
        with torch.no_grad():
            for key, weight in self.state_dict().items():
                if not key.endswith(".weight") or key == "output.weight" or not key.startswith("layers."):
                    continue
                name = key[: -len(".weight")]
                if (name + ".lora_B.weight") in lora_state_dict:
                    merged = weight + (lora_state_dict[name + ".lora_B.weight"] @ lora_state_dict[name + ".lora_A.weight"]) * scaling
                    assert self._assign(key, merged)

    @staticmethod
    def empty(args: TransformerArgs, device: Union[torch.device, str] = "cuda", dtype: torch.dtype = torch.bfloat16, **kwargs: Any) -> "Transformer":
        """A model with UNINITIALISED parameters allocated once, directly in `dtype` on `device` (shapes are laid out on `meta`
        first).  `Transformer(args)` under `torch.device("cuda")` would allocate fp32 and run the Embedding initialiser there:
        2-3x the model's bf16 bytes at the peak (Mixtral-8x7B: 187 GB)."""
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        with torch.device("meta"):
            m = Transformer(args, **kwargs)
        m = m.to(dtype=dtype).to_empty(device=dev)
        with torch.no_grad():
            for mod in m.modules():  # the packed adapters' zeros outside the segments are part of the format
                if isinstance(mod, LoraAdapter):
                    mod.a.zero_()
                    mod.b.zero_()
        return m

    @staticmethod
    def from_folder(folder: Union[Path, str], max_batch_size: int = 1, num_pipeline_ranks: int = 1,
                    device: Union[torch.device, str] = "cuda", dtype: Optional[torch.dtype] = None,
                    softmax_fp32: bool = True, expert_parallel: Optional[Tuple[int, int]] = None, expert_group: Any = None,
                    expert_weights: str = "bf16", *, kv_cache: str = "bf16", dense_weights: str = "bf16",
                    lora_slots: int = 1, prefill_compute: str = "bf16") -> "Transformer":
        """transformer.py:297-338.  Tensors stream from disk straight into the packed device buffers; with `expert_parallel`
        the experts of other ranks are skipped (never read into device memory).  With expert_weights="fp8" or "int4" each bf16
        expert tensor is copied to the device and quantised into place: the peak is the quantised model plus about one bf16 tensor.
        `kv_cache` ("bf16" | "fp8") is the format of the KV cache that generate() builds (see Transformer).  With
        dense_weights="fp8" or "int4" every bf16 layer Linear is quantised into place the same way.  `lora_slots` and
        `prefill_compute`: see Transformer; the checkpoint's adapter, if any, fills slot 0."""
        with open(Path(folder) / "params.json", "r") as f:
            model_args = TransformerArgs.from_dict(json.load(f))
        model_args.max_batch_size = max_batch_size
        pipeline_rank = torch.distributed.get_rank() if num_pipeline_ranks > 1 else 0

        pt_model_file = Path(folder) / "consolidated.00.pth"
        safetensors_model_file = Path(folder) / "consolidated.safetensors"
        assert pt_model_file.exists() or safetensors_model_file.exists(), f"Make sure either {pt_model_file} or {safetensors_model_file} exists"
        assert not (pt_model_file.exists() and safetensors_model_file.exists()), f"Both {pt_model_file} and {safetensors_model_file} cannot exist"

        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())

        def build(ck_dtype: torch.dtype) -> "Transformer":
            # shapes on `meta`, storage allocated ONCE, directly in the target dtype on the target device (the reference builds
            # on meta and assigns, transformer.py:321-331; a fp32 build followed by .to(bf16) would need 3x the model's bytes)
            return Transformer.empty(model_args, dev, dtype or ck_dtype, pipeline_rank=pipeline_rank, num_pipeline_ranks=num_pipeline_ranks,
                                     softmax_fp32=softmax_fp32, expert_parallel=expert_parallel, expert_group=expert_group,
                                     expert_weights=expert_weights, kv_cache=kv_cache, dense_weights=dense_weights, lora_slots=lora_slots,
                                     prefill_compute=prefill_compute)

        if pt_model_file.exists():
            loaded = torch.load(str(pt_model_file), mmap=True)
            model = build(next(iter(loaded.values())).dtype)
            model.load_state_dict(loaded, strict=True)
        else:
            import safetensors

            with safetensors.safe_open(str(safetensors_model_file), framework="pt", device="cpu") as f:
                keys = list(f.keys())
                probe = "norm.weight" if "norm.weight" in keys else keys[0]
                model = build(f.get_tensor(probe).dtype)
                loaded_keys = set()
                with torch.no_grad():
                    for k in keys:
                        if model._owns_key(k) and model._assign(k, f.get_tensor(k)):
                            loaded_keys.add(k)
                missing = model._missing_keys(loaded_keys)
                assert not missing, f"missing keys: {sorted(missing)[:8]}"
        return model.eval()
