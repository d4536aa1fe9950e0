"""Pixtral vision encoder, patch merger and vision-language adapter (API mirror of mistral_inference/vision_encoder.py).

The classes keep the reference's names and state-dict keys; every FLOP runs in libmb200:
  patch_conv      stride-p Conv2d = patchify kernel + plain GEMM.  The weight is stored flattened as [hidden, k_pad], the
                  Conv2d weight [hidden, C, p, p] in its own flatten order with zero columns up to a multiple of 64
                  (p = 14: 588 -> 640); `patch_conv.weight` is the unpadded [hidden, C, p, p] view.
  ln_pre          RMSNorm, eps 1e-5.
  transformer     the text model's TransformerBlock with n_kv_heads == n_heads, head_dim = hidden // heads (64 in the public
                  configs) and the 2-D RoPE table.  No cache: attention is the cache-less, unmasked mode.  The reference builds a
                  block-diagonal mask per image (vision_encoder.py:96-98), but TransformerBlock.forward never passes it on, so
                  every patch attends to every patch of every image of the call -- reproduced here, not "fixed".
  PatchMerger     gather kernel + GEMM (no bias).
  VisionLanguageAdapter  w_out(GELU(w_in(x))): GEMMs whose epilogue adds the bias and applies the exact-erf GELU.
"""
from typing import List, Optional, Tuple

import torch
from torch import nn

from . import _abi
from .args import VisionEncoderArgs
from .rope import precompute_freqs_cis_2d
from .transformer_layers import RMSNorm, TransformerBlock, _WeightView


def _pad64(k: int) -> int:
    return (k + 63) // 64 * 64


class _LinearView:
    """Stands in for an nn.Linear: `weight` and `bias` (None without bias)."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor]):
        self.weight = weight
        self.bias = bias


class VisionTransformerBlocks(nn.Module):
    """vision_encoder.py:120-144."""

    def __init__(self, args: VisionEncoderArgs):
        super().__init__()
        hd = args.hidden_size // args.num_attention_heads
        self.layers = nn.ModuleList([
            TransformerBlock(dim=args.hidden_size, hidden_dim=args.intermediate_size, n_heads=args.num_attention_heads,
                             n_kv_heads=args.num_attention_heads, head_dim=hd, norm_eps=1e-5)
            for _ in range(args.num_hidden_layers)
        ])

    def forward(self, x: torch.Tensor, rope: torch.Tensor, positions: torch.Tensor, ws: "_abi.Workspace") -> torch.Tensor:
        for layer in self.layers:
            x = layer(x, rope, positions, None, ws)
        return x


class VisionTransformer(nn.Module):
    """vision_encoder.py:31-102."""

    def __init__(self, args: VisionEncoderArgs):
        super().__init__()
        self.args = args
        self.head_dim = args.hidden_size // args.num_attention_heads
        assert self.head_dim % 2 == 0, "ROPE requires even head_dim"
        self.k_conv = args.num_channels * args.patch_size ** 2
        self.k_pad = _pad64(self.k_conv)
        self.patch_conv_weight = nn.Parameter(torch.zeros(args.hidden_size, self.k_pad), requires_grad=False)
        self.ln_pre = RMSNorm(args.hidden_size, eps=1e-5)
        self.transformer = VisionTransformerBlocks(args)
        self._rope: Optional[torch.Tensor] = None
        self._ws: Optional[_abi.Workspace] = None
        self._ws_tokens = 0

    @property
    def patch_conv(self) -> _WeightView:
        a = self.args
        return _WeightView(lambda: self.patch_conv_weight[:, : self.k_conv].view(a.hidden_size, a.num_channels, a.patch_size, a.patch_size))

    @property
    def max_patches_per_side(self) -> int:
        return self.args.image_size // self.args.patch_size

    @property
    def device(self) -> torch.device:
        return self.patch_conv_weight.device

    @property
    def rope_table(self) -> torch.Tensor:
        """fp32 [side * side, hd/2, 2]: the reference's 2-D table (built on the CPU) flattened row-major, indexed row * side + col."""
        if self._rope is None:
            side = self.max_patches_per_side
            t = precompute_freqs_cis_2d(self.head_dim, side, side, self.args.rope_theta)
            self._rope = torch.view_as_real(t).reshape(side * side, self.head_dim // 2, 2).contiguous()
        if self._rope.device != self.device:
            self._rope = self._rope.to(self.device)
        return self._rope

    def workspace(self, num_tokens: int) -> _abi.Workspace:
        if self._ws is None or self._ws_tokens < num_tokens or self._ws.buf.device != self.device:
            a = self.args
            need = _abi.workspace_bytes(num_tokens, a.hidden_size, a.num_attention_heads, a.num_attention_heads, self.head_dim,
                                        a.intermediate_size, 0, 1)
            self._ws = _abi.Workspace(need, self.device)
            self._ws_tokens = num_tokens
        return self._ws

    def patch_grid(self, images: List[torch.Tensor]) -> List[Tuple[int, int]]:
        """(rows, cols) of whole patches per image, with the reference's failures: a wrong rank or channel count, an image smaller
        than one patch (Conv2d raises RuntimeError) or more patches per side than the 2-D table has (indexing raises IndexError)."""
        a = self.args
        p, side = a.patch_size, self.max_patches_per_side
        grid = []
        for img in images:
            if img.dim() != 3 or img.shape[0] != a.num_channels:
                raise RuntimeError(f"expected an image [{a.num_channels}, H, W], got {tuple(img.shape)}")
            gh, gw = img.shape[1] // p, img.shape[2] // p
            if gh == 0 or gw == 0:
                raise RuntimeError(f"image {tuple(img.shape)} is smaller than one {p} x {p} patch")
            if gh > side or gw > side:
                raise IndexError(f"image {tuple(img.shape)} has {gh} x {gw} patches: out of bounds for the rope table of {side} x {side}")
            grid.append((gh, gw))
        return grid

    def forward(self, images: List[torch.Tensor]) -> torch.Tensor:
        """images: list of [C, H, W]; returns the features [sum of patches, hidden] of all images, in image order."""
        a = self.args
        grid = self.patch_grid(images)
        n = sum(h * w for h, w in grid)
        dev = self.device
        ws = self.workspace(n)
        patches = torch.empty(n, self.k_pad, dtype=torch.bfloat16, device=dev)
        off = 0
        for img, (h, w) in zip(images, grid):
            _abi.vision_patchify(img.to(device=dev, dtype=torch.bfloat16).contiguous(), patches[off: off + h * w], a.patch_size)
            off += h * w
        x = torch.empty(n, a.hidden_size, dtype=torch.bfloat16, device=dev)
        _abi.linear_residual(patches, self.patch_conv_weight, None, x, ws)
        x = self.ln_pre(x)
        side = self.max_patches_per_side
        positions = torch.cat([(torch.arange(h)[:, None] * side + torch.arange(w)[None, :]).reshape(-1) for h, w in grid])
        return self.transformer(x, self.rope_table, positions.to(device=dev, dtype=torch.int32), ws)


class VisionLanguageAdapter(nn.Module):
    """vision_encoder.py:105-117: w_out(GELU(w_in(x)))."""

    def __init__(self, in_dim: int, out_dim: int, bias: bool = True):
        super().__init__()
        self.w_in_weight = nn.Parameter(torch.empty(out_dim, in_dim), requires_grad=False)
        self.w_out_weight = nn.Parameter(torch.empty(out_dim, out_dim), requires_grad=False)
        self.w_in_bias = nn.Parameter(torch.empty(out_dim), requires_grad=False) if bias else None
        self.w_out_bias = nn.Parameter(torch.empty(out_dim), requires_grad=False) if bias else None

    @property
    def w_in(self) -> _LinearView:
        return _LinearView(self.w_in_weight, self.w_in_bias)

    @property
    def w_out(self) -> _LinearView:
        return _LinearView(self.w_out_weight, self.w_out_bias)

    def forward(self, x: torch.Tensor, ws: "_abi.Workspace") -> torch.Tensor:
        T, N = x.shape[0], self.w_in_weight.shape[0]
        h = torch.empty(T, N, dtype=x.dtype, device=x.device)
        _abi.linear_bias(x, self.w_in_weight, self.w_in_bias, h, True, ws)
        out = torch.empty(T, N, dtype=x.dtype, device=x.device)
        _abi.linear_bias(h, self.w_out_weight, self.w_out_bias, out, False, ws)
        return out


class PatchMerger(nn.Module):
    """vision_encoder.py:147-203: each image's s x s blocks of patch features, concatenated in the unfold order, then
    merging_layer (no bias)."""

    def __init__(self, vision_encoder_dim: int, spatial_merge_size: int) -> None:
        super().__init__()
        self.spatial_merge_size = spatial_merge_size
        self.mlp_input_dim = vision_encoder_dim * spatial_merge_size ** 2
        self.merging_layer_weight = nn.Parameter(torch.empty(vision_encoder_dim, self.mlp_input_dim), requires_grad=False)

    @property
    def merging_layer(self) -> _WeightView:
        return _WeightView(lambda: self.merging_layer_weight)

    def forward(self, x: torch.Tensor, image_sizes: List[Tuple[int, int]], ws: "_abi.Workspace") -> torch.Tensor:
        assert sum([h * w for h, w in image_sizes]) == len(x), f"{sum([h * w for h, w in image_sizes])} != {len(x)}"
        s = self.spatial_merge_size
        rows = sum((h // s) * (w // s) for h, w in image_sizes)
        permuted = torch.empty(rows, self.mlp_input_dim, dtype=x.dtype, device=x.device)
        i = o = 0
        for h, w in image_sizes:
            m = (h // s) * (w // s)
            _abi.patch_merge(x[i: i + h * w], permuted[o: o + m], h, w, s)
            i += h * w
            o += m
        out = torch.empty(rows, self.merging_layer_weight.shape[0], dtype=x.dtype, device=x.device)
        _abi.linear_residual(permuted, self.merging_layer_weight, None, out, ws)
        return out
