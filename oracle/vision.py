"""CPU restatement of the reference's vision path (TEST INFRASTRUCTURE -- see oracle/__init__.py).

mistral-inference @ 2557e12: VisionTransformer (vision_encoder.py:31-102), PatchMerger (:147-228), VisionLanguageAdapter
(:105-117) and Transformer.embed_vision_language_features (transformer.py:122-161), functional over a reference-keyed weights
dict, in plain PyTorch on the CPU with the reference's rounding points:
  patch conv      F.conv2d, stride p, no bias, one image at a time; patches flattened row-major and concatenated
  ln_pre          RMSNorm eps 1e-5
  2-D RoPE        precompute_freqs_cis_2d indexed by (row, col) of each patch
  blocks          restatement.block_forward with no cache: attention is UNMASKED over all patches of all images of the call
                  (TransformerBlock.forward drops the block-diagonal mask the encoder builds)
  projection      [RMSNorm eps 1e-5] -> [unfold-order patch merge + merging_layer] -> w_out(GELU(w_in(x)))
  splice          image features at the image-token positions, in order; tok_embeddings elsewhere
Pinned bit-exact against the reference's modules in tests/test_oracle_vision.py (fixture: oracle/make_vision_pins.py).
"""
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from . import restatement as R


def rope_table_2d(dim: int, height: int, width: int, theta: float) -> torch.Tensor:
    """rope.py:26-51: complex64 [height, width, dim/2]."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2).float() / dim))
    h = torch.arange(height, device=freqs.device)
    w = torch.arange(width, device=freqs.device)
    freqs_h = torch.outer(h, freqs[::2]).float()
    freqs_w = torch.outer(w, freqs[1::2]).float()
    freqs_2d = torch.cat([freqs_h[:, None, :].repeat(1, width, 1), freqs_w[None, :, :].repeat(height, 1, 1)], dim=-1)
    return torch.polar(torch.ones_like(freqs_2d), freqs_2d)


def patch_grid(images: List[torch.Tensor], patch: int) -> List[Tuple[int, int]]:
    return [(img.shape[1] // patch, img.shape[2] // patch) for img in images]


def encoder_forward(images: List[torch.Tensor], w: Dict[str, torch.Tensor], ve: dict) -> torch.Tensor:
    """VisionTransformer.forward: [sum of patches, hidden]."""
    p, hidden, heads = ve["patch_size"], ve["hidden_size"], ve["num_attention_heads"]
    hd = hidden // heads
    conv_w = w["vision_encoder.patch_conv.weight"]
    embeds = [F.conv2d(img[None], conv_w, stride=p)[0] for img in images]
    x = torch.cat([e.flatten(1).permute(1, 0) for e in embeds], dim=0)
    x = R.rms_norm(x, w["vision_encoder.ln_pre.weight"], 1e-5)
    side = ve["image_size"] // p
    table = rope_table_2d(hd, side, side, ve.get("rope_theta", 1e4))
    rows = torch.cat([torch.arange(e.shape[-2])[:, None].expand(-1, e.shape[-1]).reshape(-1) for e in embeds])
    cols = torch.cat([torch.arange(e.shape[-1])[None, :].expand(e.shape[-2], -1).reshape(-1) for e in embeds])
    freqs = table[rows, cols]
    n_layers = ve["num_hidden_layers"]
    args = R.OracleArgs(dim=hidden, n_layers=n_layers, head_dim=hd, hidden_dim=ve["intermediate_size"], n_heads=heads, n_kv_heads=heads,
                        norm_eps=1e-5, vocab_size=1)
    pre = "vision_encoder.transformer."
    lw = {k[len(pre):]: v for k, v in w.items() if k.startswith(pre)}
    for i in range(n_layers):
        x = R.block_forward(x, lw, i, args, freqs, [x.shape[0]], None, None, i)
    return x


def patch_merge(x: torch.Tensor, image_sizes: List[Tuple[int, int]], s: int, merging_w: torch.Tensor) -> torch.Tensor:
    """PatchMerger.forward: per image, s x s blocks in row-major block order, feature c*s^2 + ky*s + kx (unfold), then the Linear."""
    d = x.shape[-1]
    out = []
    for tokens, (h, w_) in zip(x.split([h * w_ for h, w_ in image_sizes]), image_sizes):
        grid = tokens.view(h, w_, d).permute(2, 0, 1)[None]
        sub = F.unfold(grid, kernel_size=s, stride=s).view(d * s * s, -1)
        out.append(sub.t())
    return F.linear(torch.cat(out, 0), merging_w)


def adapter(x: torch.Tensor, w: Dict[str, torch.Tensor]) -> torch.Tensor:
    """VisionLanguageAdapter.forward: w_out(GELU_erf(w_in(x))), biases when present."""
    pre = "vision_language_adapter."
    h = F.gelu(F.linear(x, w[pre + "w_in.weight"], w.get(pre + "w_in.bias")))
    return F.linear(h, w[pre + "w_out.weight"], w.get(pre + "w_out.bias"))


def image_features(images: List[torch.Tensor], w: Dict[str, torch.Tensor], ve: dict) -> torch.Tensor:
    """Encoder + projection: the rows that replace the image tokens."""
    feats = encoder_forward(images, w, ve)
    if ve.get("add_pre_mm_projector_layer_norm", False):
        feats = R.rms_norm(feats, w["pre_mm_projector_norm.weight"], 1e-5)
    if ve.get("mm_projector_id", "") == "patch_merge":
        feats = patch_merge(feats, patch_grid(images, ve["patch_size"]), ve.get("spatial_merge_size", 1),
                            w["patch_merger.merging_layer.weight"])
    return adapter(feats, w)


def embed(input_ids: torch.Tensor, images: List[torch.Tensor], w: Dict[str, torch.Tensor], ve: dict) -> torch.Tensor:
    """Transformer.embed_vision_language_features."""
    feats = image_features(images, w, ve)
    img = input_ids == ve.get("image_token_id", 10)
    assert int(img.sum()) == feats.shape[0], (int(img.sum()), feats.shape[0])
    out = torch.empty(input_ids.shape[0], feats.shape[1], dtype=feats.dtype)
    out[~img] = F.embedding(input_ids[~img], w["tok_embeddings.weight"])
    out[img] = feats
    return out


class MultimodalOracle:
    """An OracleTransformer whose first forward (the prompt) embeds `images` (flattened over the prompts, generate.py:89); every
    later forward is text.  Drives restatement.generate unchanged."""

    def __init__(self, model: R.OracleTransformer, ve: dict, images: Optional[List[torch.Tensor]]):
        self.m, self.ve, self.images = model, ve, images
        self.args = model.args

    def new_cache(self, max_seq_len: int) -> R.RingCache:
        return self.m.new_cache(max_seq_len)

    def forward(self, input_ids: torch.Tensor, seqlens: List[int], cache: Optional[R.RingCache] = None) -> torch.Tensor:
        h_in = None
        if self.images:
            h_in = embed(input_ids, self.images, self.m.w, self.ve)
            self.images = None
        return F.linear(self.m.hidden(input_ids, seqlens, cache, h_in=h_in), self.m.w["output.weight"]).float()
