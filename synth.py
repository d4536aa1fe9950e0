"""Deterministic synthetic checkpoints ("random-init" model folders) for tests and benchmarks.

Fixture generator, NOT part of the product package: imported by bench.py, tests/, oracle/make_golden.py and scripts/ only.

There is no network for real checkpoints, so every config in BASELINE.json runs on random-init
weights of the named architecture.  Values come from a counter-based integer hash (splitmix64)
evaluated with torch int64 ops, so the same (key, seed) gives bit-identical tensors on CPU and on
GPU, in any torch version -- which is what lets golden fixtures (tests/golden/) made in one
container be checked in another.  Scales follow the reference's default initialisers: nn.Linear
kaiming-uniform bound 1/sqrt(in_features), nn.Embedding unit variance, RMSNorm weight near one
(transformer_layers.py:113 uses exactly ones; a spread is used here so a dropped norm weight is
visible to parity tests).

Folder layout is the reference's on-disk contract (transformer.py:297-336): `params.json` +
`consolidated.safetensors`, state-dict keys as listed in SURVEY.md section 8b.
"""
import json
import zlib
from pathlib import Path
from typing import Dict, Iterator, Optional, Tuple, Union

import torch

_M64 = (1 << 64) - 1


def _i64(v: int) -> int:
    v &= _M64
    return v - (1 << 64) if v >= (1 << 63) else v


_GOLDEN = _i64(0x9E3779B97F4A7C15)
_C1 = _i64(0xBF58476D1CE4E5B9)
_C2 = _i64(0x94D049BB133111EB)


def _lsr(z: torch.Tensor, n: int) -> torch.Tensor:
    return (z >> n) & ((1 << (64 - n)) - 1)


def hash_uniform(numel: int, stream: int, device: Union[str, torch.device] = "cpu", offset: int = 0) -> torch.Tensor:
    """fp32 uniform in [-1, 1), element i = f(splitmix64(stream * 2^40 + offset + i))."""
    idx = torch.arange(offset, offset + numel, dtype=torch.int64, device=device)
    z = idx + _i64((stream << 40) & _M64) + _GOLDEN
    z = (z ^ _lsr(z, 30)) * _C1
    z = (z ^ _lsr(z, 27)) * _C2
    z = z ^ _lsr(z, 31)
    u24 = _lsr(z, 40)  # 24 random bits -> exactly representable in fp32
    return u24.to(torch.float32) * (2.0 / (1 << 24)) - 1.0


def _stream(key: str, seed: int) -> int:
    return ((zlib.crc32(key.encode()) & 0xFFFFFF) ^ (seed * 7919)) & 0xFFFFFF


def synth_tensor(key: str, shape: Tuple[int, ...], seed: int, dtype: torch.dtype = torch.bfloat16,
                 device: Union[str, torch.device] = "cpu") -> torch.Tensor:
    """The tensor the synthetic checkpoint holds under state-dict key `key`."""
    numel = 1
    for s in shape:
        numel *= s
    chunk = 1 << 26
    out = torch.empty(numel, dtype=dtype, device=device)
    if key.endswith("norm.weight"):
        scale, bias = 0.25, 1.0
    elif key.startswith("tok_embeddings"):
        scale, bias = 3.0 ** 0.5, 0.0
    else:
        scale, bias = float(shape[-1]) ** -0.5, 0.0
    st = _stream(key, seed)
    for o in range(0, numel, chunk):
        n = min(chunk, numel - o)
        out[o:o + n] = (hash_uniform(n, st, device, o) * scale + bias).to(dtype)
    return out.view(*shape)


def state_dict_shapes(p: dict) -> Iterator[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) for every tensor of a params.json dict `p` (single pipeline rank, no LoRA).  The vision keys only when `p` has
    a `vision_encoder` block."""
    dim, hd, hid = p["dim"], p["head_dim"], p["hidden_dim"]
    H, KV, V = p["n_heads"], p["n_kv_heads"], p["vocab_size"]
    moe = p.get("moe")
    yield "tok_embeddings.weight", (V, dim)
    if p.get("vision_encoder"):
        yield from vision_state_dict_shapes(p)
    for i in range(p["n_layers"]):
        pre = f"layers.{i}."
        yield pre + "attention.wq.weight", (H * hd, dim)
        yield pre + "attention.wk.weight", (KV * hd, dim)
        yield pre + "attention.wv.weight", (KV * hd, dim)
        yield pre + "attention.wo.weight", (dim, H * hd)
        yield pre + "attention_norm.weight", (dim,)
        yield pre + "ffn_norm.weight", (dim,)
        if moe:
            yield pre + "feed_forward.gate.weight", (moe["num_experts"], dim)
            for e in range(moe["num_experts"]):
                yield pre + f"feed_forward.experts.{e}.w1.weight", (hid, dim)
                yield pre + f"feed_forward.experts.{e}.w2.weight", (dim, hid)
                yield pre + f"feed_forward.experts.{e}.w3.weight", (hid, dim)
        else:
            yield pre + "feed_forward.w1.weight", (hid, dim)
            yield pre + "feed_forward.w2.weight", (dim, hid)
            yield pre + "feed_forward.w3.weight", (hid, dim)
    yield "norm.weight", (dim,)
    yield "output.weight", (V, dim)


def vision_state_dict_shapes(p: dict) -> Iterator[Tuple[str, Tuple[int, ...]]]:
    """The Pixtral keys (transformer.py:59-75, vision_encoder.py) with the reference's defaults for absent fields."""
    ve = p["vision_encoder"]
    d, C, ps, inter = ve["hidden_size"], ve["num_channels"], ve["patch_size"], ve["intermediate_size"]
    s = ve.get("spatial_merge_size", 1)
    yield "vision_encoder.patch_conv.weight", (d, C, ps, ps)
    yield "vision_encoder.ln_pre.weight", (d,)
    for i in range(ve["num_hidden_layers"]):
        pre = f"vision_encoder.transformer.layers.{i}."
        for n in ("wq", "wk", "wv", "wo"):
            yield pre + f"attention.{n}.weight", (d, d)
        yield pre + "attention_norm.weight", (d,)
        yield pre + "ffn_norm.weight", (d,)
        yield pre + "feed_forward.w1.weight", (inter, d)
        yield pre + "feed_forward.w2.weight", (d, inter)
        yield pre + "feed_forward.w3.weight", (inter, d)
    yield "vision_language_adapter.w_in.weight", (p["dim"], d)
    yield "vision_language_adapter.w_out.weight", (p["dim"], p["dim"])
    if ve.get("adapter_bias", True):
        yield "vision_language_adapter.w_in.bias", (p["dim"],)
        yield "vision_language_adapter.w_out.bias", (p["dim"],)
    if ve.get("add_pre_mm_projector_layer_norm", False):
        yield "pre_mm_projector_norm.weight", (d,)
    if ve.get("mm_projector_id", "") == "patch_merge":
        yield "patch_merger.merging_layer.weight", (d, d * s * s)


def synth_image(channels: int, height: int, width: int, seed: int, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """A deterministic image [C, H, W] with values in [-1, 1) (normalised pixels)."""
    return hash_uniform(channels * height * width, (seed * 6151 + 13) & 0xFFFFFF).to(dtype).view(channels, height, width)


def synth_state_dict(p: dict, seed: int = 0, dtype: torch.dtype = torch.bfloat16,
                     device: Union[str, torch.device] = "cpu") -> Dict[str, torch.Tensor]:
    return {k: synth_tensor(k, shp, seed, dtype, device) for k, shp in state_dict_shapes(p)}


LORA_LINEARS = (("attention.wq", "q"), ("attention.wk", "kv"), ("attention.wv", "kv"), ("attention.wo", "o"), ("feed_forward.w1", "h"),
                ("feed_forward.w2", "d"), ("feed_forward.w3", "h"))


def synth_lora_state_dict(p: dict, rank: int, seed: int = 0, dtype: torch.dtype = torch.bfloat16, scale: float = 1.0,
                          device: Union[str, torch.device] = "cpu") -> Dict[str, torch.Tensor]:
    """A LoRA adapter for every LoRALinear of the text layers (lora.py:22-89): `X.lora_A.weight` [rank, in] and
    `X.lora_B.weight` [out, rank], values of synth_tensor times `scale`."""
    dim, hd, hid = p["dim"], p["head_dim"], p["hidden_dim"]
    outs = {"q": p["n_heads"] * hd, "kv": p["n_kv_heads"] * hd, "o": dim, "h": hid, "d": dim}
    ins = {"q": dim, "kv": dim, "o": p["n_heads"] * hd, "h": dim, "d": hid}
    out: Dict[str, torch.Tensor] = {}
    for i in range(p["n_layers"]):
        for name, kind in LORA_LINEARS:
            for key, shp in ((f"layers.{i}.{name}.lora_A.weight", (rank, ins[kind])), (f"layers.{i}.{name}.lora_B.weight", (outs[kind], rank))):
                out[key] = (synth_tensor(key, shp, seed, torch.float32, device) * scale).to(dtype)
    return out


def write_model_folder(folder: Union[str, Path], p: dict, seed: int = 0, dtype: torch.dtype = torch.bfloat16,
                       lora: Optional[dict] = None) -> Path:
    """Writes `params.json` + `consolidated.safetensors` (the reference's on-disk contract).  `lora` = {"rank", "scaling"} adds
    the params.json block that makes every text Linear a LoRALinear; the checkpoint stays a full one (zero adapters on load)."""
    import safetensors.torch

    folder = Path(folder)
    folder.mkdir(parents=True, exist_ok=True)
    with open(folder / "params.json", "w") as f:
        json.dump(p if lora is None else dict(p, lora=lora), f)
    safetensors.torch.save_file(synth_state_dict(p, seed, dtype), str(folder / "consolidated.safetensors"))
    return folder


def synth_prompt(length: int, vocab: int, seed: int) -> list:
    """Deterministic token ids in [0, vocab)."""
    u = hash_uniform(length, (seed * 104729 + 77) & 0xFFFFFF)
    return ((u + 1.0) * 0.5 * vocab).to(torch.int64).clamp_(0, vocab - 1).tolist()


# Public params.json shapes of the BASELINE.json configs (SURVEY.md Appendix C).
SHAPES: Dict[str, dict] = {
    "mistral-7b": dict(dim=4096, n_layers=32, head_dim=128, hidden_dim=14336, n_heads=32, n_kv_heads=8,
                       norm_eps=1e-5, vocab_size=32000, sliding_window=4096),
    "mistral-nemo-12b": dict(dim=5120, n_layers=40, head_dim=128, hidden_dim=14336, n_heads=32, n_kv_heads=8,
                             norm_eps=1e-5, vocab_size=131072),
    "mixtral-8x7b": dict(dim=4096, n_layers=32, head_dim=128, hidden_dim=14336, n_heads=32, n_kv_heads=8,
                         norm_eps=1e-5, vocab_size=32000, moe=dict(num_experts=8, num_experts_per_tok=2)),
    "mixtral-8x22b": dict(dim=6144, n_layers=56, head_dim=128, hidden_dim=16384, n_heads=48, n_kv_heads=8,
                          norm_eps=1e-5, vocab_size=32768, moe=dict(num_experts=8, num_experts_per_tok=2)),
    # Mistral Large 2 (123B; also the text model of Pixtral Large): 96 query heads over 8 kv heads (H/KV = 12)
    "mistral-large-2": dict(dim=12288, n_layers=88, head_dim=128, hidden_dim=28672, n_heads=96, n_kv_heads=8,
                            norm_eps=1e-5, vocab_size=32768, rope_theta=1000000.0),
    # shapes small enough for the CPU oracle / golden fixtures (head_dim stays 128 like every real config)
    "tiny": dict(dim=256, n_layers=2, head_dim=128, hidden_dim=512, n_heads=4, n_kv_heads=2,
                 norm_eps=1e-5, vocab_size=512),
    "tiny-moe": dict(dim=256, n_layers=2, head_dim=128, hidden_dim=256, n_heads=4, n_kv_heads=2,
                     norm_eps=1e-5, vocab_size=512, moe=dict(num_experts=8, num_experts_per_tok=2)),
    # the shape the reference's own tests use (tests/test_generate.py:40-50)
    "ref-test": dict(dim=512, n_layers=1, head_dim=128, hidden_dim=2048, n_heads=4, n_kv_heads=2,
                     norm_eps=1e-5, vocab_size=32000),
    # Pixtral-12B: the Nemo-12B text model plus a 24-layer, head_dim-64 vision encoder (public params.json)
    "pixtral-12b": dict(dim=5120, n_layers=40, head_dim=128, hidden_dim=14336, n_heads=32, n_kv_heads=8, norm_eps=1e-5,
                        vocab_size=131072, rope_theta=1000000000.0,
                        vision_encoder=dict(hidden_size=1024, num_channels=3, image_size=1024, patch_size=16, intermediate_size=4096,
                                            num_hidden_layers=24, num_attention_heads=16, rope_theta=10000.0, image_token_id=10)),
    # the reference's two Pixtral test configurations (tests/test_generate.py:78-99,127-152); image_token_id 2
    "pixtral-ref-test": dict(dim=512, n_layers=1, head_dim=128, hidden_dim=2048, n_heads=4, n_kv_heads=2, norm_eps=1e-5, vocab_size=32000,
                             vision_encoder=dict(hidden_size=128, num_channels=3, image_size=4, patch_size=2, intermediate_size=256,
                                                 num_hidden_layers=1, num_attention_heads=2, rope_theta=10000, image_token_id=2)),
    "pixtral-ref-test-merge": dict(dim=512, n_layers=1, head_dim=128, hidden_dim=2048, n_heads=4, n_kv_heads=2, norm_eps=1e-5,
                                   vocab_size=32000,
                                   vision_encoder=dict(hidden_size=128, num_channels=3, image_size=8, patch_size=2, intermediate_size=256,
                                                       num_hidden_layers=1, num_attention_heads=2, rope_theta=10000, image_token_id=2,
                                                       adapter_bias=False, spatial_merge_size=2, add_pre_mm_projector_layer_norm=True,
                                                       mm_projector_id="patch_merge")),
    # tiny text model + a vision encoder at the real layer shape (hidden 1024, 16 heads of 64), small enough for the CPU oracle
    "tiny-pixtral": dict(dim=256, n_layers=2, head_dim=128, hidden_dim=512, n_heads=4, n_kv_heads=2, norm_eps=1e-5, vocab_size=512,
                         vision_encoder=dict(hidden_size=1024, num_channels=3, image_size=256, patch_size=16, intermediate_size=4096,
                                             num_hidden_layers=2, num_attention_heads=16, rope_theta=10000.0, image_token_id=10)),
}


def shape(name: str, **overrides) -> dict:
    p = dict(SHAPES[name])
    p.update(overrides)
    return p
