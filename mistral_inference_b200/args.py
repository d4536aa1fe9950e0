"""`params.json` schema (mirror of mistral_inference/args.py:29-59 and moe.py:10-13).

`simple_parsing` is not a dependency here: `from_dict` is a few lines (the reference only uses
`Serializable.from_dict`, transformer.py:306-307).
"""
from dataclasses import dataclass, fields
from typing import List, Optional, Union


@dataclass
class MoeArgs:
    num_experts: int
    num_experts_per_tok: int

    @classmethod
    def from_dict(cls, d: dict) -> "MoeArgs":
        return cls(**{f.name: d[f.name] for f in fields(cls) if f.name in d})


@dataclass
class LoraArgs:
    rank: int
    scaling: float

    @classmethod
    def from_dict(cls, d: dict) -> "LoraArgs":
        return cls(**{f.name: d[f.name] for f in fields(cls) if f.name in d})


PATCH_MERGE = "patch_merge"


@dataclass
class VisionEncoderArgs:
    """args.py:12-26 (Pixtral).  The encoder's head_dim is hidden_size // num_attention_heads."""
    hidden_size: int
    num_channels: int
    image_size: int
    patch_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int
    rope_theta: float = 1e4  # for rope-2D
    image_token_id: int = 10
    adapter_bias: bool = True
    spatial_merge_size: int = 1
    add_pre_mm_projector_layer_norm: bool = False
    mm_projector_id: str = ""

    @classmethod
    def from_dict(cls, d: dict) -> "VisionEncoderArgs":
        return cls(**{f.name: d[f.name] for f in fields(cls) if f.name in d})


@dataclass
class TransformerArgs:
    dim: int
    n_layers: int
    head_dim: int
    hidden_dim: int
    n_heads: int
    n_kv_heads: int
    norm_eps: float
    vocab_size: int

    max_batch_size: int = 0

    # For rotary embeddings. If not set, 1e6 is used (transformer.py:115).
    rope_theta: Optional[float] = None
    # If this is set, MoE layers replace the dense FeedForward.
    moe: Optional[MoeArgs] = None
    lora: Optional[LoraArgs] = None
    sliding_window: Union[None, int, List[Optional[int]]] = None
    _sliding_window: Union[None, int, List[Optional[int]]] = None
    model_type: str = "transformer"

    vision_encoder: Optional[VisionEncoderArgs] = None

    def __post_init__(self) -> None:
        assert self.model_type == "transformer", self.model_type
        assert self.sliding_window is None or self._sliding_window is None
        # same aliasing as args.py:58-59
        self.sliding_window = self.sliding_window if self.sliding_window is not None else self._sliding_window
        if isinstance(self.vision_encoder, dict):
            self.vision_encoder = VisionEncoderArgs.from_dict(self.vision_encoder)
        if isinstance(self.moe, dict):
            self.moe = MoeArgs.from_dict(self.moe)
        if isinstance(self.lora, dict):
            self.lora = LoraArgs.from_dict(self.lora)

    @classmethod
    def from_dict(cls, d: dict) -> "TransformerArgs":
        known = {f.name for f in fields(cls)}
        return cls(**{k: v for k, v in d.items() if k in known})
