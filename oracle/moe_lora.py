"""Un-merged LoRA on a mixture-of-experts checkpoint, for the CPU oracle (TEST INFRASTRUCTURE -- see oracle/__init__.py).

With `args.lora` and `args.moe` set the reference makes every expert's w1 / w2 / w3 a LoRALinear too (transformer_layers.py:151);
the router gate stays a plain nn.Linear.  oracle/lora.py's OracleLoraTransformer finds adapted Linears by the identity of their
base weight, so it runs such a checkpoint unchanged once the weights are keyed like the reference's LoRA state dict.  This module
builds those weights (`moe_lora_weights`) and the seeded adapters the tests and pins use (`synth_moe_lora_state_dict`).
"""
import re
from typing import Dict, Union

import torch

import synth

from .lora import LORA_LINEARS

_EXPERT_LINEAR = re.compile(r"^feed_forward\.experts\.\d+\.w[123]$")


def synth_moe_lora_state_dict(p: dict, rank: int, seed: int = 0, dtype: torch.dtype = torch.bfloat16, scale: float = 1.0,
                              device: Union[str, torch.device] = "cpu") -> Dict[str, torch.Tensor]:
    """synth.synth_lora_state_dict for a mixture-of-experts shape: the attention LoRALinears and every expert's w1 / w2 / w3
    (`layers.{i}.feed_forward.experts.{e}.w1.lora_A.weight`, ...), values of synth_tensor times `scale`."""
    dim, hid = p["dim"], p["hidden_dim"]
    out = {k: v for k, v in synth.synth_lora_state_dict(p, rank, seed, dtype, scale, device).items() if ".feed_forward." not in k}
    for i in range(p["n_layers"]):
        for e in range(p["moe"]["num_experts"]):
            for n, (o, inn) in (("w1", (hid, dim)), ("w2", (dim, hid)), ("w3", (hid, dim))):
                pre = f"layers.{i}.feed_forward.experts.{e}.{n}"
                for key, shp in ((pre + ".lora_A.weight", (rank, inn)), (pre + ".lora_B.weight", (o, rank))):
                    out[key] = (synth.synth_tensor(key, shp, seed, torch.float32, device) * scale).to(dtype)
    return out


def moe_lora_weights(plain: Dict[str, torch.Tensor], adapter: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """oracle/lora.py's lora_weights for a mixture-of-experts checkpoint: every attention Linear and every expert Linear of `plain`
    becomes `X.linear.weight` with the adapter's tensors, or zero ones where the adapter has none."""
    out: Dict[str, torch.Tensor] = {}
    rank = next(v.shape[0] for k, v in adapter.items() if k.endswith(".lora_A.weight"))
    for k, v in plain.items():
        name = k[: -len(".weight")]
        sub = name.split(".", 2)[2] if k.startswith("layers.") else ""
        if sub in LORA_LINEARS or _EXPERT_LINEAR.match(sub):
            out[name + ".linear.weight"] = v
            out[name + ".lora_A.weight"] = adapter.get(name + ".lora_A.weight", torch.zeros(rank, v.shape[1], dtype=v.dtype))
            out[name + ".lora_B.weight"] = adapter.get(name + ".lora_B.weight", torch.zeros(v.shape[0], rank, dtype=v.dtype))
        else:
            out[k] = v
    return out
