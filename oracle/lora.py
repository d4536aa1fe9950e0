"""CPU restatement of the reference's un-merged LoRA path (TEST INFRASTRUCTURE -- see oracle/__init__.py).

With `args.lora` set the reference builds every wq/wk/wv/wo/w1/w2/w3 of the text layers as a LoRALinear (lora.py:22-89,
transformer_layers.py:22-28) whose forward is `linear(x) + lora_B(lora_A(x)) * scaling` (lora.py:71-74).  In bf16 that is the
rounding chain
    a = bf16(x A^T);  l = bf16(a B^T);  s = bf16(l * scaling);  y = bf16(x W^T);  out = bf16(y + s)
and in fp32 the same ops without the roundings.  Everything else -- the gate, the output layer, the vision tower -- stays a
plain nn.Linear.

OracleLoraTransformer runs oracle/restatement.py unchanged: while it computes, a torch-function mode replaces each F.linear on
an adapted base weight (recognised by identity) by the chain above, so the rest of the restatement, its caches and its
`generate` are shared with the plain model.  Weights are keyed like the reference's LoRA state dict: `X.linear.weight`,
`X.lora_A.weight`, `X.lora_B.weight` for the adapted Linears (a plain `X.weight` means a zero adapter), `X.weight` elsewhere.
"""
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch.overrides import TorchFunctionMode

from .restatement import OracleArgs, OracleTransformer

LORA_LINEARS = ("attention.wq", "attention.wk", "attention.wv", "attention.wo", "feed_forward.w1", "feed_forward.w2", "feed_forward.w3")


def lora_linear(x: torch.Tensor, w: torch.Tensor, a: torch.Tensor, b: torch.Tensor, scaling: float) -> torch.Tensor:
    """LoRALinear.forward (lora.py:71-74)."""
    return F.linear(x, w) + F.linear(F.linear(x, a), b) * scaling


class _AdaptedLinears(TorchFunctionMode):
    def __init__(self, adapters: Dict[int, Tuple[torch.Tensor, torch.Tensor]], scaling: float):
        super().__init__()
        self.adapters = adapters
        self.scaling = scaling
        self.hit = set()

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is F.linear and len(args) >= 2 and not kwargs and id(args[1]) in self.adapters:
            a, b = self.adapters[id(args[1])]
            self.hit.add(id(args[1]))
            return lora_linear(args[0], args[1], a, b, self.scaling)
        return func(*args, **kwargs)


class OracleLoraTransformer(OracleTransformer):
    """OracleTransformer with un-merged adapters; `scaling` is args.lora.scaling."""

    def __init__(self, args: OracleArgs, weights: Dict[str, torch.Tensor], scaling: float, layer_ids: Optional[Sequence[int]] = None):
        base: Dict[str, torch.Tensor] = {}
        parts: Dict[str, Dict[str, torch.Tensor]] = {}
        for k, v in weights.items():
            for suffix in (".linear.weight", ".lora_A.weight", ".lora_B.weight"):
                if k.endswith(suffix):
                    parts.setdefault(k[: -len(suffix)], {})[suffix] = v
                    break
            else:
                base[k] = v
        adapters: Dict[int, Tuple[torch.Tensor, torch.Tensor]] = {}
        layer_ids = list(range(args.n_layers)) if layer_ids is None else list(layer_ids)
        for name, p in parts.items():
            if int(name.split(".")[1]) not in layer_ids:  # another pipeline stage's layer
                continue
            assert set(p) == {".linear.weight", ".lora_A.weight", ".lora_B.weight"}, f"{name}: incomplete LoRALinear {sorted(p)}"
            base[name + ".weight"] = p[".linear.weight"]
            adapters[id(p[".linear.weight"])] = (p[".lora_A.weight"], p[".lora_B.weight"])
        super().__init__(args, base, layer_ids)
        self.scaling = scaling
        self._adapters = adapters

    def hidden(self, *args, **kwargs) -> torch.Tensor:  # forward() and generate() go through here; the output layer is plain
        mode = _AdaptedLinears(self._adapters, self.scaling)
        with mode:
            out = super().hidden(*args, **kwargs)
        # the adapters are found by the identity of the base weight: a restatement that copied or converted a weight would
        # otherwise drop its adapter silently
        assert mode.hit == set(self._adapters), f"{len(set(self._adapters) - mode.hit)} adapted Linears were not reached"
        return out


def lora_weights(plain: Dict[str, torch.Tensor], adapter: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """A reference-keyed LoRA-mode weights dict from a plain checkpoint and an adapter (`X.lora_A/B.weight`): every adapted
    Linear of `plain` becomes `X.linear.weight` with the adapter's tensors, or zero ones where the adapter has none."""
    out: Dict[str, torch.Tensor] = {}
    rank = next(v.shape[0] for k, v in adapter.items() if k.endswith(".lora_A.weight"))
    for k, v in plain.items():
        name = k[: -len(".weight")]
        if k.startswith("layers.") and name.split(".", 2)[2] in LORA_LINEARS:
            out[name + ".linear.weight"] = v
            out[name + ".lora_A.weight"] = adapter.get(name + ".lora_A.weight", torch.zeros(rank, v.shape[1], dtype=v.dtype))
            out[name + ".lora_B.weight"] = adapter.get(name + ".lora_B.weight", torch.zeros(v.shape[0], rank, dtype=v.dtype))
        else:
            out[k] = v
    return out
