"""Runs the reference's own Transformer with un-merged LoRA adapters on a mixture-of-experts shape (args.lora and args.moe set;
unmodified, behind oracle/ref_shims.py) and writes tests/golden/reference/moe_lora_pins.safetensors, which
tests/test_oracle_moe_lora.py pins oracle/lora.py against (TEST INFRASTRUCTURE -- see oracle/__init__.py).

`python -m oracle.make_moe_lora_pins` (needs the reference source tree, MISTRAL_REFERENCE_SRC).
Cases (rank x scaling x dtype) on `tiny-moe`: the full checkpoint of synth.synth_state_dict(p, 3) loaded with load_state_dict (zero
adapters, lora.py:76-89), then the adapter oracle.moe_lora.synth_moe_lora_state_dict(p, rank, 7) -- the attention Linears and every expert's
w1 / w2 / w3 -- through _load_lora_state_dict, then generate(chunk_size=4) tokens and log-probabilities.  Also the reference's
state_dict() key list.
"""
import hashlib
import json
from typing import Dict

import torch

import synth

from . import ref_shims
from .make_golden import GOLDEN_DIR
from .moe_lora import synth_moe_lora_state_dict

MOE_LORA_PINS_FILE = GOLDEN_DIR / "reference" / "moe_lora_pins.safetensors"
MOE_LORA_SHAPE = "tiny-moe"
MOE_LORA_RANKS = (4, 16)
MOE_LORA_SCALINGS = (2.0, 0.5)
MOE_LORA_ADAPTER_SEED = 7
PROMPT_LENS = [11, 9, 10]


def moe_lora_key(dtype: torch.dtype, rank: int, scaling: float) -> str:
    return f"{MOE_LORA_SHAPE}/{str(dtype).split('.')[-1]}/r{rank}/s{scaling}"


def prompts_for(p: dict):
    return [synth.synth_prompt(n, p["vocab_size"], 60 + i) for i, n in enumerate(PROMPT_LENS)]


def ref_moe_lora_model(ref, p: dict, max_batch: int, dtype: torch.dtype, rank: int, scaling: float):
    args = ref.args.TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=scaling)))
    args.max_batch_size = max_batch
    m = ref.transformer.Transformer(args).to(dtype)
    m.load_state_dict(synth.synth_state_dict(p, 3, dtype), strict=True)
    m._load_lora_state_dict(synth_moe_lora_state_dict(p, rank, MOE_LORA_ADAPTER_SEED, dtype))
    return m.eval()


def run_moe_lora_pins():
    ref = ref_shims.import_reference()
    p = synth.shape(MOE_LORA_SHAPE)
    out: Dict[str, torch.Tensor] = {}
    keys = None
    for dtype in (torch.bfloat16, torch.float32):
        for rank in MOE_LORA_RANKS:
            for scaling in MOE_LORA_SCALINGS:
                m = ref_moe_lora_model(ref, p, 3, dtype, rank, scaling)
                if keys is None:
                    keys = list(m.state_dict().keys())
                toks, lps = ref.generate.generate(prompts_for(p), m, max_tokens=9, temperature=0.0, chunk_size=4)
                k = f"generate/{moe_lora_key(dtype, rank, scaling)}"
                out[f"{k}/tokens"] = torch.tensor(toks, dtype=torch.int64)
                out[f"{k}/logprobs"] = torch.tensor(sum(lps, []), dtype=torch.float64)
                out[f"{k}/lengths"] = torch.tensor([len(x) for x in lps], dtype=torch.int64)
    meta = {"torch": torch.__version__, "cpu_capability": torch.backends.cpu.get_cpu_capability(), "num_threads": str(torch.get_num_threads()),
            "state_dict_keys": json.dumps(keys), "adapter_seed": str(MOE_LORA_ADAPTER_SEED),
            "keys_sha256": hashlib.sha256(json.dumps(keys).encode()).hexdigest(),
            "reference": "mistralai/mistral-inference@2557e12 (v1.6.0) modules, unmodified, via oracle/ref_shims.py"}
    return out, meta


def main() -> None:
    import safetensors.torch

    out, meta = run_moe_lora_pins()
    MOE_LORA_PINS_FILE.parent.mkdir(parents=True, exist_ok=True)
    safetensors.torch.save_file({k: v.contiguous() for k, v in out.items()}, str(MOE_LORA_PINS_FILE), metadata=meta)
    print(f"{MOE_LORA_PINS_FILE.name}: {len(out)} tensors, {sum(v.numel() * v.element_size() for v in out.values())} bytes")


if __name__ == "__main__":
    main()
