"""Runs the reference's own Transformer with un-merged LoRA adapters (args.lora set; unmodified, behind oracle/ref_shims.py) on
seeded weights and adapters and writes tests/golden/reference/lora_pins.safetensors, which tests/test_oracle_lora.py pins
oracle/lora.py against (TEST INFRASTRUCTURE -- see oracle/__init__.py).

`python -m oracle.make_lora_pins` (needs the reference source tree, MISTRAL_REFERENCE_SRC).
Cases (LORA_CASES x rank x scaling x dtype): the full checkpoint of synth.synth_state_dict(p, 3) loaded with load_state_dict
(zero adapters, lora.py:76-89), then the adapter synth.synth_lora_state_dict(p, rank, 5) through _load_lora_state_dict, then
generate(chunk_size=4) tokens and log-probabilities.  Also: the cache-less forward, the reference's state_dict() key list, and
one case loaded with _load_lora_state_dict(..., scaling=7.0), which the un-merged path ignores.
"""
import hashlib
import json
from typing import Dict

import torch

import synth

from . import ref_shims
from .make_golden import GOLDEN_DIR, pin_key

LORA_PINS_FILE = GOLDEN_DIR / "reference" / "lora_pins.safetensors"
LORA_CASES = [("tiny", {}), ("tiny", {"sliding_window": 5}), ("tiny", {"sliding_window": [4, None]})]
LORA_RANKS = (4, 8)
LORA_SCALINGS = (2.0, 0.3)
LORA_ADAPTER_SEED = 5
PROMPT_LENS = [11, 9, 10]


def lora_key(shape: str, over: dict, dtype: torch.dtype, rank: int, scaling: float) -> str:
    return f"{pin_key(shape, over, dtype)}/r{rank}/s{scaling}"


def prompts_for(p: dict):
    return [synth.synth_prompt(n, p["vocab_size"], 40 + i) for i, n in enumerate(PROMPT_LENS)]


def ref_lora_model(ref, p: dict, max_batch: int, dtype: torch.dtype, rank: int, scaling: float, load_scaling: float = 2.0):
    args = ref.args.TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=scaling)))
    args.max_batch_size = max_batch
    m = ref.transformer.Transformer(args).to(dtype)
    m.load_state_dict(synth.synth_state_dict(p, 3, dtype), strict=True)
    m._load_lora_state_dict(synth.synth_lora_state_dict(p, rank, LORA_ADAPTER_SEED, dtype), scaling=load_scaling)
    return m.eval()


def run_lora_pins():
    ref = ref_shims.import_reference()
    out: Dict[str, torch.Tensor] = {}
    keys = None
    for dtype in (torch.bfloat16, torch.float32):
        for shape, over in LORA_CASES:
            p = synth.shape(shape, **over)
            for rank in LORA_RANKS:
                for scaling in LORA_SCALINGS:
                    m = ref_lora_model(ref, p, 3, dtype, rank, scaling)
                    if keys is None:
                        keys = list(m.state_dict().keys())
                    toks, lps = ref.generate.generate(prompts_for(p), m, max_tokens=9, temperature=0.0, chunk_size=4)
                    k = f"generate/{lora_key(shape, over, dtype, rank, scaling)}"
                    out[f"{k}/tokens"] = torch.tensor(toks, dtype=torch.int64)
                    out[f"{k}/logprobs"] = torch.tensor(sum(lps, []), dtype=torch.float64)
                    out[f"{k}/lengths"] = torch.tensor([len(x) for x in lps], dtype=torch.int64)
        p = synth.shape("tiny")
        d = str(dtype).split(".")[-1]
        m = ref_lora_model(ref, p, 2, dtype, 8, 2.0)
        with torch.inference_mode():
            out[f"forward_no_cache/{d}"] = m.forward(torch.tensor(synth.synth_prompt(13, p["vocab_size"], 5)), seqlens=[6, 7]).clone()
        m = ref_lora_model(ref, p, 3, dtype, 4, 0.3, load_scaling=7.0)  # the argument is ignored: same as r4/s0.3 above
        toks, lps = ref.generate.generate(prompts_for(p), m, max_tokens=9, temperature=0.0, chunk_size=4)
        out[f"load_scaling_7/{d}/tokens"] = torch.tensor(toks, dtype=torch.int64)
        out[f"load_scaling_7/{d}/logprobs"] = torch.tensor(sum(lps, []), dtype=torch.float64)
    meta = {"torch": torch.__version__, "cpu_capability": torch.backends.cpu.get_cpu_capability(), "num_threads": str(torch.get_num_threads()),
            "state_dict_keys": json.dumps(keys), "adapter_seed": str(LORA_ADAPTER_SEED),
            "keys_sha256": hashlib.sha256(json.dumps(keys).encode()).hexdigest(),
            "reference": "mistralai/mistral-inference@2557e12 (v1.6.0) modules, unmodified, via oracle/ref_shims.py"}
    return out, meta


def main() -> None:
    import safetensors.torch

    out, meta = run_lora_pins()
    LORA_PINS_FILE.parent.mkdir(parents=True, exist_ok=True)
    safetensors.torch.save_file({k: v.contiguous() for k, v in out.items()}, str(LORA_PINS_FILE), metadata=meta)
    print(f"{LORA_PINS_FILE.name}: {len(out)} tensors, {sum(v.numel() * v.element_size() for v in out.values())} bytes")


if __name__ == "__main__":
    main()
