"""Runs the reference's own vision modules (unmodified, behind oracle/ref_shims.py) on seeded inputs and writes their outputs to
tests/golden/reference/vision_pins.safetensors, which tests/test_oracle_vision.py pins oracle/vision.py against
(TEST INFRASTRUCTURE -- see oracle/__init__.py).

`python -m oracle.make_vision_pins` (needs the reference source tree, MISTRAL_REFERENCE_SRC).
Cases (VISION_CASES): the reference's two Pixtral test configurations (tests/test_generate.py:72-171) with their prompts and
image sizes, and a case with two images of different sizes in one prompt and none in the other.  Per case: the encoder output,
embed_vision_language_features of the whole prompt batch, and generate(images=...) tokens and log-probabilities, in bf16.
"""
import hashlib
import json
from typing import Dict, List

import numpy as np
import torch

import synth

from . import ref_shims
from .make_golden import GOLDEN_DIR

VISION_PINS_FILE = GOLDEN_DIR / "reference" / "vision_pins.safetensors"
# the 2-D RoPE table of the public encoder (head_dim 64, 1024 / 16 = 64 patches per side)
PIN_ROPE2D = dict(dim=64, side=64, theta=1e4)
PIN_ROPE2D_ROWS = [(0, 0), (0, 63), (5, 7), (63, 0), (31, 32), (63, 63)]

# name -> (synth shape, overrides, prompts (DebugTokenizer ids: bos = 1, then the numbers), image sizes [C, H, W] per prompt)
VISION_CASES = {
    "pixtral": ("pixtral-ref-test", {}, [[1, 1, 2, 2, 2, 2, 4, 5, 6, 7], [1, 12, 13, 14], [1, 2, 2, 2, 2, 7, 8, 9]],
                [[(3, 4, 4)], [], [(3, 4, 4)]]),
    "pixtral_patch_merger": ("pixtral-ref-test-merge", {}, [[1, 1, 2, 2, 2, 2, 4, 5, 6, 7], [1, 12, 13, 14], [1, 2, 2, 2, 2, 7, 8, 9]],
                             [[(3, 8, 8)], [], [(3, 8, 8)]]),
    # image 1: 4 x 3 patches (a remainder column of pixels is dropped), image 2: 2 x 4 patches -> 20 image tokens in prompt 0
    "two_images": ("pixtral-ref-test", {"image_size": 8}, [[1, 5] + [2] * 12 + [6] + [2] * 8 + [7, 8], [1, 12, 13, 14, 15]],
                   [[(3, 8, 7), (3, 5, 8)], []]),
}


def case_params(name: str) -> dict:
    shape, over, _, _ = VISION_CASES[name]
    p = synth.shape(shape)
    p["vision_encoder"] = dict(p["vision_encoder"], **over)
    return p


def case_images(name: str) -> List[List[np.ndarray]]:
    """float64 numpy images like the reference test's (np.random.default_rng(42).normal)."""
    gen = np.random.default_rng(seed=42)
    return [[gen.normal(size=s) for s in sizes] for sizes in VISION_CASES[name][3]]


def run_vision_pins():
    ref = ref_shims.import_reference()
    import mistral_inference.rope as r_rope  # type: ignore

    out: Dict[str, torch.Tensor] = {}
    for name, (_, _, prompts, _) in VISION_CASES.items():
        p = case_params(name)
        args = ref.args.TransformerArgs.from_dict(dict(p))
        args.max_batch_size = len(prompts)
        with torch.device("meta"):
            m = ref.transformer.Transformer(args)
        m.load_state_dict(synth.synth_state_dict(p, 3, torch.bfloat16), assign=True, strict=True)
        m = m.eval()
        imgs = [[torch.tensor(im, dtype=torch.bfloat16) for im in ims] for ims in case_images(name)]
        flat = sum(imgs, [])
        with torch.inference_mode():
            out[f"{name}/encoder"] = m.vision_encoder(flat).clone()
            out[f"{name}/embed"] = m.embed_vision_language_features(torch.tensor(sum(prompts, [])), flat).clone()
            toks, lps = ref.generate.generate(prompts, m, images=case_images(name), max_tokens=7, temperature=0.0)
        out[f"{name}/tokens"] = torch.tensor(toks, dtype=torch.int64)
        out[f"{name}/logprobs"] = torch.tensor(sum(lps, []), dtype=torch.float64)
        out[f"{name}/lengths"] = torch.tensor([len(x) for x in lps], dtype=torch.int64)
    t = torch.view_as_real(r_rope.precompute_freqs_cis_2d(PIN_ROPE2D["dim"], PIN_ROPE2D["side"], PIN_ROPE2D["side"], PIN_ROPE2D["theta"]))
    t = t.contiguous()
    out["rope2d_rows"] = torch.stack([t[r, c] for r, c in PIN_ROPE2D_ROWS]).clone()
    meta = {"torch": torch.__version__, "cpu_capability": torch.backends.cpu.get_cpu_capability(), "num_threads": str(torch.get_num_threads()),
            "rope2d_sha256": hashlib.sha256(t.numpy().tobytes()).hexdigest(), "cases": json.dumps(list(VISION_CASES)),
            "reference": "mistralai/mistral-inference@2557e12 (v1.6.0) modules, unmodified, via oracle/ref_shims.py"}
    return out, meta


def main() -> None:
    import safetensors.torch

    out, meta = run_vision_pins()
    VISION_PINS_FILE.parent.mkdir(parents=True, exist_ok=True)
    safetensors.torch.save_file({k: v.contiguous() for k, v in out.items()}, str(VISION_PINS_FILE), metadata=meta)
    print(f"{VISION_PINS_FILE.name}: {len(out)} tensors, {sum(v.numel() * v.element_size() for v in out.values())} bytes")


if __name__ == "__main__":
    main()
