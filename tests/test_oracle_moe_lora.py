"""Un-merged LoRA on a mixture-of-experts model, on the CPU: the oracle's rounding chain (oracle/lora.py, every expert's w1 / w2 / w3
and the attention Linears adapted) pinned against the reference's own LoRALinear model on `tiny-moe`
(tests/golden/reference/moe_lora_pins.safetensors, written by oracle/make_moe_lora_pins.py)."""
import pytest
import torch

import synth
from oracle import lora as OL
from oracle import moe_lora as OM
from oracle import restatement as R
from oracle.make_moe_lora_pins import (MOE_LORA_ADAPTER_SEED, MOE_LORA_PINS_FILE, MOE_LORA_RANKS, MOE_LORA_SCALINGS, MOE_LORA_SHAPE,
                                       moe_lora_key, prompts_for)

from .util import oracle_args, same_machine_as_golden


@pytest.fixture(scope="module")
def pins():
    import safetensors
    import safetensors.torch

    with safetensors.safe_open(str(MOE_LORA_PINS_FILE), "pt") as f:
        meta = f.metadata()
    return safetensors.torch.load_file(str(MOE_LORA_PINS_FILE)), meta


def _tol(dtype):  # tests/test_oracle_lora.py
    return 1e-4 if dtype == torch.float32 else 6e-2


def _oracle(p, dtype, rank, scaling, adapter=True):
    w = synth.synth_state_dict(p, 3, dtype)
    ad = OM.synth_moe_lora_state_dict(p, rank, MOE_LORA_ADAPTER_SEED, dtype)
    if not adapter:
        ad = {k: torch.zeros_like(v) for k, v in ad.items()}
    return OL.OracleLoraTransformer(oracle_args(p, 3), OM.moe_lora_weights(w, ad), scaling)


def _prefix_diffs(gold, key, t_or, lp_or):
    """Per sequence: |oracle - reference| of the log-probabilities up to the first token where the two generations part."""
    t_ref = gold[f"{key}/tokens"].tolist()
    lp_ref = torch.split(gold[f"{key}/logprobs"], gold[f"{key}/lengths"].tolist())
    out = []
    for tr, to, lr, lo in zip(t_ref, t_or, lp_ref, lp_or):
        n = next((i for i, (a, b) in enumerate(zip(tr, to)) if a != b), len(tr))
        m = len(lo) - len(to) + n
        out.append((torch.tensor(lo[:m], dtype=torch.float64) - lr[:m]).abs())
    return t_ref, lp_ref, out


@pytest.mark.parametrize("rank", MOE_LORA_RANKS)
@pytest.mark.parametrize("scaling", MOE_LORA_SCALINGS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_generate_vs_reference(pins, rank, scaling, dtype):
    gold, meta = pins
    p = synth.shape(MOE_LORA_SHAPE)
    key = f"generate/{moe_lora_key(dtype, rank, scaling)}"
    t_or, lp_or = R.generate(prompts_for(p), _oracle(p, dtype, rank, scaling), max_tokens=9, chunk_size=4)
    t_ref, lp_ref, diffs = _prefix_diffs(gold, key, t_or, lp_or)
    if same_machine_as_golden(meta):
        assert t_ref == t_or
        assert [x.tolist() for x in lp_ref] == lp_or
        return
    for d in diffs:
        assert d.numel() == 0 or d.max().item() <= _tol(dtype), d.max().item()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_lora_term_is_far_above_tolerance(pins, dtype):
    """Negative control: the oracle without the adapters, with the scaling doubled, or without the expert adapters alone, misses the
    pinned log-probabilities by several times the tolerance the comparison above allows (log-probabilities of short generations:
    the misses are 0.15 to 1.2 nats in bf16, against a tolerance of 0.06)."""
    gold, _ = pins
    p = synth.shape(MOE_LORA_SHAPE)
    rank, scaling = MOE_LORA_RANKS[0], MOE_LORA_SCALINGS[0]
    key = f"generate/{moe_lora_key(dtype, rank, scaling)}"
    w = synth.synth_state_dict(p, 3, dtype)
    ad = OM.synth_moe_lora_state_dict(p, rank, MOE_LORA_ADAPTER_SEED, dtype)
    experts_only_dropped = {k: (torch.zeros_like(v) if ".experts." in k else v) for k, v in ad.items()}
    wrong = [_oracle(p, dtype, rank, scaling, adapter=False), _oracle(p, dtype, rank, 2 * scaling),
             OL.OracleLoraTransformer(oracle_args(p, 3), OM.moe_lora_weights(w, experts_only_dropped), scaling)]
    for m in wrong:
        t_or, lp_or = R.generate(prompts_for(p), m, max_tokens=9, chunk_size=4)
        _, _, diffs = _prefix_diffs(gold, key, t_or, lp_or)
        assert max(d.max().item() for d in diffs if d.numel()) > 5 * _tol(dtype)


def test_zero_adapters_are_the_plain_model():
    p = synth.shape(MOE_LORA_SHAPE)
    toks = torch.tensor(synth.synth_prompt(13, p["vocab_size"], 5))
    with torch.inference_mode():
        zero = _oracle(p, torch.bfloat16, 4, 2.0, adapter=False).forward(toks, [6, 7])
        plain = R.OracleTransformer(oracle_args(p, 3), synth.synth_state_dict(p, 3)).forward(toks, [6, 7])
    assert torch.equal(zero, plain)
