"""Prompt encoding + decode loop with the per-token tail on the device (contract of mistral_inference/generate.py:43-170).

Same inputs and outputs as the reference's `generate`:
  (tokens [B][n], logprobs [B][prompt_len - 1 + n]) -- greedy when temperature == 0, otherwise nucleus sampling with the
  reference's hard-coded p = 0.8 (generate.py:126); generation stops at the first step at which every sequence has emitted
  `eos_id` (that step's tokens are not returned, generate.py:128-132); `[]` when max_tokens == 0 (generate.py:142-146).

What is different is where the work happens.  The reference materialises log_softmax over [T, V] twice per chunk and reads one
scalar per token back to the host (`.item()`), and in the decode loop it syncs three times per token.  Here:
  * the whole prompt is uploaded once; every chunk's "next token" targets are known up front, so the log-probabilities of the
    prompt are one fused log-softmax + gather kernel per block of lm-head rows (`Transformer.forward_logprobs`) -- the [T, V]
    logits of a chunk never exist at once (Nemo's 32 x 1024 x 131072 fp32 would be 17 GB);
  * the decode loop keeps tokens, log-probabilities and the eos flags on the device: pick (fused argmax of the decode kernel /
    `mb200_argmax_rows` / `mb200_sample_top_p`), `mb200_logprob_gather`, next step -- no host round trip per token; results
    come back with one copy at the end (with `eos_id` the flags are polled every EOS_POLL steps and the tail is dropped).
"""
from typing import List, Optional, Tuple

import torch

from . import _abi
from .cache import BufferCache
from .transformer import Transformer

TOP_P = 0.8     # generate.py:126
EOS_POLL = 16   # steps between host checks of the device-side "every sequence finished" flag


class _PromptPlan:
    """Chunk schedule of a ragged batch of prompts: per chunk the flattened token ids, the sequence lengths and, per token,
    the id whose log-probability the reference reports at that position (the NEXT prompt token of the same sequence, also
    across a chunk boundary: generate.py:103-107; -1 after a sequence's last prompt token)."""

    def __init__(self, prompts: List[List[int]], chunk_size: Optional[int]):
        self.B = len(prompts)
        self.lens = [len(p) for p in prompts]
        longest = max(self.lens)
        step = longest if chunk_size is None else chunk_size
        self.chunks: List[Tuple[List[int], List[int], List[int], List[Tuple[int, int]]]] = []
        for s in range(0, longest, step):
            pieces = [p[s:s + step] for p in prompts]
            assert all(len(x) > 0 for x in pieces), "every prompt needs a token in every chunk (generate.py:94)"
            flat: List[int] = []
            targets: List[int] = []
            where: List[Tuple[int, int]] = []  # (sequence, position) of each flattened token
            for b, piece in enumerate(pieces):
                for j, tok in enumerate(piece):
                    pos = s + j
                    flat.append(tok)
                    targets.append(prompts[b][pos + 1] if pos + 1 < self.lens[b] else -1)
                    where.append((b, pos))
            self.chunks.append((flat, [len(x) for x in pieces], targets, where))


@torch.inference_mode()
def generate(encoded_prompts: List[List[int]], model: Transformer, images: List[List] = [], *, max_tokens: int,  # noqa: B006
             temperature: float, chunk_size: Optional[int] = None, eos_id: Optional[int] = None,
             draft: Optional[Transformer] = None, draft_tokens: int = 4,
             lora_ids: Optional[List[int]] = None) -> Tuple[List[List[int]], List[List[float]]]:
    """`draft`: another Transformer with the same vocabulary that proposes `draft_tokens` tokens per round for the model to verify
    (speculative decoding, mistral_inference_b200/speculative.py).  Same return value and semantics as without it; greedy output
    stays the model's own argmax choices and sampled output keeps the model's nucleus distribution.
    `lora_ids`: one entry per prompt, the model's adapter slot that sequence runs through (Transformer `lora_slots`), or -1 for the
    base model; None is slot 0 for every sequence.  A sequence's result does not depend on the other sequences' ids."""
    if lora_ids is not None:
        if draft is not None:
            raise ValueError("lora_ids with a draft model (speculative decoding) is not built")
        model.check_lora_ids(lora_ids, len(encoded_prompts))
    lora_kw = {} if lora_ids is None else {"lora_ids": lora_ids}  # no ids: the model calls take no LoRA keyword
    if draft is not None:
        from .speculative import generate_speculative

        return generate_speculative(encoded_prompts, model, draft, images, max_tokens=max_tokens, temperature=temperature,
                                    chunk_size=chunk_size, eos_id=eos_id, draft_tokens=draft_tokens)
    # images[b]: the images of prompt b; the model sees all of them, in prompt order (generate.py:54-60,89)
    images_torch: List[List[torch.Tensor]] = []
    if images:
        assert chunk_size is None
        images_torch = [[torch.tensor(im, device=model.device, dtype=model.dtype) for im in images_for_sample]
                        for images_for_sample in images]
    flattened_images: List[torch.Tensor] = sum(images_torch, [])
    model = model.eval()
    dev = model.device
    plan = _PromptPlan(encoded_prompts, chunk_size)
    B, V = plan.B, model.args.vocab_size

    # one ring per layer, sized like the reference's (generate.py:68-78)
    cache = BufferCache(model.n_local_layers, model.args.max_batch_size, max(plan.lens) + max_tokens, model.args.n_kv_heads,
                        model.args.head_dim, model.args.sliding_window, kv_cache=model.kv_cache)
    cache.to(device=dev, dtype=model.dtype)
    cache.reset()

    # ---- prompt: hidden states chunk by chunk, log-probabilities fused with the lm head ----
    prompt_lp: List[torch.Tensor] = []
    last_logits: Optional[torch.Tensor] = None
    for flat, seqlens, targets, _ in plan.chunks:
        ids = torch.tensor(flat, dtype=torch.long, device=dev)
        tgt = torch.tensor(targets, dtype=torch.long, device=dev)
        lp, last_logits = model.forward_logprobs(ids, seqlens, cache, tgt, images=flattened_images, **lora_kw)
        prompt_lp.append(lp)
    assert last_logits is not None and last_logits.shape == (B, V)

    # ---- decode: everything stays on the device ----
    steps_run = 0
    gen_tok = torch.zeros(max(max_tokens, 1), B, dtype=torch.long, device=dev)       # [step, b]: each step's row is contiguous
    gen_lp = torch.zeros(max(max_tokens, 1), B, dtype=torch.float32, device=dev)
    all_done = torch.zeros(max(max_tokens, 1), dtype=torch.bool, device=dev)         # all_done[s]: every sequence finished at step s
    finished = torch.zeros(B, dtype=torch.bool, device=dev)
    stop_at = max_tokens
    for step in range(max_tokens):
        nxt = gen_tok[step]
        pick(last_logits, temperature, TOP_P, out=nxt, fused_argmax=model.last_argmax if model.last_argmax_valid_for(last_logits) else None)
        _abi.logprob_gather(last_logits, nxt, out=gen_lp[step])
        if eos_id is not None:
            finished |= nxt == eos_id
            all_done[step] = finished.all()
            if step % EOS_POLL == EOS_POLL - 1 and bool(all_done[: step + 1].any()):  # the only host sync of the loop
                break
        steps_run = step + 1
        if step + 1 < max_tokens:  # the reference runs one more forward whose result is never used; skip it
            last_logits = model.next_token_logits(nxt, cache, **lora_kw)

    # ---- one trip back to the host ----
    if eos_id is not None and max_tokens > 0:
        flags = all_done[:max(steps_run, 1)].tolist()
        stop_at = flags.index(True) if True in flags else steps_run
    else:
        stop_at = steps_run
    tokens: List[List[int]] = gen_tok[:stop_at].t().tolist() if stop_at > 0 else []
    gen_lp_host = gen_lp[:stop_at].t().tolist() if stop_at > 0 else [[] for _ in range(B)]
    logprobs: List[List[float]] = [[] for _ in range(B)]
    for (_, _, targets, where), lp in zip(plan.chunks, prompt_lp):
        for (b, _), t, v in zip(where, targets, lp.tolist()):
            if t >= 0:
                logprobs[b].append(v)
    for b in range(B):
        logprobs[b].extend(gen_lp_host[b])
    return tokens, logprobs


def pick(logits: torch.Tensor, temperature: float, top_p: float, out: Optional[torch.Tensor] = None,
         fused_argmax: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Next token per row of fp32 `logits` [B, V], on the device: greedy for temperature == 0 (`fused_argmax`, when given, is the
    decode kernel's own argmax of these logits), else one nucleus draw per row with uniforms from torch's CUDA generator."""
    out = torch.empty(logits.shape[0], dtype=torch.long, device=logits.device) if out is None else out
    if temperature > 0:
        u = torch.rand(logits.shape[0], dtype=torch.float32, device=logits.device)
        return _abi.sample_top_p(logits, u, temperature, top_p, out=out)
    if fused_argmax is not None:
        out.copy_(fused_argmax, non_blocking=True)
        return out
    return _abi.argmax_rows(logits, out=out)


def sample(logits: torch.Tensor, temperature: float, top_p: float) -> torch.Tensor:
    """Public helper with the reference's signature (generate.py:151-158): [B] token ids."""
    return pick(logits.float().contiguous(), temperature, top_p)
