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
  * per-sequence sampling controls (a list of temperatures, top_p, random_seed, presence / frequency penalties) select with
    `mb200_select_tokens` instead of pick: per-row controls, a seeded Philox stream, counts and steps all live on the device.
"""
import math
import numbers
from typing import List, Optional, Sequence, Tuple, Union

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


PENALTY_MAX = 2.0  # |presence_penalty|, |frequency_penalty| <= 2: the range of Mistral's chat API
FloatOrList = Union[float, Sequence[float]]


class SamplingControls:
    """The per-sequence controls of one generate() call on the device: temperature, top_p, presence and frequency penalty [B]
    fp32, the seeds [B] (uint64 bit patterns in int64) or None, each sequence's step [B] int32 and, with a penalty, the counts of
    its generated tokens [B, V] int32.  Allocated once per call; `select` advances steps and counts on the device."""

    def __init__(self, B: int, V: int, device, temperature: List[float], top_p: List[float], seeds: Optional[List[int]],
                 presence: List[float], frequency: List[float]):
        f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=device)  # noqa: E731
        self.temperature, self.top_p, self.presence, self.frequency = f32(temperature), f32(top_p), f32(presence), f32(frequency)
        self.seeds = None if seeds is None else torch.tensor([s - (1 << 64) if s >= 1 << 63 else s for s in seeds], dtype=torch.int64,
                                                             device=device)
        self.sampled = any(t > 0 for t in temperature)
        # without seeds and without a sampled row the kernel reads no uniform: one zero buffer keeps the generator untouched
        self.zero_u = torch.zeros(B, dtype=torch.float32, device=device) if seeds is None and not self.sampled else None
        self.step = torch.zeros(B, dtype=torch.int32, device=device)
        penalised = any(p != 0 for p in presence) or any(f != 0 for f in frequency)
        self.counts = torch.zeros(B, V, dtype=torch.int32, device=device) if penalised else None

    def select(self, logits: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        u = None
        if self.seeds is None:  # torch's CUDA generator, one draw per row and step as pick takes it
            u = torch.rand(logits.shape[0], dtype=torch.float32, device=logits.device) if self.sampled else self.zero_u
        return _abi.select_tokens(logits, self.temperature, self.top_p, self.presence, self.frequency, self.step, out, seeds=self.seeds,
                                  uniform=u, counts=self.counts)


def _per_sequence(name: str, v, B: int) -> List:
    if isinstance(v, (list, tuple)):
        if len(v) != B:
            raise ValueError(f"{name} has {len(v)} entries for {B} prompts")
        return list(v)
    return [v] * B


def sampling_controls(B: int, temperature: FloatOrList, top_p: FloatOrList, random_seed: Union[None, int, Sequence[int]],
                      presence_penalty: FloatOrList, frequency_penalty: FloatOrList):
    """Checks generate()'s sampling keywords on the host and returns None when they select today's path (every argument a scalar,
    no seed, both penalties 0), else the per-sequence lists (temperature, top_p, seeds or None, presence, frequency)."""
    lists = {}
    for name, v in (("temperature", temperature), ("top_p", top_p), ("presence_penalty", presence_penalty),
                    ("frequency_penalty", frequency_penalty)):
        vals = _per_sequence(name, v, B)
        for x in vals:
            if isinstance(x, bool) or not isinstance(x, numbers.Real) or not math.isfinite(x):
                raise ValueError(f"{name}={x!r}: a finite number is required")
            if name == "temperature" and x < 0:
                raise ValueError(f"temperature={x!r} is negative")
            if name == "top_p" and not 0 <= x <= 1:
                raise ValueError(f"top_p={x!r} lies outside [0, 1]")
            if name.endswith("penalty") and not -PENALTY_MAX <= x <= PENALTY_MAX:
                raise ValueError(f"{name}={x!r} lies outside [-{PENALTY_MAX:g}, {PENALTY_MAX:g}]")
        lists[name] = [float(x) for x in vals]
    seeds = None
    if random_seed is not None:
        per_seq = isinstance(random_seed, (list, tuple))
        given = _per_sequence("random_seed", random_seed, B) if per_seq else [random_seed]
        for x in given:
            if isinstance(x, bool) or not isinstance(x, numbers.Integral) or not 0 <= x < 1 << 64:
                raise ValueError(f"random_seed={x!r}: an int in [0, 2^64) is required")
        # one int s: sequence b runs on (s + b) mod 2^64
        seeds = [int(x) for x in given] if per_seq else [(int(random_seed) + b) % (1 << 64) for b in range(B)]
    scalars = not any(isinstance(v, (list, tuple)) for v in (temperature, top_p, presence_penalty, frequency_penalty))
    if scalars and random_seed is None and presence_penalty == 0 and frequency_penalty == 0:
        return None
    return lists["temperature"], lists["top_p"], seeds, lists["presence_penalty"], lists["frequency_penalty"]


@torch.inference_mode()
def generate(encoded_prompts: List[List[int]], model: Transformer, images: List[List] = [], *, max_tokens: int,  # noqa: B006
             temperature: FloatOrList, chunk_size: Optional[int] = None, eos_id: Optional[int] = None,
             draft: Optional[Transformer] = None, draft_tokens: int = 4,
             lora_ids: Optional[List[int]] = None, top_p: FloatOrList = TOP_P, random_seed: Union[None, int, Sequence[int]] = None,
             presence_penalty: FloatOrList = 0.0, frequency_penalty: FloatOrList = 0.0) -> Tuple[List[List[int]], List[List[float]]]:
    """`draft`: another Transformer with the same vocabulary that proposes `draft_tokens` tokens per round for the model to verify
    (speculative decoding, mistral_inference_b200/speculative.py).  Same return value and semantics as without it; greedy output
    stays the model's own argmax choices and sampled output keeps the model's nucleus distribution.
    `lora_ids`: one entry per prompt, the model's adapter slot that sequence runs through (Transformer `lora_slots`), or -1 for the
    base model; None is slot 0 for every sequence.  A sequence's result does not depend on the other sequences' ids.

    Sampling controls, each a scalar for every sequence or a list with one entry per prompt:
      `temperature` >= 0 (0: greedy), `top_p` in [0, 1] (the nucleus), `presence_penalty` and `frequency_penalty` in [-2, 2].
      Before each selection, logit v of sequence b becomes l[v] - (c[v] * frequency_penalty + presence_penalty if c[v] > 0), each
      operation rounded to fp32, with c[v] the times b has generated v (prompt tokens are not counted).
      `random_seed`: None draws the uniforms from torch's CUDA generator (torch.manual_seed applies); an int s gives sequence b the
      seed (s + b) mod 2^64, a list gives each sequence its own.  A seeded sequence's tokens depend only on its prompt, its own
      controls and its seed, not on the rest of the batch: its step-t uniform is Philox4x32-10 at counter (t, 0, 0, 0).
    The returned log-probabilities are log_softmax of the model's raw logits at the chosen token: neither temperature nor the
    penalties enter them.  With every argument a scalar, no seed and both penalties 0 the call is today's path, bit for bit."""
    controls = sampling_controls(len(encoded_prompts), temperature, top_p, random_seed, presence_penalty, frequency_penalty)
    if lora_ids is not None:
        if draft is not None:
            raise ValueError("lora_ids with a draft model (speculative decoding) is not built")
        model.check_lora_ids(lora_ids, len(encoded_prompts))
    lora_kw = {} if lora_ids is None else {"lora_ids": lora_ids}  # no ids: the model calls take no LoRA keyword
    if draft is not None:
        from .speculative import check_draft_controls, generate_speculative

        check_draft_controls(controls, top_p)
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
    ctl = None if controls is None else SamplingControls(B, V, dev, *controls)
    stop_at = max_tokens
    for step in range(max_tokens):
        nxt = gen_tok[step]
        if ctl is None:
            pick(last_logits, temperature, top_p, out=nxt, fused_argmax=model.last_argmax if model.last_argmax_valid_for(last_logits) else None)
        else:  # the decode kernel's fused argmax is of the raw logits: never used here
            ctl.select(last_logits, nxt)
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
