"""Cost of un-merged LoRA adapters: the same seeded model with and without a `lora` block, timed with CUDA events.

  python scripts/bench_lora.py [--ranks 16 64] [--steps 64] [--rounds 2] [--out DIR]

Workloads, each measured for the model without adapters and with adapters at every rank, the variants alternated `--rounds` times:
  * Mistral-7B shape, 32 layers, batch-1 greedy decode on the per-layer CUDA-graph path (the megakernel, which has no LoRA stage,
    is timed once for reference);
  * the same model's 4096-token first prefill: the 32 layers plus the final norm (forward_partial), cache preallocated and reset
    between runs, no lm head;
  * Mistral-Nemo-12B shape, 40 layers, one batch-32 decode step.
Then, per decode workload, a torch.profiler run of 16 graph-replayed steps splits the step into kernel time per kernel family and
the rest of the step (launch gaps; PDL overlap counts as kernel time of both kernels).  One JSON line per measurement, with the
card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402


def gpu_line() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def model(shape: str, rank, max_batch: int) -> Transformer:
    p = synth.shape(shape)
    d = dict(p) if rank is None else dict(p, lora=dict(rank=rank, scaling=2.0))
    args = mi.TransformerArgs.from_dict(d)
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16)
    m.load_state_dict(synth.synth_state_dict(p, 0, torch.bfloat16, "cuda"))
    if rank is not None:
        m._load_lora_state_dict(synth.synth_lora_state_dict(p, rank, 1, torch.bfloat16, 1.0, "cuda"))
    return m.eval()


def new_cache(m: Transformer, max_seq: int) -> BufferCache:
    a = m.args
    c = BufferCache(m.n_local_layers, a.max_batch_size, max_seq, a.n_kv_heads, a.head_dim, a.sliding_window)
    c.to(m.device, m.dtype)
    c.reset()
    return c


def timed(fn, n: int) -> float:
    """ms per call over n calls."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


class Decode:
    """A prefilled cache of B sequences and a decode step on it (graph path unless the megakernel applies)."""

    def __init__(self, m: Transformer, B: int, prompt_len: int, steps: int):
        self.m, self.B = m, B
        self.cache = new_cache(m, prompt_len + 8 * steps + 64)
        prompt = torch.tensor(synth.synth_prompt(prompt_len * B, m.args.vocab_size, 3), device="cuda")
        m.forward(prompt, [prompt_len] * B, self.cache)
        self.tok = torch.zeros(B, dtype=torch.long, device="cuda")
        for _ in range(4):  # warm-up and graph capture
            self.step()

    def step(self):
        self.m.next_token_logits(self.tok, self.cache)


def family(name: str) -> str:
    for f in ("lora_down_reduce_kernel", "lora_down_kernel", "skinny_linear_kernel", "attn_prefill", "gemm_streamk_kernel", "gemm_wgmma_kernel",
              "gemm_mma_kernel", "attn_decode", "rmsnorm_kernel", "decode_meta", "argmax", "kv_ring_write", "decode_megakernel"):
        if f in name:
            return f
    return "other"


def breakdown(fn, steps: int = 16) -> dict:
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    fam = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            fam[family(e.name)] += e.device_time_total / 1000.0 / steps  # ms per step
    return {k: round(v, 4) for k, v in sorted(fam.items(), key=lambda kv: -kv[1])}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    hw = gpu_line()
    lines = []

    def emit(**kw):
        kw["gpu"] = hw
        lines.append(kw)
        print(json.dumps(kw), flush=True)

    variants = [None] + a.ranks
    # ---- 7B: all variants resident, measurements alternated
    os.environ["MB200_MEGAKERNEL"] = "0"
    models = {r: model("mistral-7b", r, 1) for r in variants}
    T = 4096
    pcache = new_cache(models[None], T)
    prompt = torch.tensor(synth.synth_prompt(T, 32000, 4), device="cuda")

    def prefill(r):
        pcache.reset()
        models[r].forward_partial(prompt, [T], pcache)

    for r in variants:  # first: sizes each model's workspace for T tokens, which the decode graphs below then capture
        prefill(r)
    dec = {r: Decode(models[r], 1, 128, a.steps) for r in variants}
    for rnd in range(a.rounds):
        for r in variants:
            ms = timed(dec[r].step, a.steps)
            emit(workload="7b decode B=1 (graph path)", rank=r, round=rnd, ms_per_token=round(ms, 4), tok_s=round(1000 / ms, 1))
            emit(workload="7b prefill T=4096 (layers + final norm)", rank=r, round=rnd, ms=round(timed(lambda: prefill(r), 3), 3))
    for r in variants:
        emit(workload="7b decode B=1 (graph path) kernel ms per step", rank=r, kernels=breakdown(dec[r].step),
             step_ms=round(timed(dec[r].step, a.steps), 4))
        emit(workload="7b prefill T=4096 kernel ms per call", rank=r, kernels=breakdown(lambda: prefill(r), 2))
    os.environ["MB200_MEGAKERNEL"] = "1"
    mk = Decode(models[None], 1, 128, a.steps)
    emit(workload="7b decode B=1 (megakernel)", rank=None, ms_per_token=round(timed(mk.step, a.steps), 4))
    del dec, mk, models, pcache
    torch.cuda.empty_cache()
    # ---- Nemo B = 32: the plain model stays resident, each adapter model alternates with it
    base = model("mistral-nemo-12b", None, 32)
    dbase = Decode(base, 32, 128, a.steps)
    for r in a.ranks:
        m = model("mistral-nemo-12b", r, 32)
        d = Decode(m, 32, 128, a.steps)
        for rnd in range(a.rounds):
            for rr, dd in ((None, dbase), (r, d)):
                emit(workload="nemo decode B=32", rank=rr, round=rnd, ms_per_step=round(timed(dd.step, a.steps), 4))
        for rr, dd in ((None, dbase), (r, d)):
            emit(workload="nemo decode B=32 kernel ms per step", rank=rr, kernels=breakdown(dd.step), step_ms=round(timed(dd.step, a.steps), 4))
        del d, m, dd
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "bench_lora.jsonl").write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
