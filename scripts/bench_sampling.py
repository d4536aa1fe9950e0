"""Cost of per-sequence sampling controls (generate(temperature=[...], random_seed=..., presence_penalty=..., ...)), timed with CUDA
events, the variants alternated round by round in one process.

  python scripts/bench_sampling.py [--launches 200] [--steps 64] [--rounds 3] [--skip-steps] [--out DIR]

Kernel time of the selection tail alone, for B in {1, 8, 32} and V in {32000, 131072}, fp32 logits [B, V]:
  * pick       today's path at temperature 0.7: torch.rand(B) + mb200_sample_top_p (top_p 0.8);
  * controls   mb200_select_tokens with per-row temperature 0.7 / top_p 0.8 and Philox seeds, no count table;
  * penalties  the same with presence 0.5 / frequency 0.3 and the [B, V] int32 count table read on load.
Bytes per row: one pass over the logits (4 V) and, with penalties, over the counts (4 V more).  The nucleus search re-reads the row
32 times; at these sizes the rows stay in L2, so these are the HBM bytes, not the bytes the SMs load.

Step time of a decode loop iteration -- next_token_logits, the selection, mb200_logprob_gather -- as generate() runs it, with random
weights: the Mistral-7B shape at batch 1 (the decode megakernel) and the Mistral-Nemo-12B shape at batch 32 (the CUDA-graph path),
each with pick at temperature 0.7 and with the controls plus penalties.  One JSON line per measurement, with the card name and
power limit read in the same run.
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from bench_lora import gpu_line, new_cache, timed  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.generate import SamplingControls, pick  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

TEMP, TOP_P, PRES, FREQ = 0.7, 0.8, 0.5, 0.3


def controls(B: int, V: int, penalties: bool) -> SamplingControls:
    p = PRES if penalties else 0.0
    f = FREQ if penalties else 0.0
    return SamplingControls(B, V, "cuda", [TEMP] * B, [TOP_P] * B, [1234 + b for b in range(B)], [p] * B, [f] * B)


def selectors(B: int, V: int):
    """name -> fn(logits, out): the three selection tails."""
    ctl, pen = controls(B, V, False), controls(B, V, True)
    return {"pick": lambda lg, out: pick(lg, TEMP, TOP_P, out=out),
            "controls": lambda lg, out: ctl.select(lg, out),
            "penalties": lambda lg, out: pen.select(lg, out)}


def model(shape: str, B: int) -> Transformer:
    p = synth.shape(shape)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = B
    m = Transformer.empty(args, "cuda", torch.bfloat16)
    m.load_state_dict(synth.synth_state_dict(p, 0, torch.bfloat16, "cuda"))
    return m.eval()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py measures on the GPU; none is visible")
    hw = gpu_line()
    lines = []

    def emit(**kw):
        kw["gpu"] = hw
        lines.append(kw)
        print(json.dumps(kw), flush=True)

    # ---- the selection tail alone
    for V in (32000, 131072):
        for B in (1, 8, 32):
            logits = torch.randn(B, V, device="cuda") * 3
            out = torch.empty(B, dtype=torch.long, device="cuda")
            fns = selectors(B, V)
            for fn in fns.values():  # warm-up
                fn(logits, out)
            us = {k: [] for k in fns}
            for _ in range(a.rounds):
                for k, fn in fns.items():
                    us[k].append(1e3 * timed(lambda: fn(logits, out), a.launches))
            for k in fns:
                emit(workload="selection", variant=k, B=B, V=V, us_per_call=[round(x, 2) for x in us[k]],
                     us_median=round(statistics.median(us[k]), 2), hbm_bytes_per_row=(8 if k == "penalties" else 4) * V)

    # ---- a decode loop iteration
    if a.skip_steps:
        return
    for shape, B, path in (("mistral-7b", 1, "megakernel"), ("mistral-nemo-12b", 32, "graph")):
        torch.cuda.empty_cache()
        m = model(shape, B)
        V = m.args.vocab_size
        cache = new_cache(m, 128 + (a.rounds * 2 + 2) * (a.steps + 4) + 8)
        m.forward(torch.tensor(synth.synth_prompt(128 * B, V, 3), device="cuda"), [128] * B, cache)
        tok = torch.zeros(B, dtype=torch.long, device="cuda")
        lp = torch.zeros(B, dtype=torch.float32, device="cuda")
        fns = selectors(B, V)
        fns = {"pick": fns["pick"], "controls+penalties": fns["penalties"]}
        state = {"logits": m.next_token_logits(tok, cache)}

        def step(select):
            select(state["logits"], tok)
            _abi.logprob_gather(state["logits"], tok, out=lp)
            state["logits"] = m.next_token_logits(tok, cache)

        for fn in fns.values():  # warm-up and graph capture
            for _ in range(2):
                step(fn)
        ms = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, fn in fns.items():
                ms[k].append(timed(lambda: step(fn), a.steps))
        for k in fns:
            emit(workload=f"decode step {shape} B={B} ({path})", variant=k, ms_per_step=[round(x, 4) for x in ms[k]],
                 ms_median=round(statistics.median(ms[k]), 4), megakernel=m._megakernel_ok(B))
        del cache, m
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "bench_sampling.jsonl").write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
