"""Cost of a bank of LoRA adapter slots: the same seeded model with no adapter, one adapter (the single-adapter path, no ids) and
`lora_slots` of 2, 4, 8 and 16 with the sequences' ids spread over the slots, timed with CUDA events.

  python scripts/bench_multi_lora.py [--ranks 16 64] [--slots 2 4 8 16] [--steps 64] [--rounds 2] [--out DIR]

Workloads, per configuration (one model resident at a time; the measurements of a configuration are repeated `--rounds` times):
  * Mistral-7B shape, 32 layers: one batch-32 decode step on the CUDA-graph path, and a 4096-token prefill as 8 sequences of 512
    tokens (the 32 layers and the lm head on each sequence's last token, `last_token_logits`), cache reset between runs;
  * Mistral-Nemo-12B shape, 40 layers: one batch-32 decode step.
Sequence b uses slot b % lora_slots.  Each configuration also reports the device memory its model holds (weights and adapters) and
the peak allocated during the configuration (which includes the seeded state dict while it loads, the caches and activations).
One JSON line per measurement, with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from bench_lora import gpu_line, new_cache, timed  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

B = 32
PREFILL_SEQS, PREFILL_LEN = 8, 512


def model(shape: str, rank, slots: int, max_batch: int) -> Transformer:
    """rank None: no adapter.  Otherwise a seeded adapter (seed j) in every slot j."""
    p = synth.shape(shape)
    args = mi.TransformerArgs.from_dict(dict(p) if rank is None else dict(p, lora=dict(rank=rank, scaling=2.0)))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16, lora_slots=slots)
    m.load_state_dict(synth.synth_state_dict(p, 0, torch.bfloat16, "cuda"))
    for j in range(slots if rank is not None else 0):
        m._load_lora_state_dict(synth.synth_lora_state_dict(p, rank, 1 + j, torch.bfloat16, 1.0, "cuda"), slot=j)
    return m.eval()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--slots", type=int, nargs="+", default=[2, 4, 8, 16])
    ap.add_argument("--shapes", nargs="+", default=["mistral-7b", "mistral-nemo-12b"])
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_lora.py measures on the GPU; none is visible")
    os.environ["MB200_MEGAKERNEL"] = "0"  # batch 32 never takes it; stated for clarity
    hw = gpu_line()
    lines = []

    def emit(**kw):
        kw["gpu"] = hw
        lines.append(kw)
        print(json.dumps(kw), flush=True)

    # (rank, slots, ids): no adapter, one adapter on the single-adapter path, then the banks
    configs = [(None, 1, None)] + [(r, 1, None) for r in a.ranks] + [(r, n, [b % n for b in range(B)]) for r in a.ranks for n in a.slots]
    for shape in a.shapes:
        for rank, slots, ids in configs:
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            m = model(shape, rank, slots, B)
            resident = torch.cuda.memory_allocated()
            vocab = m.args.vocab_size
            tag = dict(shape=shape, rank=rank, lora_slots=slots if rank is not None else 0, ids="spread" if ids else None)
            kw = {} if ids is None else {"lora_ids": ids}
            if shape == "mistral-7b":  # first: sizes the workspace for the prefill, which the decode graph then captures
                pcache = new_cache(m, PREFILL_LEN)
                prompt = torch.tensor(synth.synth_prompt(PREFILL_SEQS * PREFILL_LEN, vocab, 4), device="cuda")
                pids = {} if ids is None else {"lora_ids": ids[:PREFILL_SEQS]}

                def prefill():
                    pcache.reset()
                    m.last_token_logits(prompt, [PREFILL_LEN] * PREFILL_SEQS, pcache, **pids)

                prefill()
                ms = [timed(prefill, 3) for _ in range(a.rounds)]
                emit(workload=f"prefill {PREFILL_SEQS}x{PREFILL_LEN} tokens", **tag, ms=[round(x, 3) for x in ms],
                     ms_median=round(statistics.median(ms), 3))
                del pcache
            cache = new_cache(m, 128 + a.steps * (a.rounds + 1) + 8)
            m.forward(torch.tensor(synth.synth_prompt(128 * B, vocab, 3), device="cuda"), [128] * B, cache, **kw)
            tok = torch.zeros(B, dtype=torch.long, device="cuda")
            step = lambda: m.next_token_logits(tok, cache, **kw)  # noqa: E731
            for _ in range(4):  # warm-up and graph capture
                step()
            ms = [timed(step, a.steps) for _ in range(a.rounds)]
            emit(workload=f"decode B={B} (graph path)", **tag, ms_per_step=[round(x, 4) for x in ms], ms_median=round(statistics.median(ms), 4),
                 resident_gib=round(resident / 2 ** 30, 2), peak_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
            del cache, m, step
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "bench_multi_lora.jsonl").write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
