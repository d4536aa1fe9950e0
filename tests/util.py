"""Shared helpers for the parity tests."""
import json
from pathlib import Path
from typing import Dict, List, Tuple

import torch

import synth
from oracle import restatement as R

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"
GOLDEN_CASES = sorted(p.stem for p in GOLDEN_DIR.glob("*.safetensors") if not p.stem.startswith("config1"))  # config1: its own compact format


def load_golden(name: str) -> Tuple[dict, Dict[str, torch.Tensor], dict]:
    import safetensors
    import safetensors.torch

    path = str(GOLDEN_DIR / f"{name}.safetensors")
    tensors = safetensors.torch.load_file(path)
    with safetensors.safe_open(path, "pt") as f:
        meta = f.metadata()
    return json.loads(meta["case"]), tensors, meta


def case_params_prompts(case: dict, seed: int = 1) -> Tuple[dict, List[List[int]]]:
    p = synth.shape(case["shape"], **case["over"])
    prompts = [synth.synth_prompt(n, p["vocab_size"], seed * 100 + i) for i, n in enumerate(case["prompt_lens"])]
    return p, prompts


def oracle_args(p: dict, max_batch: int) -> R.OracleArgs:
    moe = p.get("moe") or {}
    return R.OracleArgs(dim=p["dim"], n_layers=p["n_layers"], head_dim=p["head_dim"], hidden_dim=p["hidden_dim"],
                        n_heads=p["n_heads"], n_kv_heads=p["n_kv_heads"], norm_eps=p["norm_eps"], vocab_size=p["vocab_size"],
                        max_batch_size=max_batch, rope_theta=p.get("rope_theta"), num_experts=moe.get("num_experts", 0),
                        num_experts_per_tok=moe.get("num_experts_per_tok", 0), sliding_window=p.get("sliding_window"))


def oracle_model(p: dict, max_batch: int, seed: int = 1, dtype=torch.bfloat16) -> R.OracleTransformer:
    return R.OracleTransformer(oracle_args(p, max_batch), synth.synth_state_dict(p, seed, dtype))


def bf16_ulp_diff(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """|a-b| in units of bf16 ulps, per element (a, b bf16 or values that were rounded to bf16)."""
    a16 = a.to(torch.bfloat16).view(torch.int16).to(torch.int32)
    b16 = b.to(torch.bfloat16).view(torch.int16).to(torch.int32)
    # map sign-magnitude to a monotonic integer line
    a16 = torch.where(a16 < 0, -(a16 & 0x7FFF), a16)
    b16 = torch.where(b16 < 0, -(b16 & 0x7FFF), b16)
    return (a16 - b16).abs()


def same_machine_as_golden(meta: dict) -> bool:
    # the CPU's bf16 GEMMs split K by thread count: fixtures that record it are bit-exact only at the same count
    threads = meta.get("num_threads")
    return (meta.get("torch") == torch.__version__ and meta.get("cpu_capability") == torch.backends.cpu.get_cpu_capability()
            and (threads is None or threads == str(torch.get_num_threads())))


def assert_bf16_close(got: torch.Tensor, want: torch.Tensor, max_ulp: int = 1, min_exact: float = 0.97, atol: float = None, what: str = ""):
    """Element-wise comparison of two tensors of bf16-rounded values: every element within `max_ulp` bf16 ulps
    (or `atol` absolute, for values near zero where cancellation makes ulps meaningless) and at least
    `min_exact` of them bit-identical.  Default atol = 1e-5 * max(1, max|want|): the fp32 accumulation-order
    noise of a K~4k..14k dot product (this is the north-star's atol=1e-5).  Returns (exact fraction, max ulp)."""
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    if atol is None:
        atol = 1e-5 * max(1.0, want.abs().max().item())
    assert got.shape == want.shape, (got.shape, want.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite values in output"
    ulps = bf16_ulp_diff(got, want)
    ok = (ulps <= max_ulp) | ((got - want).abs() <= atol)
    exact = (ulps == 0).float().mean().item()
    worst = int(ulps[~((got - want).abs() <= atol)].max().item()) if (~((got - want).abs() <= atol)).any() else 0
    assert ok.all(), f"{what}: {(~ok).sum().item()} / {ok.numel()} elements differ by more than {max_ulp} bf16 ulp (worst {worst}); exact={exact:.4f}"
    assert exact >= min_exact, f"{what}: only {exact:.4f} of elements bit-exact (need {min_exact})"
    return exact, worst


# ----------------------------------------------------------------------------- which kernels a call launched
def launched_kernels(fn) -> List[str]:
    """Runs `fn()` and returns the attention, GEMM and MoE kernels libmb200 launched for it, in order, named like the kernels
    with their template arguments ("attn_decode_tma_kernel<8>").  The library records each launch next to the launch statement
    (mb200_debug_launch_log), so the record does not depend on a profiler being able to attach."""
    from mistral_inference_b200 import _abi

    _abi.launch_log(True)
    try:
        fn()
    finally:
        names = _abi.launch_log(False)
    return names


def assert_launched(fn, want: str, family: str, count: int) -> None:
    """Runs `fn()` and asserts that the kernels it launched whose names match the regex `family` are exactly `count` launches of
    kernels matching the regex `want` (no other kernel of the family ran in their place)."""
    import re

    mine = [n for n in launched_kernels(fn) if re.search(family, n)]
    wrong = sorted(set(n for n in mine if not re.search(want, n)))
    assert not wrong, f"expected only {want!r}, also launched: {wrong}"
    assert len(mine) == count, f"expected {count} launches of {want!r}, saw {len(mine)}"


# ----------------------------------------------------------------------------- tolerances at logit scale
def bf16_ulp_at(x: float) -> float:
    """Spacing of bf16 numbers at magnitude |x| (8 significand bits)."""
    import math

    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-30))) - 7)


def logit_tol(want: torch.Tensor, ulps: int = 2) -> float:
    """`ulps` bf16 ulps at the scale of the largest logit: logits are bf16 values (transformer.py:235) and two correct
    implementations that sum in a different order differ by one ulp on a few of them."""
    return ulps * bf16_ulp_at(float(want.abs().max()))


LOGPROB_TOL = 0.03  # log-softmax of logits that are within 2 ulps (<= 0.031 at |logit| < 4)


# ----------------------------------------------------------------------------- MoE: which tokens may legitimately flip an expert
class RouterProbe:
    """Records, for every oracle forward inside the `with` block, each token's smallest margin (in bf16 ulps of the router
    logits) between the k-th and (k+1)-th largest router logit over all MoE layers (moe.py:25-26: top-k on bf16 logits).
    A token whose margin is <= 2 ulps can be routed differently by another correct implementation (each logit may move by
    one ulp); every other token must reproduce the oracle's routing, hence its logits."""

    def __init__(self):
        self.calls = []  # one [T] tensor per forward: min margin over layers, in ulps
        self._layer_margins = []

    def __enter__(self):
        self._orig = R.moe_forward
        probe = self

        def recording(x, gate_w, experts, k):
            import torch.nn.functional as F

            logits = F.linear(x, gate_w).float()
            top = logits.topk(min(k + 1, logits.shape[-1]), dim=-1).values
            ulp = torch.pow(2.0, torch.floor(torch.log2(top[:, k - 1].abs().clamp_min(1e-30))) - 7)
            probe._layer_margins.append((top[:, k - 1] - top[:, k]) / ulp if top.shape[-1] > k else torch.full_like(ulp, 1e9))
            return probe._orig(x, gate_w, experts, k)

        R.moe_forward = recording
        return self

    def __exit__(self, *exc):
        R.moe_forward = self._orig

    def end_forward(self) -> torch.Tensor:
        """Call after each oracle forward: folds the per-layer margins of that call into one [T] tensor."""
        m = torch.stack(self._layer_margins, 0).min(0).values if self._layer_margins else torch.zeros(0)
        self._layer_margins = []
        self.calls.append(m)
        return m


# ----------------------------------------------------------------------------- MoE row plan (host restatement of csrc/moe.cuh)
def moe_route_host(x: torch.Tensor, gate_w: torch.Tensor, k: int):
    """(sel [T, k] ascending expert ids, wts [T, k] bf16) exactly as moe.py:25-27 + the ascending-expert reordering."""
    import torch.nn.functional as F

    logits = F.linear(x, gate_w)
    w, sel = torch.topk(logits, k)
    w = F.softmax(w, dim=1, dtype=torch.float).to(x.dtype)
    order = sel.argsort(dim=1)
    return sel.gather(1, order).to(torch.int32), w.gather(1, order)


def moe_plan_host(sel: torch.Tensor, E: int, tile_rows: int, shard=(0, 1)):
    """slot [T, k], segment starts [E + 1], and this rank's (expert, first row) m tiles: pairs keep token order inside an expert's
    segment, every segment is padded to a multiple of `tile_rows` (the deterministic plan of moe_plan_kernel)."""
    T, k = sel.shape
    flat = sel.reshape(-1).tolist()
    counts = [0] * E
    for e in flat:
        counts[e] += 1
    seg, tiles, rows = [], [], 0
    for e in range(E):
        seg.append(rows)
        m_tiles = -(-counts[e] // tile_rows)
        if e % shard[1] == shard[0]:
            tiles += [(e, rows + m * tile_rows) for m in range(m_tiles)]
        rows += m_tiles * tile_rows
    seg.append(rows)
    run = [0] * E
    slot = []
    for e in flat:
        slot.append(seg[e] + run[e])
        run[e] += 1
    return torch.tensor(slot, dtype=torch.int32).view(T, k), seg, tiles
