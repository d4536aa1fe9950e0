"""Twelve query heads per kv head (Mistral Large 2: 96 over 8) in the bf16-cache attention kernels.

attn_decode_tma_kernel<12> holds query heads 8..11 of a group in MMA rows 8..11 and keeps its merge arrays in the idle K/V ring;
the prefill kernels map query head h to kv head h / (H/KV).  The checks are those of tests/test_gpu_attention_edges.py at REP = 12:
the exact key set every query sees (position-coded V) at tile, window and split edges -- first prefill on both prefill kernels,
chunks on the ring, decode at B = 1 with up to 64 splits, B = 5 and B = 8 -- and the softmax weighting against float64 under
growing maxima, dominant keys and wide scores.  The launch log names the kernel each time.  The decode kernel's occupancy
(cudaOccupancyMaxActiveBlocksPerMultiprocessor, through mb200_debug_attn_decode_occupancy) is two CTAs per SM.  And a 2-layer bf16
model of the Mistral Large 2 shape against the CPU oracle: first prefill, chunked prefill on the ring, and graph decode at B = 1
(the megakernel refuses ratio 12; several KV splits) and B = 8.
"""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer
from oracle import restatement as R

from . import test_gpu_attention_edges as AE
from .test_gpu_int4_dense import run_against_oracle
from .util import oracle_args

REP = 12
DEV = "cuda"


@pytest.fixture(scope="module")
def ws():
    need = 8 * AE.KV * 64 * REP * (AE.HD + 2) * 4  # split partials at B = 8, S = 64
    return _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + need, torch.device(DEV))


def decode_cases_12():
    out = list(AE.decode_cases())
    for S in (64, 33, 7, 1):  # batch 1: a 4k ring over many splits (the Mistral Large decode), and a short one
        out.append(AE.Case("decode", (4096,), (), 4096, S))
        out.append(AE.Case("decode", (4000,), (), 4096, S))
        out.append(AE.Case("decode", (65,), (), 4096, S))
    for S, W in ((1, 300), (2, 4096), (16, 4096)):  # batch 8
        out.append(AE.Case("decode", tuple(min(n, W) for n in (1, 63, 64, 65, 127, 129, 300, W)), (), W, S))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["wgmma", "mma"])
def test_first_prefill_visible_sets_12(kernel, ws, monkeypatch):
    AE.check_visible_sets(AE.first_prefill_cases(), kernel, REP, ws, monkeypatch)


@pytest.mark.gpu
def test_ring_prefill_visible_sets_12(ws, monkeypatch):
    AE.check_visible_sets(AE.ring_cases(), "mma", REP, ws, monkeypatch)


@pytest.mark.gpu
def test_cacheless_visible_sets_12(ws, monkeypatch):
    AE.check_visible_sets(AE.nocache_cases(), "mma", REP, ws, monkeypatch)


@pytest.mark.gpu
def test_decode_visible_sets_12(ws, monkeypatch):
    AE.check_visible_sets(decode_cases_12(), "tma", REP, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["rising", "dominant", "wide"])
@pytest.mark.parametrize("kernel", ["wgmma", "mma", "tma"])
def test_softmax_weighting_vs_float64_12(kernel, pattern, ws, monkeypatch):
    case = AE.SOFTMAX_CASES[kernel]
    AE.select_kernel(kernel, monkeypatch)
    q, K, V = AE.softmax_inputs(case, pattern, REP, seed=REP)
    outs = []
    AE.assert_launched(lambda: outs.append(AE.run(case, q, K, V, REP, ws)), AE.KERNEL[kernel].format(rep=REP), AE.ATTN, 1)
    got = outs[0].double().cpu()
    o64, mag = AE.reference64(case, q, K, V, REP)
    ulp = torch.exp2(torch.floor(torch.log2(o64.abs().clamp_min(2.0 ** -126))) - 7)
    bound = 2.0 ** -8 * mag + ulp
    err = (got - o64).abs()
    assert torch.isfinite(got).all(), "non-finite output"
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{(err > bound).sum().item()} elements beyond the bound; worst err / bound = {worst:.2f}"


@pytest.mark.gpu
def test_decode_softmax_at_batch_one_with_many_splits(ws, monkeypatch):
    """The Mistral Large decode shape: one sequence, a 4096-key ring over 33 splits, wide scores."""
    case = AE.Case("decode", (4096,), (), 4096, 33)
    q, K, V = AE.softmax_inputs(case, "wide", REP, seed=5)
    outs = []
    AE.assert_launched(lambda: outs.append(AE.run(case, q, K, V, REP, ws)), AE.KERNEL["tma"].format(rep=REP), AE.ATTN, 1)
    o64, mag = AE.reference64(case, q, K, V, REP)
    ulp = torch.exp2(torch.floor(torch.log2(o64.abs().clamp_min(2.0 ** -126))) - 7)
    assert ((outs[0].double().cpu() - o64).abs() <= 2.0 ** -8 * mag + ulp).all()


@pytest.mark.gpu
def test_decode_kernel_occupancy():
    """Two CTAs of attn_decode_tma_kernel<12> per SM: its merge arrays live in the ring, not beside it (<8>, whose 16 KB of merge
    arrays sit beside the ring, fits one)."""
    occ = {rep: _abi.attn_decode_occupancy(rep) for rep in (1, 2, 4, 6, 8, 12)}
    print(f"attn_decode_tma_kernel CTAs per SM by head ratio: {occ}")
    assert occ[REP] == 2 and all(occ[REP] >= v for v in occ.values())


@pytest.mark.gpu
@pytest.mark.parametrize("lens,chunk", [([300], None), ([40, 33], 16), ([20 - (b % 3) for b in range(8)], None)],
                         ids=["prefill-decode-b1", "chunked-b2", "decode-b8"])
def test_bf16_mistral_large_vs_oracle(lens, chunk):
    p = synth.shape("mistral-large-2", n_layers=2, vocab_size=4096)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = len(lens)
    m = Transformer.empty(args, DEV, torch.bfloat16)
    sd = synth.synth_state_dict(p, 1, torch.bfloat16, DEV)
    m.load_state_dict(sd)
    om = R.OracleTransformer(oracle_args(p, len(lens)), {k: v.cpu() for k, v in sd.items()})
    assert not m.eval()._megakernel_ok(1)
    kinds = run_against_oracle(m, om, p, f"bf16 mistral-large-2 x2 {lens}", lens, chunk)
    assert "attn_decode_tma_kernel" in kinds and "decode_megakernel" not in kinds, kinds
