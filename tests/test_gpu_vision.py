"""The vision path on the GPU against the CPU oracle (oracle/vision.py): patchify + conv GEMM, head_dim-64 QKV with the 2-D RoPE
in every GEMM regime, the head_dim-64 unmasked attention kernel, the encoder at the real layer shape, merger / adapter / splice,
and the model through `generate(images=...)`.  Each kernel test asserts from the launch log that the intended kernel ran.

Exactness argument of the attention visible-set test (head_dim 64).  q = 0, so every score is 0 and every P is exactly 1: the row
sum l is the number n of visible keys (an integer, exact in fp32) and O[d] is the exact count of visible keys whose V row has a 1
in column d.  V[j, h*64 + d] = 1 iff d < 63 and (j + h) % 63 == d, or d == 63 and j >= 63, so for the unmasked mode (every
query sees keys 0..T-1) the output of head h is out[d] = c_hd / T with c_hd the number of keys j < T with a 1 in column d; the
kernel computes c * (1/l) rounded to bf16, which is within 1 bf16 ulp of c / T, and exactly 0 where c = 0.  One key more or less
changes n by one and one residue count by one: for T >= 2 the keys span at least two columns, so some value moves by a relative
(n - c) / (c (n +- 1)), at least about 1/66 (c <= ceil(4097 / 63)) -- more than the 2^-7 relative width of 1 bf16 ulp; at T = 1 the
flag column 63 separates key 0 from keys 63, 126, ... of the same residue.  Reading another head's V shifts the residues.  tests/test_oracle_vision.py checks on the CPU that the comparator rejects every such change for every T of the grid.

Softmax weighting (random q, k, v): P is rounded to bf16 before P V, so against a float64 reference each output element may be off
by at most 2^-8 * sum_j p_j |v_j| (relative rounding of each P, with p the exact weights), plus 1 bf16 ulp of the output and the
fp32 accumulation noise, which the bound's slack covers.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer
from oracle import restatement as R
from oracle import vision as V
from oracle.make_vision_pins import VISION_CASES, case_images, case_params

from .test_oracle_vision import H_VIS, VIS_T, visible_expected, visible_matches
from .util import LOGPROB_TOL, assert_bf16_close, assert_launched, launched_kernels, oracle_args

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ws(T, dim=1024, heads=16, hidden=4096):
    return _abi.Workspace(_abi.workspace_bytes(T, dim, heads, heads, 64, hidden, 0, 1), torch.device(DEV))


# ----------------------------------------------------------------------------- patchify + conv GEMM
@pytest.mark.parametrize("patch,sizes", [(16, [(3, 64, 48), (3, 37, 70), (3, 16, 16)]), (14, [(3, 56, 42), (3, 30, 62), (3, 100, 14)])])
def test_patchify_conv_vs_oracle(patch, sizes):
    hidden = 1024
    w = synth.synth_tensor("vision_encoder.patch_conv.weight", (hidden, 3, patch, patch), 1)
    k = 3 * patch * patch
    k_pad = (k + 63) // 64 * 64
    wp = torch.zeros(hidden, k_pad, dtype=torch.bfloat16)
    wp[:, :k] = w.reshape(hidden, k)
    imgs = [synth.synth_image(*s, seed=i) for i, s in enumerate(sizes)]
    grid = [(s[1] // patch, s[2] // patch) for s in sizes]
    n = sum(h * w_ for h, w_ in grid)
    patches = torch.empty(n, k_pad, dtype=torch.bfloat16, device=DEV)
    out = torch.empty(n, hidden, dtype=torch.bfloat16, device=DEV)
    ws = _ws(n)

    def run():
        o = 0
        for img, (h, w_) in zip(imgs, grid):
            _abi.vision_patchify(img.to(DEV), patches[o: o + h * w_], patch)
            o += h * w_
        _abi.linear_residual(patches, wp.to(DEV), None, out, ws)

    names = launched_kernels(run)
    assert names.count("patchify_kernel") == len(imgs)
    torch.cuda.synchronize()
    assert torch.count_nonzero(patches[:, k:]) == 0
    want = torch.cat([F.conv2d(img[None], w, stride=patch)[0].flatten(1).t() for img in imgs])
    assert_bf16_close(out, want, max_ulp=1, min_exact=0.9, what="patch conv")


# ----------------------------------------------------------------------------- head_dim-64 QKV + 2-D RoPE
@pytest.mark.parametrize("T", [1, 4, 5, 100, 128, 129, 4096])
def test_qkv_rope2d_hd64_vs_oracle(T):
    dim, H, hd, side = 1024, 16, 64, 64
    x = synth.synth_tensor("x", (T, dim), T) * 4
    nw = synth.synth_tensor("attention_norm.weight", (dim,), 2)
    wq, wk, wv = (synth.synth_tensor(f"w{c}", (dim, dim), 3) for c in "qkv")
    table = V.rope_table_2d(hd, side, side, 1e4)
    rows = (torch.arange(T) * 7) % side
    cols = (torch.arange(T) * 13 + 5) % side
    pos = (rows * side + cols).to(torch.int32)
    xn = R.rms_norm(x, nw, 1e-5)
    q_want, k_want = R.apply_rope(F.linear(xn, wq).view(T, H, hd), F.linear(xn, wk).view(T, H, hd), table[rows, cols])
    v_want = F.linear(xn, wv)
    rope = torch.view_as_real(table).reshape(side * side, hd // 2, 2).contiguous().to(DEV)
    q = torch.empty(T, dim, dtype=torch.bfloat16, device=DEV)
    k, v = torch.empty_like(q), torch.empty_like(q)
    ws = _ws(T)
    wqkv = torch.cat([wq, wk, wv]).to(DEV)
    want = "skinny_linear_kernel" if T <= 4 else ("gemm_streamk_kernel" if T <= 128 else "gemm_wgmma_kernel")
    assert_launched(lambda: _abi.attn_qkv(x.to(DEV), nw.to(DEV), wqkv, rope, pos.to(DEV), q, k, v, None, None, None, H, H, hd, 1e-5, ws),
                    want, r"gemm|skinny", 1)
    # near-zero outputs: the fp32 sums over K = 1024 cancel, so a different summation order moves them by many of their own ulps;
    # the rotation can cancel too.  Hence an absolute floor of 2 ulps at the scale of the largest value (as test_gpu_ops does for q/k)
    for got, want_t, what in ((q, q_want.reshape(T, dim), "q"), (k, k_want.reshape(T, dim), "k"), (v, v_want, "v")):
        assert_bf16_close(got, want_t, atol=2 * 2 ** -8 * want_t.abs().max().item(), what=what)


def test_hd64_rejects_causal_modes_and_other_head_dims():
    q = torch.zeros(4, 64, dtype=torch.bfloat16, device=DEV)
    qs = torch.tensor([0, 4], dtype=torch.int32, device=DEV)
    with pytest.raises(_abi.Mb200Error, match="causal=0"):
        _abi.attn_prefill(q, q, q, q, q, qs, qs, q, 1, 4, 4, 1, 1, 64, causal=True)
    with pytest.raises(_abi.Mb200Error, match="64 or 128"):
        _abi.attn_prefill(q, q, q, None, None, None, None, q, 1, 4, 0, 2, 2, 32, causal=False)


# ----------------------------------------------------------------------------- head_dim-64 attention: visible set, exact
@pytest.mark.parametrize("T", VIS_T)
def test_hd64_attention_visible_set_exact(T):
    H = H_VIS
    q = torch.zeros(T, H * 64, dtype=torch.bfloat16, device=DEV)
    k = torch.randn(T, H * 64, device=DEV).to(torch.bfloat16)
    j = torch.arange(T, device=DEV)[:, None, None]
    h = torch.arange(H, device=DEV)[None, :, None]
    d = torch.arange(64, device=DEV)[None, None, :]
    v = ((((j + h) % 63 == d) & (d < 63)) | ((d == 63) & (j >= 63))).to(torch.bfloat16).reshape(T, H * 64)
    out = torch.full((T + 3, H * 64), 7.0, dtype=torch.bfloat16, device=DEV)  # rows >= T must stay untouched
    assert_launched(lambda: _abi.attn_prefill(q, k, v, None, None, None, None, out, 1, T, 0, H, H, 64, causal=False),
                    r"^attn_full_hd64_wgmma_kernel$", r"attn", 1)
    got = out[:T].double().cpu().numpy().reshape(T, H, 64)
    want = visible_expected(T)
    for t in sorted(set([0, T - 1, T // 2] + list(range(min(T, 130))))):
        assert visible_matches(got[t], want), f"T={T} query {t}"
    assert torch.all(out[T:] == 7.0)


@pytest.mark.parametrize("T,spread", [(1, 1.0), (129, 8.0), (1000, 30.0), (4097, 60.0)])
def test_hd64_attention_softmax_weighting_bound(T, spread):
    H = 4
    g = torch.Generator().manual_seed(T)
    q = (torch.randn(T, H, 64, generator=g) * (spread / 8) ** 0.5).to(torch.bfloat16)
    k = (torch.randn(T, H, 64, generator=g) * (spread / 8) ** 0.5).to(torch.bfloat16)
    k[T // 2] *= 3  # a dominant key mid-sequence and one in the last partial tile
    k[T - 1] *= 2
    v = torch.randn(T, H, 64, generator=g).to(torch.bfloat16)
    out = torch.empty(T, H * 64, dtype=torch.bfloat16, device=DEV)
    _abi.attn_prefill(q.reshape(T, -1).to(DEV), k.reshape(T, -1).to(DEV), v.reshape(T, -1).to(DEV), None, None, None, None, out, 1, T, 0, H, H,
                      64, causal=False)
    qd, kd, vd = q.double(), k.double(), v.double()
    s = torch.einsum("thd,jhd->htj", qd, kd) * 64 ** -0.5
    p = torch.softmax(s, dim=-1)
    want = torch.einsum("htj,jhd->thd", p, vd)
    bound = 2.0 ** -8 * torch.einsum("htj,jhd->thd", p, vd.abs()) + 2.0 ** -8 * want.abs() + 1e-6
    err = (out.double().cpu().reshape(T, H, 64) - want).abs()
    assert bool((err <= bound).all()), float((err / bound).max())


# ----------------------------------------------------------------------------- encoder at the real layer shape
def _vision_model(p: dict, seed: int = 3) -> Transformer:
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 3
    m = Transformer.empty(args, DEV, torch.bfloat16)
    m.load_state_dict({k: v.to(DEV) for k, v in synth.synth_state_dict(p, seed).items()})
    return m.eval()


def _close_rel(got: torch.Tensor, want: torch.Tensor, rel_max: float, rel_mean: float, what: str) -> None:
    got, want = got.float().cpu(), want.float().cpu()
    assert torch.isfinite(got).all(), what
    diff = (got - want).abs()
    assert float(diff.max()) <= rel_max * float(want.abs().max()), (what, float(diff.max()), float(want.abs().max()))
    assert float(diff.mean()) <= rel_mean * float(want.abs().mean()), (what, float(diff.mean()), float(want.abs().mean()))


def test_encoder_real_shape_cross_image_attention_vs_oracle():
    """hidden 1024, 16 heads of 64, intermediate 4096, 2 layers; one 1024 x 1024 image (4096 patches) and two non-square images in
    ONE call: every patch attends to the patches of all three images (the reference drops its block-diagonal mask)."""
    p = synth.shape("tiny-pixtral")
    p["vision_encoder"] = dict(p["vision_encoder"], image_size=1024)
    m = _vision_model(p)
    imgs = [synth.synth_image(3, 1024, 1024, 1), synth.synth_image(3, 200, 330, 2), synth.synth_image(3, 90, 500, 3)]
    names = launched_kernels(lambda: m.vision_encoder([i.to(DEV) for i in imgs]))
    assert names.count("attn_full_hd64_wgmma_kernel") == 2 and names.count("patchify_kernel") == 3
    with torch.inference_mode():
        got = m.vision_encoder([i.to(DEV) for i in imgs])
        want = V.encoder_forward(imgs, synth.synth_state_dict(p, 3), p["vision_encoder"])
    assert got.shape == (4096 + 12 * 20 + 5 * 31, 1024)
    _close_rel(got, want, 2 ** -4, 2 ** -7, "encoder")
    # the cross-image quirk is visible: encoding the small images alone gives different features
    with torch.inference_mode():
        alone = m.vision_encoder([i.to(DEV) for i in imgs[1:]])
    assert not torch.allclose(alone.float(), got[4096:].float(), atol=1e-2)


# ----------------------------------------------------------------------------- merger, adapter, splice
@pytest.mark.parametrize("name", list(VISION_CASES))
def test_projection_and_splice_vs_oracle(name):
    """pixtral: adapter with bias; pixtral_patch_merger: pre-projector norm + 2x2 merger + adapter without bias; two_images: two
    images of different sizes in one prompt and none in the other."""
    p = case_params(name)
    m = _vision_model(p)
    prompts = VISION_CASES[name][2]
    imgs = [torch.tensor(im, dtype=torch.bfloat16) for ims in case_images(name) for im in ims]
    ids = torch.tensor(sum(prompts, []))
    names = launched_kernels(lambda: m.embed_vision_language_features(ids.to(DEV), [i.to(DEV) for i in imgs]))
    assert names.count("splice_scan_kernel") == 1 and names.count("splice_gather_kernel") == 1
    assert names.count("patch_merge_kernel") == (len(imgs) if m.patch_merger is not None else 0)
    layers = p["vision_encoder"]["num_hidden_layers"]  # conv + 4 per block (qkv, wo, gate/up, down) + merger + 2 adapter
    assert sum("gemm" in n or "skinny" in n for n in names) == 1 + 4 * layers + (1 if m.patch_merger is not None else 0) + 2
    with torch.inference_mode():
        got = m.embed_vision_language_features(ids.to(DEV), [i.to(DEV) for i in imgs])
        want = V.embed(ids, imgs, synth.synth_state_dict(p, 3), p["vision_encoder"])
    text = ids != p["vision_encoder"]["image_token_id"]
    assert torch.equal(got[text.to(DEV)].cpu(), want[text])  # text rows are copies
    # conv, ln_pre, the blocks, the optional norm, the merger and both adapter GEMMs each round to bf16: about one ulp on average
    _close_rel(got[~text.to(DEV)], want[~text], 2 ** -5, 2 ** -6, "image rows")
    with pytest.raises(AssertionError):  # one image token too many
        m.embed_vision_language_features(torch.cat([ids, ids[~text][:1]]).to(DEV), [i.to(DEV) for i in imgs])


def test_text_model_ignores_images_and_empty_list_is_text():
    p = synth.shape("pixtral-ref-test")
    m = _vision_model(p)
    ids = torch.tensor([1, 12, 13, 14, 15], device=DEV)
    a = m.forward(ids, [5])
    b = m.forward(ids, [5], images=[])
    assert torch.equal(a, b)
    t = _vision_model(synth.shape("ref-test"))
    assert torch.equal(t.forward(ids, [5]), t.forward(ids, [5], images=[torch.zeros(3, 4, 4, dtype=torch.bfloat16, device=DEV)]))


# ----------------------------------------------------------------------------- model level
@pytest.mark.parametrize("name", list(VISION_CASES))
def test_generate_with_images_vs_oracle_and_self_consistent(name):
    p = case_params(name)
    m = _vision_model(p)
    prompts = VISION_CASES[name][2]
    images = case_images(name)
    toks, lps = mi.generate(prompts, m, images=images, max_tokens=7, temperature=0.0)
    assert len(toks) == len(prompts) and all(len(t) == 7 for t in toks)
    full = [pr + t for pr, t in zip(prompts, toks)]
    # teacher-forced oracle on the GPU's tokens: log-probabilities of every prompt and generated token
    imgs = [torch.tensor(im, dtype=torch.bfloat16) for ims in images for im in ims]
    om = V.MultimodalOracle(R.OracleTransformer(oracle_args(p, len(prompts)), synth.synth_state_dict(p, 3)), p["vision_encoder"], imgs)
    _, o_lp = R.generate(full, om, max_tokens=0)
    worst = max(abs(a - b) for x, y in zip(lps, o_lp) for a, b in zip(x, y))
    assert worst <= LOGPROB_TOL, worst
    # the reference's own property (tests/test_generate.py:104-116): re-prefill prompt + output with max_tokens=0
    gen2, lps2 = mi.generate(full, m, images=images, max_tokens=0, temperature=0.0)
    assert gen2 == []
    worst2 = max(abs(a - b) for x, y in zip(lps, lps2) for a, b in zip(x, y))
    assert worst2 <= LOGPROB_TOL, worst2
