"""GPU parity, op by op: each C-ABI entry point against the oracle restatement on the same seeded inputs.

Tolerance model (written once here): every output is a bf16 value that the reference produces by rounding an
fp32 intermediate.  A different fp32 summation order moves that intermediate by ~1e-6 relative, which flips the
bf16 rounding of a small fraction of elements by ONE ulp.  So: <= 1 bf16 ulp everywhere and >= 97 % bit-identical
for GEMV/GEMM/elementwise ops.  Outputs that COMBINE two already-rounded bf16 operands (RoPE: a*c - b*d; residual:
x + y; SiLU*mul: s*b) inherit the operands' one-ulp flips: their error is one ulp of the LARGER operand, which after
cancellation can be many ulps of the (small) result -- those get an absolute tolerance of 2 ulps of the operand scale.
Attention outputs get `atol` for near-zero values, and the prefill kernel 2 ulp because P is rounded to bf16 before the
PV tensor-core product (as in any tensor-core attention).
"""

import pytest
import torch
import torch.nn.functional as F

from mistral_inference_b200 import _abi
from mistral_inference_b200.rope import precompute_freqs_cis
from oracle import restatement as R
from oracle.attention_ref import attend_block, local_causal_allowed

from .util import assert_bf16_close, assert_launched

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


@pytest.fixture(scope="module")
def ws():
    return _abi.Workspace(_abi.workspace_bytes(512, 4096, 32, 8, 128, 14336, 32000, 4), torch.device(DEV))


@pytest.fixture(scope="module")
def rope():
    table = precompute_freqs_cis(128, 8192, 1e6)
    return table, torch.view_as_real(table).contiguous().to(DEV)


@pytest.mark.parametrize("T,dim", [(1, 256), (5, 4096), (33, 5120), (2, 6144)])
def test_rmsnorm(T, dim):
    x, w = rnd(T, dim, seed=1, scale=2.0), (1 + 0.2 * rnd(dim, seed=2).float()).to(torch.bfloat16)
    got = _abi.rmsnorm(x.to(DEV), w.to(DEV), 1e-5)
    assert_bf16_close(got, R.rms_norm(x, w, 1e-5), max_ulp=1, min_exact=0.995, what="rmsnorm")


@pytest.mark.parametrize("T", [1, 2, 3, 4, 5, 37, 130])
@pytest.mark.parametrize("dim,H,KV", [(256, 4, 2), (4096, 32, 8)])
def test_attn_qkv(T, dim, H, KV, ws, rope):
    if dim == 4096 and T not in (1, 4, 130):
        pytest.skip("big shape: representative T only")
    hd = 128
    x = rnd(T, dim, seed=3)
    nw = (1 + 0.2 * rnd(dim, seed=4).float()).to(torch.bfloat16)
    wq, wk, wv = rnd(H * hd, dim, seed=5, scale=dim ** -0.5), rnd(KV * hd, dim, seed=6, scale=dim ** -0.5), rnd(KV * hd, dim, seed=7, scale=dim ** -0.5)
    positions = torch.arange(T, dtype=torch.int32) * 37 % 8000
    table, table_dev = rope
    # oracle: norm -> three linears -> rope (transformer_layers.py:165,66-70)
    xn = R.rms_norm(x, nw, 1e-5)
    q_ref, k_ref = R.apply_rope(F.linear(xn, wq).view(T, H, hd), F.linear(xn, wk).view(T, KV, hd), table[positions.long()])
    v_ref = F.linear(xn, wv)
    wqkv = torch.cat([wq, wk, wv], 0).to(DEV)
    q = torch.empty(T, H * hd, dtype=torch.bfloat16, device=DEV)
    k = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
    v = torch.empty_like(k)
    n_rows = 64
    ck = torch.full((n_rows, KV, hd), float("nan"), dtype=torch.bfloat16, device=DEV)
    cv = torch.full_like(ck, float("nan"))
    rows = torch.tensor([(5 * t) % n_rows if t % 3 else -1 for t in range(T)], dtype=torch.int32)
    if len(set(r for r in rows.tolist() if r >= 0)) < sum(r >= 0 for r in rows.tolist()):
        rows = torch.tensor([t if t % 3 and t < n_rows else -1 for t in range(T)], dtype=torch.int32)
    _abi.attn_qkv(x.to(DEV), nw.to(DEV), wqkv, table_dev, positions.to(DEV), q, k, v, ck, cv, rows.to(DEV), H, KV, hd, 1e-5, ws)
    torch.cuda.synchronize()
    assert_bf16_close(q, q_ref.reshape(T, -1), atol=2 * 2 ** -8 * q_ref.abs().max().item(), what="q")
    assert_bf16_close(k, k_ref.reshape(T, -1), atol=2 * 2 ** -8 * k_ref.abs().max().item(), what="k")
    assert_bf16_close(v, v_ref, what="v")
    # scatter: cached rows hold exactly what was written to k/v, everything else untouched (still NaN)
    for t, r in enumerate(rows.tolist()):
        if r >= 0:
            assert torch.equal(ck[r].reshape(-1), k[t]) and torch.equal(cv[r].reshape(-1), v[t])
    untouched = torch.ones(n_rows, dtype=torch.bool)
    untouched[[r for r in rows.tolist() if r >= 0]] = False
    assert torch.isnan(ck[untouched.to(DEV)].float()).all()


@pytest.mark.parametrize("T", [1, 3, 4, 7, 130, 300])
@pytest.mark.parametrize("N,K", [(256, 512), (4096, 4096), (4096, 14336), (8, 256)])
def test_linear_residual(T, N, K, ws):
    if K >= 4096 and T not in (1, 4, 130):
        pytest.skip("big shape: representative T only")
    x, w, res = rnd(T, K, seed=8), rnd(N, K, seed=9, scale=K ** -0.5), rnd(T, N, seed=10)
    out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
    _abi.linear_residual(x.to(DEV), w.to(DEV), res.to(DEV), out, ws)
    assert_bf16_close(out, res + F.linear(x, w), atol=2 * 2 ** -8 * res.abs().max().item(), what="linear+residual")
    _abi.linear_residual(x.to(DEV), w.to(DEV), None, out, ws)
    assert_bf16_close(out, F.linear(x, w), what="linear")


@pytest.mark.parametrize("T", [1, 2, 4, 6, 129])
@pytest.mark.parametrize("dim,hid", [(256, 512), (4096, 14336)])
@pytest.mark.parametrize("with_norm", [True, False])
def test_ffn_gateup(T, dim, hid, with_norm, ws):
    if dim == 4096 and T not in (1, 129):
        pytest.skip("big shape: representative T only")
    x = rnd(T, dim, seed=11)
    nw = (1 + 0.2 * rnd(dim, seed=12).float()).to(torch.bfloat16)
    w1, w3 = rnd(hid, dim, seed=13, scale=dim ** -0.5), rnd(hid, dim, seed=14, scale=dim ** -0.5)
    xin = R.rms_norm(x, nw, 1e-5) if with_norm else x
    want = F.silu(F.linear(xin, w1)) * F.linear(xin, w3)
    w13 = torch.stack([w1, w3], 1).reshape(2 * hid, dim).to(DEV)
    g = torch.empty(T, hid, dtype=torch.bfloat16, device=DEV)
    _abi.ffn_gateup(x.to(DEV), nw.to(DEV) if with_norm else None, w13, g, 1e-5, ws)
    # silu goes through exp(): CUDA expf vs the CPU's vectorised exp differ in the last fp32 bit now and then
    assert_bf16_close(g, want, max_ulp=4, min_exact=0.96, what="ffn gate/up")  # 3 chained roundings: one-ulp flips of a and b compound in s*b


@pytest.mark.parametrize("T", [1, 4, 9])
def test_lm_head(T, ws):
    dim, V = 512, 32000
    x = rnd(T, dim, seed=15)
    nw = (1 + 0.2 * rnd(dim, seed=16).float()).to(torch.bfloat16)
    wo = rnd(V, dim, seed=17, scale=dim ** -0.5)
    logits = torch.empty(T, V, dtype=torch.float32, device=DEV)
    _abi.lm_head(x.to(DEV), nw.to(DEV), wo.to(DEV), logits, 1e-5, ws)
    assert_bf16_close(logits, F.linear(R.rms_norm(x, nw, 1e-5), wo).float(), what="lm head")


def test_gemm_against_cuda_core_gemm(ws):
    """Tensor-core GEMM vs the naive CUDA-core GEMM on the GPU at a size the CPU oracle would take long for."""
    T, N, K = 515, 1536, 4096
    a, w = rnd(T, K, seed=18).to(DEV), rnd(N, K, seed=19, scale=K ** -0.5).to(DEV)
    out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
    _abi.linear_residual(a, w, None, out, ws)
    assert_bf16_close(out, _abi.test_gemm_naive(a, w).to(torch.bfloat16), what="gemm vs naive")


@pytest.mark.parametrize("bn", ["128", "192", "256"])
def test_gemm_cluster_pair_matches_single_cta(ws, bn, monkeypatch):
    """T >= 512 runs the 2-CTA cluster kernel (W tile multicast to the pair); 128-row slices of the same input run the
    single-CTA kernel.  Rows are independent and accumulate in the same k order, so the two must agree bit for bit --
    through the residual and the SiLU*mul epilogues, with a ragged last tile and an odd number of row tiles, for both tile
    widths (the launcher picks the width per shape; MB200_GEMM_BN pins it here)."""
    monkeypatch.setenv("MB200_GEMM_BN", bn)
    monkeypatch.setenv("MB200_STREAMK", "0")  # the 128-row slices below must take the single-CTA wgmma kernel, not the stream-K one
    T, dim, hid = 700, 1536, 1536  # N = 1536 / 3072: multiples of all three tile widths
    x, res = rnd(T, hid, seed=30).to(DEV), rnd(T, dim, seed=31).to(DEV)
    w2 = rnd(dim, hid, seed=32, scale=hid ** -0.5).to(DEV)
    out = torch.empty(T, dim, dtype=torch.bfloat16, device=DEV)
    _abi.linear_residual(x, w2, res, out, ws)
    xin = rnd(T, dim, seed=33).to(DEV)
    w13 = rnd(2 * hid, dim, seed=34, scale=dim ** -0.5).to(DEV)
    g = torch.empty(T, hid, dtype=torch.bfloat16, device=DEV)
    _abi.ffn_gateup(xin, None, w13, g, 1e-5, ws)
    # against the CUDA-core GEMM (independent of every tensor-core code path)
    assert_bf16_close(out, (res.float() + _abi.test_gemm_naive(x, w2).to(torch.bfloat16).float()).to(torch.bfloat16),
                      atol=2 * 2 ** -8 * res.abs().max().item(), what="cluster gemm + residual vs naive")
    for r0 in range(0, T, 128):
        n = min(128, T - r0)
        if n < 128:
            r0 = T - 128  # the single-CTA wgmma kernel needs T >= 128
            n = 128
        o1 = torch.empty(n, dim, dtype=torch.bfloat16, device=DEV)
        _abi.linear_residual(x[r0:r0 + n].contiguous(), w2, res[r0:r0 + n].contiguous(), o1, ws)
        assert torch.equal(o1, out[r0:r0 + n]), f"residual epilogue rows {r0}.."
        g1 = torch.empty(n, hid, dtype=torch.bfloat16, device=DEV)
        _abi.ffn_gateup(xin[r0:r0 + n].contiguous(), None, w13, g1, 1e-5, ws)
        assert torch.equal(g1, g[r0:r0 + n]), f"gate/up epilogue rows {r0}.."
    # the other tile widths and the single-CTA kernel at full T give the same bits
    out2 = torch.empty_like(out)
    for other in ("128", "192", "256"):
        monkeypatch.setenv("MB200_GEMM_BN", other)
        _abi.linear_residual(x, w2, res, out2, ws)
        assert torch.equal(out2, out), f"tile widths {bn} and {other} disagree"
    monkeypatch.setenv("MB200_GEMM_CLUSTER", "0")
    _abi.linear_residual(x, w2, res, out2, ws)
    assert torch.equal(out2, out), "cluster and single-CTA kernels disagree"


def test_qkv_rope_epilogue_same_bits_for_every_tile_width(ws, rope, monkeypatch):
    """Fused QKV + RoPE + ring scatter at Mistral-7B width (N = 6144 = 24 x 256 = 32 x 192 = 48 x 128) through the 2-CTA
    cluster kernel: the three tile widths must produce identical q / k / v and identical cache rows."""
    T, dim, H, KV, hd = 640, 4096, 32, 8, 128
    x = rnd(T, dim, seed=40).to(DEV)
    nw = (1 + 0.2 * rnd(dim, seed=41).float()).to(torch.bfloat16).to(DEV)
    wqkv = rnd((H + 2 * KV) * hd, dim, seed=42, scale=dim ** -0.5).to(DEV)
    positions = (torch.arange(T, dtype=torch.int32) * 3 % 8000).to(DEV)
    rows = torch.tensor([t if t % 5 else -1 for t in range(T)], dtype=torch.int32).to(DEV)
    _, table_dev = rope
    outs = {}
    for bn in ("256", "192", "128"):
        monkeypatch.setenv("MB200_GEMM_BN", bn)
        q = torch.empty(T, H * hd, dtype=torch.bfloat16, device=DEV)
        k = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
        v = torch.empty_like(k)
        ck = torch.zeros(T, KV, hd, dtype=torch.bfloat16, device=DEV)
        cv = torch.zeros_like(ck)
        _abi.attn_qkv(x, nw, wqkv, table_dev, positions, q, k, v, ck, cv, rows, H, KV, hd, 1e-5, ws)
        torch.cuda.synchronize()
        outs[bn] = (q, k, v, ck, cv)
    for bn in ("192", "128"):
        for a, b, what in zip(outs["256"], outs[bn], ("q", "k", "v", "cache_k", "cache_v")):
            assert torch.equal(a, b), f"{what}: tile width {bn} differs from 256"
    q, k, v, ck, cv = outs["192"]
    keep = rows >= 0
    assert torch.equal(ck[rows[keep].long()].reshape(-1, KV * hd), k[keep]) and torch.equal(cv[rows[keep].long()].reshape(-1, KV * hd), v[keep])


def _oracle_decode(q, ck, cv, kv_len, H, KV):
    rep = H // KV
    outs = []
    for b in range(q.shape[0]):
        n = int(kv_len[b])
        keys, vals = ck[b, :n].repeat_interleave(rep, dim=1), cv[b, :n].repeat_interleave(rep, dim=1)
        outs.append(attend_block(q[b].view(1, H, 128), keys, vals, local_causal_allowed(1, n, None)))
    return torch.cat(outs, 0).view(q.shape[0], H * 128)


@pytest.mark.parametrize("B,W,lens,S", [
    (1, 64, [1], 1), (1, 64, [5], 3), (3, 100, [100, 37, 1], 4), (2, 4096, [4096, 1000], 37), (1, 4096, [4096], 18),
    (4, 300, [300, 299, 17, 150], 9),
])
@pytest.mark.parametrize("H,KV", [(32, 8), (4, 2), (48, 8)])
@pytest.mark.parametrize("kernel", ["tma"])
def test_attn_decode(B, W, lens, S, H, KV, kernel, ws):
    """The decode attention kernel: TMA-staged K/V tiles, tensor-core scores."""
    if (H, KV) != (32, 8) and W == 4096:
        pytest.skip("long ring: 7B head layout only")
    q = rnd(B, H * 128, seed=20)
    ck, cv = rnd(B + 1, W, KV, 128, seed=21), rnd(B + 1, W, KV, 128, seed=22)  # max_batch > B like tests/test_generate.py:212
    kv_len = torch.tensor(lens, dtype=torch.int32)
    want = _oracle_decode(q, ck, cv, kv_len, H, KV)
    ck_d, cv_d = ck.to(DEV), cv.to(DEV)
    for b, n in enumerate(lens):  # slots >= kv_len are uninitialised memory in the reference (cache.py:166): poison them
        ck_d[b, n:] = float("nan")
        cv_d[b, n:] = float("nan")
    out = torch.empty(B, H * 128, dtype=torch.bfloat16, device=DEV)
    for _ in range(2):  # twice: the split counters must self-reset
        out.zero_()
        _abi.attn_decode(q.to(DEV), ck_d, cv_d, kv_len.to(DEV), out, H, KV, 128, S, ws)
        # P is rounded to bf16 for the tensor-core PV product, like the prefill kernels (and any tensor-core attention)
        assert_bf16_close(out, want, max_ulp=2, min_exact=0.5, atol=4e-3, what="decode attention (tma)")


def _oracle_prefill(q, k_new, v_new, ck, cv, seqlens, seqpos, W, H, KV):
    rep = H // KV
    outs, o = [], 0
    for b, (s, p) in enumerate(zip(seqlens, seqpos)):
        old_k, old_v = R._unrotate(ck[b], p), R._unrotate(cv[b], p)
        keys = torch.cat([old_k, k_new[o:o + s].view(s, KV, 128)], 0).repeat_interleave(rep, dim=1)
        vals = torch.cat([old_v, v_new[o:o + s].view(s, KV, 128)], 0).repeat_interleave(rep, dim=1)
        outs.append(attend_block(q[o:o + s].view(s, H, 128), keys, vals, local_causal_allowed(s, keys.shape[0], W)))
        o += s
    return torch.cat(outs, 0).view(-1, H * 128)


@pytest.mark.parametrize("seqlens,seqpos,W", [
    ([7, 3, 3, 3], [0, 0, 0, 0], 64),        # first prefill, ragged (tests/test_generate.py:39)
    ([70, 130], [0, 0], 256),                # several query/key tiles
    ([70, 130], [0, 0], 33),                 # window smaller than the chunk
    ([5, 5], [5, 5], 4),                     # chunked prefill, ring already wrapped (W < seen)
    ([65, 3], [100, 250], 128),              # chunk on top of a wrapped ring, ragged
    ([1, 9], [40, 3], 16),                   # a one-token sequence inside a prefill batch
    ([300], [0], 4096),
    ([700, 260], [0, 0], 4096),              # wgmma kernel: several 128-key tiles, ragged
    ([700, 260], [0, 0], 200),               # ... with a window smaller than the sequence
])
@pytest.mark.parametrize("H,KV", [(4, 2), (32, 8)])
def test_attn_prefill(seqlens, seqpos, W, H, KV):
    if (H, KV) == (32, 8) and sum(seqlens) > 150 and sum(seqlens) < 900:
        pytest.skip("big head count: small and wgmma-sized cases only")
    T, B = sum(seqlens), len(seqlens)
    q, k_new, v_new = rnd(T, H * 128, seed=23), rnd(T, KV * 128, seed=24), rnd(T, KV * 128, seed=25)
    ck, cv = torch.zeros(B, W, KV, 128, dtype=torch.bfloat16), torch.zeros(B, W, KV, 128, dtype=torch.bfloat16)
    valid = torch.zeros(B, W, dtype=torch.bool)
    g = torch.Generator().manual_seed(26)
    for b, p in enumerate(seqpos):  # fill the ring as if positions [0, p) had been cached
        for pos in range(max(0, p - W), p):
            ck[b, pos % W] = torch.randn(KV, 128, generator=g).to(torch.bfloat16)
            cv[b, pos % W] = torch.randn(KV, 128, generator=g).to(torch.bfloat16)
            valid[b, pos % W] = True
    want = _oracle_prefill(q, k_new, v_new, ck, cv, seqlens, seqpos, W, H, KV)
    ck_d, cv_d = ck.to(DEV), cv.to(DEV)
    ck_d[~valid.to(DEV)] = float("nan")  # never-written slots must not be read
    cv_d[~valid.to(DEV)] = float("nan")
    q_start = torch.tensor([0] + torch.tensor(seqlens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    out = torch.zeros(T, H * 128, dtype=torch.bfloat16, device=DEV)
    _abi.attn_prefill(q.to(DEV), k_new.to(DEV), v_new.to(DEV), ck_d, cv_d, q_start, torch.tensor(seqpos, dtype=torch.int32, device=DEV), out,
                      B, max(seqlens), W, H, KV, 128, causal=True, first_prefill=all(x == 0 for x in seqpos))
    assert_bf16_close(out, want, max_ulp=2, min_exact=0.5, atol=4e-3, what="prefill attention")


def test_attn_prefill_no_cache_unmasked():
    """cache=None: every query sees every key of the flattened batch (SURVEY.md Appendix E-2)."""
    T, H, KV = 77, 4, 2
    q, k, v = rnd(T, H * 128, seed=27), rnd(T, KV * 128, seed=28), rnd(T, KV * 128, seed=29)
    want = attend_block(q.view(T, H, 128), k.view(T, KV, 128).repeat_interleave(2, 1), v.view(T, KV, 128).repeat_interleave(2, 1), None)
    out = torch.zeros(T, H * 128, dtype=torch.bfloat16, device=DEV)
    _abi.attn_prefill(q.to(DEV), k.to(DEV), v.to(DEV), None, None, None, None, out, 1, T, 0, H, KV, 128, causal=False)
    assert_bf16_close(out, want.reshape(T, -1), max_ulp=2, min_exact=0.5, atol=4e-3, what="unmasked attention")


def test_kv_ring_write():
    T, KV = 9, 2
    k, v = rnd(T, KV * 128, seed=30).to(DEV), rnd(T, KV * 128, seed=31).to(DEV)
    ck = torch.zeros(16, KV, 128, dtype=torch.bfloat16, device=DEV)
    cv = torch.zeros_like(ck)
    rows = torch.tensor([-1, -1, 3, 4, 5, -1, 15, 0, 1], dtype=torch.int32, device=DEV)
    _abi.kv_ring_write(k, v, ck, cv, rows, KV, 128)
    for t, r in enumerate(rows.tolist()):
        if r >= 0:
            assert torch.equal(ck[r].reshape(-1), k[t]) and torch.equal(cv[r].reshape(-1), v[t])
    assert ck[[2, 6, 7]].abs().sum() == 0


# ----------------------------------------------------------------------------- small-batch (decode) weight-streaming wgmma GEMMs
@pytest.mark.parametrize("T", [5, 16, 32, 33, 64, 65, 127])
@pytest.mark.parametrize("N,K", [(4096, 4096),      # 7B wo / down width: 32-wide tiles (128 CTAs)
                                 (6144, 4096),      # 7B fused QKV: 64-wide tiles
                                 (5120, 14336),     # Nemo down projection, K = 14336: 224 k-blocks through the deep ring
                                 (1024, 6144)])     # fewer tiles than half the SMs: narrow tiles
def test_small_batch_gemm_vs_oracle(T, N, K, ws):
    """5 <= T <= 128 with N a multiple of 128 runs gemm_streamk_kernel (32/64/128-row A boxes by T; the MMA's upper rows read past
    the box; rows >= T are never stored): plain store and residual epilogues against the CPU oracle."""
    if K == 14336 and T not in (16, 33, 127):
        pytest.skip("long K: representative T only")
    ta = 32 if T <= 32 else 64 if T <= 64 else 128
    _small_batch_gemm_vs_oracle(T, N, K, ws, rf"gemm_streamk_kernel<\d+, {ta}>")


def _small_batch_gemm_vs_oracle(T, N, K, ws, kernel):
    x, w, res = rnd(T, K, seed=50), rnd(N, K, seed=51, scale=K ** -0.5), rnd(T, N, seed=52)
    out = torch.full((T + 3, N), float("nan"), dtype=torch.bfloat16, device=DEV)  # 3 guard rows: rows >= T must stay untouched
    out2 = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)

    def launches():
        _abi.linear_residual(x.to(DEV), w.to(DEV), res.to(DEV), out[:T], ws)
        _abi.linear_residual(x.to(DEV), w.to(DEV), None, out2, ws)

    assert_launched(launches, kernel, r"gemm_\w+_kernel", 2)
    assert_bf16_close(out[:T], res + F.linear(x, w), atol=2 * 2 ** -8 * res.abs().max().item(), what="small-batch gemm + residual")
    assert torch.isnan(out[T:].float()).all(), "rows past T were written"
    assert_bf16_close(out2, F.linear(x, w), what="small-batch gemm")


@pytest.mark.parametrize("T", [5, 32, 33, 64, 65, 127])
@pytest.mark.parametrize("N,K,streamk", [(4096, 4096, "0"),   # stream-K switched off: 32-wide tiles
                                         (1024, 6144, "0"),   # fewer tiles than half the SMs
                                         (1056, 4096, None)])  # N % 128 != 0: the default routing takes the small-batch kernel
def test_small_batch_wgmma_gemm_vs_oracle(T, N, K, streamk, ws, monkeypatch):
    """5 <= T < 128 off the stream-K path runs the small-batch gemm_wgmma_kernel with a 32-, 64- or 128-row A box (TA, the last
    template argument) chosen by T: plain store and residual epilogues against the CPU oracle."""
    if streamk is None:
        monkeypatch.delenv("MB200_STREAMK", raising=False)
    else:
        monkeypatch.setenv("MB200_STREAMK", streamk)
    ta = 32 if T <= 32 else 64 if T <= 64 else 128
    _small_batch_gemm_vs_oracle(T, N, K, ws, rf"gemm_wgmma_kernel<\d+, 1, \d+, {ta}>")


def test_small_batch_gemm_tile_widths_agree(ws, monkeypatch, rope):
    """All tile widths of the small-batch kernel give the same bits through the QKV+RoPE+ring-scatter and SiLU*mul epilogues."""
    monkeypatch.setenv("MB200_STREAMK", "0")  # the fallback for N not a multiple of 128: narrow tiles, one m tile
    T, dim, H, KV, hd, hid = 24, 1024, 8, 2, 128, 1024
    x = rnd(T, dim, seed=60).to(DEV)
    nw = (1 + 0.2 * rnd(dim, seed=61).float()).to(torch.bfloat16).to(DEV)
    wqkv = rnd((H + 2 * KV) * hd, dim, seed=62, scale=dim ** -0.5).to(DEV)
    w13 = rnd(2 * hid, dim, seed=63, scale=dim ** -0.5).to(DEV)
    positions = (torch.arange(T, dtype=torch.int32) * 7 % 8000).to(DEV)
    rows = torch.arange(T, dtype=torch.int32).to(DEV)
    _, table_dev = rope
    outs = {}
    for bn in ("32", "64", "128", "256"):
        monkeypatch.setenv("MB200_GEMM_BN", bn)
        q = torch.empty(T, H * hd, dtype=torch.bfloat16, device=DEV)
        k = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
        v = torch.empty_like(k)
        ck = torch.zeros(T, KV, hd, dtype=torch.bfloat16, device=DEV)
        cv = torch.zeros_like(ck)
        _abi.attn_qkv(x, nw, wqkv, table_dev, positions, q, k, v, ck, cv, rows, H, KV, hd, 1e-5, ws)
        g = torch.empty(T, hid, dtype=torch.bfloat16, device=DEV)
        _abi.ffn_gateup(x, nw, w13, g, 1e-5, ws)
        torch.cuda.synchronize()
        outs[bn] = (q, k, v, ck, cv, g)
    for bn in ("64", "128", "256"):
        for a, b, what in zip(outs["32"], outs[bn], ("q", "k", "v", "cache_k", "cache_v", "g")):
            assert torch.equal(a, b), f"{what}: tile width {bn} differs from 32"


# ----------------------------------------------------------------------------- device-side step state, token selection, log-probs
def test_decode_meta_matches_host_metadata():
    """mb200_decode_meta == BufferCache.build_metadata_host for one-token steps (cache.py:197-263), and it advances the positions."""
    from mistral_inference_b200.cache import BufferCache

    B, L = 5, 4
    cache = BufferCache(L, B, 64, 2, 128, sliding_window=[7, None])
    cache._kv_seqlens_host = [3, 7, 8, 20, 63]
    windows = sorted(set(cache.cache_sizes))
    seqpos = torch.tensor(cache._kv_seqlens_host, dtype=torch.int32, device=DEV)
    meta = torch.zeros(3 * B + 1 + 2 * B * len(windows), dtype=torch.int32, device=DEV)
    for _ in range(3):
        host, layout = cache.build_metadata_host([1] * B)
        assert layout["windows"] == windows
        _abi.decode_meta(seqpos, meta, windows)
        assert meta.cpu().tolist() == host.tolist()
        cache.update_seqlens([1] * B)
        assert seqpos.cpu().tolist() == cache._kv_seqlens_host


@pytest.mark.parametrize("T,V", [(1, 32000), (5, 512), (33, 131072)])
def test_argmax_and_logprob_gather(T, V):
    g = torch.Generator().manual_seed(70)
    logits = (torch.randn(T, V, generator=g) * 2).to(torch.bfloat16).float()  # bf16-valued like the lm head's output: many exact ties
    tgt = torch.randint(0, V, (T,), generator=g)
    tgt[T // 2] = -1
    got = _abi.argmax_rows(logits.to(DEV))
    assert torch.equal(got.cpu(), logits.argmax(-1)), "argmax (first index on ties)"
    out = torch.full((T,), 123.0, device=DEV)
    _abi.logprob_gather(logits.to(DEV), tgt.to(DEV), out=out)
    want = torch.log_softmax(logits, -1)
    for t in range(T):
        if tgt[t] < 0:
            assert out[t].item() == 123.0
        else:
            assert abs(out[t].item() - want[t, tgt[t]].item()) <= 2e-5, t


def _ref_top_p_keep(probs: torch.Tensor, p: float) -> torch.Tensor:
    """The kept set of the reference's sample_top_p (generate.py:161-170): sorted descending, keep while (cumsum - prob) <= p."""
    ps, idx = torch.sort(probs, dim=-1, descending=True)
    keep_sorted = ~((torch.cumsum(ps, -1) - ps) > p)
    keep = torch.zeros_like(keep_sorted)
    keep.scatter_(-1, idx, keep_sorted)
    return keep


@pytest.mark.parametrize("T,V,temp", [(4, 512, 0.7), (3, 32000, 1.0), (2, 131072, 0.3)])
def test_sample_top_p_kept_set_and_distribution(T, V, temp):
    g = torch.Generator().manual_seed(71)
    logits = torch.randn(T, V, generator=g) * 3
    probs = torch.softmax(logits / temp, -1)
    keep = _ref_top_p_keep(probs, 0.8)
    dev_logits = logits.to(DEV)
    # (a) every draw lies in the reference's kept set, for uniforms spanning [0, 1)
    us = torch.tensor([0.0, 1e-7, 0.25, 0.5, 0.75, 0.999, 0.9999999])
    picks = []
    for u in us.tolist():
        tok = _abi.sample_top_p(dev_logits, torch.full((T,), u, device=DEV), temp, 0.8).cpu()
        picks.append(tok)
        for t in range(T):
            assert keep[t, tok[t]], (t, u, int(tok[t]))
    # (b) the draw is the inverse CDF of the renormalised kept distribution in index order
    for t in range(T):
        pk = torch.where(keep[t], probs[t], torch.zeros(())).double()
        cdf = torch.cumsum(pk / pk.sum(), 0)
        for u, tok in zip(us.tolist(), picks):
            i = int(tok[t])
            lo = cdf[i - 1].item() if i > 0 else 0.0
            assert lo - 1e-4 <= u <= cdf[i].item() + 1e-4, (t, u, i, lo, cdf[i].item())
    # (c) monotone in u (index order)
    for t in range(T):
        seq = [int(x[t]) for x in picks]
        assert seq == sorted(seq)


# ----------------------------------------------------------------------------- independent attention cross-check (xformers boundary)
def _flash_attn():
    try:
        from flash_attn import flash_attn_varlen_func
        return flash_attn_varlen_func
    except Exception as e:  # pragma: no cover
        pytest.skip(f"flash_attn not importable: {e}")


@pytest.mark.parametrize("seqlens,W", [([70, 130], 256), ([70, 130], 33), ([700, 260], 4096), ([700, 260], 200)])
def test_prefill_attention_vs_flash_attn(seqlens, W):
    """The xformers boundary is unpinned in the reference tree (dependency absent).  flash_attn 2.8 (a third implementation, the
    one xformers dispatches to on GPUs) with causal + sliding-window semantics cross-checks BOTH the oracle's attention
    (oracle/attention_ref.py) and the CUDA kernels: window (i - W, i] = flash_attn window_size (W - 1, 0)."""
    fa = _flash_attn()
    H, KV = 32, 8
    T, B = sum(seqlens), len(seqlens)
    q, k, v = rnd(T, H * 128, seed=80), rnd(T, KV * 128, seed=81), rnd(T, KV * 128, seed=82)
    cu = torch.tensor([0] + torch.tensor(seqlens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    try:
        ref = fa(q.to(DEV).view(T, H, 128), k.to(DEV).view(T, KV, 128), v.to(DEV).view(T, KV, 128), cu, cu, max(seqlens), max(seqlens),
                 causal=True, window_size=(W - 1, 0)).reshape(T, H * 128)
        torch.cuda.synchronize()
    except Exception as e:
        pytest.skip(f"flash_attn does not run on this GPU: {type(e).__name__}: {e}")
    ck = torch.zeros(B, W, KV, 128, dtype=torch.bfloat16)
    want = _oracle_prefill(q, k, v, ck, ck.clone(), seqlens, [0] * B, W, H, KV)
    assert_bf16_close(ref, want, max_ulp=2, min_exact=0.5, atol=4e-3, what="flash_attn vs oracle attention")
    out = torch.zeros(T, H * 128, dtype=torch.bfloat16, device=DEV)
    ck_d = torch.full((B, W, KV, 128), float("nan"), dtype=torch.bfloat16, device=DEV)
    _abi.attn_prefill(q.to(DEV), k.to(DEV), v.to(DEV), ck_d, ck_d.clone(), cu, torch.zeros(B, dtype=torch.int32, device=DEV), out, B, max(seqlens), W,
                      H, KV, 128, causal=True, first_prefill=True)
    assert_bf16_close(out, ref, max_ulp=2, min_exact=0.5, atol=4e-3, what="attn_prefill kernel vs flash_attn")


def test_decode_attention_vs_flash_attn(ws):
    fa = _flash_attn()
    B, W, H, KV = 3, 300, 32, 8
    lens = [300, 37, 150]
    q = rnd(B, H * 128, seed=83)
    ck, cv = rnd(B, W, KV, 128, seed=84), rnd(B, W, KV, 128, seed=85)
    kv_len = torch.tensor(lens, dtype=torch.int32)
    kk = torch.cat([ck[b, :n] for b, n in enumerate(lens)], 0).to(DEV)
    vv = torch.cat([cv[b, :n] for b, n in enumerate(lens)], 0).to(DEV)
    cu_q = torch.arange(B + 1, dtype=torch.int32, device=DEV)
    cu_k = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    try:
        ref = fa(q.to(DEV).view(B, H, 128), kk, vv, cu_q, cu_k, 1, max(lens), causal=True).reshape(B, H * 128)
        torch.cuda.synchronize()
    except Exception as e:
        pytest.skip(f"flash_attn does not run on this GPU: {type(e).__name__}: {e}")
    want = _oracle_decode(q, ck, cv, kv_len, H, KV)
    assert_bf16_close(ref, want, max_ulp=2, min_exact=0.5, atol=4e-3, what="flash_attn vs oracle decode attention")
    out = torch.empty(B, H * 128, dtype=torch.bfloat16, device=DEV)
    _abi.attn_decode(q.to(DEV), ck.to(DEV), cv.to(DEV), kv_len.to(DEV), out, H, KV, 128, 4, ws)
    assert_bf16_close(out, ref, max_ulp=2, min_exact=0.5, atol=4e-3, what="attn_decode kernel vs flash_attn")


# ----------------------------------------------------------------------------- mixture of experts: device router + grouped experts
def _moe_case(T, dim, hid, E, seed):
    x = rnd(T, dim, seed=seed)
    gate_w = rnd(E, dim, seed=seed + 1, scale=dim ** -0.5)
    experts = [(rnd(hid, dim, seed=seed + 10 + 3 * e, scale=dim ** -0.5), rnd(dim, hid, seed=seed + 11 + 3 * e, scale=hid ** -0.5),
                rnd(hid, dim, seed=seed + 12 + 3 * e, scale=dim ** -0.5)) for e in range(E)]
    return x, gate_w, experts


def _router_margin_ulps(x, gate_w, k):
    logits = F.linear(x, gate_w).float()
    top = logits.topk(k + 1, dim=-1).values
    ulp = torch.pow(2.0, torch.floor(torch.log2(top[:, k - 1].abs().clamp_min(1e-30))) - 7)
    return (top[:, k - 1] - top[:, k]) / ulp


@pytest.mark.parametrize("T,dim,hid,k", [(5, 256, 256, 2), (37, 256, 256, 3), (200, 256, 512, 2), (16, 4096, 14336, 2), (300, 4096, 14336, 2),
                                         (2500, 256, 512, 2)])  # last: enough rows per expert for the 2-CTA cluster pairs of the grouped GEMM
def test_moe_route_grouped_ffn_vs_oracle(T, dim, hid, k):
    """mb200_moe_route + mb200_moe_grouped_ffn against the oracle's MoE (moe.py:24-32) + residual: routing decisions and weights
    exactly (tokens whose k-th / (k+1)-th router logits are within 2 ulps excepted), the deterministic row plan exactly, the
    output within 2 bf16 ulps."""
    from mistral_inference_b200.moe import MoeBuffers

    from .util import moe_plan_host, moe_route_host

    E = 8
    x, gate_w, experts = _moe_case(T, dim, hid, E, seed=90)
    h = rnd(T, dim, seed=89)
    want = h + R.moe_forward(x, gate_w, experts, k)
    sel_ref, wts_ref = moe_route_host(x, gate_w, k)
    safe = _router_margin_ulps(x, gate_w, k) > 2.0
    ws = _abi.Workspace(_abi.workspace_bytes(max(T, 8), dim, 32, 8, 128, hid, 0, 4), torch.device(DEV))
    b = MoeBuffers(T, dim, hid, E, k, torch.device(DEV), torch.bfloat16)
    _abi.moe_route(x.to(DEV), gate_w.to(DEV), E, k, 0, 1, b)
    torch.cuda.synchronize()
    sel = b.sel.view(T, k).cpu()
    assert torch.equal(sel[safe], sel_ref[safe]), "routing differs on tokens without a router near-tie"
    assert torch.equal(b.wts.view(T, k).cpu()[safe].float(), wts_ref[safe].float()), "routing weights"
    slot, seg, tiles = moe_plan_host(sel, E, b.tile_rows)
    plan = b.plan.cpu().tolist()
    assert torch.equal(b.slot.view(T, k).cpu(), slot), "row plan: slots"
    assert plan[0] == len(tiles) and plan[1] == seg[-1] and plan[8:8 + E + 1] == seg
    cap = plan[2]
    assert [(plan[64 + i], plan[64 + cap + i]) for i in range(len(tiles))] == tiles
    xs = b.xs.cpu()
    for t in range(T):
        for j in range(k):
            assert torch.equal(xs[slot[t, j]], x[t])
    import ctypes

    w13 = (ctypes.c_void_p * E)()
    w2 = (ctypes.c_void_p * E)()
    keep = []
    for e, (w1, w2_, w3) in enumerate(experts):
        packed = torch.stack([w1, w3], 1).reshape(2 * hid, dim).to(DEV)
        down = w2_.to(DEV)
        keep += [packed, down]
        w13[e], w2[e] = packed.data_ptr(), down.data_ptr()
    out = torch.empty(T, dim, dtype=torch.bfloat16, device=DEV)
    for _ in range(2):  # twice: stream-K flags and plan buffers must be reusable
        out.zero_()
        _abi.moe_grouped_ffn(b, w13, w2, h.to(DEV), out, T, dim, hid, E, k, None, ws)
        torch.cuda.synchronize()
        rows = safe & (sel == sel_ref).all(-1)
        assert rows.float().mean() > 0.8
        assert_bf16_close(out.cpu()[rows], want[rows], max_ulp=2, min_exact=0.9, atol=2 * 2 ** -8 * want.abs().max().item(), what="moe layer")
