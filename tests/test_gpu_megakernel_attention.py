"""The decode megakernel's own attention (csrc/decode_megakernel.cuh, phases 2a / 2b) at slice, stage and ring-wrap edges.

The megakernel splits the ring by position: with len = min(pos + 1, W) keys and G CTAs (one per SM), CTA c owns ring slots
[c*C, (c+1)*C), C = ceil(len / G), and streams them through its shared-memory ring in stages of pps = 8 or 16 positions (by
KV).  The row of the token being decoded comes from phase 1 (global memory) and is patched into its stage; V rows past the slice
are zero-filled; phase 2b merges the n_slices = ceil(len / C) partials.  `geometry` below restates that arithmetic, and every
grid here is built from the SM count of the device it runs on, so each edge lands where that device puts it.

Each test drives `_abi.decode_step` directly on a synthetic model (dim = hidden = 256, vocab 512, head_dim 128, H = KV * REP) and
reads the last layer's q and attention output from the workspace (`_abi.decode_scratch`).  The embedding row and the norms are
all ones, so the normed input is exactly 1.0 in every column and column 0 of wq / wk / wv *is* the fresh q / k (before RoPE) / v.

Visible sets (exact), as in test_gpu_attention_edges.py: q = 0, so every P is exactly 1 and O = count / n per element, within one
bf16 ulp, exactly 0 where the count is 0.  Two V encodings:
  * "codes": the position code of the edges test, keyed by ring slot (neighbouring heads and batch rows differ in offsets and
    scale).  It resolves single keys while every bucket holds at most ~64 keys.
  * "probes": V is zero except at the first and last slot of every slice and at the current slot; each probe owns one
    (KV head, dim) cell with weight 2^8 (3 * 2^8 for a second probe in a cell, when there are more probes than cells).  A
    dropped, duplicated or misplaced probe moves its cell by a third or more, exactly, at any n.  Used where n = W (no slot
    beyond the visible set exists) and the codes cannot resolve a single key.
test_comparator_rejects_every_single_key_change proves, on the CPU and for G = 132 and 114, that the chosen encoding catches
every single-key change the kernel could make at the slice and stage edges of every case, and the neighbouring KV head or batch
row.  The cache holds NaN at slots >= len, at the current slot (the producer streams its stale contents before phase 1 rewrites
it, so a missed patch is NaN) and the other batch rows hold their own sequences' encodings.

Softmax weighting against float64 uses the bound derived in test_gpu_attention_edges.py's docstring,
|O - O64| <= 2^-8 * sum_j p_j |v_j| + ulp: the megakernel also rounds P to bf16 for P.V while l sums the unrounded fp32 P.
"""
import functools
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from mistral_inference_b200 import _abi
from mistral_inference_b200.rope import precompute_freqs_cis
from oracle import restatement as R

from .test_gpu_attention_edges import LOG2E, Case, bf16_round, code_params, reference64, rows_off
from .util import assert_bf16_close, assert_launched

DEV = "cuda"
HD = 128
DIM = HIDDEN = 256
VOCAB = 512
EPS = 1e-5
MAX_BATCH = 3
G_SXM, G_PCIE = 132, 114  # SM counts of the H100 SXM and PCIe
STAGE_BYTES = 16 * 1024 + 16 * 16  # MK_STAGE_BYTES: one ring stage holds pps padded K or V position rows
ROPE_LEN = 65_600
PROBE = 256.0
KV_REPS = [(8, 1), (8, 2), (8, 4), (8, 6), (8, 8), (2, 1), (2, 2), (2, 4), (2, 6), (2, 8), (5, 2)]
MK = r"decode_megakernel"


# ----------------------------------------------------------------------------- slice geometry (attn_slice restated)
def pps_of(KV: int) -> int:
    return min(16, (STAGE_BYTES // (KV * HD * 2 + 16)) & ~7)


class Geom(NamedTuple):
    n: int         # keys: min(pos + 1, W)
    C: int         # slots per CTA
    n_slices: int  # CTAs with a non-empty range
    pps: int       # positions per K / V stage
    cur: int       # ring slot of the token being decoded


def geometry(G: int, KV: int, pos: int, W: int) -> Geom:
    n = min(pos + 1, W)
    C = -(-n // G)
    return Geom(n, C, -(-n // C), pps_of(KV), pos % W)


def slices(g: Geom):
    """[(first, end)] slot range of every non-empty slice (CTA c = index)."""
    return [(c * g.C, min((c + 1) * g.C, g.n)) for c in range(g.n_slices)]


def stages(g: Geom, lo: int, hi: int):
    """[(first, end)] of the K / V stages of the slice [lo, hi)."""
    return [(k, min(k + g.pps, hi)) for k in range(lo, hi, g.pps)]


def edge_slots(g: Geom, with_stages: bool) -> np.ndarray:
    out = {g.cur} if g.cur < g.n else set()
    for lo, hi in slices(g):
        out |= {lo, hi - 1}
        if with_stages:
            for a, b in stages(g, lo, hi):
                out |= {a, b - 1}
    return np.array(sorted(out))


# ----------------------------------------------------------------------------- the grid
class MkCase(NamedTuple):
    pos: int
    W: int
    batch_row: int


def mk_cases(G: int, KV: int):
    pps = pps_of(KV)
    C4096 = -(-4096 // G)
    pw = [(n - 1, 8192) for n in (1, G - 1, G, G + 1, 2 * G + 1, 8 * G, 8 * G + 1, 16 * G, 16 * G + 1, 4096, 8192)]
    pw += [(p, 300) for p in (299, 300, 302, 303, 1000)]
    pw += [(p, 100) for p in (99, 100, 250)]
    pw += [(4096 + d, 4096) for d in (-1, 0, pps - 1, pps, C4096 - 1, C4096)] + [(3 * 4096 + 4095, 4096)]
    return [MkCase(p, W, 2 * (i % 2)) for i, (p, W) in enumerate(pw)]


def encoding(case: MkCase) -> str:
    return "codes" if min(case.pos + 1, case.W) <= 4096 else "probes"


def case_id(c: MkCase) -> str:
    return f"pos{c.pos}-W{c.W}-b{c.batch_row}"


# ----------------------------------------------------------------------------- V encodings (by ring slot)
def code_rows(W: int, KV: int, b: int) -> torch.Tensor:
    """[W, KV, 128] float32: the edges test's position code of every ring slot for KV head g and sequence b."""
    v = torch.zeros(W, KV, HD)
    j = torch.arange(W)
    for g in range(KV):
        a, c, s = code_params(g, b)
        v[j, g, (j + a) % 64] = s
        v[j, g, 64 + (j // 64 + c) % 64] = s
    return v


def probe_rows(W: int, KV: int, b: int, slots: np.ndarray) -> torch.Tensor:
    """[W, KV, 128] float32: zero except one cell per probe slot (KV head k % KV, a dim that also depends on the head and b)."""
    v = torch.zeros(W, KV, HD)
    cells = KV * HD
    assert len(slots) <= 2 * cells, "more probes than two per cell"
    for k, j in enumerate(slots.tolist()):
        r = k // cells
        kk = k % cells
        g = kk % KV
        v[j, g, (kk // KV + 17 * g + 29 * b) % HD] = PROBE * (1 + 2 * r)
    return v


def v_rows(case: MkCase, G: int, KV: int, b: int) -> torch.Tensor:
    """V of batch row b at slots [0, min(len + 1, W)) (the visible set and the slot after it)."""
    g = geometry(G, KV, case.pos, case.W)
    rows = min(g.n + 1, case.W)
    if encoding(case) == "codes":
        return code_rows(rows, KV, b)
    return probe_rows(rows, KV, b, edge_slots(g, with_stages=False))


@functools.lru_cache(maxsize=None)
def expected(case: MkCase, G: int, KV: int):
    """(counts [KV, 128] float64 over slots [0, n) of the case's batch row, n)."""
    g = geometry(G, KV, case.pos, case.W)
    return v_rows(case, G, KV, case.batch_row)[:g.n].double().sum(0).numpy(), g.n


def single_key_changes(case: MkCase, G: int, KV: int):
    """(name, counts [m, KV, 128], n [m]) for every change the kernel's slice walk could make."""
    g = geometry(G, KV, case.pos, case.W)
    V = v_rows(case, G, KV, case.batch_row).double().numpy()
    counts, n = expected(case, G, KV)
    e = edge_slots(g, with_stages=encoding(case) == "codes")
    if n > 1:  # with one key, dropping it leaves nothing and duplicating it leaves the output unchanged
        yield "drop an edge slot", counts[None] - V[e], np.full(len(e), n - 1)
        yield "drop the current row", (counts - V[g.cur])[None], np.array([n - 1])
        yield "duplicate an edge slot", counts[None] + V[e], np.full(len(e), n + 1)
    if g.n < case.W:
        yield "one key more (slot len)", (counts + V[g.n])[None], np.array([n + 1])
    # the current slot holds NaN in the cache until phase 1 writes it: a stale row makes the output NaN
    yield "a stale current row", np.full_like(counts, np.nan)[None], np.array([n])
    if KV > 1:
        yield "the neighbouring KV head", np.roll(counts, -1, axis=0)[None], np.array([n])
    other = 1  # batch rows 0 and 2 both neighbour row 1
    yield "the neighbouring batch row", v_rows(case, G, KV, other)[:g.n].double().sum(0).numpy()[None], np.array([n])


ALL_CPU = [(G, KV, c) for G in (G_SXM, G_PCIE) for KV in sorted({kv for kv, _ in KV_REPS}) for c in mk_cases(G, KV)]


def assert_comparator_catches(G: int, KV: int, case: MkCase):
    counts, n = expected(case, G, KV)
    assert not rows_off(bf16_round(counts / n)[None], counts[None], np.array([n])).any()
    if encoding(case) == "probes":
        assert min(case.pos + 1, case.W) == case.W
    for what, wrong, wn in single_key_changes(case, G, KV):
        got = bf16_round(wrong / wn[:, None, None])
        caught = rows_off(got, np.repeat(counts[None], len(wn), 0), np.full(len(wn), n))
        assert caught.all(), f"G={G} KV={KV} {case}: '{what}' not detected in {int((~caught).sum())} of {len(caught)} variants"


@pytest.mark.parametrize("G,KV,case", ALL_CPU, ids=[f"G{G}-KV{KV}-{case_id(c)}" for G, KV, c in ALL_CPU])
def test_comparator_rejects_every_single_key_change(G, KV, case):
    """CPU check of the comparator for every case the GPU tests run, at the SM counts of both H100 models: the correct answer
    passes, and every dropped / duplicated edge slot, one key beyond the set, a dropped or stale current row, and the keys of
    the neighbouring KV head or batch row would be caught."""
    assert_comparator_catches(G, KV, case)


@pytest.mark.parametrize("G", [G_SXM, G_PCIE])
def test_grid_reaches_every_edge(G):
    """The grid, built from G, reaches every edge of the slice walk for each KV."""
    for KV in (8, 2, 5):
        gs = [(c, geometry(G, KV, c.pos, c.W)) for c in mk_cases(G, KV)]
        pps = pps_of(KV)
        assert pps == {8: 8, 2: 16, 5: 8}[KV]
        has = lambda f: any(f(c, g) for c, g in gs)  # noqa: E731
        assert has(lambda c, g: g.n == 1)
        assert has(lambda c, g: g.C == 1 and g.n_slices == G) and has(lambda c, g: g.C == 2 and g.n == G + 1)
        assert has(lambda c, g: g.C == 1 and g.n_slices == G - 1)
        assert has(lambda c, g: g.C == 2 and g.n_slices < G)  # idle CTAs after a full-C split
        assert has(lambda c, g: g.C == 3 and c.W > g.n)
        assert has(lambda c, g: g.C == pps + 1)  # a second stage of one row
        assert has(lambda c, g: g.C == pps and g.n_slices == G)  # exactly one full stage per CTA
        assert has(lambda c, g: g.C == 8 + 1) and has(lambda c, g: g.C == 16 + 1)  # both pps edges, whatever KV
        assert has(lambda c, g: g.n == 4096 and g.C // pps >= 2)  # several stages per CTA
        assert has(lambda c, g: g.n == 8192 and g.n % g.C != 0)  # a short last slice
        assert has(lambda c, g: c.W < G and c.pos >= c.W)  # a wrapped ring with fewer slots than CTAs
        assert has(lambda c, g: c.W == 300 and c.pos >= c.W and g.C == 3)
        wrapped = [(c, g) for c, g in gs if c.W == 4096 and c.pos >= c.W]
        rows = {(g.cur % g.C, (g.cur % g.C) % pps) for c, g in wrapped}
        assert any(r == 0 for r, _ in rows)                                      # first row of a slice (and stage)
        assert any(r == g.C - 1 for c, g in wrapped for r in [g.cur % g.C])      # last row of a slice
        assert any(s == pps - 1 for _, s in rows) and any(s == 0 and r > 0 for r, s in rows)  # last / first row of an inner stage
        assert any(g.cur == c.W - 1 for c, g in wrapped)
        assert {c.batch_row for c, _ in gs} == {0, 2}
    c32 = geometry(G, 8, 32767, 32768)
    if G == G_SXM:
        assert (c32.C, c32.n - (c32.n_slices - 1) * c32.C) == (249, 149)
    assert len(edge_slots(c32, with_stages=False)) <= 8 * HD


def test_probe_comparator_32k():
    """The 32k-slot ring (len 32768, no window): the probe encoding catches every change at the slice edges and the current slot."""
    for G in (G_SXM, G_PCIE):
        assert_comparator_catches(G, 8, MkCase(32767, 32768, 2))


# ----------------------------------------------------------------------------- the synthetic model
@pytest.fixture(scope="module")
def rope():
    table = precompute_freqs_cis(HD, ROPE_LEN, 1e6)
    return table, torch.view_as_real(table).contiguous().to(DEV)


@pytest.fixture(scope="module")
def ws():
    return _abi.Workspace(_abi.workspace_bytes(1, DIM, 64, 8, HD, HIDDEN, VOCAB, MAX_BATCH), torch.device(DEV))


class Model:
    """1 or 2 layers; everything but the caches and column 0 of wqkv is fixed: ones for the embedding and the norms, zeros for
    wo, w13 and w2 (so a later layer sees the same all-ones input), and w_out as given."""

    def __init__(self, KV: int, rep: int, windows, w_out=None):
        self.KV, self.rep, self.H = KV, rep, KV * rep
        self.windows = list(windows)
        bf = dict(dtype=torch.bfloat16, device=DEV)
        self.emb = torch.ones(VOCAB, DIM, **bf)
        self.ones = torch.ones(DIM, **bf)
        self.w_out = torch.zeros(VOCAB, DIM, **bf) if w_out is None else w_out.to(**bf)
        self.wqkv = [torch.zeros((self.H + 2 * KV) * HD, DIM, **bf) for _ in windows]
        self.wo = torch.zeros(DIM, self.H * HD, **bf)
        self.w13 = torch.zeros(2 * HIDDEN, DIM, **bf)
        self.w2 = torch.zeros(DIM, HIDDEN, **bf)
        self.ck = [torch.full((MAX_BATCH, W, KV, HD), float("nan"), **bf) for W in windows]
        self.cv = [torch.full((MAX_BATCH, W, KV, HD), float("nan"), **bf) for W in windows]
        desc = [[self.wqkv[i].data_ptr(), self.wo.data_ptr(), self.w13.data_ptr(), self.w2.data_ptr(), self.ones.data_ptr(),
                 self.ones.data_ptr(), self.ck[i].data_ptr(), self.cv[i].data_ptr()] for i in range(len(windows))]
        self.layers = torch.tensor(desc, dtype=torch.int64, device=DEV)
        self.win = torch.tensor(self.windows, dtype=torch.int32, device=DEV)
        self.token = torch.zeros(1, dtype=torch.long, device=DEV)
        self.logits = torch.empty(VOCAB, dtype=torch.float32, device=DEV)
        self.next = torch.full((1,), -1, dtype=torch.long, device=DEV)

    def set_fresh(self, layer: int, q=None, k=None, v=None):
        """Column 0 of wq / wk / wv: the fresh q and k before RoPE, and v (the input is exactly 1.0 in every column)."""
        w = self.wqkv[layer]
        qd, kd = self.H * HD, self.KV * HD
        for lo, x in ((0, q), (qd, k), (qd + kd, v)):
            if x is not None:
                w[lo:lo + x.numel(), 0] = x.reshape(-1).to(w)

    def step(self, pos: int, batch_row: int, ws, rope_dev):
        _abi.decode_step(self.layers, self.win, len(self.windows), self.emb, self.ones, self.w_out, rope_dev, self.token, pos, batch_row,
                         self.logits, self.next, DIM, HIDDEN, self.H, self.KV, HD, VOCAB, EPS, ws)

    def scratch(self, ws):
        """(q [H, 128], attention output [H, 128]) of the last layer, bf16 on the host, as the step left them in the workspace."""
        qo, ao = _abi.decode_scratch(DIM, HIDDEN, self.H, self.KV, HD)
        nb = self.H * HD * 2
        return (ws.buf[qo:qo + nb].view(torch.bfloat16).view(self.H, HD).cpu(),
                ws.buf[ao:ao + nb].view(torch.bfloat16).view(self.H, HD).cpu())


def rope_fp32(x: torch.Tensor, pos: int, table: torch.Tensor) -> torch.Tensor:
    """The QKV epilogue's RoPE, bit for bit: bf16 pairs (a, b) times (c, d) from the fp32 table, re = ac - bd and im = ad + bc with
    every product and sum rounded to fp32 (no FMA), then rounded to bf16."""
    a, b = x.float().reshape(-1, HD // 2, 2).unbind(-1)
    cd = torch.view_as_real(table[pos])
    c, d = cd[:, 0].numpy(), cd[:, 1].numpy()
    a, b = a.numpy(), b.numpy()
    re = (a * c).astype(np.float32) - (b * d).astype(np.float32)
    im = (a * d).astype(np.float32) + (b * c).astype(np.float32)
    return torch.from_numpy(np.stack([re, im], -1).reshape(-1)).to(torch.bfloat16)


def unrope(x: torch.Tensor, pos: int, table: torch.Tensor) -> torch.Tensor:
    """A pre-RoPE vector whose rotation at `pos` is close to x ([..., 128], float64 then bf16)."""
    z = torch.view_as_complex(x.double().reshape(*x.shape[:-1], HD // 2, 2).contiguous())
    return torch.view_as_real(z * table[pos].to(torch.complex128).conj()).reshape(x.shape).to(torch.bfloat16)


# ----------------------------------------------------------------------------- visible sets
def fill_case(m: Model, layer: int, case: MkCase, G: int, gen: torch.Generator):
    """Caches of one layer: the case's V encoding and random K at slots < len of every batch row, NaN elsewhere and at the
    current slot of the case's row; the fresh K / V row through wk / wv.  Returns the intended K and V of the current slot."""
    KV, W = m.KV, case.W
    g = geometry(G, KV, case.pos, W)
    ck = torch.full((MAX_BATCH, W, KV, HD), float("nan"), dtype=torch.bfloat16)
    cv = ck.clone()
    for b in range(MAX_BATCH):
        ck[b, :g.n] = torch.randn(g.n, KV, HD, generator=gen).to(torch.bfloat16)
        cv[b, :g.n] = v_rows(case, G, KV, b)[:g.n].to(torch.bfloat16)
    v_cur = v_rows(case, G, KV, case.batch_row)[g.cur].to(torch.bfloat16)
    k_pre = torch.randn(KV * HD, generator=gen).to(torch.bfloat16)
    ck[case.batch_row, g.cur] = float("nan")
    cv[case.batch_row, g.cur] = float("nan")
    m.ck[layer].copy_(ck)
    m.cv[layer].copy_(cv)
    m.set_fresh(layer, k=k_pre, v=v_cur)
    return k_pre, v_cur


def check_ring_write(m: Model, layer: int, before_k, before_v, case: MkCase, k_cur, v_cur):
    """The current slot of the case's row holds exactly k_cur / v_cur; every other slot and row is bit for bit unchanged."""
    cur = case.pos % case.W
    for name, before, after, want in (("K", before_k, m.ck[layer], k_cur), ("V", before_v, m.cv[layer], v_cur)):
        after = after.cpu()
        assert torch.equal(after[case.batch_row, cur].reshape(-1).view(torch.int16), want.reshape(-1).view(torch.int16)), \
            f"{case}: the current {name} row is not what phase 1 computed"
        after[case.batch_row, cur] = before[case.batch_row, cur]
        assert torch.equal(after.view(torch.int16), before.view(torch.int16)), f"{case}: {name} ring changed outside the current slot"


def check_output(out: torch.Tensor, case: MkCase, G: int, KV: int, rep: int, what: str = ""):
    counts, n = expected(case, G, KV)
    H = KV * rep
    want = np.repeat(counts, rep, axis=0)  # query head h reads KV head h // rep
    off = rows_off(out.view(1, H, HD), want[None], np.array([n]))
    if off.any():
        got = out.float().cpu() * n
        bad = (got - torch.from_numpy(want)).abs().sum(1)
        h = int(bad.argmax())
        raise AssertionError(f"{what}G={G} KV={KV} REP={rep} {case} ({encoding(case)}, {geometry(G, KV, case.pos, case.W)}): "
                             f"head {h} sees the wrong keys; n * O differs from the counts by {bad[h]:.3f} in total")


def run_visible_case(m: Model, case: MkCase, G: int, ws, rope, seed: int):
    table, rope_dev = rope
    gen = torch.Generator().manual_seed(seed)
    layer = len(m.windows) - 1
    for l, W in enumerate(m.windows[:-1]):  # earlier layers: their own finite rings, checked for the ring write only
        fill_case(m, l, MkCase(case.pos, W, case.batch_row), G, gen)
    k_pre, v_cur = fill_case(m, layer, case, G, gen)
    before = [(k.cpu(), v.cpu()) for k, v in zip(m.ck, m.cv)]
    m.step(case.pos, case.batch_row, ws, rope_dev)
    q, out = m.scratch(ws)
    assert torch.equal(q.float(), torch.zeros_like(q.float())), "q must be 0"
    for l, W in enumerate(m.windows):
        c = MkCase(case.pos, W, case.batch_row)
        kp = m.wqkv[l][m.H * HD:(m.H + m.KV) * HD, 0].cpu()
        vc = m.wqkv[l][(m.H + m.KV) * HD:, 0].cpu()
        check_ring_write(m, l, before[l][0], before[l][1], c, rope_fp32(kp, case.pos, table), vc)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("KV,rep", KV_REPS)
def test_megakernel_visible_sets(KV, rep, ws, rope):
    """Every case of the grid, one launch each, on one workspace: exact visible set of every query head, and the ring write."""
    G = _abi.device_info()[0]
    cases = mk_cases(G, KV)
    outs = []

    def launches():
        for i, case in enumerate(cases):
            outs.append(run_visible_case(Model(KV, rep, [case.W]), case, G, ws, rope, seed=i))

    assert_launched(launches, rf"decode_megakernel<{rep}>", MK, len(cases))
    for case, out in zip(cases, outs):
        check_output(out, case, G, KV, rep)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", [1, 4])
def test_megakernel_32k_ring_probes(rep, ws, rope):
    """Nemo's ring (no window: max_seq_len slots) full at 32768 keys: slice edges and the current slot, by sparse probes."""
    G = _abi.device_info()[0]
    case = MkCase(32767, 32768, 2)
    outs = []

    def launch():
        m = Model(8, rep, [case.W])
        outs.append(run_visible_case(m, case, G, ws, rope, seed=7))

    assert_launched(launch, rf"decode_megakernel<{rep}>", MK, 1)
    check_output(outs[0], case, G, 8, rep)


@pytest.mark.gpu
@pytest.mark.parametrize("KV,rep", [(8, 4), (2, 2)])
@pytest.mark.parametrize("windows", [(100, 4096), (4096, 100)])
def test_megakernel_per_layer_windows(windows, KV, rep, ws, rope):
    """Two layers with different windows; layer 0's wo and w2 are zero, so layer 1 sees the same all-ones input.  The observed
    layer 1 must walk its own ring (producer and consumers) and layer 0 must write its own."""
    G = _abi.device_info()[0]
    outs = []
    cases = [MkCase(p, windows[1], b) for p, b in ((5000, 0), (4096 + 99, 2))]

    def launches():
        for i, case in enumerate(cases):
            m = Model(KV, rep, windows)
            outs.append(run_visible_case(m, case, G, ws, rope, seed=100 + i))

    assert_launched(launches, rf"decode_megakernel<{rep}>", MK, len(cases))
    for case, out in zip(cases, outs):
        check_output(out, case, G, KV, rep, f"windows {windows}: ")


@pytest.mark.gpu
def test_megakernel_merge_ignores_stale_partials(ws, rope):
    """On one workspace: G slices (C = 1), then 1 slice, then ceil((G + 1) / 2) slices.  The merge must read only this launch's."""
    G = _abi.device_info()[0]
    cases = [MkCase(G - 1, 8192, 0), MkCase(0, 8192, 2), MkCase(G, 8192, 0)]
    assert [geometry(G, 8, c.pos, c.W).n_slices for c in cases] == [G, 1, -(-(G + 1) // 2)]
    outs = []

    def launches():
        for i, case in enumerate(cases):
            m = Model(8, 2, [case.W])
            outs.append(run_visible_case(m, case, G, ws, rope, seed=200 + i))

    assert_launched(launches, r"decode_megakernel<2>", MK, len(cases))
    for case, out in zip(cases, outs):
        check_output(out, case, G, 8, 2)


# ----------------------------------------------------------------------------- softmax weighting against float64
SCORE_LOG2_PER_UNIT = HD * HD ** -0.5 * LOG2E  # q = k = all-ones vectors: score in log2 units


def dominant_slots(g: Geom):
    """Slice and stage boundaries computed from the geometry, and the current slot."""
    sl = slices(g)
    picks = []
    for lo, hi in (sl[0], sl[1], sl[len(sl) // 2], sl[-1]):
        picks += [lo, hi - 1]
        st = stages(g, lo, hi)
        if len(st) > 1:
            picks += [st[1][0], st[0][1] - 1]
    picks.append(g.cur)
    return list(dict.fromkeys(picks))


@pytest.mark.gpu
@pytest.mark.parametrize("ring", ["4096-wrapped", "32768"])
@pytest.mark.parametrize("pattern", ["rising", "dominant", "wide"])
@pytest.mark.parametrize("rep", [1, 4, 8])
@pytest.mark.parametrize("KV", [8, 2])
def test_megakernel_softmax_vs_float64(KV, rep, pattern, ring, ws, rope):
    """Online softmax and the slice merge under stress: a running max that grows in every stage and slice, dominant keys on
    slice / stage boundaries and at the current slot, scores spanning about +-60 log2 units.  q is the one the kernel used
    (from the workspace) and K / V are the ring after the step, so phase 1's rounding does not enter the bound."""
    table, rope_dev = rope
    G = _abi.device_info()[0]
    pos, W = (3 * 4096 + 1234, 4096) if ring == "4096-wrapped" else (32767, 32768)
    g = geometry(G, KV, pos, W)
    H = KV * rep
    gen = torch.Generator().manual_seed(1000 * KV + 10 * rep + len(pattern))
    u = torch.sign(torch.randn(HD, generator=gen))
    n = g.n
    if pattern == "rising":  # by ring slot, the order the slices walk
        K = (torch.arange(n, dtype=torch.float64) * (0.07 / SCORE_LOG2_PER_UNIT))[:, None, None].expand(n, KV, HD).clone()
        q_rot = torch.ones(H, HD, dtype=torch.float64)
    elif pattern == "dominant":
        K = torch.randn(n, KV, HD, generator=gen, dtype=torch.float64) * 0.25
        for i, j in enumerate(dominant_slots(g)):
            K[j] = u * (18 + 2 * i) / SCORE_LOG2_PER_UNIT
        q_rot = u + 0.3 * torch.randn(H, HD, generator=gen, dtype=torch.float64)
    else:
        K = torch.randn(n, KV, HD, generator=gen, dtype=torch.float64) * 3.7
        q_rot = torch.randn(H, HD, generator=gen, dtype=torch.float64) * 3.7
    V = torch.randn(n, KV, HD, generator=gen).to(torch.bfloat16)
    m = Model(KV, rep, [W])
    ck = torch.full((MAX_BATCH, W, KV, HD), float("nan"), dtype=torch.bfloat16)
    cv = ck.clone()
    ck[1, :n] = K.to(torch.bfloat16)
    cv[1, :n] = V
    ck[1, g.cur] = cv[1, g.cur] = float("nan")
    m.ck[0].copy_(ck)
    m.cv[0].copy_(cv)
    m.set_fresh(0, q=unrope(q_rot, pos, table), k=unrope(K[g.cur], pos, table), v=V[g.cur])
    assert_launched(lambda: m.step(pos, 1, ws, rope_dev), rf"decode_megakernel<{rep}>", MK, 1)
    q, out = m.scratch(ws)
    Kc, Vc = m.ck[0][1, :n].cpu(), m.cv[0][1, :n].cpu()
    assert torch.isfinite(Kc.float()).all() and torch.isfinite(Vc.float()).all()
    case = Case("decode", (n,), (), n)
    o64 = torch.empty(H, HD, dtype=torch.float64)
    mag = torch.empty_like(o64)
    for kv in range(KV):  # one KV head at a time keeps the float64 reference small at 32k keys
        hs = slice(kv * rep, (kv + 1) * rep)
        o, mg = reference64(case, q[hs][None], [Kc[:, kv:kv + 1]], [Vc[:, kv:kv + 1]], rep)
        o64[hs], mag[hs] = o[0], mg[0]
    got = out.double().cpu()
    ulp = torch.exp2(torch.floor(torch.log2(o64.abs().clamp_min(2.0 ** -126))) - 7)
    bound = 2.0 ** -8 * mag + ulp
    err = (got - o64).abs()
    assert torch.isfinite(got).all(), "non-finite output"
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{g}: {(err > bound).sum().item()} elements beyond the bound; worst err / bound = {worst:.2f}"


# ----------------------------------------------------------------------------- phase 1 at large and wrapped positions
PHASE1_POS = [4095, 4096, 4096 + 7, 4096 + 8, 3 * 4096 + 4095, 32767, 32768 + 131, 65_000]


@pytest.mark.gpu
@pytest.mark.parametrize("KV,rep", [(8, 4), (2, 8)])
def test_megakernel_phase1_at_large_positions(KV, rep, ws, rope):
    """q and the fresh K / V row against R.apply_rope(F.linear(...)) with random weights and input, within the ulps that
    test_attn_qkv allows, at the positions the attention tests use and up to 65 000 (a 4096-slot ring)."""
    table, rope_dev = rope
    gen = torch.Generator().manual_seed(KV * 10 + rep)
    W = 4096
    m = Model(KV, rep, [W])
    H = m.H
    x = torch.randn(DIM, generator=gen).to(torch.bfloat16)
    m.emb.copy_(x[None].expand(VOCAB, DIM))
    wq = (torch.randn(H * HD, DIM, generator=gen) * DIM ** -0.5).to(torch.bfloat16)
    wk = (torch.randn(KV * HD, DIM, generator=gen) * DIM ** -0.5).to(torch.bfloat16)
    wv = (torch.randn(KV * HD, DIM, generator=gen) * DIM ** -0.5).to(torch.bfloat16)
    m.wqkv[0].copy_(torch.cat([wq, wk, wv], 0))
    m.ck[0].zero_()
    m.cv[0].zero_()
    xn = R.rms_norm(x[None], torch.ones(DIM, dtype=torch.bfloat16), EPS)
    got = []

    def launches():
        for pos in PHASE1_POS:
            m.step(pos, 2, ws, rope_dev)
            q, _ = m.scratch(ws)
            got.append((q, m.ck[0][2, pos % W].clone(), m.cv[0][2, pos % W].clone()))

    assert_launched(launches, rf"decode_megakernel<{rep}>", MK, len(PHASE1_POS))
    v_ref = F.linear(xn, wv)
    for pos, (q, k, v) in zip(PHASE1_POS, got):
        q_ref, k_ref = R.apply_rope(F.linear(xn, wq).view(1, H, HD), F.linear(xn, wk).view(1, KV, HD), table[[pos]])
        assert_bf16_close(q.reshape(1, -1), q_ref.reshape(1, -1), atol=2 * 2 ** -8 * q_ref.abs().max().item(), what=f"q @ {pos}")
        assert_bf16_close(k.reshape(1, -1), k_ref.reshape(1, -1), atol=2 * 2 ** -8 * k_ref.abs().max().item(), what=f"k @ {pos}")
        assert_bf16_close(v.reshape(1, -1), v_ref, what=f"v @ {pos}")


# ----------------------------------------------------------------------------- fused greedy argmax
ARGMAX_TIES = {
    # name: (value of the tied maximum rows, indices of the tied rows); every other row sums to about -128
    "negative-across-ctas": (-0.4, [300, 17, 509]),
    "negative-in-one-pair": (-0.4, [263, 262]),
    "zero-across-ctas": (0.0, [41, 256, 40]),
    "zero-pair-and-far": (0.0, [511, 200, 201]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ARGMAX_TIES))
def test_megakernel_fused_argmax_ties(name, ws, rope):
    """w_out with duplicated rows, so that the largest logit ties at indices in different CTAs' vocab slices and inside one row
    pair, with all logits negative or a maximum of exactly 0: next_token is torch.argmax of the kernel's own logits."""
    _, rope_dev = rope
    value, idx = ARGMAX_TIES[name]
    gen = torch.Generator().manual_seed(len(name))
    w = (torch.randn(VOCAB, DIM, generator=gen) * 0.1 - 0.5).to(torch.bfloat16)
    top = torch.zeros(DIM) if value == 0.0 else (torch.randn(DIM, generator=gen) * 0.1 + value)
    w[idx] = top.to(torch.bfloat16)
    m = Model(8, 4, [64], w_out=w)
    m.ck[0].zero_()
    m.cv[0].zero_()
    assert_launched(lambda: m.step(10, 0, ws, rope_dev), r"decode_megakernel<4>", MK, 1)
    logits = m.logits.cpu()
    assert (logits[idx] == logits.max()).all(), "the duplicated rows must tie at the maximum"
    assert (logits < 0).all() if value < 0 else logits.max().item() == 0.0
    assert int(m.next.item()) == int(logits.argmax().item()) == min(idx)
