"""Mixture-of-experts layer (API mirror of mistral_inference/moe.py:16-32).

Batch-1 decode runs the router and the selected experts INSIDE the decode megakernel (csrc/decode_megakernel.cuh).  Everything
else -- prefill and batched decode -- goes through two C-ABI calls per layer with no host synchronisation (csrc/moe.cuh):

  mb200_moe_route        gate GEMV, top-k on the bf16 router logits, fp32 softmax over the k selected (moe.py:25-27), a
                         deterministic expert-sorted row plan, gather of the token rows
  mb200_moe_grouped_ffn  grouped wgmma GEMMs over the experts (gate/up + SiLU*mul, down) and the combine:
                         out = h + sum_j bf16(w_j * y_j) taken in ascending expert index, rounded to bf16 at every step exactly
                         like the reference's `results[idx] += w * expert(x)` loop (moe.py:28-31)

Expert parallelism (SURVEY.md 8e): with `expert_shard = (g, G)` this rank owns the experts `e % G == g` and holds no weights of
the others.  Every rank evaluates the router and the row plan redundantly (deterministic, identical on all ranks), runs the
grouped GEMMs for its own experts, and the DOWN PROJECTION'S EPILOGUE stores each weighted output row into the row buffer of
every rank over NVLink (peer memory mapped with CUDA IPC, `ExpertComm`): the exchange is an all-gather of rows fused into the
GEMM, not a collective call after it.  After a flag handshake every rank combines all k rows of every token in the reference's
order, so the result is bit-identical to the unsharded model for any k -- no reduction order is left to a library.
"""
import ctypes
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _abi
from .args import LoraArgs, MoeArgs

MOE_BLOCK_TOKENS = 16384  # prefill goes through the experts in blocks of this many tokens (bounds the row buffers: ~2 GB at 8x22B)


class _GateView:
    def __init__(self, layer: "MoeLayer"):
        self._layer = layer

    @property
    def weight(self) -> torch.Tensor:
        return self._layer.gate_weight


EXPERT_WEIGHTS = ("bf16", "fp8", "int4")


class Fp8Expert(nn.Module):
    """One expert with FP8 (e4m3) weights, the storage format of include/mistral_b200.h: `w13_q` [2*hidden, dim] (row 2i = w1[i],
    row 2i + 1 = w3[i], like FeedForward.w13) and `w2_q` [dim, hidden] hold the e4m3 bit patterns as uint8, with one fp32 scale
    per row.  The scales are stored as their int32 bit patterns (`w13_scale` / `w2_scale` are the fp32 views): `Module.to(dtype)`
    casts every floating tensor, and these must keep their bits.  Weights arrive as bf16 and are quantised in place on the device.
    With `lora` set the expert's w1 / w2 / w3 are LoRALinears (lora.py:22-89) on W': `w13_lora` and `w2_lora` hold their bf16
    adapters, packed like FeedForward's."""

    def __init__(self, dim: int, hidden_dim: int, lora: Optional[LoraArgs] = None):
        super().__init__()
        self.dim = dim
        self.hidden_dim = hidden_dim
        self.w13_q = nn.Parameter(torch.empty(2 * hidden_dim, dim, dtype=torch.uint8), requires_grad=False)
        self.w2_q = nn.Parameter(torch.empty(dim, hidden_dim, dtype=torch.uint8), requires_grad=False)
        self.w13_scale_bits = nn.Parameter(torch.empty(2 * hidden_dim, dtype=torch.int32), requires_grad=False)
        self.w2_scale_bits = nn.Parameter(torch.empty(dim, dtype=torch.int32), requires_grad=False)
        self.lora = lora
        if lora is not None:
            from .transformer_layers import LoraAdapter  # (transformer_layers imports this module)

            self.w13_lora = LoraAdapter(dim, [hidden_dim, hidden_dim], lora, interleaved=True)
            self.w2_lora = LoraAdapter(hidden_dim, [dim], lora)

    def adapter(self, name: str):
        """(packed adapter, segment) of the reference Linear `name` (w1, w2 or w3)."""
        if name in ("w1", "w3"):
            return self.w13_lora, 0 if name == "w1" else 1
        if name == "w2":
            return self.w2_lora, 0
        raise ValueError(f"expert Linear {name!r}")

    @property
    def w13_scale(self) -> torch.Tensor:
        return self.w13_scale_bits.view(torch.float32)

    @property
    def w2_scale(self) -> torch.Tensor:
        return self.w2_scale_bits.view(torch.float32)

    def _slots(self, name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        """(q rows, scale entries) of the reference Linear `name` (w1, w2 or w3): zero-copy, strided for w1 / w3."""
        h, d = self.hidden_dim, self.dim
        if name in ("w1", "w3"):
            seg = 0 if name == "w1" else 1
            return self.w13_q.view(h, 2, d)[:, seg], self.w13_scale.view(h, 2)[:, seg]
        if name == "w2":
            return self.w2_q, self.w2_scale
        raise ValueError(f"expert Linear {name!r}")

    def weight_e4m3(self, name: str) -> torch.Tensor:
        return self._slots(name)[0].view(torch.float8_e4m3fn)

    def weight_scale(self, name: str) -> torch.Tensor:
        return self._slots(name)[1]

    def quantize_(self, name: str, w: torch.Tensor) -> None:
        """Quantises the bf16 weight `w` of Linear `name` into place (one bf16 copy of `w` on the device while it runs)."""
        quantize_rows_(name, w, *self._slots(name))


def quantize_rows_(name: str, w: torch.Tensor, q: torch.Tensor, s: torch.Tensor) -> None:
    """q, s (e4m3 rows as uint8 and fp32 row scales, both possibly strided views) of the bf16 weight `w` of Linear `name`."""
    assert tuple(w.shape) == tuple(q.shape), f"{name}: shape {tuple(w.shape)} != expected {tuple(q.shape)}"
    _abi.quantize_e4m3_rows(w.to(device=q.device, dtype=torch.bfloat16).contiguous(), q, s)


class _Int4Rows:
    """INT4 storage of a module's packed matrices: `<m>` is uint8 [N, K/2] (two codes per byte, low nibble = even k), and
    `<m>_gscale_bits` int16 [N, K/128] the bit patterns of the bf16 group scales (`Module.to(dtype)` casts every floating tensor;
    these must keep their bits).  The module's `_slots` maps a reference Linear name to its (code rows, scale rows): zero-copy views,
    strided where rows interleave."""

    def _int4_params(self, name: str, n: int, k: int) -> nn.Parameter:
        assert k % 128 == 0, f"{name}: K={k} is not a multiple of the 128-wide scale groups"
        setattr(self, name + "_gscale_bits", nn.Parameter(torch.empty(n, k // 128, dtype=torch.int16), requires_grad=False))
        return nn.Parameter(torch.empty(n, k // 2, dtype=torch.uint8), requires_grad=False)

    def weight_int4(self, name: str) -> torch.Tensor:
        return self._slots(name)[0]

    def weight_gscale(self, name: str) -> torch.Tensor:
        return self._slots(name)[1]

    def quantize_int4_(self, name: str, w: torch.Tensor) -> None:
        """Quantises the bf16 weight `w` of Linear `name` into place (one bf16 copy of `w` on the device while it runs)."""
        q, s = self._slots(name)
        assert tuple(w.shape) == (q.shape[0], 2 * q.shape[1]), f"{name}: shape {tuple(w.shape)} != expected {(q.shape[0], 2 * q.shape[1])}"
        _abi.quantize_int4_groups(w.to(device=q.device, dtype=torch.bfloat16).contiguous(), q, s)


class Int4Expert(nn.Module, _Int4Rows):
    """One expert with INT4 weights, the format of the INT4 dense Linears (include/mistral_b200.h): `w13` uint8 [2*hidden, dim/2]
    (row 2i = w1[i], row 2i + 1 = w3[i], like FeedForward.w13) and `w2_weight` uint8 [dim, hidden/2] hold the packed codes, with one
    bf16 scale per group of 128 k of a row in `w13_gscale_bits` / `w2_gscale_bits` (int16 bit patterns; `w13_gscale` / `w2_gscale`
    are the bf16 views).  Weights arrive as bf16 and are quantised in place on the device."""

    def __init__(self, dim: int, hidden_dim: int):
        super().__init__()
        self.dim = dim
        self.hidden_dim = hidden_dim
        self.w13 = self._int4_params("w13", 2 * hidden_dim, dim)
        self.w2_weight = self._int4_params("w2", dim, hidden_dim)

    @property
    def w13_gscale(self) -> torch.Tensor:
        return self.w13_gscale_bits.view(torch.bfloat16)

    @property
    def w2_gscale(self) -> torch.Tensor:
        return self.w2_gscale_bits.view(torch.bfloat16)

    def _slots(self, name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        """(code rows, scale rows) of the reference Linear `name` (w1, w2 or w3): zero-copy, strided for w1 / w3."""
        h, d = self.hidden_dim, self.dim
        if name in ("w1", "w3"):
            seg = 0 if name == "w1" else 1
            return self.w13.view(h, 2, d // 2)[:, seg], self.w13_gscale.view(h, 2, d // 128)[:, seg]
        if name == "w2":
            return self.w2_weight, self.w2_gscale
        raise ValueError(f"expert Linear {name!r}")


class MoeBuffers:
    """Row buffers of one MoE call for up to `T` tokens (shared by all layers of a model; sizes from mb200_moe_sizes)."""

    def __init__(self, T: int, dim: int, hidden: int, E: int, k: int, device: torch.device, dtype: torch.dtype, yw_ptr: Optional[int] = None,
                 lora_cols: int = 0):
        self.T = T
        self.tile_rows, self.rows_cap, self.plan_words = _abi.moe_sizes(T, E, k)
        i32 = dict(dtype=torch.int32, device=device)
        self.sel = torch.empty(T * k, **i32)
        self.slot = torch.empty(T * k, **i32)
        self.plan = torch.zeros(self.plan_words, **i32)
        self.wts = torch.empty(T * k, dtype=dtype, device=device)
        self.row_w = torch.zeros(self.rows_cap, dtype=dtype, device=device)
        self.xs = torch.zeros(self.rows_cap, dim, dtype=dtype, device=device)  # zero once: padded rows stay finite
        self.g = torch.zeros(self.rows_cap, hidden, dtype=dtype, device=device)
        # weighted expert output rows: a local tensor, or (expert parallel) this rank's IPC-exported region that peers write too
        self.yw = torch.zeros(self.rows_cap, dim, dtype=dtype, device=device) if yw_ptr is None else None
        self.yw_ptr = self.yw.data_ptr() if yw_ptr is None else yw_ptr
        # un-merged expert adapters (lora_cols = the w13 adapter's rank columns, the wider one): the down projection's output and the
        # up projection's L, shared by w13 and w2 (include/mistral_b200.h); l_buf doubles as the down projection's split partials
        self.lora_a = torch.empty(self.rows_cap, lora_cols, dtype=dtype, device=device) if lora_cols else None
        self.lora_l = torch.empty(self.rows_cap, max(2 * hidden, dim), dtype=dtype, device=device) if lora_cols else None


class ExpertComm:
    """NVLink peer memory of an expert-parallel group: per rank ONE cudaMalloc'ed region exported with CUDA IPC, holding two row
    buffers (consecutive MoE layers alternate, so a rank that runs ahead never overwrites rows a peer is still combining) and
    the handshake flags.  Handles travel through torch.distributed (`all_gather_object`)."""

    FLAG_BYTES = 4096  # [2 parities][n_ranks] uint32, padded

    def __init__(self, rank: int, world: int, group, rows_cap: int, dim: int, device: torch.device):
        import torch.distributed as dist

        self.rank, self.world, self.rows_cap, self.dim = rank, world, rows_cap, dim
        self.buf_bytes = (rows_cap * dim * 2 + 255) & ~255
        self.total = self.FLAG_BYTES + 2 * self.buf_bytes
        self.base = _abi.comm_alloc(self.total)
        handle = _abi.comm_export(self.base)
        handles: List[Optional[bytes]] = [None] * world
        dist.all_gather_object(handles, handle, group=group)
        self.peers: List[int] = []  # mapped base pointers of the other ranks, in rank order
        for r in range(world):
            if r != rank:
                self.peers.append(_abi.comm_open(handles[r]))
        self.state = torch.zeros(2, 64, dtype=torch.int32, device=device)  # per parity: [0] epoch, [32] done counter (separate lines)
        self.calls = 0
        self._structs: Dict[int, "_abi.MoeCommStruct"] = {}
        dist.barrier(group=group)  # nobody writes a peer before every rank has mapped everything

    def yw_ptr(self, parity: int) -> int:
        """Device pointer of this rank's row buffer of `parity` (inside the IPC-exported allocation)."""
        return self.base + self.FLAG_BYTES + parity * self.buf_bytes

    def struct(self, parity: int) -> "_abi.MoeCommStruct":
        s = self._structs.get(parity)
        if s is None:
            s = _abi.MoeCommStruct()
            s.n_ranks, s.my_rank = self.world, self.rank
            for i, pb in enumerate(self.peers):
                s.peer_yw[i] = pb + self.FLAG_BYTES + parity * self.buf_bytes
                s.peer_flags[i] = pb + parity * 4 * 64
            s.my_flags = self.base + parity * 4 * 64
            s.epoch = self.state[parity].data_ptr()
            s.done_counter = self.state[parity].data_ptr() + 32 * 4
            self._structs[parity] = s
        return s

    def close(self) -> None:
        for pb in self.peers:
            _abi.comm_close(pb)
        self.peers = []
        if self.base:
            _abi.comm_free(self.base)
            self.base = 0


class MoeLayer(nn.Module):
    def __init__(self, experts: Dict[int, nn.Module], gate_weight: nn.Parameter, moe_args: MoeArgs,
                 expert_shard: Tuple[int, int] = (0, 1), expert_group=None):
        """`experts`: the LOCAL experts keyed by global expert id (all of them when unsharded; a list is accepted too)."""
        super().__init__()
        if not isinstance(experts, dict):
            experts = dict(enumerate(experts))
        assert len(experts) > 0
        # keyed by the GLOBAL expert id so that the reference's key names `experts.{e}.w1.weight` stay valid on every rank
        self.experts = nn.ModuleDict({str(e): m for e, m in sorted(experts.items())})
        self.gate_weight = gate_weight  # [E, dim]
        self.args = moe_args
        self.expert_shard = expert_shard
        self.expert_group = expert_group
        self.layer_parity = 0  # set by the model: consecutive MoE layers alternate the exchange buffer
        first = self.experts[str(self.local_expert_ids[0])]
        # the experts' storage format, one of EXPERT_WEIGHTS: which grouped entry point runs and which tensors it reads
        self.expert_weights = "fp8" if isinstance(first, Fp8Expert) else ("int4" if isinstance(first, Int4Expert) else "bf16")
        self.lora = first.lora if isinstance(first, Fp8Expert) else None  # un-merged adapters: FP8 experts only
        self._ptrs = None
        self._lora_ptrs = None

    @property
    def gate(self) -> _GateView:
        return _GateView(self)

    @property
    def local_expert_ids(self) -> List[int]:
        return sorted(int(e) for e in self.experts.keys())

    @property
    def sharded(self) -> bool:
        return self.expert_shard[1] > 1

    @property
    def fp8(self) -> bool:
        return self.expert_weights == "fp8"

    def _weight_tables(self):
        """HOST arrays of E device pointers (NULL for experts of other ranks), rebuilt when a weight moved: (w13, w2), for FP8
        experts (w13_q, w13 scales, w2_q, w2 scales), for INT4 experts (w13 codes, w13 group scales, w2 codes, w2 group scales)."""
        if self.expert_weights == "fp8":
            tensors = lambda ex: (ex.w13_q, ex.w13_scale_bits, ex.w2_q, ex.w2_scale_bits)  # noqa: E731
        elif self.expert_weights == "int4":
            tensors = lambda ex: (ex.w13, ex.w13_gscale_bits, ex.w2_weight, ex.w2_gscale_bits)  # noqa: E731
        else:
            tensors = lambda ex: (ex.w13, ex.w2_weight)  # noqa: E731
        return self._pointer_tables("_ptrs", tensors)

    def _adapter_tables(self):
        """The same for the FP8 experts' packed adapters: (w13 A, w13 B, w2 A, w2 B)."""
        return self._pointer_tables("_lora_ptrs", lambda ex: (ex.w13_lora.a, ex.w13_lora.b, ex.w2_lora.a, ex.w2_lora.b))

    def _pointer_tables(self, cache: str, tensors):
        """One HOST array of E device pointers per tensor that `tensors(expert)` returns, cached in attribute `cache` until a pointer
        changes."""
        E = self.args.num_experts
        key = tuple((e, *(t.data_ptr() for t in tensors(self.experts[str(e)]))) for e in self.local_expert_ids)
        cached = getattr(self, cache)
        if cached is None or cached[0] != key:
            tables = [(ctypes.c_void_p * E)() for _ in key[0][1:]]
            for e in self.local_expert_ids:
                for tab, t in zip(tables, tensors(self.experts[str(e)])):
                    tab[e] = t.data_ptr()
            cached = (key, tables)
            setattr(self, cache, cached)
        return cached[1]

    def run(self, hn: torch.Tensor, residual: Optional[torch.Tensor], ws: "_abi.Workspace") -> torch.Tensor:
        """`hn` = ffn_norm(h) [T, dim]; returns residual + moe(hn) (or moe(hn) when residual is None)."""
        T, dim = hn.shape
        first = self.experts[str(self.local_expert_ids[0])]
        E, k = self.args.num_experts, self.args.num_experts_per_tok
        out = torch.empty_like(hn)
        tables = self._weight_tables()
        lora_tables = self._adapter_tables() if self.lora is not None else None
        lora_cols = first.w13_lora.rank_cols if self.lora is not None else 0
        g, G = self.expert_shard
        for r0 in range(0, T, MOE_BLOCK_TOKENS):
            r1 = min(T, r0 + MOE_BLOCK_TOKENS)
            n = r1 - r0
            comm = ws.expert_comm(self, n, dim) if self.sharded else None
            b = ws.moe_buffers(n, dim, first.hidden_dim, E, k, hn.dtype, comm, self.layer_parity, lora_cols)
            assert comm is None or b.rows_cap <= comm.rows_cap
            _abi.moe_route(hn[r0:r1], self.gate_weight, E, k, g, G, b)
            res = residual[r0:r1] if residual is not None else None
            cs = comm.struct(self.layer_parity) if comm is not None else None
            if lora_tables is not None:
                a13, b13, a2, b2 = lora_tables
                l13 = _abi.moe_lora_struct(a13, b13, first.w13_lora.rank_cols, first.w13_lora.scaling, b.lora_a, b.lora_l)
                r2 = first.w2_lora.rank_cols
                l2 = _abi.moe_lora_struct(a2, b2, r2, first.w2_lora.scaling, b.lora_a.view(-1)[: b.rows_cap * r2].view(b.rows_cap, r2), b.lora_l)
                _abi.moe_grouped_ffn_fp8_lora(b, *tables, res, out[r0:r1], n, dim, first.hidden_dim, E, k, cs, ws, l13, l2)
            elif self.expert_weights == "fp8":
                _abi.moe_grouped_ffn_fp8(b, *tables, res, out[r0:r1], n, dim, first.hidden_dim, E, k, cs, ws)
            elif self.expert_weights == "int4":
                _abi.moe_grouped_ffn_int4(b, *tables, res, out[r0:r1], n, dim, first.hidden_dim, E, k, cs, ws)
            else:
                _abi.moe_grouped_ffn(b, *tables, res, out[r0:r1], n, dim, first.hidden_dim, E, k, cs, ws)
        return out

    def forward(self, inputs: torch.Tensor, ws: Optional["_abi.Workspace"] = None) -> torch.Tensor:
        """`inputs` = ffn_norm(h) [T, dim] (already normed, like the reference's MoeLayer.forward); returns the expert mixture."""
        T, dim = inputs.shape
        first = self.experts[str(self.local_expert_ids[0])]
        ws = ws or _abi.Workspace(_abi.workspace_bytes(T, dim, 1, 1, 128, first.hidden_dim, 0, 1), inputs.device)
        return self.run(inputs, None, ws)
