"""Row-sharded SpMM across GPUs (one process per GPU, torch.distributed / NCCL over NVLink).

SpMM output rows are independent, so the path shards naturally by 1-D row blocks of A
(SURVEY §8e): rank r owns rows [r*M/P, (r+1)*M/P) of A (a `narrow_rows` slice, the reference's
torch_sparse/narrow.py:15-42) and the matching row block of the dense operand X. X must be visible
to every rank; the product stays row-sharded — no reduction. Backward: grad_value is local;
grad_X = A^T grad_out is a full-height partial per rank, so it is reduce-scattered back to row blocks.

Two ways to make X visible:

  * `RowShardedSpMM`: all-gather X once (NCCL), then any number of steps run `local_spmm` with no
    collective inside the step ("broadcast once", BASELINE north_star) — the steady state.
  * `PipelinedRowShardedSpMM`: X changes every step (chained layers), so the gather is part of the
    step. The gather is cut into C chunks issued back to back on NCCL's stream (every rank contributes
    to every chunk, so every NVLink stays busy throughout) and the SpMM of chunk c is launched as soon
    as chunk c has landed — the multiply of chunk c overlaps the transfer of chunks c+1.. . The chunks
    are FEATURE slices of X by default (no partial sums; see the class), column chunks of A optionally.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from . import ops
from .matmul import matmul
from .tensor import SparseTensor


def _world(group) -> int:
    return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1


def _rank(group) -> int:
    return dist.get_rank(group) if dist.is_available() and dist.is_initialized() else 0


class _AllGatherRows(torch.autograd.Function):
    """forward: concatenate every rank's row block (all_gather); backward: reduce_scatter.
    Every rank must hold the same number of rows (pad the last block: `RowShardedSpMM.pad_rows`)."""

    @staticmethod
    def forward(ctx, x_local: Tensor, group) -> Tensor:
        ctx.group = group
        world = _world(group)
        ctx.rows = x_local.size(0)
        if world == 1:
            return x_local
        x_local = x_local.contiguous()
        out = x_local.new_empty((world * x_local.size(0),) + tuple(x_local.shape[1:]))
        dist.all_gather_into_tensor(out, x_local, group=group)
        return out

    @staticmethod
    def backward(ctx, grad_full: Tensor):
        world = _world(ctx.group)
        if world == 1:
            return grad_full, None
        grad_full = grad_full.contiguous()
        out = grad_full.new_empty((ctx.rows,) + tuple(grad_full.shape[1:]))
        dist.reduce_scatter_tensor(out, grad_full, op=dist.ReduceOp.SUM, group=ctx.group)
        return out, None


class RowShardedSpMM:
    """`a_local` is this rank's row block of A with FULL column extent (cols index the gathered X).

    The dense operand is sharded by the SAME block height on every rank: `block_rows(N, world)` =
    ceil(N / world); a rank whose share is shorter pads it with zero rows (`pad_rows`), so that the
    gathered operand has world * block_rows >= N rows, the first N of which are X."""

    def __init__(self, a_local: SparseTensor, reduce: str = "sum", group=None):
        self.a = a_local
        self.reduce = reduce
        self.group = group

    @staticmethod
    def block_rows(n: int, world: int) -> int:
        return (n + world - 1) // world

    @staticmethod
    def partition(a: SparseTensor, rank: int, world: int) -> SparseTensor:
        """Contiguous row block `rank` of `world` (ceil(M / world) rows, the last blocks may be shorter or empty)."""
        M = a.sparse_size(0)
        per = RowShardedSpMM.block_rows(M, world)
        start = min(rank * per, M)
        return a.narrow_rows(start, min(per, M - start))

    @staticmethod
    def pad_rows(x_local: Tensor, rows: int) -> Tensor:
        """Zero-pad a dense row block to `rows` rows (no copy when it already has them)."""
        if x_local.size(0) == rows:
            return x_local
        assert x_local.size(0) < rows
        pad = x_local.new_zeros((rows - x_local.size(0),) + tuple(x_local.shape[1:]))
        return torch.cat([x_local, pad], dim=0)

    def gather_dense(self, x_local: Tensor) -> Tensor:
        world = _world(self.group)
        if world > 1:
            n = self.a.sparse_size(1)
            per = self.block_rows(n, world)
            assert x_local.size(0) <= per, (
                f"dense row block has {x_local.size(0)} rows, expected at most ceil({n} / {world}) = {per}")
            x_local = self.pad_rows(x_local, per)   # equal block heights: what all_gather / reduce_scatter need
        return _AllGatherRows.apply(x_local, self.group)

    def local_spmm(self, x_full: Tensor) -> Tensor:
        n = self.a.sparse_size(1)
        if x_full.size(-2) > n:      # rows added by the padding of the last block
            x_full = x_full.narrow(-2, 0, n)
        return matmul(self.a, x_full, self.reduce)

    def __call__(self, x_local: Tensor) -> Tensor:
        return self.local_spmm(self.gather_dense(x_local))


def split_column_chunks(rowptr: Tensor, col: Tensor, value: Optional[Tensor], block: int, world: int,
                        chunks: int) -> Tuple[List[Tuple[Tensor, Tensor, Optional[Tensor]]], int]:
    """Split a CSR row block (columns over world * block dense rows) into `chunks` column chunks for the pipelined
    gather. Chunk c holds the entries whose column lies in rows [c*mc, (c+1)*mc) of SOME rank's block (mc = block /
    chunks), with the columns re-indexed to the chunk-major layout of the gathered operand:
        col = p * block + c * mc + i   ->   c * (world * mc) + p * mc + i.
    Returns ([(rowptr_c, col_c, value_c)], mc). Entry order inside a row is preserved. Structure-only set-up work."""
    assert block % chunks == 0, f"block height {block} is not divisible by {chunks} chunks"
    mc = block // chunks
    M = rowptr.numel() - 1
    counts = rowptr[1:] - rowptr[:-1]
    row = torch.repeat_interleave(torch.arange(M, device=col.device), counts)
    p = torch.div(col, block, rounding_mode="floor")
    within = col - p * block
    c = torch.div(within, mc, rounding_mode="floor")
    new_col = c * (world * mc) + p * mc + (within - c * mc)
    out = []
    for k in range(chunks):
        sel = (c == k).nonzero().view(-1)
        rp = torch.zeros(M + 1, dtype=torch.long, device=col.device)
        torch.cumsum(torch.bincount(row[sel], minlength=M), 0, out=rp[1:])
        out.append((rp, new_col[sel].contiguous(), None if value is None else value[sel].contiguous()))
    return out, mc


class PipelinedRowShardedSpMM:
    """Sum-SpMM of this rank's row block with a dense operand that is gathered INSIDE the step, chunk by chunk,
    while the chunks that have already landed are being multiplied (forward only; CUDA / NCCL).

    `block` = rows of the dense operand every rank holds (all equal); `chunks` = pipeline depth C.

    split="feature" (default): the operand travels in C FEATURE slices. Slice c is all-gathered as a contiguous
    [world * block, F / C] matrix and multiplied by the whole of A with the ordinary SpMM kernel into slice c of the
    result — no partial sums, the only extra work is that A's index arrays are re-read C times. The fast path keeps
    the slice-major layout on both sides (`forward_sliced`: [C, block, F/C] in, [C, M, F/C] out), which is what a
    chain of layers wants: the output of one step is already laid out for the gather of the next.
    split="column": A's columns are split instead (`split_column_chunks`) and the chunks share an fp32 partial
    (tsb200_spmm_fw_acc). Every chunk re-walks the row structure and read-modify-writes the partial, so it is kept
    for operands that cannot be sliced by features.

    transport="peer" (default on CUDA/NCCL groups): every rank keeps its slices in a symmetric-memory buffer and PULLS
    the peers' slices with cudaMemcpyAsync over NVLink — copy engines only. The SpMM kernel is a persistent grid that
    fills every SM, so a transfer that needs SMs (NCCL's all-gather kernel) cannot run beside it and the "overlap"
    serialises; DMA pulls do overlap. transport="nccl": chunked all_gather_into_tensor."""

    def __init__(self, a_local: SparseTensor, block: int, chunks: int = 4, group=None, split: str = "feature",
                 transport: str = "auto"):
        assert split in ("feature", "column") and transport in ("auto", "peer", "nccl")
        if transport == "auto":   # peer-memory copies need CUDA tensors and the symmetric-memory allocator
            transport = "peer" if (a_local.is_cuda() and split == "feature" and _world(group) > 1
                                   and dist.get_backend(group) == "nccl") else "nccl"
        self.transport = transport
        # concurrent DMA streams of the pulls (default one: concurrent peer copies contend)
        self.peer_streams = int(os.environ.get("TSB200_PEER_STREAMS", "1"))
        self.group = group
        self.world = _world(group)
        self.block = block
        self.chunks = chunks
        self.split = split
        rowptr, col, value = a_local.csr()
        assert a_local.sparse_size(1) == self.world * block
        self.M = a_local.sparse_size(0)
        self.csr = (rowptr, col, value)
        if split == "column":
            self.parts, self.mc = split_column_chunks(rowptr, col, value, block, self.world, chunks)
        self._x = None
        self._partial = None

    # ------------------------------------------------------------------ feature slices
    def to_sliced(self, x: Tensor) -> Tensor:
        """[rows, F] -> slice-major [C, rows, F / C]."""
        rows, F = x.shape
        assert F % self.chunks == 0
        return x.view(rows, self.chunks, F // self.chunks).permute(1, 0, 2).contiguous()

    @staticmethod
    def from_sliced(xs: Tensor) -> Tensor:
        """slice-major [C, rows, Fc] -> [rows, C * Fc]."""
        C, rows, Fc = xs.shape
        return xs.permute(1, 0, 2).reshape(rows, C * Fc)

    # ---- transport 1: copy engines over peer memory (torch symmetric memory), no SM is used by the transfer ----
    def _peer_setup(self, like: Tensor, Fc: int):
        """Collective. Two symmetric input buffers (alternating steps) + views of every peer's buffers."""
        import torch.distributed._symmetric_memory as symm
        group = self.group if self.group is not None else dist.group.WORLD
        self._sym, self._hdl, self._peer = [], [], []
        for _ in range(2):
            buf = symm.empty((self.chunks, self.block, Fc), dtype=like.dtype, device=like.device)
            hdl = symm.rendezvous(buf, group)
            self._sym.append(buf)
            self._hdl.append(hdl)
            self._peer.append([hdl.get_buffer(r, (self.chunks, self.block, Fc), like.dtype)
                               for r in range(self.world)])
        self._copy_streams = [torch.cuda.Stream(device=like.device) for _ in range(self.world)]
        self._step = 0

    def input_buffer(self, like: Tensor, Fc: int) -> Tensor:
        """The symmetric [C, block, Fc] buffer the NEXT step will be gathered from: a producer that writes its slices
        straight into it saves the staging copy `forward_sliced` would otherwise make."""
        if getattr(self, "_sym", None) is None or self._sym[0].dtype != like.dtype or self._sym[0].size(-1) != Fc:
            self._peer_setup(like, Fc)
        return self._sym[self._step & 1]

    def _gather_peer(self, x_sliced: Tensor, xg: Tensor):
        """Pull every peer's slices with cudaMemcpyAsync over NVLink (one copy stream per peer, copy engines only),
        slice by slice; returns per-slice lists of events the compute stream waits on."""
        C, Fc = self.chunks, x_sliced.size(-1)
        mine = self.input_buffer(x_sliced, Fc)
        if x_sliced.data_ptr() != mine.data_ptr():
            mine.copy_(x_sliced)
        k = self._step & 1
        self._step += 1
        # every rank has written buffer k and is done with the step that last read buffer k
        self._hdl[k].barrier()
        me = _rank(self.group)
        cur = torch.cuda.current_stream()
        ready = torch.cuda.Event()
        ready.record(cur)
        events = [[] for _ in range(C)]
        # Peer order is staggered by rank (at hop h every rank pulls from rank me + h: a permutation, so no source
        # serves two pullers in the same hop) and spread round-robin over `peer_streams` copy streams.
        ns = max(1, min(self.peer_streams, self.world - 1))
        for st in self._copy_streams[:ns]:
            st.wait_event(ready)
        for c in range(C):
            for h in range(1, self.world):
                r = (me + h) % self.world
                st = self._copy_streams[(h - 1) % ns]
                with torch.cuda.stream(st):
                    xg[c, r * self.block:(r + 1) * self.block].copy_(self._peer[k][r][c], non_blocking=True)
            for st in self._copy_streams[:ns]:
                ev = torch.cuda.Event()
                ev.record(st)
                events[c].append(ev)
        for c in range(C):   # own rows: a local copy on the compute stream
            xg[c, me * self.block:(me + 1) * self.block].copy_(mine[c], non_blocking=True)
        return events

    def forward_sliced(self, x_sliced: Tensor) -> Tensor:
        """x_sliced [C, block, Fc] (this rank's rows of every feature slice) -> [C, M, Fc]."""
        C, rows, Fc = x_sliced.shape
        assert C == self.chunks and rows == self.block and x_sliced.is_contiguous()
        if self._x is None or self._x.dtype != x_sliced.dtype or self._x.size(-1) != Fc:
            self._x = x_sliced.new_empty((C, self.world * self.block, Fc))
        xg = self._x
        works, events = [], None
        if self.world > 1 and self.transport == "peer":
            events = self._gather_peer(x_sliced, xg)
        else:
            for c in range(C):
                if self.world > 1:
                    works.append(dist.all_gather_into_tensor(xg[c], x_sliced[c], group=self.group, async_op=True))
                else:
                    xg[c].copy_(x_sliced[c])
        rowptr, col, value = self.csr
        value = None if value is None else value.to(x_sliced.dtype)
        out = []
        for c in range(C):
            if works:
                works[c].wait()          # the compute stream waits for slice c only
            if events is not None:
                cur = torch.cuda.current_stream()
                for ev in events[c]:
                    cur.wait_event(ev)
            out.append(ops.spmm_fw(rowptr, col, value, xg[c], "sum")[0])
        return torch.stack(out, dim=0)

    # ------------------------------------------------------------------ column chunks
    def _buffers(self, x_local: Tensor):
        F = x_local.size(1)
        if self._x is None or self._x.dtype != x_local.dtype or self._x.size(-1) != F:
            self._x = x_local.new_empty((self.chunks, self.world * self.mc, F))
            self._partial = torch.empty((self.M, F), dtype=torch.float32, device=x_local.device)
        return self._x, self._partial

    def _forward_columns(self, x_local: Tensor) -> Tensor:
        xg, partial = self._buffers(x_local)
        mc, C = self.mc, self.chunks
        works = []
        for c in range(C):
            src = x_local[c * mc:(c + 1) * mc]
            if self.world > 1:
                works.append(dist.all_gather_into_tensor(xg[c], src, group=self.group, async_op=True))
            else:
                xg[c].copy_(src)
        out = torch.empty((self.M, x_local.size(1)), dtype=x_local.dtype, device=x_local.device)
        x_flat = xg.view(C * self.world * mc, x_local.size(1))
        parts = [(rp, cl, None if v is None else v.to(x_local.dtype)) for rp, cl, v in self.parts]
        for c in range(C):
            if works:
                works[c].wait()          # the compute stream waits for chunk c only
            mode = 1 if c == 0 else (3 if c == C - 1 else 2)
            rp, cl, v = parts[c]
            if C == 1:
                return ops.spmm_fw(rp, cl, v, x_flat, "sum")[0]
            ops.spmm_fw_acc(rp, cl, v, x_flat, partial, out, mode)
        return out

    def __call__(self, x_local: Tensor) -> Tensor:
        """x_local [block, F] -> [M, F] (row-major on both sides; the feature split converts the layout on the way
        in and out — use `forward_sliced` to keep the slice-major layout across steps)."""
        assert x_local.dim() == 2 and x_local.size(0) == self.block and x_local.is_contiguous()
        if self.split == "column":
            return self._forward_columns(x_local)
        return self.from_sliced(self.forward_sliced(self.to_sliced(x_local)))
