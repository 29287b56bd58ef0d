"""Multi-GPU use of the projector: one process per GPU, crops sharded across ranks, weights replicated.

The projector itself needs no collective (every crop is independent, builder.py:107-137 has no cross-crop op), and the
crops normally arrive already sharded because the CLIP tower upstream is data parallel.  The only exchange step of the
path is the reassembly of per-image HD token sequences (llava_arch.py:139-155) when an image's crops live on different
ranks: one all-gather of the projected crop blocks over NVLink (NCCL), then the packed assembly on every rank.
Host logic only — works with the gloo backend on CPU tensors for tests; device work goes through the C ABI.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, world: int, rank: int):
    """Contiguous block partition [lo, hi) of n_items over world ranks (sizes differ by at most one)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_counts(n_items: int, world: int):
    return [shard_bounds(n_items, world, r)[1] - shard_bounds(n_items, world, r)[0] for r in range(world)]


def all_gather_crops(local: torch.Tensor, counts: Sequence[int], group=None) -> torch.Tensor:
    """All-gather per-rank crop blocks [n_r, M, H] (n_r = counts[r]) into [sum(counts), M, H] on every rank.

    Equal counts take the single-buffer NCCL path (all_gather_into_tensor); ragged counts are padded to the maximum."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if len(counts) != world or local.shape[0] != counts[rank]:
        raise ValueError(f"rank {rank}: local block has {local.shape[0]} crops, counts say {list(counts)}")
    local = local.contiguous()
    tail = tuple(local.shape[1:])
    if len(set(counts)) == 1 and dist.get_backend(group) == "nccl":
        out = local.new_empty((sum(counts),) + tail)
        dist.all_gather_into_tensor(out, local, group=group)
        return out
    mx = max(counts)
    padded = local
    if local.shape[0] != mx:
        padded = local.new_zeros((mx,) + tail)
        padded[: local.shape[0]] = local
    bufs = [local.new_empty((mx,) + tail) for _ in range(world)]
    dist.all_gather(bufs, padded, group=group)
    return torch.cat([b[:c] for b, c in zip(bufs, counts)], dim=0)


class ShardedTokenPacker:
    """Data-parallel wrapper: ``projector`` is a (replicated) TokenPackerB200 on this rank's GPU."""

    def __init__(self, projector, group=None):
        self.projector = projector
        self.group = group

    def forward_local(self, x_local):
        """This rank's crops only — no communication."""
        return self.projector(x_local)

    def forward_gathered(self, x_local, counts: Sequence[int]):
        """Project this rank's crops, then all-gather so every rank holds all [N, M, H] crop blocks."""
        return all_gather_crops(self.forward_local(x_local), counts, self.group)

    def forward_hd(self, x_local, counts: Sequence[int], h_block, w_block, sep_row, ret_row):
        """HD path across ranks: local projection -> all-gather -> per-image packed assembly (every rank gets all images)."""
        from .hd import hd_assemble
        feats = self.forward_gathered(x_local, counts)
        return hd_assemble(feats, h_block, w_block, sep_row, ret_row)


class FusedGatherTokenPacker:
    """Projector whose last GEMM stores straight into every rank's output buffer over NVLink (TMA stores to peer-mapped
    memory from ``torch.distributed._symmetric_memory``): compute and the all-gather are ONE kernel, transfers overlap the
    remaining tiles' math.  ``forward_hd`` goes one step further: the stores land in the PACKED per-image rows of
    llava_arch.py:139-155 on every rank (uniform crop stride M + 1, see ``tp_forward_packed``), so there is no gathered
    intermediate and no assembly pass — each rank only fills the separator rows of its own copy.  CUDA + NCCL-capable ranks of
    one NVLink domain only; inference only.  ``forward_hd`` needs crops of a multiple of 4 tokens: scale factors 8 and 24 (9 and 1
    tokens) raise TokenPackerError (invalid argument) from tp_forward_allgather, which launches no projector work for them;
    ``forward_gathered`` serves them.

    Two buffers alternate between calls, so ONE cross-rank barrier per call is enough: the barrier of call i+1 (which
    every rank reaches only after its stream has consumed call i's buffer) is what licenses call i+2 to overwrite that buffer."""

    def __init__(self, projector, group=None):
        self.projector = projector
        self.group = group if group is not None else dist.group.WORLD
        self._bufs = {}
        self._calls = {}

    def _buffers(self, shape, device):
        import torch.distributed._symmetric_memory as symm_mem
        if shape not in self._bufs:
            bufs = []
            for _ in range(2):
                t = symm_mem.empty(shape, dtype=torch.bfloat16, device=device)
                bufs.append((t, symm_mem.rendezvous(t, self.group)))
            bufs[0][1].barrier(channel=0)        # nobody starts writing before everybody has mapped the buffers
            self._bufs[shape], self._calls[shape] = bufs, 0
        i = self._calls[shape]
        self._calls[shape] = i + 1
        return self._bufs[shape][i % 2]

    def forward_gathered(self, x_local, counts: Sequence[int]):
        """Returns the gathered [sum(counts), M, H] crop blocks — a view of a symmetric buffer that stays valid until the call
        after next."""
        rank = dist.get_rank(self.group)
        device = x_local[0].device
        buf, hdl = self._buffers((int(sum(counts)), self.projector.num_queries, self.projector.hidden_size), device)
        if counts[rank] > 0:            # a rank may own no crops of a small batch: it still takes part in the barrier
            self.projector.forward_into_peers(x_local, list(hdl.buffer_ptrs), int(sum(counts[:rank])))
        hdl.barrier(channel=0)          # every rank's stores have landed everywhere
        return buf

    def forward_hd(self, x_local, counts: Sequence[int], h_block, w_block, sep_row, ret_row):
        """HD path across ranks in ONE pass: returns (packed [sum(L_i), H], cu_seqlens) — the packed tensor is a view of a
        symmetric buffer that stays valid until the call after next."""
        from .hd import fill_separators, hd_layout
        proj = self.projector
        rank = dist.get_rank(self.group)
        device = x_local[0].device
        m, hidden = proj.num_queries, proj.hidden_size
        total_crops = int(sum(counts))
        plan, _, sep_rows, ret_rows, total_rows = hd_layout(h_block, w_block, m, device, total_crops, "the ranks hold {}")
        assert total_rows == total_crops * (m + 1)
        buf, hdl = self._buffers((total_rows, hidden), device)
        with torch.cuda.device(device):
            # separator rows of MY copy (local stores; peers only ever write crop rows)
            fill_separators(buf, sep_row, ret_row, sep_rows, ret_rows)
        if counts[rank] > 0:
            proj.forward_into_peers(x_local, list(hdl.buffer_ptrs), int(sum(counts[:rank])), out_crop_rows=m + 1)
        hdl.barrier(channel=0)          # every rank's stores have landed everywhere
        return buf, plan.cu_seqlens
