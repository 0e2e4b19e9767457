"""Multi-GPU plumbing: one process per GPU (torchrun), frames sharded by contiguous ranges, no
data-path collective except ONE all-gather of the output vertices (NCCL over NVLink on GPUs, gloo
in the CPU tests).  The reference's only parallelism is a single-process nn.DataParallel wrapper
(/root/reference/acr/main.py:61) that degenerates to one GPU (SURVEY.md F6)."""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [begin, end) of frames owned by `rank`; remainders go to the low ranks."""
    base, rem = divmod(total, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def gather_vertices(verts: torch.Tensor, counts: torch.Tensor, out: torch.Tensor = None,
                    counts_out: torch.Tensor = None):
    """All-gather the dense per-rank vertex buffers (R, 778, 3) (R = worst-case rows, identical on
    every rank) and the (8,) int32 count vectors.  Returns (world, R, 778, 3), (world, 8).
    Asynchronous w.r.t. the host on NCCL (enqueued on the current stream)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if out is None:
        out = torch.empty((world,) + tuple(verts.shape), dtype=verts.dtype, device=verts.device)
    if counts_out is None:
        counts_out = torch.empty((world,) + tuple(counts.shape), dtype=counts.dtype, device=counts.device)
    if world == 1:
        out[0].copy_(verts)
        counts_out[0].copy_(counts)
        return out, counts_out
    dist.all_gather_into_tensor(out.view(-1), verts.contiguous().view(-1))
    dist.all_gather_into_tensor(counts_out.view(-1), counts.contiguous().view(-1))
    return out, counts_out


def compact_gathered(gathered: torch.Tensor, counts: torch.Tensor) -> List[torch.Tensor]:
    """Valid rows of every rank's shard, in rank order (counts[:, 2] = L+R of each shard)."""
    n = counts[:, 2].tolist()
    return [gathered[r, : int(n[r])] for r in range(gathered.shape[0])]


def parse_rows(batch: int, hands_per_side: int = 1) -> int:
    """Worst-case parse rows of one shard, the ``rows`` a gather buffer needs: 2 * K * batch (K hands per image and
    side, ``max_hands_per_side``), so always even as PeerVertexGather requires."""
    return 2 * int(hands_per_side) * int(batch)


def gather_layout(world: int, rows: int) -> dict:
    """Byte layout of the symmetric gather allocation (include/acr_b200.h, acr_b200_gather): two slots of
    verts[world][rows][778][3] fp32 + counts[world][8] int32, then flags[world] uint64."""
    if rows % 2 or rows <= 0 or not 1 <= world <= 8:
        raise ValueError("gather_layout: rows per rank must be even and positive, world in 1..8")
    verts_bytes = world * rows * 778 * 3 * 4
    counts_offset = (verts_bytes + 15) // 16 * 16
    slot_bytes = (counts_offset + world * 32 + 255) // 256 * 256
    return dict(counts_offset=counts_offset, slot_bytes=slot_bytes, flags_offset=2 * slot_bytes,
                total_bytes=2 * slot_bytes + 256, verts_bytes=verts_bytes)


class PeerVertexGather:
    """Vertex all-gather fused into the MANO kernel (``acr_b200_mano_forward_gather``, protocol in
    include/acr_b200.h).  One symmetric-memory allocation per rank holds TWO gather slots -- each
    ``verts (world, rows, 778, 3)`` fp32 + ``counts (world, 8)`` int32 -- and one arrival flag per rank.
    Launch s writes slot s & 1 of every rank over NVLink (16-byte ``multimem.st`` through the NVLS multicast
    mapping when there is one, 16-byte peer stores otherwise), row counts included, and its last CTA publishes
    s in every rank's flag word.  There is no barrier and no NCCL call: the kernel itself waits (on flags in
    its own memory) until the slot it is about to overwrite has been released, which with two slots is a
    dependency on the PREVIOUS step of the peers.

    ``rows`` is the shard's worst-case parse rows, ``parse_rows(batch, max_hands_per_side)`` = 2KB.

    Contract: consume step k's gathered data (``gathered()`` / ``counts()`` after ``finish()``) on the
    launching stream before the next fused launch -- then no peer can overwrite it while it is read.
    torch symmetric memory only provides the mapped addresses."""

    NV3 = 778 * 3

    def __init__(self, rows: int, device, group=None, use_multicast: bool = True):
        import ctypes as C

        import torch.distributed._symmetric_memory as symm_mem

        from . import lib as L
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.rows = int(rows)
        if self.rows % 2 or self.world > 8:
            raise ValueError("PeerVertexGather: rows per rank must be even and world <= 8")
        self.device = torch.device(device)
        lay = gather_layout(self.world, self.rows)
        self.counts_offset, self.slot_bytes, self.flags_offset = lay["counts_offset"], lay["slot_bytes"], lay["flags_offset"]
        self.buf = symm_mem.empty(lay["total_bytes"], dtype=torch.uint8, device=self.device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, self.group)
        self.local_state = torch.zeros(2, dtype=torch.int64, device=self.device)
        mc = 0
        if use_multicast:
            try:
                if self.hdl.has_multicast_support:
                    mc = int(self.hdl.multicast_ptr or 0)
            except Exception:
                mc = 0
        self.multicast_ptr = mc
        d = L.Gather()
        for r, ptr in enumerate(self.hdl.buffer_ptrs):
            d.peer_base[r] = int(ptr)
        d.multicast_base, d.world, d.rank, d.rows = mc, self.world, self.rank, self.rows
        d.slot_bytes, d.counts_offset, d.flags_offset = self.slot_bytes, self.counts_offset, self.flags_offset
        d.local_state = self.local_state.data_ptr()
        self.desc = d
        self.step = 0            # host mirror of the device step counter (which slot holds the latest data)
        torch.cuda.synchronize(self.device)
        dist.barrier(self.group)          # every rank's flags are zero before anybody publishes

    @property
    def mode(self) -> str:
        return "16-byte multimem.st (NVLS multicast)" if self.multicast_ptr else "16-byte peer stores"

    def note_launch(self) -> None:
        self.step += 1

    def finish(self) -> None:
        """Stream-ordered: returns (on the device) once the latest step of EVERY rank has landed here."""
        from . import lib as L
        with L.on(self.device):
            L.check(L.load().acr_b200_gather_wait(self.desc, L.current_stream(self.device)), "gather_wait")

    def _slot(self) -> torch.Tensor:
        s = self.step & 1
        return self.buf[s * self.slot_bytes: (s + 1) * self.slot_bytes]

    def gathered(self) -> torch.Tensor:
        """(world, rows, 778, 3) view of the slot written by the latest launch (valid after ``finish()``)."""
        n = self.world * self.rows * self.NV3
        return self._slot()[: n * 4].view(torch.float32).view(self.world, self.rows, 778, 3)

    def counts(self) -> torch.Tensor:
        """(world, 8) int32 row counts of every shard, same slot."""
        return self._slot()[self.counts_offset: self.counts_offset + self.world * 32].view(torch.int32).view(self.world, 8)
