"""
Multi-GPU plumbing (one process per GPU, torch.distributed).

The planning path shards trivially: scenarios are independent, there is NO data-path collective (SURVEY 8(e)).  What
crosses GPUs is bookkeeping around it:
  * ``broadcast_lattice``  -- rank 0 packs the read-only lattice blob once, every other rank receives the bytes
    (NCCL broadcast on the device, over NVLink / NVSwitch) and builds its own handle on them;
  * ``PeerGather``         -- the gather of the action sets into ONE consumer rank without a collective call: every rank's
    exporting kernels (k_vel_res on first ticks, k_export on stateful ticks, k_emergency) store their fp32 rows straight
    into the consumer's HBM through a peer pointer
    (symmetric memory over NVLink), so only LIVE rows cross the fabric, fused into the kernel that produces them; one
    small peer copy of the per-path arrays and one device-side barrier per tick complete it;
  * ``gather_rows``        -- the same gather with point-to-point sends of the live rows (row counts are exchanged
    first): fallback where peer memory is not available, and the path the world_size-2 ``gloo`` tests cover on CPU.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import capi
from .lattice_blob import pack_lattice

_CAP_KEYS = ("h_max", "max_window_edges", "p0_max", "p_max", "max_plan_layers")


def shard_indices(n: int, rank: int, world: int) -> np.ndarray:
    """scenario i is planned by rank i % world."""
    return np.arange(rank, n, world)


def broadcast_lattice(lattice, device, src: int = 0) -> tuple:
    """returns (LatticeHeader, capacities dict, blob tensor on `device`).  `lattice` is only needed on rank `src`."""
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    hsize = C.sizeof(capi.LatticeHeader)
    if rank == src:
        header, blob, cap = pack_lattice(lattice)
        meta = np.zeros(hsize + 8 * len(_CAP_KEYS), dtype=np.uint8)
        meta[:hsize] = np.frombuffer(bytes(header), dtype=np.uint8)
        meta[hsize:] = np.array([cap[k] for k in _CAP_KEYS], dtype=np.int64).view(np.uint8)
        meta_t = torch.from_numpy(meta).to(device)
    else:
        meta_t = torch.zeros(hsize + 8 * len(_CAP_KEYS), dtype=torch.uint8, device=device)
    if world > 1:
        dist.broadcast(meta_t, src=src)
    meta_h = meta_t.cpu().numpy()
    header = capi.LatticeHeader.from_buffer_copy(meta_h[:hsize].tobytes())
    cap = dict(zip(_CAP_KEYS, (int(v) for v in meta_h[hsize:].view(np.int64))))
    if rank == src:
        blob_t = torch.from_numpy(blob).to(device)
    else:
        blob_t = torch.empty(int(header.blob_bytes), dtype=torch.uint8, device=device)
    if world > 1:
        dist.broadcast(blob_t, src=src)
    return header, cap, blob_t


def gather_rows(rows: torch.Tensor, n_rows: int, dst: int = 0, out: torch.Tensor = None) -> tuple:
    """gather the first ``n_rows`` rows of every rank's ``rows`` tensor on rank ``dst``: the counts are all-gathered, then
    every rank sends exactly its live rows.  Returns (gathered tensor on ``dst`` -- rank r's rows at
    [offsets[r], offsets[r] + counts[r]) -- or None elsewhere, counts).  Works with nccl (device tensors) and gloo."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return rows[:n_rows], [int(n_rows)]
    world, rank = dist.get_world_size(), dist.get_rank()
    cnt = torch.tensor([int(n_rows)], dtype=torch.int64, device=rows.device)
    all_cnt = torch.empty(world, dtype=torch.int64, device=rows.device)
    dist.all_gather_into_tensor(all_cnt, cnt)
    counts = [int(v) for v in all_cnt.cpu().tolist()]
    total = sum(counts)
    ops = []
    if rank == dst:
        if out is None or out.shape[0] < total or out.shape[1:] != rows.shape[1:] or out.dtype != rows.dtype:
            out = torch.empty((max(total, 1),) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
        off = 0
        for r in range(world):
            if r == dst:
                out[off:off + counts[r]].copy_(rows[:counts[r]])
            elif counts[r]:
                ops.append(dist.P2POp(dist.irecv, out[off:off + counts[r]], r))
            off += counts[r]
    elif counts[rank]:
        ops.append(dist.P2POp(dist.isend, rows[:counts[rank]].contiguous(), dst))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    return (out[:total] if rank == dst else None), counts


class PeerGather(object):
    """Action sets of all ranks in the consumer rank's HBM, written there by the producing kernels themselves.

    Every rank owns one region of a symmetric-memory buffer on ``dst``: [rows_cap][n_export][7] fp32 rows followed by a
    copy of the packed per-path arrays (BatchPlanner.d_meta_raw: traj_len, traj_id, action_id, traj_row, queue_cnt, ...).
    ``attach`` binds the planner's export rows (LtplBuffers.traj) to the peer region through
    BatchPlanner.set_export_rows, which every later binding keeps until ``detach``, so the exporting kernels store
    their rows over NVLink while they compute them -- the compact row index comes from the rank-local counter, only
    live rows move.  ``finish`` (on the planner's stream, after the tick) copies the per-path arrays into the region and
    runs the device-side barrier of the symmetric-memory handle; behind it the consumer may read every region."""

    def __init__(self, planner, group=None, dst: int = 0):
        import torch.distributed._symmetric_memory as symm_mem
        self.pl = planner
        self.dst = dst
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        d = planner.dims
        self.rows_cap = (capi.NSLOT + 1) * int(d.batch)
        self.row_bytes = int(d.n_export) * 7 * 4
        rows_bytes = (self.rows_cap * self.row_bytes + 255) // 256 * 256
        self.meta_bytes = int(planner.d_meta_raw.numel())
        self.region_bytes = rows_bytes + (self.meta_bytes + 255) // 256 * 256
        sizes = torch.tensor([self.region_bytes, -self.region_bytes], dtype=torch.int64, device=planner.device)
        dist.all_reduce(sizes, op=dist.ReduceOp.MAX, group=group)
        if int(sizes[0].item()) != -int(sizes[1].item()):   # the consumer parses every region with its own layout
            raise ValueError("PeerGather needs equal shard sizes on all ranks (use gather_rows otherwise)")
        self.rows_bytes = rows_bytes
        self.buf = symm_mem.empty(self.world * self.region_bytes, dtype=torch.uint8, device=planner.device)
        self.hdl = symm_mem.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        # tensor views of this rank's rows and meta slot inside the consumer's buffer (peer memory)
        self.peer_rows = self.hdl.get_buffer(dst, (self.rows_cap * self.row_bytes,), torch.uint8,
                                             self.rank * self.region_bytes).view(torch.float32) \
            .view(self.rows_cap, int(d.n_export), 7)
        self.peer_meta = self.hdl.get_buffer(dst, (self.meta_bytes,), torch.uint8,
                                             self.rank * self.region_bytes + rows_bytes)

    def attach(self) -> None:
        self.pl.set_export_rows(self.peer_rows)

    def detach(self) -> None:
        self.pl.set_export_rows(None)

    def finish(self) -> None:
        self.peer_meta.copy_(self.pl.d_meta_raw, non_blocking=True)
        self.hdl.barrier(channel=0)

    def regions(self) -> list:
        """consumer side: per rank (rows [rows_cap][n_export][7] fp32, packed per-path arrays uint8) views."""
        out = []
        ne = int(self.pl.dims.n_export)
        for r in range(self.world):
            o = r * self.region_bytes
            rows = self.buf[o:o + self.rows_cap * self.row_bytes].view(torch.float32).view(self.rows_cap, ne, 7)
            meta = self.buf[o + self.rows_bytes:o + self.rows_bytes + self.meta_bytes]
            out.append((rows, meta))
        return out
