"""Sphere-per-rank sharding (SURVEY.md section 8(e)).

Tet-spheres share no vertices (``geometry/tetmesh_geometry.py:305-331`` concatenates them with
index offsets), so every operator is block-diagonal by sphere: each rank owns a contiguous range
of spheres with their vertices, tets and gradient slice -- no halo, no gradient exchange.  The
only cross-rank quantity is the scalar energy: one ``all_reduce(SUM)`` of 3 floats (total,
smoothness, barrier), issued asynchronously so it stays off the critical path of the next
iteration's kernel.

One process per GPU, ``torch.distributed`` (NCCL over NVLink on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from .mesh import TetPack

__all__ = ["partition_spheres", "shard_pack", "ShardedEnergy", "allreduce_energy"]


def partition_spheres(tets_per_sphere: Sequence[int], world_size: int) -> List[Tuple[int, int]]:
    """Contiguous sphere ranges [lo, hi) per rank, balanced by tet count (greedy prefix split).

    Every rank gets a (possibly empty) range; ranges are disjoint and cover all spheres.
    """
    w = np.asarray(tets_per_sphere, dtype=np.int64)
    S = len(w)
    if world_size <= 0:
        raise ValueError("world_size must be positive")
    csum = np.concatenate([[0], np.cumsum(w)])
    total = int(csum[-1])
    bounds = [0]
    for r in range(1, world_size):
        target = total * r / world_size
        j = int(np.searchsorted(csum, target, side="left"))
        # pick the closer of the two neighbouring boundaries, never going backwards
        if j > 0 and abs(csum[j - 1] - target) <= abs(csum[min(j, S)] - target):
            j -= 1
        bounds.append(min(max(j, bounds[-1]), S))
    bounds.append(S)
    return [(bounds[r], bounds[r + 1]) for r in range(world_size)]


def shard_pack(pack: TetPack, rank: int, world_size: int) -> Tuple[TetPack, Tuple[int, int]]:
    """This rank's self-contained sub-pack and its sphere range."""
    sizes = np.diff(pack.tet_offsets)
    lo, hi = partition_spheres(sizes, world_size)[rank]
    return pack.slice_spheres(lo, hi), (lo, hi)


def allreduce_energy(energy: torch.Tensor, group=None, async_op: bool = True):
    """SUM the per-rank energy terms in place.  Returns the work handle (or None if not
    distributed).  4-12 bytes: latency-bound, so callers overlap it with the next launch."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return None
    return dist.all_reduce(energy, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


class ShardedEnergy:
    """Per-rank fused energy+gradient over this rank's spheres plus the scalar all-reduce.

    ``energy_grad(x_local)`` returns (energy[3] device tensor holding the GLOBAL sums once
    ``wait()`` has been called, local gradient [n_local,3]).

    ``deterministic=True`` makes each rank's gradient and local energies bitwise repeatable
    (``TetSpheres(..., deterministic=True)``); the NCCL all-reduce of the energies is outside that guarantee.
    """

    def __init__(self, pack: TetPack, rank: Optional[int] = None, world_size: Optional[int] = None,
                 device=None, group=None, warps_per_cta: int = 0, deterministic: bool = False):
        from . import tet_spheres_ext as ext   # needs the CUDA library + a GPU
        self.group = group
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world_size = dist.get_world_size(group) if world_size is None else world_size
        self.local, self.sphere_range = shard_pack(pack, self.rank, self.world_size)
        self.tet_sp = ext.TetSpheres(self.local.verts.reshape(-1), self.local.tets.reshape(-1),
                                     device=device, warps_per_cta=warps_per_cta,
                                     deterministic=deterministic) if self.local.nele else None
        self._work = None
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = self.tet_sp.device if self.tet_sp is not None else torch.device(device)
        self._comm_stream = torch.cuda.Stream(device=self.device)

    def energy_grad(self, x_local: torch.Tensor, c1: float, c2: float, order: int, gradH=1.0):
        """A rank that owns no spheres (more ranks than spheres) still takes part in the collective: it
        contributes zeros and returns an empty gradient, so the other ranks never wait on it."""
        if self.tet_sp is None:
            energy = torch.zeros(3, dtype=torch.float32, device=self.device)
            grad = torch.empty((0, 3), dtype=torch.float32, device=self.device)
        else:
            energy, grad = self.tet_sp.energy_grad(x_local, c1, c2, order, gradH)
            energy = energy.clone()                 # the all-reduce must not write into the handle's energy ring
        if self.world_size > 1:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self._comm_stream):
                self._comm_stream.wait_event(ev)
                energy.record_stream(self._comm_stream)
                self._work = allreduce_energy(energy, self.group, async_op=True)
        return energy, grad

    def wait(self):
        """Block the current stream until the pending scalar all-reduce has landed."""
        if self._work is not None:
            self._work.wait()
            torch.cuda.current_stream(self.device).wait_stream(self._comm_stream)
            self._work = None
