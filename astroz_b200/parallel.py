"""Satellite-axis sharding across the GPUs of one box (SURVEY.md section 8e).

One process per GPU (torch.distributed, NCCL over NVLink between GPUs, gloo in CPU tests).  Cells are
independent and SDP4 couples only along time *within* a satellite, so the satellite axis shards with no
data-path collective.  The one collective the north star names -- an all-gather of the satellite-major
position/velocity block so every rank holds the whole result -- is `ShardedPropagator.all_gather`.
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np

TILE = 8  # satellites per element tile (astroz_b200/csrc/az_device.cuh kTileSats; src/Constellation.zig:23)


def shard_rows(n_sats: int, world: int, align: int = TILE) -> int:
    """Rows per rank: equal for every rank (an in-place all-gather needs equal counts), tile aligned."""
    per = -(-n_sats // world)
    return -(-per // align) * align


def shard_bounds(n_sats: int, world: int, align: int = TILE) -> list[tuple[int, int]]:
    """Contiguous satellite range [begin, end) of each rank; trailing ranks may be short or empty."""
    rows = shard_rows(n_sats, world, align)
    return [(min(r * rows, n_sats), min((r + 1) * rows, n_sats)) for r in range(world)]


class ShardedPropagator:
    """Rank-local constellation over this rank's satellite range of one catalog.

    backend(tles, grav, device) must provide numSatellites, numSgp4, epochs, classes, referenceEpochJd
    (settable) and propagate_device(jd, fr, pos, vel, status, outputMode, layout, out_num_sats,
    out_sat_offset, stream) -- astroz_b200.Constellation on a GPU.
    """

    def __init__(self, tles: Sequence, rank: int, world: int, device: int = 0, grav: int = 1,
                 backend: Callable | None = None, dist=None):
        if backend is None:
            from .constellation import Constellation as backend
        self.rank, self.world, self.dist = rank, world, dist
        self.n_total = len(tles)
        self.rows = shard_rows(self.n_total, world)
        self.begin, self.end = shard_bounds(self.n_total, world)[rank]
        self.n_local = self.end - self.begin
        self.local = backend(list(tles[self.begin:self.end]), grav, device) if self.n_local else None
        self.reference_epoch = self._agree_reference_epoch()

    def _agree_reference_epoch(self) -> float:
        """The whole catalog's reference epoch = epoch of its first near-earth satellite
        (src/Constellation.zig:139-140); every shard must use the same one so tsince rounds identically."""
        mine = np.array([float("inf"), 0.0])
        if self.local is not None and self.local.numSgp4 > 0:
            first = int(np.flatnonzero(np.asarray(self.local.classes) == 0)[0])
            mine = np.array([float(self.begin + first), float(self.local.epochs[first])])
        if self.dist is not None and self.world > 1:
            import torch

            t = torch.from_numpy(mine.copy())
            dev = None
            if self.dist.get_backend() == "nccl":
                dev = torch.device("cuda", torch.cuda.current_device())
                t = t.to(dev)
            got = [torch.empty_like(t) for _ in range(self.world)]
            self.dist.all_gather(got, t)
            cand = np.stack([g.cpu().numpy() for g in got])
        else:
            cand = mine[None, :]
        best = cand[np.argmin(cand[:, 0])]
        ref = float(best[1]) if np.isfinite(best[0]) else 0.0
        if self.local is not None and np.isfinite(best[0]):
            self.local.referenceEpochJd = ref
        return ref

    @property
    def padded_rows(self) -> int:
        return self.rows * self.world

    def propagate_into_full(self, jd, fr, full_pos, full_vel=None, mode: int = 0, stream: int = 0) -> None:
        """Write this rank's rows into the full satellite-major block [padded_rows, n_times, 3]."""
        if self.local is None:
            return
        self.local.propagate_device(jd, fr, full_pos, full_vel, None, mode, 0, self.padded_rows,
                                    self.rank * self.rows, stream)

    def all_gather(self, full_block) -> None:
        """In-place all-gather of the rank-contiguous row blocks: full_block is [padded_rows, ...] (or
        [k, padded_rows, ...] is NOT supported -- gather pos and vel as one [padded_rows, n_times, 6]-style
        block or call twice)."""
        if self.dist is None or self.world == 1:
            return
        mine = full_block[self.rank * self.rows:(self.rank + 1) * self.rows]
        self.dist.all_gather_into_tensor(full_block, mine)


class SymmetricBlock:
    """The whole (padded_rows, n_times, 3) position and velocity blocks in NVLink-symmetric memory
    (torch.distributed._symmetric_memory): every rank allocates the same buffer, rendezvous maps all
    peers' copies (and, where NVLS is available, one multicast address) into this process.  The fused
    kernels write each rank's rows into every copy, so after `barrier()` all ranks hold the whole block."""

    def __init__(self, padded_rows: int, n_times: int, device, group=None):
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem

        self.torch = torch
        group = group if group is not None else dist.group.WORLD
        self.block = symm_mem.empty((2, padded_rows, n_times, 3), dtype=torch.float64, device=device)
        name = group.group_name if hasattr(group, "group_name") else group
        self.handle = symm_mem.rendezvous(self.block, name)
        self.pos, self.vel = self.block[0], self.block[1]
        vel_off = self.block[1].data_ptr() - self.block[0].data_ptr()
        self.peer_pos = [int(p) for p in self.handle.buffer_ptrs]
        self.peer_vel = [int(p) + vel_off for p in self.handle.buffer_ptrs]
        mc = int(getattr(self.handle, "multicast_ptr", 0) or 0)
        self.mc_pos = mc
        self.mc_vel = mc + vel_off if mc else 0

    @property
    def has_multicast(self) -> bool:
        return self.mc_pos != 0

    def barrier(self) -> None:
        self.handle.barrier(channel=0)


def propagate_gather(sp: ShardedPropagator, sym: SymmetricBlock, jd, fr, velocities: bool = True, stream: int = 0,
                     use_multicast: bool = True) -> None:
    """One fused launch per rank: propagate this rank's satellites and deliver the rows to every GPU
    (multimem.st through the NVSwitch when multicast is mapped, peer stores otherwise)."""
    if sp.local is None:
        return
    if use_multicast and sym.has_multicast:
        sp.local.propagate_gather(jd, fr, mc_pos=sym.mc_pos, mc_vel=sym.mc_vel if velocities else 0,
                                  out_num_sats=sp.padded_rows, out_sat_offset=sp.rank * sp.rows, stream=stream)
    else:
        sp.local.propagate_gather(jd, fr, peer_pos=sym.peer_pos, peer_vel=sym.peer_vel if velocities else None,
                                  out_num_sats=sp.padded_rows, out_sat_offset=sp.rank * sp.rows, stream=stream)


def bind_to_gpu_numa_node(device_index: int) -> dict:
    """Pin this process to the CPUs of the NUMA node its GPU hangs off, so pinned host buffers are allocated
    (first touch) next to the GPU's PCIe root.  Each GPU has its own Gen5 x16 link; with one process per GPU
    and node-local staging the per-GPU device->host rate holds as N grows.  Best effort: returns what it did."""
    import glob
    import os

    info = {"device": device_index, "numa_node": None, "cpus": None}
    try:
        import torch

        props = torch.cuda.get_device_properties(device_index)
        bus = f"{getattr(props, 'pci_domain_id', 0):04x}:{props.pci_bus_id:02x}:{props.pci_device_id:02x}.0"
        path = f"/sys/bus/pci/devices/{bus}/numa_node"
        if not os.path.exists(path):
            cands = glob.glob(f"/sys/bus/pci/devices/*:{props.pci_bus_id:02x}:{props.pci_device_id:02x}.0/numa_node")
            path = cands[0] if cands else path
        node = int(open(path).read().strip())
        if node < 0:
            return info
        cpulist = open(f"/sys/devices/system/node/node{node}/cpulist").read().strip()
        cpus = set()
        for part in cpulist.split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        allowed = cpus & os.sched_getaffinity(0)
        if allowed:
            os.sched_setaffinity(0, allowed)
            info.update(numa_node=node, cpus=len(allowed))
    except Exception as exc:  # sysfs layout differs / no permission: keep the default affinity
        info["error"] = repr(exc)[:120]
    return info
