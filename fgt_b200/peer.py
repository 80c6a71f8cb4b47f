"""Peer-mapped device buffers and the device-side barrier for the multi-GPU exchange (one process per GPU).

Buffers come from the C-ABI (`fgt_peer_alloc`: cudaMalloc, IPC-capable), their 64-byte CUDA IPC handles are
exchanged over the torch.distributed group (any backend — only host bytes travel) and imported by every
peer, after which kernels store straight into the peers' memory over NVLink / NVSwitch
(`fgt_rownorm_bcast`) and order those stores with `fgt_peer_barrier` (release / acquire at system scope,
graph-replayable). The reference has no counterpart: its inference is single-device (SURVEY §8e).
"""
import ctypes

import torch
import torch.distributed as dist

from . import lib


class _Raw:
    """CUDA array interface over a raw device allocation, so torch can view it without copying."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class PeerGroup:
    def __init__(self, group=None, rank=None, world=None):
        self.group = group
        self.world = world if world is not None else (dist.get_world_size(group) if dist.is_initialized() else 1)
        self.rank = rank if rank is not None else (dist.get_rank(group) if dist.is_initialized() else 0)
        if self.world > 8:
            raise ValueError("PeerGroup: at most 8 ranks (one NVSwitch domain)")
        self._local, self._imported, self._keep = [], [], []
        # flags: world uint64 written by the peers + this rank's epoch counter
        self.flag_ptrs, _ = self.alloc(8 * (self.world + 1))
        self.epoch_ptr = self.flag_ptrs[self.rank] + 8 * self.world
        self._flag_arr = (ctypes.c_void_p * self.world)(*self.flag_ptrs)

    def alloc(self, nbytes):
        """Collective: every rank allocates `nbytes` (zeroed). Returns ([address on this rank of rank q's buffer
        for q in ranks], uint8 torch view of the local buffer)."""
        p = ctypes.c_void_p()
        lib.call("fgt_peer_alloc", nbytes, ctypes.byref(p))
        self._local.append(p.value)
        handle = ctypes.create_string_buffer(64)
        lib.call("fgt_peer_export", p, handle)
        handles = [None] * self.world
        if self.world > 1:
            dist.all_gather_object(handles, handle.raw, group=self.group)
        ptrs = []
        for q in range(self.world):
            if q == self.rank:
                ptrs.append(p.value)
                continue
            r = ctypes.c_void_p()
            lib.call("fgt_peer_import", handles[q], ctypes.byref(r))
            self._imported.append(r.value)
            ptrs.append(r.value)
        raw = _Raw(p.value, nbytes)
        self._keep.append(raw)
        view = torch.as_tensor(raw, device=torch.device("cuda", torch.cuda.current_device()))
        return ptrs, view

    def barrier(self):
        """Enqueue the device-side barrier on the current stream (no host synchronisation)."""
        lib.call("fgt_peer_barrier", self._flag_arr, self.world, self.rank, self.epoch_ptr)

    def close(self):
        """Unimports the peers' buffers and frees this rank's, attempting every one; raises the first failure."""
        torch.cuda.synchronize()
        failed = []
        for r in self._imported:
            try:
                lib.call("fgt_peer_unimport", r)
            except RuntimeError as e:
                failed.append(e)
        if self.world > 1:
            dist.barrier(group=self.group)  # nobody frees memory a peer still has mapped
        for p in self._local:
            try:
                lib.call("fgt_peer_free", p)
            except RuntimeError as e:
                failed.append(e)
        self._imported, self._local, self._keep = [], [], []
        if failed:
            raise failed[0]
