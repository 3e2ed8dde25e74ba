"""Peer-memory plumbing of the fused SyncBN kernels (libb3d b3d_cbn_prepare_sync / b3d_cbn_bwd_reduce_sync: a one-shot
all-reduce over NVLink / NVSwitch fused into the kernel that consumes the statistics — sync_batchnorm/batchnorm.py:68-150
of the reference does a thread rendezvous + two comm ops per layer; round 1 here did one NCCL all-reduce per layer).

One process per GPU (torch.distributed, NCCL): a symmetric buffer from torch's symmetric-memory allocator is mapped into
every peer; the kernels get the table of peer pointers.  Falls back to NCCL collectives (b3d.ew) when the backend is not
NCCL or symmetric memory is unavailable."""
import ctypes

import torch
import torch.distributed as dist

from . import lib

lib.b3d_sync_buffer_bytes.restype = ctypes.c_size_t
lib.b3d_sync_flag_offset.restype = ctypes.c_size_t

_state = {"inst": None}


class PeerSync:
    def __init__(self, device):
        import torch.distributed._symmetric_memory as symm_mem
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        if self.world > 8:
            raise RuntimeError("fused SyncBN: at most 8 ranks")
        nbytes = int(lib.b3d_sync_buffer_bytes(self.world))
        group = dist.group.WORLD
        if hasattr(symm_mem, "enable_symm_mem_for_group"):
            try:
                symm_mem.enable_symm_mem_for_group(group.group_name)
            except Exception:
                pass
        self.buf = symm_mem.empty((nbytes + 3) // 4, dtype=torch.float32, device=device)
        self.handle = symm_mem.rendezvous(self.buf, group.group_name)
        self.buf.zero_()
        torch.cuda.synchronize(device)
        dist.barrier()                                          # every rank's flags are zero before the first call
        ptrs = [int(p) for p in self.handle.buffer_ptrs]
        off = int(lib.b3d_sync_flag_offset(self.world))
        self.data = (ctypes.c_void_p * self.world)(*ptrs)
        self.flag = (ctypes.c_void_p * self.world)(*[p + off for p in ptrs])
        self.epoch = torch.zeros(1, device=device, dtype=torch.int32)
        self.err = torch.zeros(1, device=device, dtype=torch.int32)

    def check(self):
        """Host-side check (outside the timed / captured region): a peer timed out inside a fused kernel."""
        if int(self.err.item()) != 0:
            raise RuntimeError("fused SyncBN: a peer did not arrive within 4 s (see csrc/ew_kernels.cu peer_allreduce)")


def peer_sync(device):
    """The process-wide PeerSync, or None (single process, another backend, or symmetric memory unavailable -> NCCL path)."""
    if _state["inst"] is None:
        inst = False
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 \
                and dist.get_backend() == "nccl":
            try:
                inst = PeerSync(device)
            except Exception as e:                              # noqa: BLE001 — any failure of the optional fast path
                if dist.get_rank() == 0:
                    print(f"[b3d.sync] fused SyncBN unavailable ({type(e).__name__}: {e}); using NCCL all-reduces", flush=True)
                inst = False
            # all ranks must agree, or the collective sequences diverge
            flag = torch.tensor([1 if inst else 0], device=device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
            if int(flag.item()) == 0:
                inst = False
        _state["inst"] = inst
    return _state["inst"] or None
