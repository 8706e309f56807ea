"""
Multi-GPU plumbing (one process per GPU, torch.distributed): the image is partitioned by scanline — row y
belongs to rank y % world — every rank renders its rows with the scene replicated, and ONE gather of the
radiance slabs to rank 0 ends the frame (BASELINE.json north_star; SURVEY 8e).  No other collective exists
on the data path.  Backend "nccl" on the GPUs (NVLink / NVSwitch), "gloo" in the CPU tests.

A rank's slab is local_rows x width float4, local row r = image row rank + r * world.  Ranks can own one row
less than rank 0 when world does not divide the height, so slabs are padded to rows_max for the gather.
"""
import numpy as np
import torch
import torch.distributed as dist


def local_rows(height: int, rank: int, world: int) -> int:
    return (height - rank + world - 1) // world if height > rank else 0


def rows_max(height: int, world: int) -> int:
    return (height + world - 1) // world


class RadianceGather:
    """Pre-allocated buffers for the per-frame gather; `slab` is the rank's radiance as a (n_local, 4) float32 tensor
    (zero-copy view of the device buffer on GPU)."""

    def __init__(self, width: int, height: int, rank: int, world: int, device):
        self.width, self.height, self.rank, self.world = width, height, rank, world
        self.n_local = local_rows(height, rank, world) * width
        self.n_pad = rows_max(height, world) * width
        self.send = torch.zeros((self.n_pad, 4), dtype=torch.float32, device=device)
        # rank 0 receives into ONE contiguous (world, n_pad, 4) buffer: slab r at recv_all[r], the layout
        # rt_resolve_gathered reads through (recv_ptr, recv_stride_bytes)
        self.recv_all = torch.zeros((world, self.n_pad, 4), dtype=torch.float32, device=device) if rank == 0 else None
        self.recv = list(self.recv_all.unbind(0)) if rank == 0 else None
        self.recv_ptr = self.recv_all.data_ptr() if rank == 0 and self.recv_all.is_cuda else None
        self.recv_stride_bytes = self.n_pad * 16

    def gather(self, slab: torch.Tensor):
        """The one collective of the frame.  Returns the list of padded slabs on rank 0, None elsewhere."""
        if self.world == 1:
            return [slab]
        if self.n_local == self.n_pad and slab.shape[0] == self.n_pad:
            dist.gather(slab, self.recv, dst=0)                 # every rank owns rows_max rows: gather straight from the device slab
        else:
            self.send[: self.n_local].copy_(slab[: self.n_local])
            dist.gather(self.send, self.recv, dst=0)
        return self.recv

    def reassemble(self, slabs) -> np.ndarray:
        """Rank 0: padded slabs -> full height x width x 4 image (host)."""
        img = np.zeros((self.height, self.width, 4), dtype=np.float32)
        for r, s in enumerate(slabs):
            n = local_rows(self.height, r, self.world)
            img[r::self.world] = s[: n * self.width].reshape(n, self.width, 4).cpu().numpy()
        return img


class SharedHostImage:
    """One width x height RGBA32F image in POSIX shared memory, mapped by every rank of the node and (on a GPU box)
    page-locked in every process, so that each rank's rt_resolve writes ITS rows straight into the final image over its own
    PCIe link (rt_resolve leaves the rows of other ranks untouched).  After `complete()` — one barrier — rank 0 holds the
    whole frame on the host.  This is the parallel read-back path; the alternative is rt_resolve_gathered on rank 0 after
    the NCCL gather (one PCIe link).  Collective: construct and close on all ranks."""

    def __init__(self, width: int, height: int, rank: int, world: int, register_cuda: bool = True):
        from multiprocessing import shared_memory
        self.rank, self.world = rank, world
        self.shm, self.image, self.pinned = None, None, False
        nbytes = width * height * 16
        name = [None]
        if rank == 0:
            try:
                self.shm = shared_memory.SharedMemory(create=True, size=nbytes)
                name[0] = self.shm.name
            except Exception:
                name[0] = None
        if world > 1:
            dist.broadcast_object_list(name, src=0)
        ok = name[0] is not None
        if ok and rank != 0:
            try:
                self.shm = shared_memory.SharedMemory(name=name[0])
                try:    # the creating rank owns the segment; keep this process's resource tracker from unlinking it at exit
                    from multiprocessing import resource_tracker
                    resource_tracker.unregister(self.shm._name, "shared_memory")
                except Exception:
                    pass
            except Exception:
                ok = False
        if world > 1:   # every rank learns whether every rank mapped the segment (no rank is left waiting in a later barrier)
            dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
            flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=dev)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
            ok = bool(int(flag[0]))
        if not ok:
            self._release()
            raise RuntimeError("SharedHostImage: the shared-memory image could not be created / mapped on every rank")
        self.image = np.ndarray((height, width, 4), dtype=np.float32, buffer=self.shm.buf)
        if register_cuda and torch.cuda.is_available():
            err = torch.cuda.cudart().cudaHostRegister(self.image.ctypes.data, nbytes, 0)
            self.pinned = int(err) == 0         # not fatal: an unregistered mapping is read back through a staging copy

    def _release(self):
        self.image = None
        if self.shm is not None:
            self.shm.close()
            if self.rank == 0:
                try:
                    self.shm.unlink()
                except Exception:
                    pass
            self.shm = None

    def complete(self):
        """Every rank has finished writing its rows (each rank calls this after its blocking rt_resolve)."""
        if self.world > 1:
            dist.barrier()

    def close(self):
        if self.world > 1:
            dist.barrier()
        if self.pinned:
            torch.cuda.cudart().cudaHostUnregister(self.image.ctypes.data)
            self.pinned = False
        self._release()


class FusedGather:
    """The frame's one collective done by the frame kernels themselves (include/rt_b200.h, rt_set_gather_target): rank 0 owns a
    buffer of `world` radiance slabs + completion flags on its GPU, every other rank maps it through CUDA IPC (NVLink peer
    memory) and its frame kernel stores a pixel's radiance there the moment the pixel's path ends.  torch.distributed only
    carries the 64-byte IPC handle at set-up; no collective runs per frame.  `ok` is False (on every rank) when the mapping could
    not be set up on some rank — callers then fall back to RadianceGather (NCCL)."""

    def __init__(self, ctx, rank: int, world: int):
        from . import capi
        self.ctx, self.rank, self.world = ctx, rank, world
        self.ptr = self.stride = None
        err = None
        handle = [None]
        try:
            if rank == 0:
                self.ptr, self.stride, _ = ctx.gather_buffer()
                handle = [(capi.ipc_export(self.ptr), self.stride)]
        except Exception as e:          # noqa: BLE001
            err = repr(e)
        if world > 1:
            dist.broadcast_object_list(handle, src=0)
        try:
            if err is None and rank != 0:
                if handle[0] is None:
                    raise RuntimeError("rank 0 could not export the buffer")
                self.stride = handle[0][1]
                self.ptr = ctx.ipc_open(handle[0][0])
            if err is None:
                ctx.set_gather_target(self.ptr, self.stride)
        except Exception as e:          # noqa: BLE001
            err = repr(e)
        flags = [err]
        if world > 1:
            all_err = [None] * world
            dist.all_gather_object(all_err, err)
            flags = all_err
        self.errors = [e for e in flags if e]
        self.ok = not self.errors
        if not self.ok:
            try:
                ctx.set_gather_target(None)
            except Exception:           # noqa: BLE001
                pass

    def wait(self):
        """Rank 0: the render stream waits until every rank has delivered the frame rendered last."""
        if self.rank == 0:
            self.ctx.gather_wait()

    def close(self):
        try:
            self.ctx.set_gather_target(None)
        except Exception:               # noqa: BLE001
            pass
