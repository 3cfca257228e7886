"""Data parallelism over collocation points (SURVEY.md §8e): every rank owns a contiguous slice of the batch, weights
and optimizer state are replicated, the per-rank partial gradients -- computed with ``loss_scale = 2 / (N_global n_eq)``
so that they simply add up -- and the partial sums of squared residuals travel in ONE flat buffer ``[grad | sum r^2]``
that is summed over the ranks once per optimizer step: on the GPUs of one node by the hand-written one-shot kernel over
NVLink peer memory (``csrc/pinnjet_comm.cu``, ``pj_allreduce_oneshot``; torch symmetric memory only provides the
peer-mapped allocation), otherwise by the process group's all-reduce (NCCL across nodes, gloo in the CPU tests)."""
import ctypes
import os

import torch


def shard_bounds(n_points, rank, world_size):
    """Half-open slice of rank ``rank`` of a batch of ``n_points`` (slices tile the batch, sizes differ by <= 1)."""
    return (n_points * rank) // world_size, (n_points * (rank + 1)) // world_size


def shard_coords(coords, rank, world_size):
    lo, hi = shard_bounds(coords[0].shape[0], rank, world_size)
    return [c[lo:hi].contiguous() for c in coords]


def all_reduce_gradbuf(gradbuf, dist=None):
    """Sum ``[grad_theta | sum r^2]`` over the ranks, in place.  No-op without an initialised process group."""
    dist = dist or torch.distributed
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(gradbuf)
    return gradbuf


class GradBufReducer:
    """SUM of one flat float32 (or float64) buffer over the ranks, in place; ``mode`` says how: ``"single"`` (no process group),
    ``"oneshot-nvlink"`` (one launch of ``pj_allreduce_oneshot``: every rank reads its peers' copies over NVLink and adds
    them in rank order -- bit-identical results everywhere, CUDA-graph capturable) or ``"process-group"``
    (``dist.all_reduce``).  ``PINNJET_ALLREDUCE=nccl`` forces the last one, and so does a float64 buffer: the NVLink
    collectives push 64-bit {epoch, float32} words.

    ``fused_args`` (one-shot mode only, else ``None``): ``(peer pointers, rank, world)`` of a SECOND symmetric buffer, for
    ``pj_backward_allreduce`` -- the reverse kernel's partial reduction and this collective as one launch
    (``FusedProblem.residual_grad(reducer=...)``); ``PINNJET_FUSED_AR=0`` keeps the two launches."""

    def __init__(self, buf, dist=None):
        dist = dist or torch.distributed
        self.dist, self.mode, self.why, self.fused_args, self.n = dist, "single", "", None, buf.numel()
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        self.mode = "process-group"
        world = dist.get_world_size()
        if not buf.is_cuda:
            self.why = "buffer not on a GPU"
            return
        if buf.dtype == torch.float64:
            self.why = "float64 buffer (the NVLink collectives are float32 only)"
            return
        if os.environ.get("PINNJET_ALLREDUCE", "").lower() in ("nccl", "process-group"):
            self.why = "PINNJET_ALLREDUCE"
            return
        if world > 8:
            self.why = "more than 8 ranks"
            return
        try:
            import torch.distributed._symmetric_memory as symm
            from .engine import load_library
            lib = load_library()
            lib.pj_allreduce_bytes.argtypes = [ctypes.c_int64]
            lib.pj_allreduce_bytes.restype = ctypes.c_int64
            lib.pj_allreduce_oneshot.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                                                 ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]
            lib.pj_allreduce_oneshot.restype = ctypes.c_int
            n = buf.numel()
            words = int(lib.pj_allreduce_bytes(n)) // 4
            self._sym = symm.empty(words, dtype=torch.float32, device=buf.device)
            self._sym.zero_()
            group = dist.group.WORLD
            self._hdl = symm.rendezvous(self._sym, group.group_name)
            if self._hdl.world_size != world:
                raise RuntimeError("symmetric-memory world size mismatch")
            self._ptrs = (ctypes.c_uint64 * world)(*[int(p) for p in self._hdl.buffer_ptrs])
            self._rank, self._world, self._n, self._lib = dist.get_rank(), world, n, lib
            fused = None
            if os.environ.get("PINNJET_FUSED_AR", "1") != "0":   # every rank reads the same environment: same rendezvous count
                words_f = int(lib.pj_backward_allreduce_bytes(n, world)) // 4
                self._sym_f = symm.empty(words_f, dtype=torch.float32, device=buf.device)
                self._sym_f.zero_()
                self._hdl_f = symm.rendezvous(self._sym_f, group.group_name)
                fused = ((ctypes.c_uint64 * world)(*[int(p) for p in self._hdl_f.buffer_ptrs]), self._rank, world)
            torch.cuda.synchronize(buf.device)
            dist.barrier()                      # every rank's flags are zero before anyone signals
            self.mode, self.fused_args = "oneshot-nvlink", fused
        except Exception as exc:  # noqa: BLE001  -- no peer access / symmetric memory: the process group still works
            self.why = f"{type(exc).__name__}: {exc}"

    def __call__(self, buf):
        if self.mode == "oneshot-nvlink" and buf.dtype != torch.float64:
            if buf.numel() != self._n or buf.dtype != torch.float32 or not buf.is_contiguous():
                raise ValueError("GradBufReducer: buffer does not match the one it was built for")
            rc = self._lib.pj_allreduce_oneshot(self._ptrs, self._rank, self._world, buf.data_ptr(), buf.data_ptr(), self._n,
                                                ctypes.c_void_p(torch.cuda.current_stream(buf.device).cuda_stream))
            if rc != 0:
                raise RuntimeError(f"pj_allreduce_oneshot failed ({rc})")
        elif self.mode != "single":
            self.dist.all_reduce(buf)
        return buf
