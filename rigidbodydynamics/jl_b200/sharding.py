"""Batch sharding across the GPUs of one box (SURVEY 8(e)): samples are independent, the flattened mechanism is
replicated in every process, so the data path has NO collective.  The only optional communication is the final gather of
v̇ (``gather_columns``), an NCCL all-gather over NVLink on GPUs (gloo on CPU in the tests).

One process per GPU, launched by ``torchrun``; each rank evaluates ``shard_bounds(B, world, rank)``.

``GatheredResult`` + ``dynamics_gather_`` are the fused form of that gather (BASELINE config 5): the result array of every GPU is
peer-mapped into every process (torch symmetric memory = CUDA VMM over NVLink) and the forward-dynamics kernel stores each v̇ row
into all of them -- the output store is the gather, no collective runs after the kernel (``rbd_dynamics_gather``).
"""
from __future__ import annotations

from typing import Tuple

import torch


def shard_bounds(B: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of the batch owned by ``rank``: sizes differ by at most one, earlier ranks get the extra."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    base, rem = divmod(B, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_columns(local: torch.Tensor, B: int, group=None) -> torch.Tensor:
    """All-gather ``[rows, n_local]`` shards (batch index fastest) into the full ``[rows, B]`` array on every rank.

    The result layout keeps the batch fastest, so the gather is done on the transposed ``[n_local, rows]`` view: shards are
    then contiguous slabs of the output and no post-gather transpose pass over the full array is needed on the receive side
    other than the final ``.t()`` view."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    rows = local.shape[0]
    sizes = [shard_bounds(B, world, r) for r in range(world)]
    nmax = max(hi - lo for lo, hi in sizes)
    lo, hi = sizes[rank]
    if local.shape[1] != hi - lo:
        raise ValueError("local shard has the wrong number of samples")
    send = torch.zeros((nmax, rows), dtype=local.dtype, device=local.device)
    send[: hi - lo] = local.t()
    recv = torch.empty((world * nmax, rows), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(recv, send, group=group)
    out = torch.empty((B, rows), dtype=local.dtype, device=local.device)
    for r, (a, b) in enumerate(sizes):
        out[a:b] = recv[r * nmax: r * nmax + (b - a)]
    return out.t()


class GatheredResult:
    """``[rows, world * B_local]`` array that exists on every GPU of the group, each one peer-mapped into every process.
    Rank r owns columns ``[r * B_local, (r + 1) * B_local)``; after ``dynamics_gather_`` + ``barrier()`` every GPU holds all of them.
    PyTorch only supplies the memory mapping and the rendezvous (``torch.distributed._symmetric_memory``)."""

    def __init__(self, rows: int, B_local: int, dtype: torch.dtype, group=None, use_multicast: bool = True):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        group = dist.group.WORLD if group is None else group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.rows, self.B_local = int(rows), int(B_local)
        dev = torch.device("cuda", torch.cuda.current_device())
        self.tensor = symm.empty((self.rows, self.world * self.B_local), dtype=dtype, device=dev)
        self.handle = symm.rendezvous(self.tensor, group.group_name)
        self.ptrs = [int(p) for p in self.handle.buffer_ptrs]
        mc = getattr(self.handle, "multicast_ptr", 0) or 0          # NVLS multicast mapping (NVSwitch systems), else 0
        self.multicast_ptr = int(mc) if use_multicast else 0

    @property
    def ld(self) -> int:
        return self.world * self.B_local

    def barrier(self):
        """All GPUs of the group have finished what they enqueued before this point (device-side barrier on the current stream)."""
        self.handle.barrier()


def dynamics_gather_(gathered: GatheredResult, state, torques=None):
    """``dynamics!`` on this rank's shard with the result gather fused into the kernel: v̇ of local sample b is written to column
    ``rank * B_local + b`` of the gathered array of EVERY GPU (``rbd_dynamics_gather``).  Call ``gathered.barrier()`` before
    reading columns owned by other ranks."""
    import ctypes
    from . import _cabi
    from .algorithms import _check, _ptr, _require_tree, _stream
    from .state import _DT
    _require_tree(state, "dynamics_gather_")
    state.check_modcount()
    if state.batch != gathered.B_local or gathered.rows != state.nv or gathered.tensor.dtype != state.dtype:
        raise ValueError("gathered array does not match the state (rows = nv, B_local = state.batch, same dtype)")
    _check(torques, state.nv, state, "torques")
    lib = _cabi.load_library()
    arr = (ctypes.c_void_p * gathered.world)(*gathered.ptrs)
    _cabi.check(lib.rbd_dynamics_gather(state.handle.ptr, _DT[state.dtype], state.batch, state.batch, _ptr(state.q), _ptr(state.v),
                                        _ptr(torques), gathered.world, arr, gathered.multicast_ptr or None, gathered.ld,
                                        gathered.rank * gathered.B_local, _stream()))
    return gathered
