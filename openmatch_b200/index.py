"""HBM-resident exact inner-product index: the drop-in for ``faiss.IndexFlatIP`` as the reference uses it
(``src/openmatch/retriever/dense_retriever.py:38-41`` construct, ``:105`` add, ``:133-137`` reset,
``:180`` search) plus the row-sharded multi-GPU search that replaces
``faiss.index_cpu_to_gpu_multiple(shard=True)`` (``:43-58``).

All arithmetic runs in libopenmatch_b200.so (csrc/search.cu); this file only marshals pointers.
"""
from __future__ import annotations

import ctypes
from typing import Tuple

import numpy as np
import torch

from . import _lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class FlatIPIndex:
    """``faiss.IndexFlatIP`` duck type (``d``, ``ntotal``, ``add``, ``search``, ``reset``) living on the
    current CUDA device."""

    def __init__(self, d: int):
        self._lib = _lib.load()
        h = ctypes.c_void_p()
        _lib.check(self._lib.om_index_create(int(d), ctypes.byref(h)))
        self._h = h
        self.d = int(d)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.om_index_destroy(h)

    # ---- faiss surface ----
    @property
    def ntotal(self) -> int:
        return int(self._lib.om_index_ntotal(self._h))

    def add(self, x) -> None:
        """x: float32 [n, d]; numpy (host) or torch tensor (host or CUDA)."""
        if isinstance(x, torch.Tensor) and x.is_cuda:
            x = x.contiguous()
            if x.dtype not in (torch.float32, torch.bfloat16, torch.float16):
                x = x.float()
            dt = {torch.float32: _lib.OM_F32, torch.bfloat16: _lib.OM_BF16, torch.float16: _lib.OM_F16}[x.dtype]
            self._check_shape(x.shape)
            _lib.check(self._lib.om_index_add(self._h, x.data_ptr(), _lib.OM_DEVICE, dt, x.shape[0], _stream()))
            torch.cuda.current_stream().synchronize()  # the caller's tensor may be freed right after
            return
        if isinstance(x, torch.Tensor):
            x = x.detach().cpu().numpy()
        x = np.ascontiguousarray(x, dtype=np.float32)
        self._check_shape(x.shape)
        _lib.check(self._lib.om_index_add(self._h, x.ctypes.data, _lib.OM_HOST, _lib.OM_F32, x.shape[0], _stream()))

    def reset(self) -> None:
        _lib.check(self._lib.om_index_reset(self._h))

    def search(self, q, k: int, id_offset: int = 0) -> Tuple[np.ndarray, np.ndarray]:
        """``D, I = index.search(q, k)`` with numpy outputs (float32 [nq, k], int64 [nq, k])."""
        if isinstance(q, torch.Tensor) and q.is_cuda:
            D, I = self.search_device(q, k, id_offset)
            return D.cpu().numpy(), I.cpu().numpy()
        if isinstance(q, torch.Tensor):
            q = q.detach().cpu().numpy()
        q = np.ascontiguousarray(q, dtype=np.float32)
        self._check_shape(q.shape)
        nq = q.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        _lib.check(self._lib.om_index_search(self._h, q.ctypes.data, _lib.OM_HOST, nq, int(k), D.ctypes.data,
                                             I.ctypes.data, _lib.OM_HOST, int(id_offset), _stream()))
        return D, I

    # ---- device-resident variants ----
    @staticmethod
    def _outputs(nq: int, k: int, device, out):
        if out is None:
            return (torch.empty((nq, k), dtype=torch.float32, device=device),
                    torch.empty((nq, k), dtype=torch.int64, device=device))
        D, I = out
        if D.shape != (nq, k) or I.shape != (nq, k) or D.dtype != torch.float32 or I.dtype != torch.int64 or \
                not (D.is_cuda and I.is_cuda and D.is_contiguous() and I.is_contiguous()):
            raise ValueError("out must be contiguous CUDA tensors (float32 [nq, k], int64 [nq, k])")
        return D, I

    def search_device(self, q: torch.Tensor, k: int, id_offset: int = 0, out=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``out=(D, I)``: write into caller-owned CUDA tensors (no allocation on the search path)."""
        q = q.contiguous().float()
        self._check_shape(q.shape)
        nq = q.shape[0]
        D, I = self._outputs(nq, int(k), q.device, out)
        _lib.check(self._lib.om_index_search(self._h, q.data_ptr(), _lib.OM_DEVICE, nq, int(k), D.data_ptr(),
                                             I.data_ptr(), _lib.OM_DEVICE, int(id_offset), _stream()))
        return D, I

    def search_sharded_device(self, comm: "Comm", q: torch.Tensor, k: int, id_offset: int = 0, out=None):
        """This rank's call of the row-sharded search (``om_index_search_sharded``): collective over ``comm``; every
        rank passes the same queries and receives the same global (D, I) [nq, k] on its device."""
        q = q.contiguous().float()
        self._check_shape(q.shape)
        nq = q.shape[0]
        D, I = self._outputs(nq, int(k), q.device, out)
        _lib.check(self._lib.om_index_search_sharded(self._h, comm._h, q.data_ptr(), _lib.OM_DEVICE, nq, int(k),
                                                     D.data_ptr(), I.data_ptr(), _lib.OM_DEVICE, int(id_offset), _stream()))
        return D, I

    def search_sharded_pinned(self, comm: "Comm", q_host: torch.Tensor, k: int, D_out: torch.Tensor, I_out: torch.Tensor,
                              id_offset: int = 0) -> None:
        """Host (pinned) queries in; results into ``D_out`` / ``I_out`` (pinned host on the rank that wants them,
        device tensors elsewhere)."""
        nq = q_host.shape[0]
        kind = _lib.OM_DEVICE if D_out.is_cuda else _lib.OM_HOST
        _lib.check(self._lib.om_index_search_sharded(self._h, comm._h, q_host.data_ptr(), _lib.OM_HOST, nq, int(k),
                                                     D_out.data_ptr(), I_out.data_ptr(), kind, int(id_offset), _stream()))

    def search_pinned(self, q_host: torch.Tensor, k: int, D_host: torch.Tensor, I_host: torch.Tensor,
                      id_offset: int = 0) -> None:
        """Host (pinned) in, host (pinned) out — the end-to-end call the benchmark times."""
        nq = q_host.shape[0]
        _lib.check(self._lib.om_index_search(self._h, q_host.data_ptr(), _lib.OM_HOST, nq, int(k), D_host.data_ptr(),
                                             I_host.data_ptr(), _lib.OM_HOST, int(id_offset), _stream()))

    def reserve_rows(self, n: int) -> torch.Tensor:
        """Zero-copy ingest: a float32 CUDA tensor view [n, d] of the next n rows of the shard; fill it
        (e.g. as the encoder's output buffer) and call ``commit_rows(n)``."""
        p = ctypes.c_void_p()
        _lib.check(self._lib.om_index_reserve(self._h, int(n), ctypes.byref(p)))
        return _wrap_device_f32(p.value, (int(n), self.d))

    def master_rows(self) -> torch.Tensor:
        """float32 CUDA view [ntotal, d] of the shard's master rows (no copy)."""
        n = self.ntotal
        p = ctypes.c_void_p()
        _lib.check(self._lib.om_index_reserve(self._h, 0, ctypes.byref(p)))  # address one past the last row
        if n == 0:
            return torch.empty((0, self.d), dtype=torch.float32, device="cuda")
        return _wrap_device_f32(p.value - n * self.d * 4, (n, self.d))

    def commit_rows(self, n: int) -> None:
        _lib.check(self._lib.om_index_commit(self._h, int(n), _stream()))

    def set_param(self, name: str, value: int) -> None:
        _lib.check(self._lib.om_index_set_param(self._h, name.encode(), int(value)))

    def stat(self, name: str) -> int:
        return int(self._lib.om_index_get_stat(self._h, name.encode()))

    def _check_shape(self, shape):
        if len(shape) != 2 or shape[1] != self.d:
            raise ValueError("expected a [n, %d] matrix, got %s" % (self.d, tuple(shape)))


class _CudaArrayView:
    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 3, "strides": None}


def _wrap_device_f32(ptr: int, shape) -> torch.Tensor:
    return torch.as_tensor(_CudaArrayView(ptr, shape), device="cuda")


class Comm:
    """NCCL communicator owned by libopenmatch_b200 for the row-sharded search (``om_comm_init``).  The 128-byte
    unique id is created on rank 0 and shipped to the other ranks of the torch.distributed ``group`` (any backend),
    then every rank joins collectively on its current CUDA device."""

    def __init__(self, group=None):
        import torch.distributed as dist
        self._lib = _lib.load()
        self._h = None
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        uid = ctypes.create_string_buffer(128)
        if self.rank == 0:
            _lib.check(self._lib.om_comm_unique_id(uid))
        box = [uid.raw]
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        h = ctypes.c_void_p()
        _lib.check(self._lib.om_comm_init(ctypes.create_string_buffer(box[0], 128), self.rank, self.world, ctypes.byref(h)))
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.om_comm_destroy(h)


_COMMS = {}


def comm_for(group=None):
    """One library communicator per process group (created collectively on first use)."""
    key = id(group) if group is not None else 0
    if key not in _COMMS:
        _COMMS[key] = Comm(group)
    return _COMMS[key]


def merge_topk_device(D_parts: torch.Tensor, I_parts: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """[nparts, nq, k_in] per-shard results (shards in increasing id order) -> global (D, I) [nq, k]."""
    lib = _lib.load()
    nparts, nq, k_in = D_parts.shape
    assert I_parts.shape == D_parts.shape
    D_parts = D_parts.contiguous().float()
    I_parts = I_parts.contiguous().long()
    D = torch.empty((nq, k), dtype=torch.float32, device=D_parts.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=D_parts.device)
    _lib.check(lib.om_topk_merge_n(D_parts.data_ptr(), I_parts.data_ptr(), nparts, nq, k_in, k, D.data_ptr(),
                                   I.data_ptr(), _stream()))
    return D, I


def sharded_search_device(index: "FlatIPIndex", q: torch.Tensor, k: int, id_offset: int, group=None):
    """Row-sharded exact search: every rank passes the same queries and its own shard's ``id_offset`` and receives
    the same global (D, I) [nq, k].  Scan, exchange, merge and the exactness certificate run inside the library
    (``om_index_search_sharded``) over the library's NCCL communicator for ``group``, which is created on first
    use whatever the group's backend.  Without a process group, or with one rank: the single-shard search."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return index.search_device(q, k, id_offset=id_offset)
    return index.search_sharded_device(comm_for(group), q, k, id_offset)


def shard_offsets(n_local: int, group=None):
    """(global id of this rank's first row, total rows) for rank-major contiguous shards."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 0, n_local
    counts = [None] * dist.get_world_size(group)
    dist.all_gather_object(counts, int(n_local), group=group)
    return sum(counts[: dist.get_rank(group)]), sum(counts)


class ShardedFlatIPIndex:
    """Row-sharded index: rank r of ``torch.distributed`` holds rows [offset_r, offset_r + n_r) in its own
    HBM.  ``search`` = replicate queries -> local fused scan/top-k with global ids -> all-gather of the
    per-shard [nq, k] (score, id) lists over NCCL/NVLink -> merge (score desc, id asc) on every rank."""

    def __init__(self, d: int, group=None):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.local = FlatIPIndex(d)
        self.d = d
        self.offset = 0
        self._ntotal = 0

    def add_local(self, x) -> None:
        self.local.add(x)

    def finalize_offsets(self) -> None:
        """Call once after all ranks added their rows: computes global id offsets (rank-major)."""
        self.offset, self._ntotal = shard_offsets(self.local.ntotal, self.group)

    @property
    def ntotal(self) -> int:
        return self._ntotal

    def search_device(self, q: torch.Tensor, k: int):
        return sharded_search_device(self.local, q, k, self.offset, self.group)

    def search(self, q, k: int):
        if not isinstance(q, torch.Tensor):
            q = torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32))
        D, I = self.search_device(q.cuda(), k)
        return D.cpu().numpy(), I.cpu().numpy()
