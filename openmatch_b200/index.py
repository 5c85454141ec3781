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


_STORAGE = {torch.float32: _lib.OM_F32, torch.float16: _lib.OM_F16, torch.int8: _lib.OM_I8}


# ---- search filters (om_search_filter): the allowed-row bitmap and the per-query excluded ids ----
def _as_tensor(a) -> torch.Tensor:
    if isinstance(a, np.ndarray):
        if a.dtype == np.uint32:
            a = a.view(np.int32)
        return torch.from_numpy(np.ascontiguousarray(a))
    if isinstance(a, torch.Tensor):
        return a.detach()
    raise TypeError("expected a torch tensor or a numpy array, got %s" % type(a).__name__)


def pack_allow(allow, n: int, device=None) -> torch.Tensor:
    """The allowed-row bitmap of ``n`` rows as int32 words (bit ``r & 31`` of word ``r >> 5`` = row ``r``), packed on
    ``device`` with torch ops.  ``allow``: a bool tensor or ndarray ``[n]``, or words already packed (int32 / uint32,
    at least ``ceil(n / 32)`` of them), which are passed as they are."""
    a = _as_tensor(allow)
    if device is not None:
        a = a.to(device)
    if a.dim() != 1:
        raise ValueError("allow must be one-dimensional, got shape %s" % (tuple(a.shape),))
    if a.dtype == torch.int32:
        if a.numel() < (n + 31) // 32:
            raise ValueError("allow holds %d packed words; %d rows need %d" % (a.numel(), n, (n + 31) // 32))
        return a.contiguous()
    if a.dtype != torch.bool:
        raise ValueError("allow must be bool [%d] or packed int32 words, got %s" % (n, a.dtype))
    if a.numel() != n:
        raise ValueError("allow has %d entries for %d rows" % (a.numel(), n))
    words = (n + 31) // 32
    bits = torch.zeros(words * 32, dtype=torch.int64, device=a.device)
    bits[:n] = a.to(torch.int64)
    w = (bits.view(words, 32) << torch.arange(32, device=a.device)).sum(1)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)


def unpack_allow(words: torch.Tensor, n: int) -> torch.Tensor:
    """Inverse of :func:`pack_allow`: bool ``[n]`` on the words' device."""
    w = words.to(torch.int64) & 0xFFFFFFFF
    bits = (w.view(-1, 1) >> torch.arange(32, device=w.device)) & 1
    return bits.view(-1)[:n].bool()


def exclusion_csr(exclude, nq: int, device=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(offsets int64 [nq + 1], ids int64) of the per-query excluded ids.  ``exclude``: a list of ``nq`` id lists, or an
    ``(offsets, ids)`` pair of tensors / ndarrays that is passed as it is."""
    if isinstance(exclude, tuple):
        if len(exclude) != 2:
            raise ValueError("exclude as a tuple must be (offsets, ids)")
        off, ids = (_as_tensor(t) for t in exclude)
        if off.dim() != 1 or off.numel() != nq + 1 or ids.dim() != 1:
            raise ValueError("exclude offsets must be [nq + 1] = [%d] and ids one-dimensional" % (nq + 1))
        if off.is_floating_point() or ids.is_floating_point() or off.dtype == torch.bool or ids.dtype == torch.bool:
            raise ValueError("exclude offsets and ids must be integer tensors")
    else:
        exclude = list(exclude)
        if len(exclude) != nq:
            raise ValueError("exclude has %d id lists for %d queries" % (len(exclude), nq))
        lens = [len(e) for e in exclude]
        off = torch.from_numpy(np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).astype(np.int64))
        ids = torch.from_numpy(np.fromiter((int(i) for e in exclude for i in e), dtype=np.int64, count=sum(lens)))
    off, ids = off.to(torch.int64).contiguous(), ids.to(torch.int64).contiguous()
    if device is not None:
        off, ids = off.to(device), ids.to(device)
    return off, ids


def _filter(n: int, nq: int, device, allow, exclude):
    """(om_search_filter or None, the tensors it points into, to be kept alive for the call)"""
    if allow is None and exclude is None:
        return None, ()
    f = _lib.SearchFilter()
    keep = []
    if allow is not None:
        words = pack_allow(allow, n, device)
        f.allow_bits, f.allow_words = words.data_ptr() or None, words.numel()
        keep.append(words)
    if exclude is not None:
        off, ids = exclusion_csr(exclude, nq, device)
        f.exclude_offsets, f.exclude_ids = off.data_ptr(), ids.data_ptr() if ids.numel() else None
        keep += [off, ids]
    return f, keep


def _cuda_queries(q) -> torch.Tensor:
    """Queries given as a numpy array or a tensor, as a contiguous float32 tensor on the current CUDA device."""
    if not isinstance(q, torch.Tensor):
        q = torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32))
    return q.detach().cuda().contiguous().float()


def range_radius(radius, nq: int, device=None) -> torch.Tensor:
    """The per-query radii of a range search as float32 ``[nq]``: a number is broadcast, an array must hold ``nq``."""
    if isinstance(radius, (int, float, np.floating, np.integer)):
        r = torch.full((nq,), float(radius), dtype=torch.float32)
    else:
        r = _as_tensor(np.asarray(radius, dtype=np.float32) if isinstance(radius, (list, tuple)) else radius)
        if r.dim() == 0:
            r = r.reshape(1).expand(nq)
        if r.dim() != 1 or r.numel() != nq:
            raise ValueError("radius must be a number or hold one value per query ([%d]), got shape %s"
                             % (nq, tuple(r.shape)))
        r = r.float()
    r = r.contiguous()
    return r.to(device) if device is not None else r


class FlatIPIndex:
    """``faiss.IndexFlatIP`` duck type (``d``, ``ntotal``, ``add``, ``search``, ``reset``) living on the
    current CUDA device.

    ``dtype`` is the row storage.  ``torch.float32`` (default): fp32 master rows plus an fp16 scan copy (6 bytes per
    element); search is exact over the rows as added.  ``torch.float16``: the fp16 rows only (2 bytes per element);
    added rows are rounded to fp16 (nearest even) and search is exact with respect to the STORED values: the exact
    top-k by fp32 inner product of the fp32 query with the fp16 rows, ties by ascending id, bitwise what a float32
    index of the fp16-rounded rows returns.  fp16 storage refuses what it cannot hold: ``add`` of a NaN or of a value
    that rounds to +-inf in fp16 (|x| >= 65520) raises and adds nothing; rows written in place through ``reserve_rows``
    and committed with such values make ``search`` raise until ``reset`` (``stat("nonfinite_rows")``).

    ``torch.int8``: one byte per element plus a per-row fp32 scale (rows of ``dpad + 16`` bytes, ``dpad`` = d rounded up
    to 16; the scale sits at byte ``dpad``).  A row x is stored as ``s = max|x| / 127`` and ``c = clamp(rint(x / s),
    -127, 127)`` (a zero row: s = 0); search is exact with respect to the dequantised values ``fp32(s * c)``, bitwise
    what a float32 index of ``rows_f32()`` returns.  ``add`` of a row holding inf or NaN raises and adds nothing; rows
    written in place (the encoder quantises into an int8 ``reserve_rows`` view) and committed with a non-finite scale
    make ``search`` raise until ``reset``.

    ``memory="host"`` (``om_index_create_host``) keeps the stored rows in pinned host memory, for corpora larger than
    the GPU's memory: a search streams them through the GPU ``window_rows`` rows at a time (a multiple of 256; 0 = sized
    from the free device memory) and returns bitwise what the ``memory="device"`` index of the same adds returns.
    ``add``, ``search`` (filters included), ``search_device``, ``search_pinned``, ``reset``, ``set_param`` and
    ``stat`` work as for a device index; the calls that need device rows (``reserve_rows``, ``commit_rows``,
    ``master_rows``, ``rows_f32``), range search and the sharded searches raise the library's error."""

    def __init__(self, d: int, dtype: torch.dtype = torch.float32, memory: str = "device", window_rows: int = 0):
        if dtype not in _STORAGE:
            raise ValueError("index storage must be torch.float32, torch.float16 or torch.int8, got %s" % dtype)
        if memory not in ("device", "host"):
            raise ValueError("index memory must be 'device' or 'host', got %r" % (memory,))
        self._lib = _lib.load()
        h = ctypes.c_void_p()
        if memory == "host":
            _lib.check(self._lib.om_index_create_host(int(d), _STORAGE[dtype], int(window_rows), ctypes.byref(h)))
        else:
            _lib.check(self._lib.om_index_create_typed(int(d), _STORAGE[dtype], ctypes.byref(h)))
        self._h = h
        self.d = int(d)
        self.dtype = dtype
        self.memory = memory

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.om_index_destroy(h)

    # ---- faiss surface ----
    @property
    def ntotal(self) -> int:
        return int(self._lib.om_index_ntotal(self._h))

    def add(self, x) -> None:
        """x: [n, d]; numpy (host) or torch tensor (host or CUDA); float32, bfloat16 or float16 tensors are passed as they
        are, anything else as float32."""
        if isinstance(x, torch.Tensor) and (x.is_cuda or (self.dtype != torch.float32 and x.dtype in _ADD_DTYPES)):
            x = x.detach().contiguous()
            if x.dtype not in _ADD_DTYPES:
                x = x.float()
            kind = _lib.OM_DEVICE if x.is_cuda else _lib.OM_HOST
            self._check_shape(x.shape)
            _lib.check(self._lib.om_index_add(self._h, x.data_ptr(), kind, _ADD_DTYPES[x.dtype], x.shape[0], _stream()))
            torch.cuda.current_stream().synchronize()  # the caller's tensor may be freed right after
            return
        if isinstance(x, torch.Tensor):
            x = x.detach().cpu().numpy()
        if self.dtype != torch.float32 and isinstance(x, np.ndarray) and x.dtype == np.float16:
            x = np.ascontiguousarray(x)
            self._check_shape(x.shape)
            _lib.check(self._lib.om_index_add(self._h, x.ctypes.data, _lib.OM_HOST, _lib.OM_F16, x.shape[0], _stream()))
            return
        x = np.ascontiguousarray(x, dtype=np.float32)
        self._check_shape(x.shape)
        _lib.check(self._lib.om_index_add(self._h, x.ctypes.data, _lib.OM_HOST, _lib.OM_F32, x.shape[0], _stream()))

    def reset(self) -> None:
        _lib.check(self._lib.om_index_reset(self._h))

    def search(self, q, k: int, id_offset: int = 0, allow=None, exclude=None) -> Tuple[np.ndarray, np.ndarray]:
        """``D, I = index.search(q, k)`` with numpy outputs (float32 [nq, k], int64 [nq, k]).

        Filtered search (``om_index_search_filtered``): ``allow`` restricts the result to the rows it allows (bool
        ``[ntotal]``, tensor or ndarray, or int32 words packed as :func:`pack_allow` does); ``exclude`` drops ids per
        query (a list of ``nq`` id lists, or an ``(offsets, ids)`` CSR pair; at most 128 ids per query; ids are
        ``id_offset`` + row).  The result is the exact top-k among the eligible rows, bitwise what an index of those rows
        alone returns with ids mapped back; missing slots hold id -1.  ``None`` keeps the unfiltered search."""
        if allow is not None or exclude is not None or (isinstance(q, torch.Tensor) and q.is_cuda):
            D, I = self.search_device(_cuda_queries(q), k, id_offset, allow=allow, exclude=exclude)
            return D.cpu().numpy(), I.cpu().numpy()
        if isinstance(q, torch.Tensor):
            q = q.detach().cpu().numpy()
        q = np.ascontiguousarray(q, dtype=np.float32)
        self._check_shape(q.shape)
        nq = q.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        self._call("search", None, None, q.ctypes.data, _lib.OM_HOST, nq, int(k), D.ctypes.data, I.ctypes.data,
                   _lib.OM_HOST, int(id_offset))
        return D, I

    def _call(self, kind: str, comm, f, *args) -> None:
        """One call of the C ABI's ``om_index_<kind>`` (``search`` or ``range_search``), ``_sharded`` with ``comm``,
        ``_filtered`` with the filter ``f``; ``args`` go between the handles and the filter.  An unfiltered call never
        takes a ``_filtered`` entry: with more than one rank that would add a collective filter check."""
        name = "om_index_" + kind + ("" if comm is None else "_sharded") + ("" if f is None else "_filtered")
        head = (self._h,) if comm is None else (self._h, comm._h)
        tail = (_stream(),) if f is None else (ctypes.byref(f), _stream())
        _lib.check(getattr(self._lib, name)(*head, *args, *tail))

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

    def search_device(self, q: torch.Tensor, k: int, id_offset: int = 0, out=None, allow=None,
                      exclude=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``out=(D, I)``: write into caller-owned CUDA tensors (no allocation on the search path).  ``allow`` /
        ``exclude``: the filter of :meth:`search`, packed on the query's device."""
        return self._search(None, q, k, id_offset, allow, exclude, out)

    def search_sharded_device(self, comm: "Comm", q: torch.Tensor, k: int, id_offset: int = 0, out=None, allow=None,
                              exclude=None):
        """This rank's call of the row-sharded search (``om_index_search_sharded``): collective over ``comm``; every
        rank passes the same queries and receives the same global (D, I) [nq, k] on its device.  ``allow`` covers THIS
        rank's rows (``ntotal`` of them); ``exclude`` holds global ids and may be the same on every rank.  Every rank
        passes a filter or none does; a rank's filter may be empty (a shard without rows packs to no words), which
        still takes the filtered call, so the ranks' collectives stay in step."""
        return self._search(comm, q, k, id_offset, allow, exclude, out)

    def _search(self, comm, q: torch.Tensor, k: int, id_offset: int, allow, exclude, out=None):
        q = q.detach().contiguous().float()
        self._check_shape(q.shape)
        nq, k = q.shape[0], int(k)
        f, _keep = _filter(self.ntotal, nq, q.device, allow, exclude)
        D, I = self._outputs(nq, k, q.device, out)
        self._call("search", comm, f, q.data_ptr(), _lib.OM_DEVICE, nq, k, D.data_ptr(), I.data_ptr(), _lib.OM_DEVICE,
                   int(id_offset))
        return D, I

    def search_sharded_pinned(self, comm: "Comm", q_host: torch.Tensor, k: int, D_out: torch.Tensor, I_out: torch.Tensor,
                              id_offset: int = 0) -> None:
        """Host (pinned) queries in; results into ``D_out`` / ``I_out`` (pinned host on the rank that wants them,
        device tensors elsewhere)."""
        self._search_pinned(comm, q_host, k, D_out, I_out, id_offset)

    def search_pinned(self, q_host: torch.Tensor, k: int, D_host: torch.Tensor, I_host: torch.Tensor,
                      id_offset: int = 0) -> None:
        """Host (pinned) in, host (pinned) out — the end-to-end call the benchmark times."""
        self._search_pinned(None, q_host, k, D_host, I_host, id_offset)

    def _search_pinned(self, comm, q_host: torch.Tensor, k: int, D_out: torch.Tensor, I_out: torch.Tensor,
                       id_offset: int) -> None:
        kind = _lib.OM_DEVICE if D_out.is_cuda else _lib.OM_HOST
        self._call("search", comm, None, q_host.data_ptr(), _lib.OM_HOST, q_host.shape[0], int(k), D_out.data_ptr(),
                   I_out.data_ptr(), kind, int(id_offset))

    # ---- range search ----
    def range_search(self, q, radius, id_offset: int = 0, allow=None,
                     exclude=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """``lims, D, I = index.range_search(q, radius)`` (faiss's signature): for query i every row whose score is
        strictly greater than ``radius`` (a float, or one per query), at ``D[lims[i]:lims[i + 1]]`` /
        ``I[lims[i]:lims[i + 1]]`` ordered by (score desc, id asc).  The first j results of a query are bitwise
        ``search(q, j)``'s for j <= 4096.  numpy outputs (int64 [nq + 1], float32, int64).

        ``allow`` / ``exclude``: the filter of :meth:`search` (``om_index_range_search_filtered``).  The result is then
        every eligible row above the radius, bitwise what an index of the eligible rows alone returns with ids mapped
        back, and its first j results are ``search(q, j, allow=allow, exclude=exclude)``'s.  ``None`` keeps the
        unfiltered range search."""
        lims, D, I = self.range_search_device(_cuda_queries(q), radius, id_offset, allow=allow, exclude=exclude)
        return lims.cpu().numpy(), D.cpu().numpy(), I.cpu().numpy()

    def range_search_device(self, q: torch.Tensor, radius, id_offset: int = 0, allow=None, exclude=None):
        """:meth:`range_search` with CUDA tensors in and out: (lims int64 [nq + 1], D float32, I int64).  ``allow`` /
        ``exclude``: the filter of :meth:`range_search`, packed on the query's device."""
        return self._range(None, q, radius, id_offset, allow, exclude)

    def range_search_sharded_device(self, comm: "Comm", q: torch.Tensor, radius, id_offset: int = 0, allow=None,
                                    exclude=None):
        """This rank's call of the row-sharded range search (``om_index_range_search_sharded``): collective over
        ``comm``; every rank passes the same queries and radii and receives the same global (lims, D, I).  ``allow``
        covers THIS rank's rows and ``exclude`` holds global ids, as for :meth:`search_sharded_device`; every rank
        passes a filter or none does."""
        return self._range(comm, q, radius, id_offset, allow, exclude)

    def _range(self, comm, q: torch.Tensor, radius, id_offset: int, allow, exclude):
        q = q.detach().contiguous().float()
        self._check_shape(q.shape)
        nq = q.shape[0]
        rho = range_radius(radius, nq, q.device)
        f, _keep = _filter(self.ntotal, nq, q.device, allow, exclude)
        lims = torch.empty(nq + 1, dtype=torch.int64)
        self._call("range_search", comm, f, q.data_ptr(), _lib.OM_DEVICE, nq, rho.data_ptr(), lims.data_ptr(), _lib.OM_HOST,
                   int(id_offset))
        total = int(lims[-1])
        D = torch.empty(total, dtype=torch.float32, device=q.device)
        I = torch.empty(total, dtype=torch.int64, device=q.device)
        _lib.check(self._lib.om_index_range_results(self._h, D.data_ptr() or None, I.data_ptr() or None, _lib.OM_DEVICE,
                                                    _stream()))
        return lims.to(q.device), D, I

    def _rows_at(self, n: int):
        """(device address, row pitch in elements) of the shard's rows after reserving room for n more"""
        p, pitch = ctypes.c_void_p(), ctypes.c_int64()
        _lib.check(self._lib.om_index_reserve_rows(self._h, int(n), ctypes.byref(p), ctypes.byref(pitch)))
        return p.value, pitch.value

    def reserve_rows(self, n: int) -> torch.Tensor:
        """Zero-copy ingest: a CUDA tensor view [n, d] of the next n rows of the shard in the index's dtype (float16
        rows have row stride dpad = d rounded up to 8, int8 rows dpad + 16 with dpad = d rounded up to 16 and the row's
        scale beyond the view); fill it (e.g. as the encoder's output buffer) and call ``commit_rows(n)``."""
        p, pitch = self._rows_at(n)
        return _wrap_device(p, (int(n), self.d), pitch, self.dtype)

    def master_rows(self) -> torch.Tensor:
        """CUDA view [ntotal, d] of the shard's stored rows in the index's dtype (no copy).  Exported embedding files
        upcast it to float32, so an fp16 index writes its fp16-rounded values."""
        n = self.ntotal
        p, pitch = self._rows_at(0)  # address one past the last row
        if n == 0:
            return torch.empty((0, self.d), dtype=self.dtype, device="cuda")
        return _wrap_device(p - n * pitch * self.dtype.itemsize, (n, self.d), pitch, self.dtype)

    def rows_f32(self, chunk_rows: int = 1 << 16):
        """The stored rows as float32 CUDA blocks of at most ``chunk_rows`` rows (int8: the dequantised values
        ``fp32(s * c)``, computed block by block).  Exported embedding files hold these values, so a float32 index
        rebuilt from them answers bitwise like this one."""
        n = self.ntotal
        if self.dtype != torch.int8:
            rows = self.master_rows()
            for lo in range(0, n, chunk_rows):
                yield rows[lo:lo + chunk_rows].float()
            return
        p, pitch = self._rows_at(0)
        if n == 0:
            return
        full = _wrap_device(p - n * pitch, (n, pitch), pitch, torch.int8)  # whole rows: codes, padding, scale
        dpad = (self.d + 15) // 16 * 16
        for lo in range(0, n, chunk_rows):
            part = full[lo:lo + chunk_rows]
            scale = part[:, dpad:dpad + 4].contiguous().view(torch.float32)  # [rows, 1]
            yield part[:, :self.d].float() * scale

    def commit_rows(self, n: int) -> None:
        _lib.check(self._lib.om_index_commit(self._h, int(n), _stream()))

    def set_param(self, name: str, value: int) -> None:
        _lib.check(self._lib.om_index_set_param(self._h, name.encode(), int(value)))

    def stat(self, name: str) -> int:
        return int(self._lib.om_index_get_stat(self._h, name.encode()))

    def _check_shape(self, shape):
        if len(shape) != 2 or shape[1] != self.d:
            raise ValueError("expected a [n, %d] matrix, got %s" % (self.d, tuple(shape)))


_ADD_DTYPES = {torch.float32: _lib.OM_F32, torch.bfloat16: _lib.OM_BF16, torch.float16: _lib.OM_F16}


class _CudaArrayView:
    def __init__(self, ptr, shape, typestr, strides):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 3, "strides": strides}


def _wrap_device(ptr: int, shape, pitch: int, dtype: torch.dtype) -> torch.Tensor:
    size = dtype.itemsize
    strides = None if pitch == shape[1] else (pitch * size, size)
    typestr = "|i1" if dtype == torch.int8 else "<f%d" % size
    return torch.as_tensor(_CudaArrayView(ptr, shape, typestr, strides), device="cuda")


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


def local_allow(allow, id_offset: int, n_local: int, device=None):
    """A shard's slice ``[id_offset, id_offset + n_local)`` of an allowed-row bitmap over global ids (bool, or int32 words
    packed as :func:`pack_allow` does), as bool ``[n_local]``; ``None`` stays ``None``."""
    if allow is None:
        return None
    a = _as_tensor(allow)
    if device is not None:
        a = a.to(device)
    if a.dtype == torch.int32:
        a = unpack_allow(a, a.numel() * 32)
    if a.dtype != torch.bool or a.dim() != 1:
        raise ValueError("allow must be bool [ntotal] or packed int32 words, got %s %s" % (a.dtype, tuple(a.shape)))
    if a.numel() < id_offset + n_local:
        raise ValueError("allow covers %d ids; this shard holds ids [%d, %d)" % (a.numel(), id_offset, id_offset + n_local))
    return a[id_offset:id_offset + n_local]


def sharded_search_device(index: "FlatIPIndex", q: torch.Tensor, k: int, id_offset: int, group=None, allow=None,
                          exclude=None):
    """Row-sharded exact search: every rank passes the same queries and its own shard's ``id_offset`` and receives
    the same global (D, I) [nq, k].  Scan, exchange, merge and the exactness certificate run inside the library
    (``om_index_search_sharded``) over the library's NCCL communicator for ``group``, which is created on first
    use whatever the group's backend.  Without a process group, or with one rank: the single-shard search.
    ``allow`` (over global ids; each rank takes its slice) and ``exclude`` (global ids) filter as in
    :meth:`FlatIPIndex.search`."""
    return _on_shards(index._search, index, q, k, id_offset, group, allow, exclude)


def sharded_range_search_device(index: "FlatIPIndex", q: torch.Tensor, radius, id_offset: int, group=None, allow=None,
                                exclude=None):
    """Row-sharded exact range search: every rank passes the same queries and radii and its own shard's ``id_offset``
    and receives the same global (lims, D, I), bitwise one index's range search over the concatenated shards.  Without
    a process group, or with one rank: the single-shard range search.  ``allow`` (over global ids; each rank takes its
    slice) and ``exclude`` (global ids) filter as in :meth:`FlatIPIndex.range_search`."""
    return _on_shards(index._range, index, q, radius, id_offset, group, allow, exclude)


def _on_shards(call, index: "FlatIPIndex", q: torch.Tensor, arg, id_offset: int, group, allow, exclude):
    """``call(comm, q, arg, id_offset, allow, exclude)`` (``FlatIPIndex._search`` or ``_range``) on this rank's shard,
    with its slice of the bitmap ``allow``: without a process group, or with one rank, the single-shard call (``comm``
    None), else the sharded one over the library's communicator for ``group``."""
    import torch.distributed as dist
    allow = local_allow(allow, int(id_offset), index.ntotal, q.device)
    sharded = dist.is_initialized() and dist.get_world_size(group) > 1
    return call(comm_for(group) if sharded else None, q, arg, id_offset, allow, exclude)


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

    def __init__(self, d: int, group=None, dtype: torch.dtype = torch.float32):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.local = FlatIPIndex(d, dtype)  # every rank must pass the same dtype
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

    def search_device(self, q: torch.Tensor, k: int, allow=None, exclude=None):
        """``allow``: bitmap over the global ids (each rank uses its slice); ``exclude``: global ids per query."""
        return sharded_search_device(self.local, q, k, self.offset, self.group, allow=allow, exclude=exclude)

    def search(self, q, k: int, allow=None, exclude=None):
        D, I = self.search_device(_cuda_queries(q), k, allow=allow, exclude=exclude)
        return D.cpu().numpy(), I.cpu().numpy()

    def range_search_device(self, q: torch.Tensor, radius, allow=None, exclude=None):
        """``allow``: bitmap over the global ids (each rank uses its slice); ``exclude``: global ids per query."""
        return sharded_range_search_device(self.local, q, radius, self.offset, self.group, allow=allow, exclude=exclude)

    def range_search(self, q, radius, allow=None, exclude=None):
        """(lims, D, I) numpy over the global ids, the same on every rank."""
        lims, D, I = self.range_search_device(_cuda_queries(q), radius, allow=allow, exclude=exclude)
        return lims.cpu().numpy(), D.cpu().numpy(), I.cpu().numpy()
