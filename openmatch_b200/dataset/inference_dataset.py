"""Streaming inference datasets (reference: ``src/openmatch/dataset/inference_dataset.py``).

Same contract as the reference: ``InferenceDataset.load`` dispatches on the file extension (``.json`` ->
JSON lines, ``.tsv``/``.txt`` -> tab separated with the configured column names), examples are rendered
through the query / doc template, tokenised to a fixed ``max_length`` padding, and ranks take interleaved
blocks of ``batch_size`` examples (:99-115).  Files are streamed with plain Python I/O.
``PretokenizedDataset`` is the device-friendly ingest format: int32 token ids in a ``.npy`` memory map.
"""
from __future__ import annotations

import json
import os
from typing import Dict, Iterator

import numpy as np
from torch.utils.data import IterableDataset

from ..arguments import DataArguments
from ..utils import fill_template, find_all_markers


def get_idx(obj) -> str:
    example_id = obj.get("_id", None) or obj.get("id", None)
    return str(example_id) if example_id is not None else None


def _ragged_prefix(path: str):
    """``<name>`` when ``path`` is ``<name>.tokens.npy`` next to ``<name>.offsets.npy`` (a ragged store), else None"""
    if path.endswith(".tokens.npy") and os.path.exists(path[:-len(".tokens.npy")] + ".offsets.npy"):
        return path[:-len(".tokens.npy")]
    return None


def write_ragged_store(prefix: str, ids_2d, names=None, pad_id: int = 0) -> str:
    """Writes the rows of an int ``[n, L]`` id matrix (``pad_id`` = padding, dropped: the tokenizer's pad id, 1 for
    RoBERTa) as a ragged store ``<prefix>.tokens.npy`` + ``<prefix>.offsets.npy`` (+ ``<prefix>.ids.txt`` when ``names``
    is given); returns the path to hand to ``PretokenizedDataset`` (``data_args.corpus_path`` / ``query_path``).  Every
    row needs at least one token."""
    ids_2d = np.asarray(ids_2d)
    keep = ids_2d != pad_id
    lens = keep.sum(1).astype(np.int64)
    if ids_2d.shape[0] and lens.min() < 1:
        raise ValueError("row %d holds no token" % int(np.argmin(lens)))
    offsets = np.zeros(ids_2d.shape[0] + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    np.save(prefix + ".tokens.npy", ids_2d[keep].astype(np.int32))
    np.save(prefix + ".offsets.npy", offsets)
    if names is not None:
        with open(prefix + ".ids.txt", "w") as f:
            f.write("\n".join(str(x) for x in names))
    return prefix + ".tokens.npy"


class InferenceDataset(IterableDataset):
    def __init__(self, tokenizer, data_args: DataArguments, is_query: bool = False, final: bool = True,
                 stream: bool = True, batch_size: int = 1, num_processes: int = 1, process_index: int = 0,
                 cache_dir: str = None):
        super().__init__()
        self.tokenizer = tokenizer
        self.data_files = [data_args.query_path] if is_query else [data_args.corpus_path]
        self.max_len = data_args.q_max_len if is_query else data_args.p_max_len
        self.template = data_args.query_template if is_query else data_args.doc_template
        self.all_markers = find_all_markers(self.template)
        self.final, self.stream = final, stream
        self.batch_size, self.num_processes, self.process_index = batch_size, num_processes, process_index

    @classmethod
    def load(cls, tokenizer, data_args: DataArguments, is_query: bool = False, final: bool = True, stream: bool = True,
             batch_size: int = 1, num_processes: int = 1, process_index: int = 0, cache_dir: str = None):
        path = data_args.query_path if is_query else data_args.corpus_path
        ext = os.path.splitext(path)[1]
        target = {".json": JsonlDataset, ".jsonl": JsonlDataset, ".tsv": TsvDataset, ".txt": TsvDataset,
                  ".npy": PretokenizedDataset}.get(ext)
        if target is None:
            raise ValueError("Unsupported dataset file extension {}".format(ext))
        return target(tokenizer=tokenizer, data_args=data_args, is_query=is_query, final=final, stream=stream,
                      batch_size=batch_size, num_processes=num_processes, process_index=process_index,
                      cache_dir=cache_dir)

    def _records(self) -> Iterator[Dict]:
        raise NotImplementedError

    def process_one(self, example):
        text = fill_template(self.template, example, self.all_markers, allow_not_found=True)
        tok = self.tokenizer(text, add_special_tokens=self.final, padding="max_length" if self.final else False,
                             truncation=True, max_length=self.max_len, return_attention_mask=self.final,
                             return_token_type_ids=self.final)
        return {"text_id": get_idx(example), **tok}

    def __iter__(self):
        group = self.batch_size * self.num_processes
        lo, hi = self.process_index * self.batch_size, (self.process_index + 1) * self.batch_size
        pending = []
        for rec in self._records():
            pending.append(rec)
            if len(pending) == group:
                for rec_ in pending[lo:hi]:
                    yield self.process_one(rec_)
                pending = []
        for rec_ in pending[lo:hi]:
            yield self.process_one(rec_)


class JsonlDataset(InferenceDataset):
    def _records(self):
        with open(self.data_files[0]) as f:
            for line in f:
                if line.strip():
                    yield json.loads(line)


class TsvDataset(InferenceDataset):
    def __init__(self, tokenizer, data_args: DataArguments, is_query: bool = False, **kwargs):
        super().__init__(tokenizer, data_args, is_query, **kwargs)
        self.all_columns = (data_args.query_column_names if is_query else data_args.doc_column_names).split(",")

    def _records(self):
        with open(self.data_files[0]) as f:
            for line in f:
                yield dict(zip(self.all_columns, line.rstrip("\n").split("\t")))


class PretokenizedDataset(InferenceDataset):
    """``<name>.npy``: int32 ``[n, L]`` token ids, padded with the tokenizer's pad id (``pad_id``: 0 for BERT and T5, 1
    for RoBERTa; 0 without a tokenizer); optional ``<name>.ids.txt`` with one id per row.  The tokenizer is not run:
    rows are sliced to ``max_len``, padded with ``pad_id`` and the mask is ``ids != pad_id``.

    Two ways out: the reference's per-example iterator (``__iter__`` -> DataLoader + DRInferenceCollator, same
    interleaving of ``batch_size`` blocks over the ranks, :99-115), and ``iter_batches()``, which hands whole
    ``[B, L]`` int32 slices of the memory map to ``Retriever`` (one memcpy into a pinned buffer per batch, no
    per-row Python objects) — the ingest path that can feed the encoder at tens of thousands of passages/s.

    A ragged store (``write_ragged_store``) holds the same rows without padding: ``<name>.tokens.npy`` (int32, the rows
    back to back) and ``<name>.offsets.npy`` (int64 ``[n + 1]``, row i = ``tokens[offsets[i]:offsets[i + 1]]``), with
    the same optional ``<name>.ids.txt``; its path is ``<name>.tokens.npy``.  ``iter_batches()`` then yields
    ``(text_ids, tokens int32 [sum(seqlens)], seqlens int32 [b])`` (rows truncated to ``max_len``) for
    ``DRModel.encode_packed_into``, and ``__iter__`` yields padded examples as for the padded store."""

    @property
    def pad_id(self) -> int:
        pad = getattr(self.tokenizer, "pad_token_id", None) if self.tokenizer is not None else None
        return int(pad) if pad is not None else 0

    @property
    def is_ragged(self) -> bool:
        return _ragged_prefix(self.data_files[0]) is not None

    def _open(self):
        prefix = _ragged_prefix(self.data_files[0])
        if prefix is not None:
            tokens = np.load(prefix + ".tokens.npy", mmap_mode="r")
            offsets = np.load(prefix + ".offsets.npy")
            if tokens.ndim != 1 or tokens.dtype != np.int32 or offsets.ndim != 1 or offsets.dtype != np.int64 \
                    or offsets.shape[0] < 1 or offsets[0] != 0 or offsets[-1] != tokens.shape[0] \
                    or (np.diff(offsets) < 0).any():
                raise ValueError("%s: expected int32 tokens [T] and int64 offsets [n + 1] from 0 to T" % prefix)
            rows, n, names_path = (tokens, offsets), offsets.shape[0] - 1, prefix + ".ids.txt"
        else:
            rows = np.load(self.data_files[0], mmap_mode="r")
            if rows.ndim != 2 or rows.dtype != np.int32:
                raise ValueError("%s: expected an int32 [n, L] array, got %s %s" % (self.data_files[0], rows.dtype,
                                                                                   rows.shape))
            n, names_path = rows.shape[0], os.path.splitext(self.data_files[0])[0] + ".ids.txt"
        names = None
        if os.path.exists(names_path):
            with open(names_path) as f:
                names = f.read().split("\n")
            if len(names) < n:
                raise ValueError("%s holds %d ids for %d rows" % (names_path, len(names), n))
        return rows, names

    def _num_rows(self) -> int:
        prefix = _ragged_prefix(self.data_files[0])
        if prefix is not None:
            return np.load(prefix + ".offsets.npy", mmap_mode="r").shape[0] - 1
        return np.load(self.data_files[0], mmap_mode="r").shape[0]

    def _records(self):
        rows, names = self._open()
        if isinstance(rows, tuple):
            tokens, offsets = rows
            for i in range(offsets.shape[0] - 1):
                yield {"id": names[i] if names else str(i), "row": tokens[offsets[i]:offsets[i + 1]]}
            return
        for i in range(rows.shape[0]):
            yield {"id": names[i] if names else str(i), "row": rows[i]}

    def num_local_rows(self) -> int:
        """rows this rank will see (blocks ``process_index, process_index + W, ...`` of ``batch_size`` rows)"""
        n = self._num_rows()
        bs, W, r = self.batch_size, self.num_processes, self.process_index
        full, rest = divmod(n, bs * W)
        return full * bs + max(0, min(bs, rest - r * bs))

    def iter_batches(self):
        """Yields ``(text_ids: list[str], ids: int32 [b, max_len] C-contiguous view or padded copy)`` for this rank's
        blocks, in the order ``__iter__`` would produce the same examples.  A ragged store yields
        ``(text_ids, tokens, seqlens)`` instead (see the class docstring)."""
        ids, names = self._open()
        if isinstance(ids, tuple):
            yield from self._iter_ragged_batches(*ids, names)
            return
        n, width = ids.shape
        bs, W, r = self.batch_size, self.num_processes, self.process_index
        for b0 in range(r * bs, n, W * bs):
            b1 = min(n, b0 + bs)
            block = ids[b0:b1, : self.max_len]
            if width < self.max_len:  # stored narrower than the model's padded length: pad like the reference does
                padded = np.full((b1 - b0, self.max_len), self.pad_id, dtype=np.int32)
                padded[:, :width] = block
                block = padded
            yield (names[b0:b1] if names else [str(i) for i in range(b0, b1)]), block

    def _iter_ragged_batches(self, tokens, offsets, names):
        n = offsets.shape[0] - 1
        bs, W, r = self.batch_size, self.num_processes, self.process_index
        for b0 in range(r * bs, n, W * bs):
            b1 = min(n, b0 + bs)
            starts = offsets[b0:b1]
            lens = np.minimum(offsets[b0 + 1:b1 + 1] - starts, self.max_len)
            if (lens < 1).any():
                raise ValueError("%s: row %d is empty" % (self.data_files[0], b0 + int(np.argmin(lens))))
            if (lens == offsets[b0 + 1:b1 + 1] - starts).all():  # nothing truncated: one contiguous slice
                block = tokens[offsets[b0]:offsets[b1]]
            else:
                ends = np.cumsum(lens)
                block = tokens[np.repeat(starts - (ends - lens), lens) + np.arange(int(ends[-1]))]
            yield (names[b0:b1] if names else [str(i) for i in range(b0, b1)]), block, lens.astype(np.int32)

    def process_one(self, example):
        pad = self.pad_id
        row = np.asarray(example["row"][: self.max_len], dtype=np.int64)
        if row.shape[0] < self.max_len:
            row = np.pad(row, (0, self.max_len - row.shape[0]), constant_values=pad)
        return {"text_id": get_idx(example), "input_ids": row.tolist(), "attention_mask": (row != pad).astype(np.int64).tolist(),
                "token_type_ids": [0] * self.max_len}
