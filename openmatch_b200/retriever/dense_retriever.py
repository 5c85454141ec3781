"""Dense retriever with the reference's public surface (``src/openmatch/retriever/dense_retriever.py``):
``Retriever`` (``doc_embedding_inference``, ``init_index_and_add``, ``build_all``, ``build_embeddings``,
``from_embeddings``, ``reset_index``, ``query_embedding_inference``, ``search``, ``retrieve``) and
``SuccessiveRetriever``; ``FaissRetriever`` is the successor repo's name for the same class.

What changed underneath:
  * embeddings come from the sm_90a encoder and are written straight into this rank's HBM index shard
    (zero-copy ``reserve_rows``/``commit_rows``); one D2H copy per *corpus* (for the reference-compatible
    pickle), not one blocking ``.cpu()`` per batch (reference :81);
  * the index is ``openmatch_b200.index.FlatIPIndex`` (fused wgmma scan + top-k) instead of faiss;
    with ``world_size > 1`` every rank keeps the rows it encoded, searches all queries against its shard and
    the per-shard top-k lists are all-gathered over NCCL and merged (the reference instead idles all ranks
    but 0 and lets faiss shard inside one process, :43-58,200-203);
  * the on-disk format is unchanged: ``embeddings.{corpus,query}.rank.{r}`` = pickle protocol 4 of
    ``(float32 [n, d], list[str])`` (:84-86,160-161), so either implementation can read the other's files.
"""
from __future__ import annotations

import glob
import logging
import os
import pickle
from typing import Dict, List

import numpy as np
import torch
from torch.utils.data import DataLoader, IterableDataset
from tqdm import tqdm

from ..arguments import InferenceArguments as EncodingArguments
from ..dataset import DRInferenceCollator
from ..embedding_store import EmbeddingFile, write_embedding_file
from ..index import FlatIPIndex, comm_for, range_radius, shard_offsets
from ..modeling import DRModelForInference
from ..utils import merge_retrieval_results_by_score

logger = logging.getLogger(__name__)


def _results_dict(query_ids: List[str], doc_lookup: np.ndarray, D: np.ndarray, I: np.ndarray) -> Dict[str, Dict[str, float]]:
    """{qid: {docid: score}} in rank order.  Padding slots (id -1, k > ntotal) are dropped."""
    out = {}
    scores = D.tolist()
    for qi, qid in enumerate(query_ids):
        row = I[qi]
        valid = row >= 0
        names = doc_lookup[row[valid]].tolist()
        out[str(qid)] = dict(zip(names, scores[qi][: len(names)])) if valid.all() else \
            dict(zip(names, np.asarray(scores[qi])[valid].tolist()))
    return out


def _range_dict(query_ids: List[str], doc_lookup: np.ndarray, lims: np.ndarray, D: np.ndarray, I: np.ndarray):
    """{qid: {docid: score}} of a range search, each query's documents in rank order."""
    scores = D.tolist()
    names = doc_lookup[I].tolist() if len(I) else []
    return {str(qid): dict(zip(names[lims[qi]:lims[qi + 1]], scores[lims[qi]:lims[qi + 1]]))
            for qi, qid in enumerate(query_ids)}


def doc_filter(doc_lookup, query_ids, allowed_docs=None, exclude=None, id_offset: int = 0):
    """Maps a search filter over doc-id strings onto index rows: ``(allow, excluded)`` with ``allow`` a bool array over
    the rows of ``doc_lookup`` (None: every row) and ``excluded`` one list of ids (``id_offset`` + row) per query of
    ``query_ids`` (None: no exclusions).  ``allowed_docs``: iterable of doc ids; ``exclude``: ``{qid: [doc ids]}``.  Doc
    ids the lookup does not hold are ignored, so every rank of a sharded index maps the same arguments on its own rows."""
    if allowed_docs is None and exclude is None:
        return None, None
    row = {d: i for i, d in enumerate(doc_lookup)}
    allow = None
    if allowed_docs is not None:
        allow = np.zeros(len(doc_lookup), dtype=bool)
        allow[[row[d] for d in allowed_docs if d in row]] = True
    excluded = None
    if exclude is not None:
        excluded = [[id_offset + row[d] for d in exclude.get(q, ()) if d in row] for q in query_ids]
    return allow, excluded


def _index_dtype(args) -> torch.dtype:
    name = getattr(args, "index_dtype", "float32")
    dtypes = {"float32": torch.float32, "float16": torch.float16, "int8": torch.int8}
    if name not in dtypes:
        raise ValueError("--index_dtype must be 'float32', 'float16' or 'int8', got %r" % name)
    return dtypes[name]


def _index_memory(args, writes_rows: bool = False) -> str:
    """``--index_memory``: 'device' (the rows in HBM) or 'host' (the rows in pinned host memory, streamed through the GPU
    by every search).  A host-resident index is built from embedding files on one process: the paths that write rows in
    place on the GPU (``writes_rows``) and row-sharded retrieval need the device index."""
    memory = getattr(args, "index_memory", "device")
    if memory not in ("device", "host"):
        raise ValueError("--index_memory must be 'device' or 'host', got %r" % (memory,))
    if memory == "host" and args.world_size > 1:
        raise ValueError("--index_memory host searches on one process; world_size is %d (row-sharded retrieval needs "
                         "--index_memory device)" % args.world_size)
    if memory == "host" and writes_rows:
        raise ValueError("--index_memory host: a host-resident index is built from embedding files (driver.retrieve); "
                         "encoding the corpus into the index writes its rows in place on the GPU and needs "
                         "--index_memory device")
    return memory


class RankArrays:
    """Search output kept as arrays (``Retriever.search(..., as_arrays=True)``): row ``i`` of ``I`` / ``D`` holds the
    ranked rows of ``doc_names`` / scores for ``query_ids[i]``; ``to_dict()`` gives the reference's dict-of-dicts."""

    def __init__(self, query_ids, doc_names, D, I):
        self.query_ids, self.doc_names, self.D, self.I = list(query_ids), np.asarray(doc_names), D, I

    def to_dict(self) -> Dict[str, Dict[str, float]]:
        return _results_dict(self.query_ids, self.doc_names, self.D, self.I)

    def unique_doc_ids(self) -> bool:
        return len(set(self.doc_names.tolist())) == self.doc_names.shape[0]

    def save_trec(self, path: str, run_id: str = "OpenMatch"):
        from ..utils import save_as_trec, save_trec_arrays
        if self.unique_doc_ids():
            save_trec_arrays(self.query_ids, self.doc_names, self.I, self.D, path, run_id)
        else:  # duplicated doc-id strings collapse in the reference's dict (dense_retriever.py:186-187)
            save_as_trec(self.to_dict(), path, run_id)

    def __len__(self):
        return len(self.query_ids)


class Retriever:

    def __init__(self, model: DRModelForInference, corpus_dataset: IterableDataset, args: EncodingArguments):
        logger.info("Initializing retriever")
        self.model = model
        self.corpus_dataset = corpus_dataset
        self.args = args
        self.doc_lookup: List[str] = []
        self.query_lookup: List[str] = []
        self.index = None
        self._resident_rows = 0  # rows of self.index that were written in place by doc_embedding_inference
        self.model.to(self.args.device)
        self.model.eval()

    # ------------------------------------------------------------------ index plumbing
    def _initialize_faiss_index(self, dim: int):
        """Name kept from the reference (:38-41); the index is the HBM-resident flat IP index with the row storage
        ``--index_dtype`` names (float32, float16 or int8), in the memory ``--index_memory`` names."""
        self.index = FlatIPIndex(dim, dtype=_index_dtype(self.args), memory=_index_memory(self.args))

    def _move_index_to_gpu(self):
        """The reference clones a CPU faiss index to all GPUs here (:43-58).  Ours is born in HBM, one row
        shard per process, so there is nothing to move."""
        logger.info("Index already resident in HBM (%d rows on this rank)", 0 if self.index is None else self.index.ntotal)

    def _loader(self, dataset):
        return DataLoader(dataset, batch_size=self.args.per_device_eval_batch_size, collate_fn=DRInferenceCollator(),
                          num_workers=self.args.dataloader_num_workers, pin_memory=self.args.dataloader_pin_memory)

    def _encode_dataset(self, dataset, is_query: bool, into_index: bool):
        """Shared encode loop: H2D of the id tensors, CUDA encoder, embeddings stay on the device.  With
        ``into_index`` the encoder writes its output rows IN PLACE into this rank's index shard
        (``reserve_rows`` -> ``DRModel.encode_into`` -> ``commit_rows``: no intermediate tensor, no copy).
        Datasets that can hand out whole ``[B, L]`` blocks (``PretokenizedDataset.iter_batches``) skip the per-example
        DataLoader / collator path altogether."""
        if hasattr(dataset, "iter_batches") and hasattr(self.model, "encode_into"):
            return self._encode_blocks(dataset, is_query, into_index)
        ids: List[str] = []
        chunks: List[torch.Tensor] = []
        device = self.args.device
        in_place = into_index and hasattr(self.model, "encode_into")
        for batch_ids, batch in tqdm(self._loader(dataset), disable=self.args.local_process_index > 0):
            ids.extend(batch_ids)
            batch = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
            if in_place:
                self._encode_rows_in_place(batch, is_query)
                continue
            out = self.model(query=batch) if is_query else self.model(passage=batch)
            reps = out.q_reps if is_query else out.p_reps
            if into_index:  # foreign model object without encode_into: one device-to-device copy
                if self.index is None:
                    self._initialize_faiss_index(reps.shape[1])
                if self.index.dtype == torch.int8:  # the index quantises what it adds
                    self.index.add(reps)
                else:
                    rows = self.index.reserve_rows(reps.shape[0])
                    rows.copy_(reps)
                    self.index.commit_rows(reps.shape[0])
            else:
                chunks.append(reps.float())
        return ids, chunks

    def _encode_rows_in_place(self, batch, is_query: bool):
        if self.index is None:
            self._initialize_faiss_index(self.model.rep_dim(is_query))
        n = batch["input_ids"].shape[0]
        rows = self.index.reserve_rows(n)
        self.model.encode_into(batch, rows, is_query)
        self.index.commit_rows(n)

    def _encode_blocks(self, dataset, is_query: bool, into_index: bool):
        """Block ingest: memory-mapped int32 ``[b, L]`` slice -> pinned staging buffer (double-buffered) -> async H2D
        -> int64 ids + mask (``ids != dataset.pad_id``) built on the device -> encoder (-> index rows in place)."""
        if getattr(dataset, "is_ragged", False) and hasattr(self.model, "encode_packed_into"):
            return self._encode_ragged_blocks(dataset, is_query, into_index)
        device = self.args.device
        pad_id = getattr(dataset, "pad_id", 0)
        ids: List[str] = []
        chunks: List[torch.Tensor] = []
        bs, L = dataset.batch_size, dataset.max_len
        stage = [torch.empty((bs, L), dtype=torch.int32).pin_memory() for _ in range(2)]
        busy = [None, None]
        if into_index:
            if self.index is None:
                self._initialize_faiss_index(self.model.rep_dim(is_query))
            if hasattr(dataset, "num_local_rows"):
                self.index.reserve_rows(dataset.num_local_rows())  # capacity only: no re-allocation while encoding
        dim = self.model.rep_dim(is_query)
        for bi, (names, block) in enumerate(tqdm(dataset.iter_batches(), disable=self.args.local_process_index > 0)):
            slot = bi & 1
            if busy[slot] is not None:
                busy[slot].synchronize()  # the H2D copy that last read this pinned buffer has finished
            n = block.shape[0]
            np.copyto(stage[slot][:n].numpy(), block)
            d_ids = stage[slot][:n].to(device, non_blocking=True)
            busy[slot] = torch.cuda.Event()
            busy[slot].record()
            batch = {"input_ids": d_ids.long(), "attention_mask": (d_ids != pad_id).long()}
            ids.extend(names)
            if into_index:
                self._encode_rows_in_place(batch, is_query)
            else:
                out = torch.empty((n, dim), dtype=torch.float32, device=device)
                self.model.encode_into(batch, out, is_query)
                chunks.append(out)
        return ids, chunks

    def _encode_ragged_blocks(self, dataset, is_query: bool, into_index: bool):
        """Block ingest of a ragged store: the block's tokens without padding -> pinned staging buffer (double-buffered)
        -> async H2D -> ``encode_packed_into`` (-> index rows in place, fp32 or fp16 storage alike)."""
        device = self.args.device
        ids: List[str] = []
        chunks: List[torch.Tensor] = []
        stage = [torch.empty((dataset.batch_size * dataset.max_len,), dtype=torch.int32).pin_memory() for _ in range(2)]
        busy = [None, None]
        if into_index:
            if self.index is None:
                self._initialize_faiss_index(self.model.rep_dim(is_query))
            self.index.reserve_rows(dataset.num_local_rows())  # capacity only: no re-allocation while encoding
        dim = self.model.rep_dim(is_query)
        for bi, (names, tokens, seqlens) in enumerate(tqdm(dataset.iter_batches(),
                                                           disable=self.args.local_process_index > 0)):
            slot = bi & 1
            if busy[slot] is not None:
                busy[slot].synchronize()  # the H2D copy that last read this pinned buffer has finished
            n, t = seqlens.shape[0], tokens.shape[0]
            np.copyto(stage[slot][:t].numpy(), tokens)
            d_tokens = stage[slot][:t].to(device, non_blocking=True)
            busy[slot] = torch.cuda.Event()
            busy[slot].record()
            ids.extend(names)
            if into_index:
                rows = self.index.reserve_rows(n)
                self.model.encode_packed_into(d_tokens, seqlens, rows, is_query)
                self.index.commit_rows(n)
            else:
                out = torch.empty((n, dim), dtype=torch.float32, device=device)
                self.model.encode_packed_into(d_tokens, seqlens, out, is_query)
                chunks.append(out)
        return ids, chunks

    # ------------------------------------------------------------------ corpus side
    def doc_embedding_inference(self):
        if self.corpus_dataset is None:
            raise ValueError("No corpus dataset provided")
        _index_memory(self.args, writes_rows=True)
        ids, _ =self._encode_dataset(self.corpus_dataset, is_query=False, into_index=True)
        self.doc_lookup = list(ids)
        self._resident_rows = len(ids)
        os.makedirs(self.args.output_dir, exist_ok=True)
        path = os.path.join(self.args.output_dir, "embeddings.corpus.rank.{}".format(self.args.process_index))
        if self.index is None or self.index.ntotal == 0:
            with open(path, "wb") as f:
                pickle.dump((np.zeros((0, 0), dtype=np.float32), ids), f, protocol=4)
        else:
            # same bytes-on-disk contract as the reference's pickle.dump((encoded, lookup), protocol=4) (:84-86), but the
            # shard is streamed out of HBM through one pinned chunk instead of materialising [n, d] twice on the host
            rows = self.index.rows_f32() if self.index.dtype == torch.int8 else self.index.master_rows()
            write_embedding_file(path, rows, ids, n=self.index.ntotal, d=self.index.d)
        if self.args.world_size > 1:
            torch.distributed.barrier()

    def init_index_and_add(self, partition: str = None):
        logger.info("Initializing index from pre-computed document embeddings")
        files = [partition] if partition is not None else sorted(
            glob.glob(os.path.join(self.args.output_dir, "embeddings.corpus.rank.*")))
        for i, part in enumerate(files):
            # reference: pickle.load of the whole (matrix, ids) tuple (:96-101); here the matrix payload is memory-mapped
            # and fed to the index chunk by chunk (files written by the reference, by us or by split_embeddings.py)
            ef = EmbeddingFile(part)
            encoded, lookup = ef, ef.ids
            # (The reference re-creates its index on the first file of every call, :102-103; a rank of a row-sharded
            # retriever calls this once per file it owns, so rows must accumulate — start afresh with reset_index().)
            if ef.shape[0] == 0:
                continue
            if self.index is None or self.index.d != encoded.shape[1]:
                self._initialize_faiss_index(encoded.shape[1])
            if getattr(self.index, "memory", "device") == "device":
                self.index.reserve_rows(ef.shape[0])  # capacity for the whole file: one allocation
            for chunk in ef.chunks():
                self.index.add(np.ascontiguousarray(chunk))
            self.doc_lookup.extend(lookup)

    @classmethod
    def build_all(cls, model: DRModelForInference, corpus_dataset: IterableDataset, args: EncodingArguments):
        _index_memory(args, writes_rows=True)
        retriever = cls(model, corpus_dataset, args)
        retriever.doc_embedding_inference()  # leaves this rank's rows in its HBM shard
        if args.world_size > 1:
            torch.distributed.barrier()
        return retriever

    @classmethod
    def build_embeddings(cls, model: DRModelForInference, corpus_dataset: IterableDataset, args: EncodingArguments):
        _index_memory(args, writes_rows=True)
        retriever = cls(model, corpus_dataset, args)
        retriever.doc_embedding_inference()
        return retriever

    @classmethod
    def from_embeddings(cls, model: DRModelForInference, args: EncodingArguments):
        _index_memory(args)
        retriever = cls(model, None, args)
        if args.world_size > 1:
            # rank r loads the files r, r+W, ... : the corpus ends up row-sharded across the GPUs
            files = sorted(glob.glob(os.path.join(args.output_dir, "embeddings.corpus.rank.*")))
            for part in files[args.process_index::args.world_size]:
                retriever.init_index_and_add(part)
            torch.distributed.barrier()
        else:
            retriever.init_index_and_add()
        return retriever

    def reset_index(self):
        if self.index:
            self.index.reset()
        self.doc_lookup = []
        self.query_lookup = []
        self._resident_rows = 0

    # ------------------------------------------------------------------ query side
    def query_embedding_inference(self, query_dataset: IterableDataset):
        ids, chunks = self._encode_dataset(query_dataset, is_query=True, into_index=False)
        self._q_ids = list(ids)
        self._q_reps = torch.cat(chunks) if chunks else torch.zeros((0, 0), device=self.args.device)
        encoded = self._q_reps.cpu().numpy()
        os.makedirs(self.args.output_dir, exist_ok=True)
        with open(os.path.join(self.args.output_dir, "embeddings.query.rank.{}".format(self.args.process_index)), "wb") as f:
            pickle.dump((encoded, ids), f, protocol=4)
        if self.args.world_size > 1:
            torch.distributed.barrier()

    def _load_queries(self):
        encoded = []
        self.query_lookup = []
        for i in range(self.args.world_size):
            with open(os.path.join(self.args.output_dir, "embeddings.query.rank.{}".format(i)), "rb") as f:
                reps, lookup = pickle.load(f)
            encoded.append(reps)
            self.query_lookup.extend(lookup)
        return np.concatenate(encoded)

    def search(self, topk: int = 100, as_arrays: bool = False, allowed_docs=None, exclude=None):
        """Reference contract (:166-192): ``{qid: {docid: score}}``.  ``as_arrays=True`` returns the same ranking as
        a :class:`RankArrays` (no per-result Python objects; rank 0 only when sharded).

        ``allowed_docs`` (doc ids) restricts the ranking to those documents and ``exclude`` (``{qid: [doc ids]}``, at
        most 128 per query) drops documents per query, e.g. the query's positives or the query itself; the ranking is the
        exact top-k among the remaining documents (``FlatIPIndex.search``'s filter).  Unknown doc ids are ignored."""
        logger.info("Searching")
        out = self._search_index(lambda q, **f: self.index.search(q, topk, **f),
                                 lambda comm, q, offset, **f: self.index.search_sharded_device(comm, q, topk, offset, **f),
                                 allowed_docs, exclude)
        if out is None:
            return RankArrays([], [], None, None) if as_arrays else {}
        names, (D, I) = out
        result = RankArrays(self.query_lookup, names, D, I)
        logger.info("End searching with %d queries", len(result))
        return result if as_arrays else result.to_dict()

    def range_search(self, radius, allowed_docs=None, exclude=None):
        """Every document whose score is strictly above ``radius`` (a float, or one per query in query order) as
        ``{qid: {docid: score}}``, each query's documents in rank order (``FlatIPIndex.range_search``).  Sharded: every
        rank takes part and rank 0 builds the result; the other ranks return ``{}``.

        ``allowed_docs`` / ``exclude`` filter as in :meth:`search`: only the allowed documents, less each query's
        excluded ones (at most 128 per query, e.g. the query itself in near-duplicate detection), are returned."""
        def radii(q):
            return range_radius(radius, q.shape[0]).numpy()

        out = self._search_index(lambda q, **f: self.index.range_search(q, radii(q), **f),
                                 lambda comm, q, offset, **f: self.index.range_search_sharded_device(
                                     comm, q, torch.from_numpy(radii(q)), offset, **f),
                                 allowed_docs, exclude)
        if out is None:
            return {}
        names, (lims, D, I) = out
        return _range_dict(self.query_lookup, names, lims, D, I)

    def _search_index(self, local, sharded, allowed_docs, exclude):
        """One search of the saved queries, with the filter mapped onto this rank's rows.  One process:
        ``local(queries, **filter)`` with numpy queries and results.  ``world_size > 1``: every rank searches all queries
        against its row shard, ``sharded(comm, queries, id_offset, **filter)`` with CUDA tensors, and the doc-id strings
        are gathered to rank 0, which alone builds the result (like the reference, :200-203).  Returns (doc names, numpy
        results), or None on the other ranks.  An unfiltered search passes no filter arguments."""
        if self.index is None:
            raise ValueError("Index is not initialized")
        encoded = self._load_queries()
        W = self.args.world_size
        offset = shard_offsets(len(self.doc_lookup))[0] if W > 1 else 0
        # each rank maps the filter on its own rows (its slice of the bitmap, exclusions among its own documents)
        allow, excluded = doc_filter(self.doc_lookup, self.query_lookup, allowed_docs, exclude, offset)
        f = {} if allow is None and excluded is None else {"allow": allow, "exclude": excluded}
        if W <= 1:
            return np.array(self.doc_lookup), local(encoded, **f)
        q = torch.from_numpy(np.ascontiguousarray(encoded, dtype=np.float32)).to(self.args.device)
        results = sharded(comm_for(None), q, offset, **f)
        rank0 = self.args.process_index == 0
        lookups = [None] * W if rank0 else None
        torch.distributed.gather_object(self.doc_lookup, lookups, dst=0)
        if not rank0:
            return None
        return np.array([d for part in lookups for d in part]), tuple(t.cpu().numpy() for t in results)

    def retrieve(self, query_dataset: IterableDataset, topk: int = 100, as_arrays: bool = False, allowed_docs=None,
                 exclude=None):
        """Encodes the queries and searches them; ``allowed_docs`` / ``exclude`` filter as in :meth:`search`."""
        self.query_embedding_inference(query_dataset)
        self.model.cpu()
        del self.model
        torch.cuda.empty_cache()
        if self.args.world_size > 1:
            # collective: every rank takes part, rank 0 gets the result
            results = self.search(topk, as_arrays, allowed_docs, exclude)
            torch.distributed.barrier()
            return results
        return self.search(topk, as_arrays, allowed_docs, exclude)


class SuccessiveRetriever(Retriever):
    """Partition-at-a-time search for corpora larger than the index memory (reference :209-236)."""

    @classmethod
    def from_embeddings(cls, model: DRModelForInference, args: EncodingArguments):
        return cls(model, None, args)

    def retrieve(self, query_dataset: IterableDataset, topk: int = 100):
        self.query_embedding_inference(query_dataset)
        del self.model
        torch.cuda.empty_cache()
        final_result = {}
        if self.args.process_index == 0:
            encoded = self._load_queries()
            for partition in sorted(glob.glob(os.path.join(self.args.output_dir, "embeddings.corpus.rank.*"))):
                logger.info("Loading partition %s", partition)
                self.init_index_and_add(partition)
                D, I = self.index.search(encoded, topk)
                cur = _results_dict(self.query_lookup, np.array(self.doc_lookup), D, I)
                self.reset_index()
                self.query_lookup = []
                for i in range(self.args.world_size):  # reset_index cleared the ids; restore them
                    with open(os.path.join(self.args.output_dir, "embeddings.query.rank.{}".format(i)), "rb") as f:
                        self.query_lookup.extend(pickle.load(f)[1])
                final_result = merge_retrieval_results_by_score([final_result, cur], topk)
        if self.args.world_size > 1:
            torch.distributed.barrier()
        return final_result


FaissRetriever = Retriever  # name used by OpenMatch's successor repo and by BASELINE.json's north_star
