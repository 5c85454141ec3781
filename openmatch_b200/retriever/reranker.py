"""Cross-encoder re-ranking of a run (reference: ``src/openmatch/retriever/reranker.py``):
``Reranker(model, tokenizer, corpus_dataset, args).rerank(query_dataset, run) -> {qid: {did: score}}``.

The reference re-tokenises every (query, passage) pair on the host (``encode_plus``) and scores padded batches of
``q_max_len + p_max_len + 2`` tokens.  Here every query and passage the run references is tokenised once (or read from
a pretokenised store), the rows go to the device once per call as two int32 token stores, and each batch of pairs is
assembled on the device and encoded without padding (``RRModel.encode_pairs`` -> ``om_encode_pairs``).  Scores stay
on the device until one copy at the end.

Pair content (``DESIGN.md`` §6): the query / passage ids of ``InferenceDataset(final=False)``, i.e. the text rendered
through its template and tokenised without special tokens, truncated to ``q_max_len`` / ``p_max_len``; a pretokenised
row without its padding (the tokenizer's pad id) and, when it starts with the tokenizer's prefix and ends with its suffix, without those.
"""
from __future__ import annotations

import logging
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from ..arguments import InferenceArguments as EncodingArguments
from ..dataset.inference_dataset import PretokenizedDataset, get_idx

logger = logging.getLogger(__name__)


def special_tokens(tokenizer) -> Tuple[List[int], List[int]]:
    """(prefix, suffix): the ids the tokenizer puts around one sequence, ``tokenizer(x) = prefix ++ tokenizer(x,
    add_special_tokens=False) ++ suffix`` ([CLS] / [SEP] for BERT, nothing / </s> for T5)."""
    for probe in ("hello world", "a"):
        full = list(tokenizer(probe)["input_ids"])
        bare = list(tokenizer(probe, add_special_tokens=False)["input_ids"])
        for i in range(len(full) - len(bare) + 1):
            if bare and full[i:i + len(bare)] == bare:
                return full[:i], full[i + len(bare):]
    raise ValueError("cannot find the special tokens of %s" % type(tokenizer).__name__)


def encode_pair(prefix: Sequence[int], suffix: Sequence[int], item1: Sequence[int], item2: Sequence[int]) -> List[int]:
    """The tokens of the reference's ``encode_pair(tokenizer, item1, item2, q_max, p_max)`` (reranker.py:23-29) without
    its padding: ``encode_plus(item1 + item2, truncation='longest_first', padding='max_length', max_length=q_max +
    p_max + 2)`` is ``prefix ++ item1 ++ item2 ++ suffix`` with token types 0, and never truncates because ``len(item1)
    <= q_max`` and ``len(item2) <= p_max``.  Restated because transformers 5 has no ``encode_plus`` on id lists."""
    return list(prefix) + list(item1) + list(item2) + list(suffix)


def assemble_pairs(a_tokens: np.ndarray, b_tokens: np.ndarray, spans: np.ndarray, prefix: Sequence[int],
                   suffix: Sequence[int]) -> Tuple[np.ndarray, np.ndarray]:
    """Host assembly of what ``om_encode_pairs`` assembles on the device: (int64 tokens back to back, int32 lengths)."""
    rows = [encode_pair(prefix, suffix, a_tokens[a0:a0 + al], b_tokens[b0:b0 + bl]) for a0, al, b0, bl in spans]
    lens = np.array([len(r) for r in rows], dtype=np.int32)
    return np.array([t for r in rows for t in r], dtype=np.int64), lens


def _content(row: np.ndarray, prefix: Sequence[int], suffix: Sequence[int], max_len: int, pad_id: int = 0) -> np.ndarray:
    """a pretokenised row's pair content: the padding (the tokenizer's pad id) dropped, a dense-retrieval row's special
    tokens stripped"""
    row = np.asarray(row)
    row = row[row != pad_id]
    npre, nsuf = len(prefix), len(suffix)
    if (npre or nsuf) and row.shape[0] >= npre + nsuf and list(row[:npre]) == list(prefix) \
            and list(row[row.shape[0] - nsuf:]) == list(suffix):
        row = row[npre:row.shape[0] - nsuf]
    return row[:max_len]


def token_store(dataset, ids: Sequence[str], prefix: Sequence[int], suffix: Sequence[int]):
    """One int32 row per id in ``ids`` (each once) from an ``InferenceDataset`` loaded with ``final=False``: (tokens back
    to back, {id: (start, length)}).  Raises ``KeyError`` naming an id the source does not hold."""
    want = set(ids)
    rows: Dict[str, np.ndarray] = {}
    if isinstance(dataset, PretokenizedDataset):
        store, names = dataset._open()
        n = store[1].shape[0] - 1 if isinstance(store, tuple) else store.shape[0]
        index = {name: i for i, name in enumerate(names[:n])} if names else {str(i): i for i in range(n)}
        for name in want:
            i = index.get(name)
            if i is None:
                continue
            row = store[0][store[1][i]:store[1][i + 1]] if isinstance(store, tuple) else store[i]
            rows[name] = _content(row, prefix, suffix, dataset.max_len, dataset.pad_id)
    else:  # text: tokenised once per id, as InferenceDataset(final=False) does
        for rec in dataset._records():
            name = get_idx(rec)
            if name in want and name not in rows:
                rows[name] = np.asarray(dataset.process_one(rec)["input_ids"], dtype=np.int32)
    missing = [name for name in ids if name not in rows]
    if missing:
        raise KeyError("id %r of the run is not in %s" % (missing[0], dataset.data_files[0]))
    where, parts, off = {}, [], 0
    for name in dict.fromkeys(ids):
        r = rows[name].astype(np.int32)
        where[name] = (off, int(r.shape[0]))
        parts.append(r)
        off += int(r.shape[0])
    return (np.concatenate(parts) if parts else np.zeros(0, np.int32)), where


def local_pair_indices(n: int, block: int, world: int, rank: int) -> np.ndarray:
    """the pairs of rank ``rank``: blocks ``rank, rank + world, ...`` of ``block`` pairs in run order (the reference's
    ``IterableDatasetShard`` blocks, without its wrap-around padding)"""
    idx = np.arange(n)
    return idx[(idx // block) % world == rank]


class Reranker:
    def __init__(self, model, tokenizer, corpus_dataset, args: EncodingArguments):
        logger.info("Initializing reranker")
        self.tokenizer = tokenizer
        self.corpus_dataset = corpus_dataset
        self.args = args
        self.model = model.to(args.device)
        self.model.eval()

    def _score(self, a_tokens: np.ndarray, b_tokens: np.ndarray, spans: np.ndarray, prefix, suffix) -> np.ndarray:
        """fp32 scores of the pairs ``spans`` [n, 4] over the two token stores, batches of per_device_eval_batch_size"""
        dev = self.args.device
        a = torch.from_numpy(a_tokens).to(dev)
        b = torch.from_numpy(b_tokens).to(dev)
        out = torch.empty((spans.shape[0], 1), dtype=torch.float32, device=dev)
        bs = self.args.per_device_eval_batch_size
        for lo in range(0, spans.shape[0], bs):
            self.model.encode_pairs(a, b, spans[lo:lo + bs], prefix, suffix, out=out[lo:lo + bs])
        return out[:, 0].cpu().numpy()

    def rerank(self, query_dataset, run: Dict[str, Dict[str, float]]) -> Dict[str, Dict[str, float]]:
        prefix, suffix = special_tokens(self.tokenizer)
        q_max, p_max = query_dataset.max_len, self.corpus_dataset.max_len
        limit = self.model.max_pair_len()
        if q_max + p_max + len(prefix) + len(suffix) > limit:
            raise ValueError("q_max_len %d + p_max_len %d + %d special tokens exceed the model's %d tokens" % (
                q_max, p_max, len(prefix) + len(suffix), limit))
        pairs = [(qid, did) for qid, docs in run.items() for did in docs]
        world, rank = self.args.world_size, self.args.process_index
        bs = self.args.per_device_eval_batch_size
        mine = local_pair_indices(len(pairs), bs, world, rank)
        local = [pairs[i] for i in mine]
        a_tokens, qwhere = token_store(query_dataset, [q for q, _ in local], prefix, suffix)
        b_tokens, dwhere = token_store(self.corpus_dataset, [d for _, d in local], prefix, suffix)
        spans = np.array([qwhere[q] + dwhere[d] for q, d in local], dtype=np.int64).reshape(-1, 4)
        scores = self._score(a_tokens, b_tokens, spans, prefix, suffix) if local else np.zeros(0, np.float32)
        if world > 1:
            # every rank holds the same run: rank 0 puts each rank's scores back at that rank's pair indices and
            # returns the union of all pairs (no per-query cut)
            parts = [None] * world if rank == 0 else None
            dist.gather_object(scores, parts, dst=0)
            if rank == 0:
                full = np.zeros(len(pairs), dtype=np.float32)
                for r, part in enumerate(parts):
                    full[local_pair_indices(len(pairs), bs, world, r)] = part
                local, scores = pairs, full
        result: Dict[str, Dict[str, float]] = {}
        for (qid, did), s in zip(local, scores.tolist()):
            result.setdefault(qid, {})[did] = s
        return result
