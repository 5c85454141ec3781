"""CPU: the host side of cross-encoder re-ranking (openmatch_b200.retriever.reranker, driver.rerank).

Pair assembly from spans over the token stores must reproduce the reference's own pairs (tests/golden/rerank_small.npz,
made by tests/golden/make_golden_rerank.py) for TSV text, for padded and ragged pretokenised stores of the content rows
and for dense-retrieval rows with their special tokens; the run cut, missing ids, the length limit, and the multi-rank
gather (the union of all pairs on rank 0, no per-query cut, one TREC file)."""
import os
import socket
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _fixture(golden_dir, tmp_path):
    from transformers import BertTokenizer
    z = np.load(os.path.join(golden_dir, "rerank_small.npz"))
    (tmp_path / "vocab.txt").write_text("\n".join(z["vocab"].tolist()))
    tok = BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)
    (tmp_path / "queries.tsv").write_text("".join(x + "\n" for x in z["queries"].tolist()))
    (tmp_path / "corpus.tsv").write_text("".join(x + "\n" for x in z["corpus"].tolist()))
    run = {}
    for q, d, s in zip(z["run_qid"].tolist(), z["run_did"].tolist(), z["run_score"].tolist()):
        run.setdefault(q, {})[d] = s
    return z, tok, run


def _data_args(tmp_path, z, query_path=None, corpus_path=None):
    from openmatch_b200.arguments import DataArguments
    return DataArguments(query_path=str(query_path or tmp_path / "queries.tsv"),
                         corpus_path=str(corpus_path or tmp_path / "corpus.tsv"), q_max_len=int(z["q_max_len"]),
                         p_max_len=int(z["p_max_len"]), query_template="<text>", query_column_names="id,text",
                         doc_template="<title> <text>", doc_column_names="id,title,text")


def _datasets(tok, dargs):
    from openmatch_b200.dataset import InferenceDataset
    return (InferenceDataset.load(tok, dargs, is_query=True, final=False, stream=False),
            InferenceDataset.load(tok, dargs, is_query=False, final=False, stream=False))


def _assembled(tok, qds, cds, run):
    from openmatch_b200.retriever.reranker import assemble_pairs, special_tokens, token_store
    prefix, suffix = special_tokens(tok)
    pairs = [(q, d) for q, docs in run.items() for d in docs]
    a, qw = token_store(qds, [q for q, _ in pairs], prefix, suffix)
    b, dw = token_store(cds, [d for _, d in pairs], prefix, suffix)
    spans = np.array([qw[q] + dw[d] for q, d in pairs], dtype=np.int64)
    tokens, lens = assemble_pairs(a, b, spans, prefix, suffix)
    return np.split(tokens, np.cumsum(lens)[:-1])


def _want(z):
    m = z["attention_mask"].astype(bool)
    return [z["input_ids"][i][m[i]].astype(np.int64) for i in range(m.shape[0])]


def test_special_tokens_and_encode_pair(golden_dir, tmp_path):
    from openmatch_b200.retriever.reranker import encode_pair, special_tokens
    _, tok, _ = _fixture(golden_dir, tmp_path)
    prefix, suffix = special_tokens(tok)
    assert (prefix, suffix) == ([tok.cls_token_id], [tok.sep_token_id])
    assert encode_pair(prefix, suffix, [8, 9], [10]) == [2, 8, 9, 10, 3]
    assert encode_pair(prefix, suffix, [], []) == [2, 3]


def test_text_pairs_match_reference(golden_dir, tmp_path):
    z, tok, run = _fixture(golden_dir, tmp_path)
    qds, cds = _datasets(tok, _data_args(tmp_path, z))
    got, want = _assembled(tok, qds, cds, run), _want(z)
    assert len(got) == len(want) == 24
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert max(len(w) for w in want) == 2 + int(z["q_max_len"]) + int(z["p_max_len"])  # premise: truncation happened


def _content_rows(tok, path, cols, template, max_len, special):
    from openmatch_b200.utils import fill_template
    names, rows = [], []
    for line in open(path):
        rec = dict(zip(cols, line.rstrip("\n").split("\t")))
        names.append(rec["id"])
        text = fill_template(template, rec, allow_not_found=True)
        rows.append(tok(text, add_special_tokens=special, truncation=True, max_length=max_len)["input_ids"])
    return names, rows


def _write_store(tmp_path, stem, names, rows, ragged):
    from openmatch_b200.dataset import write_ragged_store
    width = max(len(r) for r in rows) + 3
    arr = np.zeros((len(rows), width), np.int32)
    for i, r in enumerate(rows):
        arr[i, :len(r)] = r
    if ragged:
        return write_ragged_store(str(tmp_path / stem), arr, names)
    np.save(tmp_path / (stem + ".npy"), arr)
    (tmp_path / (stem + ".ids.txt")).write_text("\n".join(names))
    return str(tmp_path / (stem + ".npy"))


@pytest.mark.parametrize("kind", ["padded", "ragged", "dr_padded", "dr_ragged"])
def test_store_pairs_match_reference(golden_dir, tmp_path, kind):
    z, tok, run = _fixture(golden_dir, tmp_path)
    qmax, pmax = int(z["q_max_len"]), int(z["p_max_len"])
    dr = kind.startswith("dr")
    # content rows, or dense-retrieval rows ([CLS] content [SEP]) tokenised long enough that nothing was cut
    extra = 2 if dr else 0
    qn, qr = _content_rows(tok, tmp_path / "queries.tsv", ["id", "text"], "<text>", qmax + extra, dr)
    dn, drows = _content_rows(tok, tmp_path / "corpus.tsv", ["id", "title", "text"], "<title> <text>", pmax + extra, dr)
    ragged = kind.endswith("ragged")
    qp = _write_store(tmp_path, "q_" + kind, qn, qr, ragged)
    cp = _write_store(tmp_path, "c_" + kind, dn, drows, ragged)
    qds, cds = _datasets(tok, _data_args(tmp_path, z, qp, cp))
    for g, w in zip(_assembled(tok, qds, cds, run), _want(z)):
        assert np.array_equal(g, w)


def test_dr_rows_cut_with_their_special_tokens(golden_dir, tmp_path):
    # the documented divergence: a DR row truncated at p_max_len together with [CLS] / [SEP] keeps 2 content tokens less
    from openmatch_b200.retriever.reranker import special_tokens, token_store
    z, tok, run = _fixture(golden_dir, tmp_path)
    pmax = int(z["p_max_len"])
    dn, drows = _content_rows(tok, tmp_path / "corpus.tsv", ["id", "title", "text"], "<title> <text>", pmax, True)
    cp = _write_store(tmp_path, "c_cut", dn, drows, False)
    _, cds = _datasets(tok, _data_args(tmp_path, z, None, cp))
    _, cds_text = _datasets(tok, _data_args(tmp_path, z))
    prefix, suffix = special_tokens(tok)
    _, where = token_store(cds, dn, prefix, suffix)
    _, where_text = token_store(cds_text, dn, prefix, suffix)
    cut = [d for d in dn if where_text[d][1] == pmax]
    assert cut, "premise: some passage is longer than p_max_len"
    assert all(where[d][1] == pmax - 2 for d in cut)
    assert all(where[d][1] == where_text[d][1] for d in dn if where_text[d][1] <= pmax - 2)


def test_reranking_depth_cuts_the_run(tmp_path):
    from openmatch_b200.arguments import InferenceArguments
    from openmatch_b200.utils import load_from_trec
    with open(tmp_path / "run.trec", "w") as f:
        for q in range(3):
            for r in range(10):
                f.write("q%d Q0 d%d %d %f OpenMatch\n" % (q, (q * 7 + r) % 13, r + 1, 10.0 - r))
    args = InferenceArguments(reranking_depth=4)
    run = load_from_trec(str(tmp_path / "run.trec"), max_len_per_q=args.reranking_depth)
    assert list(run) == ["q0", "q1", "q2"]
    for q in range(3):
        assert list(run["q%d" % q]) == ["d%d" % ((q * 7 + r) % 13) for r in range(4)]
    assert InferenceArguments().reranking_depth is None


class _FakeModel(torch.nn.Module):
    def __init__(self, limit=512):
        super().__init__()
        self.limit = limit

    def max_pair_len(self):
        return self.limit


class _FakeScorer:
    """A deterministic stand-in for the GPU scorer: a function of each pair's assembled tokens."""

    def _score(self, a_tokens, b_tokens, spans, prefix, suffix):
        from openmatch_b200.retriever.reranker import assemble_pairs
        tokens, lens = assemble_pairs(a_tokens, b_tokens, spans, prefix, suffix)
        rows = np.split(tokens, np.cumsum(lens)[:-1])
        return np.array([float((r * np.arange(1, len(r) + 1)).sum() % 9973) / 97.0 for r in rows], dtype=np.float32)


def _fake_reranker(tok, cds, world=1, rank=0, limit=512):
    from openmatch_b200.retriever.reranker import Reranker

    class FakeReranker(_FakeScorer, Reranker):
        pass

    args = types.SimpleNamespace(device=torch.device("cpu"), world_size=world, process_index=rank,
                                 per_device_eval_batch_size=16)
    return FakeReranker(_FakeModel(limit), tok, cds, args)


def test_missing_id_and_length_limit(golden_dir, tmp_path):
    z, tok, run = _fixture(golden_dir, tmp_path)
    qds, cds = _datasets(tok, _data_args(tmp_path, z))
    bad = dict(run)
    bad["q1"] = dict(bad["q1"], d_missing=1.0)
    with pytest.raises(KeyError, match="d_missing"):
        _fake_reranker(tok, cds).rerank(qds, bad)
    with pytest.raises(KeyError, match="q_missing"):
        _fake_reranker(tok, cds).rerank(qds, {"q_missing": {"d0": 1.0}})
    # 16 + 64 + [CLS] + [SEP] = 82 tokens: a model limit of 81 refuses the run before any scoring
    with pytest.raises(ValueError, match="exceed"):
        _fake_reranker(tok, cds, limit=81).rerank(qds, run)
    assert len(_fake_reranker(tok, cds, limit=82).rerank(qds, run)) == 4


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _big_run_inputs(tmp_path, write=True):
    """2 queries x 150 passages (more than the reference's top-100 merge keeps).  Only the caller that passes
    write=True writes the files: a rank that rewrote them could truncate the corpus while another rank reads it."""
    from transformers import BertTokenizer
    words = ["river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky"]
    rng = np.random.default_rng(11)
    corpus = "".join("d%d\t%s\t%s\n" % (i, words[i % 10], " ".join(rng.choice(words, 1 + i % 37))) for i in range(150))
    if write:
        (tmp_path / "vocab.txt").write_text("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words))
        (tmp_path / "corpus.tsv").write_text(corpus)
        (tmp_path / "queries.tsv").write_text("qa\triver bank\nqb\tgreen tree sky water\n")
    run = {q: {"d%d" % i: float(-i) for i in rng.permutation(150)} for q in ("qa", "qb")}
    z = {"q_max_len": 8, "p_max_len": 32}
    tok = BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)
    return tok, _datasets(tok, _data_args(tmp_path, z)), run


def _worker(rank, world, port, tmp):
    import pathlib
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openmatch_b200.utils import save_as_trec
        tok, (qds, cds), run = _big_run_inputs(pathlib.Path(tmp), write=False)
        result = _fake_reranker(tok, cds, world, rank).rerank(qds, run)
        if rank == 0:
            save_as_trec(result, os.path.join(tmp, "out", "rerank.trec"))
    finally:
        dist.destroy_process_group()


def test_two_ranks_return_the_union_on_rank_0(tmp_path):
    from openmatch_b200.utils import load_from_trec, save_as_trec
    tok, (qds, cds), run = _big_run_inputs(tmp_path)
    want = _fake_reranker(tok, cds).rerank(qds, run)
    assert [len(v) for v in want.values()] == [150, 150]
    os.makedirs(tmp_path / "out")
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert os.listdir(tmp_path / "out") == ["rerank.trec"]  # written once, no per-rank files left behind
    got = load_from_trec(str(tmp_path / "out" / "rerank.trec"))
    save_as_trec(want, str(tmp_path / "want.trec"))
    assert got == load_from_trec(str(tmp_path / "want.trec"))
    assert {q: set(v) for q, v in got.items()} == {q: set(v) for q, v in run.items()}
