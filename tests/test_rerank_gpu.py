"""GPU: cross-encoder re-ranking (om_encode_pairs / CudaEncoder.encode_pairs / RRModel / Reranker / driver.rerank).

om_encode_pairs must return bitwise what om_encode_packed returns for the host-assembled pair sequences; its scores are
held to the float64-oracle bound of tests/test_encoder_numerics_gpu.py and to the reference's own scores
(tests/golden/rerank_small.npz); invalid input, side streams, reuse of the host arrays, RRModel's padded and autograd
paths, and the rerank driver end to end on a run from the retrieve driver."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from test_encoder_gpu import _check, _rand_bert_sd, _rand_t5_sd
from test_encoder_numerics_gpu import F64, _bert_spec, _judge, _ospec, _t5_spec

pytestmark = pytest.mark.gpu

TARGET_LENS = [1, 127, 128, 129, 162, 255, 256, 257, 512]


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


def _model(name, gen):
    if name == "bert":
        return _bert_spec(2, 128, 2, 512), _rand_bert_sd(gen, 2, 128, 512, 2000, 512)
    if name == "bert_hd32":
        return _bert_spec(2, 128, 4, 512), _rand_bert_sd(gen, 2, 128, 512, 2000, 512)
    return _t5_spec(2, 128, 2, 512), _rand_t5_sd(gen, 2, 128, 2, 512, 2000)


def _stores(gen, na=3000, nb=30000):
    return (torch.randint(5, 2000, (na,), generator=gen, dtype=torch.int32),
            torch.randint(5, 2000, (nb,), generator=gen, dtype=torch.int32))


def _spans(gen, a, b, lens, n_special):
    """one span per assembled length (a query part of up to 32 tokens, the rest from b), plus a_len = 0 / b_len = 0"""
    rows = []
    for l in lens:
        body = l - n_special
        if body < 0:
            continue
        al = int(torch.randint(0, min(32, body) + 1, (1,), generator=gen))
        bl = body - al
        rows.append((int(torch.randint(0, a.numel() - al + 1, (1,), generator=gen)), al,
                     int(torch.randint(0, b.numel() - bl + 1, (1,), generator=gen)), bl))
    rows += [(7, 0, 100, 40), (9, 20, 5, 0), (0, 0, 0, 0)] if n_special else [(7, 0, 100, 40), (9, 20, 5, 0)]
    return np.array(rows, dtype=np.int64)


def _host_stream(a, b, spans, prefix, suffix):
    from openmatch_b200.retriever.reranker import assemble_pairs
    tokens, lens = assemble_pairs(a.numpy(), b.numpy(), spans, prefix, suffix)
    return torch.from_numpy(tokens), lens


SPECIALS = [([101], [102]), ([], [1]), ([5, 6, 7, 8], [9, 10, 11, 12])]
# (model, pooling, head, out dtype)
CONFIGS = [("bert", "first", True, torch.float32), ("bert", "mean", False, torch.bfloat16),
           ("bert_hd32", "first", True, torch.float16), ("bert_hd32", "mean", True, torch.float32),
           ("t5", "first", False, torch.float16), ("t5", "mean", True, torch.bfloat16)]


@pytest.mark.parametrize("name,pooling,has_head,dtype", CONFIGS)
def test_pairs_bitwise_equal_packed(enc_mod, name, pooling, has_head, dtype):
    gen = torch.Generator().manual_seed(4000 + CONFIGS.index((name, pooling, has_head, dtype)))
    spec, sd = _model(name, gen)
    head = torch.randn(1, spec["hidden"], generator=gen) * spec["hidden"] ** -0.5 if has_head else None
    a, b = _stores(gen)
    ad, bd = a.cuda(), b.cuda()
    big = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, max_batch_tokens=1 << 15)
    small = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, max_batch_tokens=1024)
    for prefix, suffix in SPECIALS:
        lens = TARGET_LENS + torch.randint(1, 513, (12,), generator=gen).tolist()
        spans = _spans(gen, a, b, lens, len(prefix) + len(suffix))
        tokens, seqlens = _host_stream(a, b, spans, prefix, suffix)
        if not prefix and not suffix[1:]:
            assert 1 in seqlens.tolist()
        for enc in (big, small):  # small: the layout takes several row groups of 1024 rows
            want = enc.encode_packed(tokens.cuda(), seqlens, out_dtype=dtype)
            got = enc.encode_pairs(ad, bd, spans, prefix, suffix, out_dtype=dtype)
            assert got.dtype == dtype and torch.isfinite(got.float()).all()
            assert torch.equal(got, want), "%s %s: pairs differ from packed" % (name, (prefix, suffix))
    # more sequences than max_batch_tokens: encoded in chunks of sequences
    tiny = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, max_batch_tokens=64)
    spans = _spans(gen, a, b, torch.randint(2, 40, (150,), generator=gen).tolist(), 2)
    tokens, seqlens = _host_stream(a, b, spans, [101], [102])
    assert torch.equal(tiny.encode_pairs(ad, bd, spans, [101], [102]), tiny.encode_packed(tokens.cuda(), seqlens))
    # into a strided buffer
    buf = torch.full((spans.shape[0], tiny.rep_dim + 16), 7.0, device="cuda")
    tiny.encode_pairs(ad, bd, spans, [101], [102], out=buf[:, 8:8 + tiny.rep_dim])
    assert torch.equal(buf[:, 8:8 + tiny.rep_dim], tiny.encode_packed(tokens.cuda(), seqlens))
    assert (buf[:, :8] == 7).all() and (buf[:, 8 + tiny.rep_dim:] == 7).all()


@pytest.mark.parametrize("name,pooling", [("bert", "first"), ("bert_hd32", "mean"), ("t5", "mean")])
def test_pair_scores_vs_oracle(enc_mod, name, pooling):
    gen = torch.Generator().manual_seed(4100)
    spec, sd = _model(name, gen)
    head = torch.randn(1, spec["hidden"], generator=gen) * spec["hidden"] ** -0.5
    a, b = _stores(gen)
    prefix, suffix = ([101], [102]) if spec["arch"] == "bert" else ([], [1])
    spans = _spans(gen, a, b, [2, 30, 100, 162, 162, 200, 300, 512] + torch.randint(40, 163, (16,), generator=gen).tolist(),
                   len(prefix) + len(suffix))
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, max_batch_tokens=1 << 14)
    got = enc.encode_pairs(a.cuda(), b.cuda(), spans, prefix, suffix).cpu().numpy()
    tokens, lens = _host_stream(a, b, spans, prefix, suffix)
    ospec = _ospec(spec, pooling, False)
    want, auto = [], []
    for s in torch.split(tokens, lens.tolist()):
        for emulate, dst in ((False, want), (True, auto)):
            dst.append(oracle.encode_reps(sd, ospec, s[None], torch.ones(1, len(s), dtype=torch.long), None, head,
                                          dtype=F64, emulate_bf16=emulate)[1][0].numpy())
    # one score per pair: judged as one vector over the batch
    _judge("%s %s pair scores" % (name, pooling), got.reshape(1, -1), np.stack(want).reshape(1, -1),
           np.stack(auto).reshape(1, -1))


def _golden_model(golden_dir):
    z = np.load(os.path.join(golden_dir, "rerank_small.npz"))
    sd = {k[2:]: torch.from_numpy(z[k].astype(np.float32) * z["s." + k[2:]]) for k in z.files if k.startswith("q.")}
    return z, sd


def test_golden_scores(enc_mod, golden_dir, tmp_path):
    from test_rerank_cpu import _data_args, _datasets, _fixture

    from openmatch_b200.retriever.reranker import special_tokens, token_store
    z, sd = _golden_model(golden_dir)
    _, tok, run = _fixture(golden_dir, tmp_path)
    head = sd.pop("head.linear.weight")
    spec = _bert_spec(2, 128, 2, 256, vocab=len(z["vocab"]), max_pos=256)
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling="first", max_batch_tokens=4096)
    qds, cds = _datasets(tok, _data_args(tmp_path, z))
    prefix, suffix = special_tokens(tok)
    pairs = [(q, d) for q, docs in run.items() for d in docs]
    a, qw = token_store(qds, [q for q, _ in pairs], prefix, suffix)
    b, dw = token_store(cds, [d for _, d in pairs], prefix, suffix)
    spans = np.array([qw[q] + dw[d] for q, d in pairs], dtype=np.int64)
    got = enc.encode_pairs(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), spans, prefix, suffix)
    got = got[:, 0].cpu().numpy()
    want = z["scores"]
    _check(got.reshape(1, -1), want.reshape(1, -1), "reference rerank scores")
    eps = 1e-2 * float(np.abs(want).max())
    qids = np.array([q for q, _ in pairs])
    for q in set(qids.tolist()):
        i = np.nonzero(qids == q)[0]
        for x in i:
            for y in i:
                if want[x] - want[y] > 2 * eps:
                    assert got[x] > got[y], "query %s: order differs where the golden gap exceeds the bound" % q


def test_invalid_input(enc_mod):
    from openmatch_b200 import _lib
    gen = torch.Generator().manual_seed(4200)
    spec = _bert_spec(1, 128, 2, 256, vocab=100, max_pos=200)
    enc = enc_mod.CudaEncoder(spec, _rand_bert_sd(gen, 1, 128, 256, 100, 200), max_batch_tokens=4096)
    lib, stream = _lib.load(), _lib.current_stream_ptr()
    a = torch.randint(5, 100, (50,), device="cuda", dtype=torch.int32)
    b = torch.randint(5, 100, (500,), device="cuda", dtype=torch.int32)
    out = torch.full((3, 128), float("nan"), device="cuda")
    pre, suf = np.array([101, 1, 2, 3], np.int32), np.array([102, 4, 5, 6], np.int32)

    def call(rows, B=3, n_pre=1, n_suf=1, **over):
        sp = np.ascontiguousarray(np.asarray(rows, dtype=np.int64).reshape(-1, 4))
        args = dict(enc=enc._h, a=a.data_ptr(), na=50, b=b.data_ptr(), nb=500, spans=sp.ctypes.data, B=B,
                    pre=pre.ctypes.data, n_pre=n_pre, suf=suf.ctypes.data, n_suf=n_suf, out=out.data_ptr(), dtype=_lib.OM_F32, stride=128, stream=stream)
        args.update(over)
        return lib.om_encode_pairs(*args.values())

    ok = [[0, 10, 0, 100]] * 3
    bad_spans = [[[-1, 1, 0, 1]] + ok[1:], [[0, -1, 0, 1]] + ok[1:], [[0, 1, -1, 1]] + ok[1:], [[0, 1, 0, -1]] + ok[1:],
                 ok[:2] + [[45, 6, 0, 1]], ok[:2] + [[0, 1, 499, 2]], ok[:2] + [[0, 0, 0, 0]],  # 50 + 1 > 50; 501 > 500
                 ok[:2] + [[0, 50, 0, 149]]]  # 201 tokens > max_position_embeddings
    for i, s in enumerate(bad_spans):
        over = dict(n_pre=0, n_suf=0) if i == 6 else {}  # an assembled length of 0
        assert call(s, **over) == -1, s
        assert b"pair" in lib.om_last_error()
    for over in (dict(enc=None), dict(a=None), dict(b=None), dict(spans=None), dict(out=None), dict(pre=None),
                 dict(suf=None), dict(B=-1), dict(n_pre=5), dict(n_suf=-1), dict(n_pre=-1), dict(n_suf=5),
                 dict(na=-1), dict(dtype=7), dict(stride=64)):
        assert call(ok, **over) == -1, over
    assert call(ok[:1], B=0) == 0  # empty batch: nothing to do
    long_enc = enc_mod.CudaEncoder(spec, _rand_bert_sd(gen, 1, 128, 256, 100, 200), max_batch_tokens=150)
    assert call(ok[:2] + [[0, 20, 0, 140]], enc=long_enc._h) == -1  # 162 > max_batch_tokens
    torch.cuda.synchronize()
    assert torch.isnan(out).all(), "a refused call wrote to the output"
    with pytest.raises(RuntimeError, match="pair 1"):
        enc.encode_pairs(a, b, [[0, 1, 0, 1], [0, 51, 0, 1]], [101], [102])
    assert call(ok) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()


def test_side_stream_poisoned_workspace_and_reuse(enc_mod):
    gen = torch.Generator().manual_seed(4300)
    for name in ("bert", "t5"):
        spec, sd = _model(name, gen)
        a, b = _stores(gen)
        ad, bd = a.cuda(), b.cuda()
        spans = _spans(gen, a, b, [3, 512, 40, 129, 77, 2, 128, 300, 64, 65, 162], 2)
        want = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=4096).encode_pairs(ad, bd, spans, [3], [4])
        torch.cuda.synchronize()
        os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
        try:  # the pair workspace is allocated (poisoned) on the first call
            enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=4096)
            got = enc.encode_pairs(ad, bd, spans, [3], [4])
        finally:
            del os.environ["OPENMATCH_B200_POISON_ALLOC"]
        assert torch.isfinite(got).all() and torch.equal(got, want), name + ": poisoned workspace changes the result"
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            sp = spans.copy()
            sr = enc.encode_pairs(ad, bd, sp, [3], [4])
            sp[:] = 0  # the host spans may be reused as soon as the call returns
            sr2 = enc.encode_pairs(ad, bd, spans, [3], [4])
        side.synchronize()
        assert torch.equal(sr, want), name + ": side stream differs"
        assert torch.equal(sr2, want), name + ": reused spans change the result"


def _tiny_rr(max_pos=256, hidden=128, heads=2):
    from transformers import BertConfig, BertModel

    from openmatch_b200.modeling import LinearHead, RRModel
    torch.manual_seed(4400)
    lm = BertModel(BertConfig(vocab_size=300, hidden_size=hidden, num_hidden_layers=2, num_attention_heads=heads,
                              intermediate_size=256, max_position_embeddings=max_pos))
    return RRModel(lm=lm, head=LinearHead(hidden, 1), pooling="first")


def test_rrmodel_padded_and_autograd_paths(enc_mod):
    from openmatch_b200.retriever.reranker import encode_pair
    model = _tiny_rr().cuda().eval()
    gen = torch.Generator().manual_seed(4401)
    a, b = _stores(gen, 400, 4000)
    a, b = a % 300, b % 300
    spans = _spans(gen, a, b, torch.randint(2, 163, (40,), generator=gen).tolist(), 2)
    spans[:, 1] = np.minimum(spans[:, 1], 32)
    spans[:, 3] = np.minimum(spans[:, 3], 128)
    rows = [encode_pair([2], [3], a[x:x + al].tolist(), b[y:y + bl].tolist()) for x, al, y, bl in spans]
    L = 162
    ids = torch.zeros(len(rows), L, dtype=torch.long)
    mask = torch.zeros_like(ids)
    for i, r in enumerate(rows):
        ids[i, :len(r)], mask[i, :len(r)] = torch.tensor(r), 1
    items = {"input_ids": ids.cuda(), "attention_mask": mask.cuda(), "token_type_ids": torch.zeros_like(ids).cuda()}
    with torch.no_grad():
        padded = model.encode(items)
    pairs = model.encode_pairs(a.cuda(), b.cuda(), spans, [2], [3])
    assert padded.shape == (len(rows), 1) and torch.equal(padded, pairs)
    with torch.no_grad():
        hf = model.head(model.lm(**items).last_hidden_state[:, 0])
    _check(padded.cpu().numpy().reshape(1, -1), hf.cpu().numpy().reshape(1, -1), "RRModel.encode vs HF fp32")
    left = {k: v.flip(1) for k, v in items.items()}
    with pytest.raises(ValueError, match="right padding"), torch.no_grad():
        model.encode(left)
    # training mode under autograd: the HF module, pooling and head, with gradients
    model.train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    s = model.encode(items)
    assert s.requires_grad
    with torch.no_grad():
        ref = model.head(model.lm(**items, return_dict=True).last_hidden_state[:, 0])
    assert torch.allclose(s.detach(), ref, rtol=1e-5, atol=1e-6)
    s.sum().backward()
    assert model.head.linear.weight.grad is not None and torch.isfinite(model.head.linear.weight.grad).all()
    with pytest.raises(NotImplementedError, match="training"):
        model(items, items)
    model.cpu()


def _run(main, argv):
    old = sys.argv
    sys.argv = ["prog"] + [str(x) for x in argv]
    try:
        main()
    finally:
        sys.argv = old


def test_rerank_driver_end_to_end(enc_mod, tmp_path):
    from transformers import BertConfig, BertModel, BertTokenizer

    from openmatch.arguments import ModelArguments
    from openmatch.driver import build_index, rerank, retrieve
    from openmatch.utils import load_from_trec
    from openmatch_b200.dataset import write_ragged_store
    from openmatch_b200.modeling import LinearHead, RRModel
    from openmatch_b200.retriever.reranker import encode_pair, special_tokens
    words = ["the", "a", "of", "river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky", "rain",
             "city", "road", "car", "train", "music", "piano"]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    (tmp_path / "vocab.txt").write_text("\n".join(vocab))
    tok = BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)
    torch.manual_seed(4500)
    cfg = BertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                     intermediate_size=256, max_position_embeddings=256)
    dr_dir, rr_dir = tmp_path / "dr", tmp_path / "rr"
    BertModel(cfg).save_pretrained(str(dr_dir))
    tok.save_pretrained(str(dr_dir))
    os.makedirs(rr_dir)
    rr = RRModel(lm=BertModel(cfg), head=LinearHead(128, 1), pooling="first")
    rr.save(str(rr_dir))
    tok.save_pretrained(str(rr_dir))
    assert json.load(open(rr_dir / "openmatch_config.json"))["pooling"] == "first"
    rng = np.random.default_rng(4500)
    corpus = {"d%d" % i: (" ".join(rng.choice(words, 2)), " ".join(rng.choice(words, int(rng.integers(1, 60)))))
              for i in range(80)}
    queries = {"q%d" % i: " ".join(rng.choice(words, int(rng.integers(1, 12)))) for i in range(9)}
    with open(tmp_path / "corpus.tsv", "w") as f:
        f.writelines("%s\t%s\t%s\n" % (k, t, x) for k, (t, x) in corpus.items())
    with open(tmp_path / "queries.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in queries.items())
    with open(tmp_path / "queries.jsonl", "w") as f:
        f.writelines(json.dumps({"id": k, "text": v}) + "\n" for k, v in queries.items())
    emb = tmp_path / "emb"
    common = ["--output_dir", emb, "--model_name_or_path", dr_dir, "--per_device_eval_batch_size", 16, "--q_max_len", 16,
              "--p_max_len", 64, "--dataloader_num_workers", 0]
    _run(build_index.main, common + ["--corpus_path", tmp_path / "corpus.tsv", "--doc_template", "<title> <text>",
                                     "--doc_column_names", "id,title,text"])
    run_path = tmp_path / "run.trec"
    _run(retrieve.main, common + ["--query_path", tmp_path / "queries.tsv", "--query_template", "<text>",
                                  "--query_column_names", "id,text", "--trec_save_path", run_path,
                                  "--retrieve_depth", 30, "--use_gpu"])
    depth = 20
    run = load_from_trec(str(run_path), max_len_per_q=depth)

    def rerank_with(query_path, corpus_path, out):
        _run(rerank.main, ["--output_dir", tmp_path / "rr_out", "--model_name_or_path", rr_dir, "--query_path", query_path,
                           "--corpus_path", corpus_path, "--query_template", "<text>", "--query_column_names", "id,text",
                           "--doc_template", "<title> <text>", "--doc_column_names", "id,title,text", "--q_max_len", 16,
                           "--p_max_len", 64, "--per_device_eval_batch_size", 24, "--trec_run_path", run_path,
                           "--trec_save_path", out, "--reranking_depth", depth, "--fp16", "--dataloader_num_workers", 0])
        return load_from_trec(str(out))

    got = rerank_with(tmp_path / "queries.tsv", tmp_path / "corpus.tsv", tmp_path / "rr_tsv.trec")
    assert {q: set(v) for q, v in got.items()} == {q: set(v) for q, v in run.items()}
    for docs in got.values():
        s = list(docs.values())
        assert s == sorted(s, reverse=True)
    # HF fp32 RRModel.encode on the reference's padded pairs
    prefix, suffix = special_tokens(tok)
    model = RRModel.build(ModelArguments(model_name_or_path=str(rr_dir))).cuda().eval()
    assert torch.equal(model.head.linear.weight.cpu(), rr.head.linear.weight)

    def content(text, n):
        return tok(text, add_special_tokens=False, truncation=True, max_length=n)["input_ids"]

    pairs = [(q, d) for q, docs in run.items() for d in docs]
    rows = [encode_pair(prefix, suffix, content(queries[q], 16), content(" ".join(corpus[d]), 64)) for q, d in pairs]
    ids = torch.zeros(len(rows), 16 + 64 + 2, dtype=torch.long)
    for i, r in enumerate(rows):
        ids[i, :len(r)] = torch.tensor(r)
    items = {"input_ids": ids.cuda(), "attention_mask": (ids != 0).long().cuda(), "token_type_ids": torch.zeros_like(ids).cuda()}
    with torch.no_grad():
        hf = model.head(model.lm(**items).last_hidden_state[:, 0])[:, 0].cpu().numpy()
    mine = np.array([got[q][d] for q, d in pairs])
    _check(mine.reshape(1, -1), hf.reshape(1, -1), "rerank driver vs HF fp32")
    # JSON lines queries, and ragged pretokenised stores of the same (untruncated) texts: identical scores
    assert max(len(content(v, 100)) for v in queries.values()) <= 16
    assert max(len(content(" ".join(v), 100)) for v in corpus.values()) <= 64
    assert rerank_with(tmp_path / "queries.jsonl", tmp_path / "corpus.tsv", tmp_path / "rr_jsonl.trec") == got

    def ragged(stem, names, texts):
        arr = np.zeros((len(texts), 100), np.int32)
        for i, t in enumerate(texts):
            r = tok(t)["input_ids"]  # dense-retrieval rows, with [CLS] / [SEP]
            arr[i, :len(r)] = r
        return write_ragged_store(str(tmp_path / stem), arr, names)

    qp = ragged("q", list(queries), list(queries.values()))
    cp = ragged("c", list(corpus), [" ".join(v) for v in corpus.values()])
    assert rerank_with(qp, cp, tmp_path / "rr_ragged.trec") == got
    model.cpu()
