"""GPU: RoBERTa / XLM-RoBERTa encoders (ANCE, multilingual-e5, RoBERTa cross-encoders) on the sm_90a encoder.

RoBERTa is BERT's encoder with position ids computed from the token ids by roberta_pos_kernel (padding_idx 1): a pad id
inside a sequence's content takes position 1 and does not advance the count.  Reps and attended hidden rows are held to
the float64-oracle bound of tests/test_encoder_numerics_gpu.py (err_kernel <= 2 err_autocast + 2e-4, plus rel-L2 <= 1e-2
and cosine >= 0.9999) on the padded and the packed path; the reference's own golden vectors, the HF module, device pair
assembly, the length limit of max_position_embeddings - 2, handles of both families in one process, side streams,
poisoned workspaces and the drivers end to end."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import roberta_oracle as ro
from test_encode_packed_gpu import EDGE_LENS
from test_encoder_gpu import _check, _rand_bert_sd
from test_encoder_numerics_gpu import F64, _judge, _ospec
from test_encoder_roberta_cpu import GOLDEN_HEADS, golden_spec, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


# (hidden, heads, ffn, vocab): roberta-base / ANCE and multilingual-e5-small widths, 2 layers, max_position_embeddings 514
SHAPES = {"roberta_base": (768, 12, 3072, 50265), "me5_small": (384, 12, 1536, 250002)}


def _spec(H, heads, F, vocab, layers=2, max_pos=514):
    return dict(arch="roberta", layers=layers, hidden=H, heads=heads, ffn=F, vocab=vocab, max_pos=max_pos, type_vocab=1,
                ln_eps=1e-5)


def _rand_sd(gen, layers, H, F, vocab, max_pos=514):
    sd = _rand_bert_sd(gen, layers, H, F, 8, max_pos)
    sd["embeddings.word_embeddings.weight"] = torch.randn(vocab, H, generator=gen) * 0.02
    sd["embeddings.token_type_embeddings.weight"] = sd["embeddings.token_type_embeddings.weight"][:1]
    return sd


def _model(name, gen):
    H, heads, F, vocab = SHAPES[name]
    return _spec(H, heads, F, vocab), _rand_sd(gen, 2, H, F, vocab)


def _seq(gen, n, vocab, inner_pad=True):
    """<s> content </s> with ids >= 3 (no accidental pad), a few content tokens replaced by the pad id 1"""
    s = torch.randint(3, vocab, (n,), generator=gen)
    s[0] = 0
    if n > 1:
        s[-1] = 2
    if inner_pad and n > 4:
        s[torch.randint(1, n - 1, (max(1, n // 50),), generator=gen)] = 1
    return s


def _padded(seqs, L):
    ids = torch.ones(len(seqs), L, dtype=torch.long)  # right padding with id 1
    mask = torch.zeros(len(seqs), L, dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = s
        mask[i, :len(s)] = 1
    return ids, mask


def _packed(enc, seqs, **kw):
    lens = np.array([len(s) for s in seqs], dtype=np.int32)
    return enc.encode_packed(torch.cat(seqs).cuda(), lens, **kw)


def _oracles(sd, ospec, ids, mask, head):
    return (ro.encode_reps(sd, ospec, ids, mask, head, dtype=F64),
            ro.encode_reps(sd, ospec, ids, mask, head, dtype=F64, emulate_bf16=True))


# ------------------------------------------------------------------------------------------------------------------
# the reference's golden vectors
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(GOLDEN_HEADS))
def test_reference_golden(enc_mod, golden_dir, cfg):
    z, sd, head, ids, mask = load_golden(golden_dir, cfg)
    m = mask.bool()
    lens = m.sum(1).numpy().astype(np.int32)
    ids, mask = ids.cuda(), mask.cuda()
    for pooling, normalize, hw, key in (("first", False, head, "reps_first_head"), ("mean", True, None, "reps_mean_norm")):
        enc = enc_mod.CudaEncoder(golden_spec(cfg), sd, head_weight=hw, pooling=pooling, normalize=normalize,
                                  max_batch_tokens=1024)
        hidden, reps = enc.encode(ids, mask, return_hidden=True)
        what = "roberta %s %s" % (cfg, key)
        _check(reps.cpu().numpy(), z["%s.%s" % (cfg, key)], what)
        _check(hidden[m.cuda()].cpu().numpy(), z[cfg + ".hidden_attended"], what + " hidden")
        ph, preps = enc.encode_packed(ids[m.cuda()], lens, return_hidden=True)
        _check(preps.cpu().numpy(), z["%s.%s" % (cfg, key)], what + " packed")
        _check(ph.cpu().numpy(), z[cfg + ".hidden_attended"], what + " packed hidden")


# ------------------------------------------------------------------------------------------------------------------
# float64 oracle at roberta-base and multilingual-e5-small width
# ------------------------------------------------------------------------------------------------------------------
PADDED = [("roberta_base", 32, 12, "first", False, False), ("roberta_base", 128, 6, "mean", True, True),
          ("roberta_base", 512, 2, "mean", False, True), ("me5_small", 32, 12, "mean", False, True),
          ("me5_small", 128, 6, "first", True, False), ("me5_small", 512, 2, "first", False, False)]


@pytest.mark.parametrize("name,L,B,pooling,has_head,normalize", PADDED)
def test_padded_vs_float64_oracle(enc_mod, name, L, B, pooling, has_head, normalize):
    gen = torch.Generator().manual_seed(8000 + PADDED.index((name, L, B, pooling, has_head, normalize)))
    spec, sd = _model(name, gen)
    H = spec["hidden"]
    head = torch.randn(96, H, generator=gen) * H ** -0.5 if has_head else None
    lens = [L] + torch.randint(1, L + 1, (B - 1,), generator=gen).tolist()
    ids, mask = _padded([_seq(gen, n, spec["vocab"]) for n in lens], L)
    assert ((ids == 1) & (mask == 1)).any()  # pad ids inside content
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize, max_batch_tokens=B * L)
    hidden, reps = enc.encode(ids.cuda(), mask.cuda(), return_hidden=True)
    (oh, oreps), (ah, areps) = _oracles(sd, _ospec(dict(spec, arch="bert"), pooling, normalize), ids, mask, head)
    m = mask.numpy().astype(bool)
    what = "roberta %s L=%d %s" % (name, L, pooling)
    _judge(what + " reps", reps.cpu().numpy(), oreps.numpy(), areps.numpy())
    _judge(what + " hidden", hidden.cpu().numpy()[m], oh.numpy()[m], ah.numpy()[m])


@pytest.mark.parametrize("name,pooling,has_head,normalize", [("roberta_base", "mean", False, True),
                                                             ("me5_small", "first", True, False)])
def test_packed_vs_float64_oracle(enc_mod, name, pooling, has_head, normalize):
    gen = torch.Generator().manual_seed(8100 + len(name))
    spec, sd = _model(name, gen)
    H = spec["hidden"]
    head = torch.randn(64, H, generator=gen) * H ** -0.5 if has_head else None
    lens = EDGE_LENS + torch.randint(1, 513, (3,), generator=gen).tolist() + torch.randint(1, 60, (8,), generator=gen).tolist()
    lens = [lens[i] for i in torch.randperm(len(lens), generator=gen).tolist()]
    seqs = [_seq(gen, n, spec["vocab"]) for n in lens]
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                              max_batch_tokens=len(seqs) * 512)
    hidden, reps = _packed(enc, seqs, return_hidden=True)
    ids, mask = _padded(seqs, 512)
    (oh, oreps), (ah, areps) = _oracles(sd, _ospec(dict(spec, arch="bert"), pooling, normalize), ids, mask, head)
    m = mask.numpy().astype(bool)
    what = "roberta %s packed %s" % (name, pooling)
    _judge(what + " reps", reps.cpu().numpy(), oreps.numpy(), areps.numpy())
    _judge(what + " hidden", hidden.cpu().numpy(), oh.numpy()[m], ah.numpy()[m])


# ------------------------------------------------------------------------------------------------------------------
# HF parity through DRModel, device pair assembly
# ------------------------------------------------------------------------------------------------------------------
def _hf_roberta(seed=9, heads=2, max_pos=514, vocab=1000):
    from transformers import RobertaConfig, RobertaModel
    torch.manual_seed(seed)
    cfg = RobertaConfig(vocab_size=vocab, hidden_size=128, num_hidden_layers=2, num_attention_heads=heads,
                        intermediate_size=512, max_position_embeddings=max_pos, type_vocab_size=1, pad_token_id=1)
    return RobertaModel(cfg).eval()


@pytest.mark.parametrize("pooling,normalize", [("first", False), ("mean", True)])
def test_hf_parity_through_drmodel(enc_mod, pooling, normalize):
    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    lm = _hf_roberta().cuda()
    model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling=pooling, normalize=normalize,
                                model_args=ModelArguments("unused", pooling=pooling, normalize=normalize))
    gen = torch.Generator().manual_seed(8200)
    for L, B in ((96, 7), (512, 2)):
        ids, mask = _padded([_seq(gen, n, 1000) for n in [L] + torch.randint(1, L, (B - 1,), generator=gen).tolist()], L)
        assert ((ids == 1) & (mask == 1)).any()
        batch = {"input_ids": ids.cuda(), "attention_mask": mask.cuda()}
        hidden, reps = model.encode_passage(batch)
        with torch.no_grad():
            want_h = lm(**batch).last_hidden_state.float()
        if pooling == "first":
            want = want_h[:, 0]
        else:
            mf = mask.cuda().unsqueeze(-1).float()
            want = (want_h * mf).sum(1) / mf.sum(1).clamp(min=1e-9)
        if normalize:
            want = torch.nn.functional.normalize(want, dim=1)
        m = mask.bool()
        _check(reps.cpu().numpy(), want.cpu().numpy(), "roberta DRModel vs HF reps L=%d" % L)
        _check(hidden.float().cpu()[m].numpy(), want_h.cpu()[m].numpy(), "roberta DRModel vs HF hidden L=%d" % L)


def test_pairs_bitwise_equal_packed(enc_mod):
    gen = torch.Generator().manual_seed(8300)
    H, F, vocab = 256, 512, 1000
    sd = _rand_sd(gen, 2, H, F, vocab)
    head = torch.randn(1, H, generator=gen) * H ** -0.5
    for heads in (4, 8):  # 64- and 32-wide heads
        enc = enc_mod.CudaEncoder(_spec(H, heads, F, vocab), sd, head_weight=head, pooling="first",
                                  max_batch_tokens=2048)
        a = [_seq(gen, int(n), vocab)[1:-1] for n in torch.randint(2, 40, (9,), generator=gen)]
        b = [_seq(gen, int(n), vocab)[1:-1] for n in torch.randint(2, 480, (9,), generator=gen)]
        a[3] = torch.ones(0, dtype=torch.long)  # an empty query side
        b[5][:3] = 1  # pad ids at the start of the passage content
        a_store, b_store = torch.cat(a).to(torch.int32), torch.cat(b).to(torch.int32)
        a0 = np.cumsum([0] + [len(x) for x in a])[:-1]
        b0 = np.cumsum([0] + [len(x) for x in b])[:-1]
        pairs = [(i, j) for i in range(9) for j in range(9) if (i + j) % 4 == 0]
        spans = np.array([(a0[i], len(a[i]), b0[j], len(b[j])) for i, j in pairs], dtype=np.int64)
        got = enc.encode_pairs(a_store.cuda(), b_store.cuda(), spans, [0], [2, 2])
        seqs = [torch.cat([torch.tensor([0]), a[i], b[j], torch.tensor([2, 2])]) for i, j in pairs]
        want = _packed(enc, seqs)
        assert torch.equal(got, want), "heads=%d: encode_pairs differs from encode_packed" % heads


# ------------------------------------------------------------------------------------------------------------------
# the length limit: max_position_embeddings - 2
# ------------------------------------------------------------------------------------------------------------------
def test_length_limit_refused_before_any_write(enc_mod):
    gen = torch.Generator().manual_seed(8400)
    H, F, vocab, max_pos = 128, 256, 500, 66
    enc = enc_mod.CudaEncoder(_spec(H, 2, F, vocab, layers=1, max_pos=max_pos), _rand_sd(gen, 1, H, F, vocab, max_pos),
                              pooling="mean", max_batch_tokens=4096)
    out = torch.full((2, H), 7.0, device="cuda")
    ok = [_seq(gen, 64, vocab), _seq(gen, 10, vocab)]
    ids, mask = _padded(ok, 64)
    enc.encode(ids.cuda(), mask.cuda(), out=out)  # 64 = max_position_embeddings - 2 tokens: accepted
    _packed(enc, ok, out=out)
    out.fill_(7.0)
    ids, mask = _padded(ok, 65)
    with pytest.raises(RuntimeError, match="max_position_embeddings - 2"):
        enc.encode(ids.cuda(), mask.cuda(), out=out)
    long = [_seq(gen, 65, vocab), _seq(gen, 10, vocab)]
    with pytest.raises(RuntimeError, match="max_position_embeddings - 2"):
        _packed(enc, long, out=out)
    store = torch.cat(long).to(torch.int32).cuda()
    with pytest.raises(RuntimeError, match="max_position_embeddings - 2"):
        enc.encode_pairs(store, store, np.array([[0, 60, 0, 3], [0, 2, 0, 2]]), [0], [2], out=out)
    torch.cuda.synchronize()
    assert (out == 7.0).all()
    from openmatch_b200 import _lib
    lib = _lib.load()
    desc = _lib.EncoderDesc(arch=_lib.OM_ARCH_ROBERTA, layers=1, hidden=H, heads=2, ffn=F, vocab=vocab, max_pos=2,
                            type_vocab=1, ln_eps=1e-5, pooling=_lib.OM_POOL_FIRST, has_head=0, head_out=0, normalize=0,
                            rel_buckets=32, rel_max_distance=128, max_batch_tokens=1024)
    h = ctypes.c_void_p()
    assert lib.om_encoder_create(ctypes.byref(desc), ctypes.byref(h)) == -1 and not h.value  # OM_EINVAL
    assert "max_position_embeddings=2" in lib.om_last_error().decode()


# ------------------------------------------------------------------------------------------------------------------
# BERT and RoBERTa handles in one process, side streams, poisoned workspaces
# ------------------------------------------------------------------------------------------------------------------
def _run_all(enc, gen_seed, vocab=1000):
    gen = torch.Generator().manual_seed(gen_seed)
    res = []
    for L, B in ((32, 11), (100, 7), (256, 3)):
        ids, mask = _padded([_seq(gen, int(n), vocab) for n in [L] + torch.randint(1, L, (B - 1,), generator=gen).tolist()], L)
        res.append(enc.encode(ids.cuda(), mask.cuda(), return_hidden=True))
    res.append(_packed(enc, [_seq(gen, n, vocab) for n in (3, 512, 40, 129, 77, 1, 128, 300, 64, 65)], return_hidden=True))
    a = torch.randint(3, vocab, (300,), generator=gen).to(torch.int32).cuda()
    a[::7] = 1
    spans = np.array([[0, 20, 20, 200], [5, 0, 40, 3], [100, 30, 0, 90]], dtype=np.int64)
    res.append((enc.encode_pairs(a, a, spans, [0], [2]), torch.zeros(1, device="cuda")))
    return [(h.clone(), r.clone()) for h, r in res]


def _same(got, want, what):
    for (gh, gr), (wh, wr) in zip(got, want):
        assert torch.isfinite(gr).all() and torch.isfinite(gh).all(), what + ": non-finite output"
        assert torch.equal(gr, wr) and torch.equal(gh, wh), what


def test_bert_and_roberta_interleaved_side_stream_poison(enc_mod):
    gen = torch.Generator().manual_seed(8500)
    H, F, vocab = 256, 512, 1000
    sd = _rand_sd(gen, 2, H, F, vocab)
    bert_sd = dict(sd, **{"embeddings.token_type_embeddings.weight": torch.randn(2, H, generator=gen) * 0.02})
    specs = {"roberta": (_spec(H, 4, F, vocab), sd),
             "bert": (dict(_spec(H, 8, F, vocab), arch="bert", max_pos=514, type_vocab=2), bert_sd)}

    def make(k):
        return enc_mod.CudaEncoder(specs[k][0], specs[k][1], head_weight=torch.ones(1, H) / H, pooling="mean",
                                   max_batch_tokens=4096)

    live = {k: make(k) for k in specs}
    for rnd in range(2):  # calls alternate between the two handles, each against a fresh handle of its kind
        for k in ("roberta", "bert", "roberta"):
            got = _run_all(live[k], 8600 + rnd)
            fresh = make(k)
            _same(got, _run_all(fresh, 8600 + rnd), "%s round %d: live handle differs from a fresh one" % (k, rnd))
            del fresh
    want = _run_all(live["roberta"], 8700)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = _run_all(live["roberta"], 8700)
    side.synchronize()
    _same(got, want, "side stream differs from the default stream")
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        enc = make("roberta")
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]
    _same(_run_all(enc, 8700), want, "poisoned workspace changes the result")


# ------------------------------------------------------------------------------------------------------------------
# drivers end to end: a saved RoBERTa checkpoint with a byte-level tokenizer
# ------------------------------------------------------------------------------------------------------------------
def _run(main, argv):
    old = sys.argv
    sys.argv = ["prog"] + [str(a) for a in argv]
    try:
        main()
    finally:
        sys.argv = old


WORDS = ["the", "a", "of", "river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky", "rain",
         "city", "road", "car", "train", "music", "piano"]


def _eps_equal_runs(got, want, scores, eps):
    """same queries, each ranking equal up to ties within eps of the wanted scores"""
    assert sorted(got) == sorted(want)
    for q in want:
        g, w = list(got[q]), list(want[q])
        assert len(g) == len(w)
        for r, (dg, dw) in enumerate(zip(g, w)):
            assert dg == dw or abs(scores[q][dg] - scores[q][dw]) <= eps, (q, r, dg, dw)


def test_build_index_retrieve_and_rerank(enc_mod, tmp_path):
    from openmatch.arguments import ModelArguments
    from openmatch.dataset import write_ragged_store
    from openmatch.driver import build_index, rerank, retrieve
    from openmatch.utils import load_from_trec
    from openmatch_b200.modeling import LinearHead, RRModel
    from openmatch_b200.retriever.reranker import encode_pair, special_tokens
    tok = ro.offline_tokenizer(str(tmp_path))
    assert tok.pad_token_id == 1 and special_tokens(tok) == ([0], [2])
    dr_dir, rr_dir = tmp_path / "dr", tmp_path / "rr"
    _hf_roberta(seed=10, vocab=len(tok), max_pos=130).save_pretrained(str(dr_dir))
    tok.save_pretrained(str(dr_dir))
    os.makedirs(rr_dir)
    rr = RRModel(lm=_hf_roberta(seed=11, heads=4, vocab=len(tok), max_pos=130), head=LinearHead(128, 1), pooling="first")
    rr.save(str(rr_dir))
    tok.save_pretrained(str(rr_dir))
    rng = np.random.default_rng(8800)
    corpus = {"d%d" % i: " ".join(rng.choice(WORDS, int(rng.integers(1, 14)))) for i in range(60)}
    queries = {"q%d" % i: " ".join(rng.choice(WORDS, int(rng.integers(1, 4)))) for i in range(7)}
    with open(tmp_path / "corpus.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in corpus.items())
    with open(tmp_path / "queries.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in queries.items())
    q_max, p_max = 24, 96
    assert max(len(tok(t)["input_ids"]) for t in corpus.values()) <= p_max

    def padded_store(stem, texts, width):
        arr = np.full((len(texts), width), 1, np.int32)  # padded with RoBERTa's pad id 1
        for i, t in enumerate(texts.values()):
            r = tok(t)["input_ids"]
            arr[i, :len(r)] = r
        np.save(tmp_path / (stem + ".npy"), arr)
        (tmp_path / (stem + ".ids.txt")).write_text("\n".join(texts))
        return arr

    def retrieve_with(tag, corpus_args):
        emb = tmp_path / ("emb_" + tag)
        common = ["--output_dir", emb, "--model_name_or_path", dr_dir, "--per_device_eval_batch_size", 16, "--q_max_len",
                  q_max, "--p_max_len", p_max, "--dataloader_num_workers", 0]
        _run(build_index.main, common + corpus_args)
        out = tmp_path / ("run_%s.trec" % tag)
        _run(retrieve.main, common + ["--query_path", tmp_path / "queries.tsv", "--query_template", "<text>",
                                      "--query_column_names", "id,text", "--trec_save_path", out, "--retrieve_depth",
                                      20, "--use_gpu"])
        return load_from_trec(str(out))

    text_run = retrieve_with("text", ["--corpus_path", tmp_path / "corpus.tsv", "--doc_template", "<text>",
                                      "--doc_column_names", "id,text"])
    arr = padded_store("corpus_tok", corpus, p_max)
    padded_run = retrieve_with("padded", ["--corpus_path", tmp_path / "corpus_tok.npy"])
    ragged_path = write_ragged_store(str(tmp_path / "corpus_rag"), arr, list(corpus), pad_id=1)
    assert np.load(ragged_path)[0] == 0  # <s> kept
    ragged_run = retrieve_with("ragged", ["--corpus_path", ragged_path])
    assert len(text_run) == 7 and all(len(v) == 20 for v in text_run.values())
    eps = 2e-3  # the bf16 encoder's score error; ranks compared up to ties within it
    _eps_equal_runs(padded_run, text_run, text_run, eps)
    _eps_equal_runs(ragged_run, text_run, {q: {**text_run[q], **ragged_run[q]} for q in text_run}, eps)
    for q in text_run:  # scores of the documents both runs hold agree within eps
        for d in set(text_run[q]) & set(ragged_run[q]):
            assert abs(text_run[q][d] - ragged_run[q][d]) <= eps

    depth = 12
    out = tmp_path / "rr.trec"
    _run(rerank.main, ["--output_dir", tmp_path / "rr_out", "--model_name_or_path", rr_dir, "--query_path",
                       tmp_path / "queries.tsv", "--corpus_path", tmp_path / "corpus.tsv", "--query_template", "<text>",
                       "--query_column_names", "id,text", "--doc_template", "<text>", "--doc_column_names", "id,text",
                       "--q_max_len", q_max, "--p_max_len", p_max, "--per_device_eval_batch_size", 24,
                       "--trec_run_path", tmp_path / "run_text.trec", "--trec_save_path", out, "--reranking_depth",
                       depth, "--dataloader_num_workers", 0])
    got = load_from_trec(str(out))
    run = load_from_trec(str(tmp_path / "run_text.trec"), max_len_per_q=depth)
    assert {q: set(v) for q, v in got.items()} == {q: set(v) for q, v in run.items()}
    # HF fp32 RRModel.encode on the reference's pairs, padded with 1
    model = RRModel.build(ModelArguments(model_name_or_path=str(rr_dir))).cuda().eval()
    pairs = [(q, d) for q, docs in run.items() for d in docs]

    def content(text, n):
        return tok(text, add_special_tokens=False, truncation=True, max_length=n)["input_ids"]

    rows = [encode_pair([0], [2], content(queries[q], q_max), content(corpus[d], p_max)) for q, d in pairs]
    ids = torch.ones(len(rows), q_max + p_max + 2, dtype=torch.long)
    mask = torch.zeros_like(ids)
    for i, r in enumerate(rows):
        ids[i, :len(r)] = torch.tensor(r)
        mask[i, :len(r)] = 1
    with torch.no_grad():
        hf = model.head(model.lm(input_ids=ids.cuda(), attention_mask=mask.cuda()).last_hidden_state[:, 0])[:, 0]
    mine = np.array([got[q][d] for q, d in pairs])
    _check(mine.reshape(1, -1), hf.cpu().numpy().reshape(1, -1), "roberta rerank driver vs HF fp32")
    # the padded-store path of the cross-encoder: the same scores as the text path
    qarr = padded_store("queries_tok", queries, q_max)
    assert qarr.shape[1] == q_max
    out2 = tmp_path / "rr_store.trec"
    _run(rerank.main, ["--output_dir", tmp_path / "rr_out", "--model_name_or_path", rr_dir, "--query_path",
                       tmp_path / "queries_tok.npy", "--corpus_path", tmp_path / "corpus_tok.npy", "--q_max_len", q_max,
                       "--p_max_len", p_max, "--per_device_eval_batch_size", 24, "--trec_run_path",
                       tmp_path / "run_text.trec", "--trec_save_path", out2, "--reranking_depth", depth,
                       "--dataloader_num_workers", 0])
    assert load_from_trec(str(out2)) == got
    model.cpu()
