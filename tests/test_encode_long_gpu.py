"""GPU: sequences of 513 - 8192 tokens on the sm_90a encoder (attn_stream_kernel), BERT and RoBERTa, head widths 64 and 32.

Every batch below mixes bins (<= 128 tokens, attn_kernel), 129 - 512-token sequences and longer ones (both
attn_stream_kernel), so both attention kernels run in every layer.  Reps and attended hidden rows are held to the
float64-oracle bound of tests/test_encoder_numerics_gpu.py (err_kernel <= 2 err_autocast + 2e-4, plus rel-L2 <= 1e-2 and
cosine >= 0.9999), one sequence per oracle call; the online softmax at 8192 tokens with the row maxima in the first,
the last and a moving key tile; bitwise batch invariance, pair assembly and the padded DRModel path; refusals before any
write; poisoned workspaces and side streams; HF fp32 parity at bge-m3 width; the drivers end to end at 2048 tokens."""
import os
import sys

import numpy as np
import pytest
import torch

import oracle
import roberta_oracle as ro
from test_encoder_gpu import _check, _rand_bert_sd
from test_encoder_numerics_gpu import F64, _judge, _Logits, _ospec, _tile_gap

pytestmark = pytest.mark.gpu

SHORT = [1, 77, 128, 129, 300, 512]  # both sides of the one-tile limit of attn_kernel, up to 512 tokens


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


def _spec(arch, H, heads, F, vocab, max_pos, layers=2):
    return dict(arch=arch, layers=layers, hidden=H, heads=heads, ffn=F, vocab=vocab, max_pos=max_pos,
                type_vocab=2 if arch == "bert" else 1, ln_eps=1e-12 if arch == "bert" else 1e-5)


def _model(gen, arch, heads, max_pos, H=128, F=256, vocab=1000, layers=2, q_scale=20.0):
    """random weights; the query weights scaled so that attention rows are peaked, not uniform over 8192 keys"""
    sd = _rand_bert_sd(gen, layers, H, F, vocab, max_pos)
    if arch == "roberta":
        sd["embeddings.token_type_embeddings.weight"] = sd["embeddings.token_type_embeddings.weight"][:1]
    for i in range(layers):
        for n in ("weight", "bias"):
            sd[f"encoder.layer.{i}.attention.self.query.{n}"] *= q_scale
    return _spec(arch, H, heads, F, vocab, max_pos, layers), sd


def _seq(gen, arch, n, vocab):
    """RoBERTa: <s> content </s> with a few pad ids 1 inside the content; BERT: ids >= 5"""
    s = torch.randint(5, vocab, (n,), generator=gen)
    if arch == "roberta":
        s[0] = 0
        if n > 1:
            s[-1] = 2
        if n > 4:
            s[torch.randint(1, n - 1, (max(1, n // 50),), generator=gen)] = 1
    return s


def _packed(enc, seqs, **kw):
    lens = np.array([len(s) for s in seqs], dtype=np.int32)
    return enc.encode_packed(torch.cat(seqs).cuda(), lens, **kw)


def _oracle(arch, sd, ospec, seq, head, emulate):
    ids, mask = seq[None], torch.ones(1, len(seq), dtype=torch.long)
    if arch == "roberta":
        return ro.encode_reps(sd, ospec, ids, mask, head, dtype=F64, emulate_bf16=emulate)
    return oracle.encode_reps(sd, ospec, ids, mask, None, head, dtype=F64, emulate_bf16=emulate)


def _vs_oracle(what, arch, sd, spec, seqs, got_h, got, head, pooling, normalize):
    """judge every sequence's reps and hidden rows against the float64 oracle, one sequence per oracle call"""
    ospec = _ospec(dict(spec, arch="bert"), pooling, normalize)  # RoBERTa: the BERT oracle with its position ids
    offs = np.cumsum([0] + [len(s) for s in seqs])
    want, auto, wh, ah = [], [], [], []
    for s in seqs:
        (h0, r0), (h1, r1) = _oracle(arch, sd, ospec, s, head, False), _oracle(arch, sd, ospec, s, head, True)
        want.append(r0[0].numpy())
        auto.append(r1[0].numpy())
        wh.append(h0[0].numpy())
        ah.append(h1[0].numpy())
    got, got_h = got.float().cpu().numpy(), got_h.cpu().numpy()
    for i, s in enumerate(seqs):
        if len(s) > 512:
            _judge("%s L=%d reps" % (what, len(s)), got[i:i + 1], want[i][None], auto[i][None])
            _judge("%s L=%d hidden" % (what, len(s)), got_h[offs[i]:offs[i + 1]], wh[i], ah[i])
    _judge(what + " all reps", got, np.stack(want), np.stack(auto))
    _judge(what + " all hidden", got_h, np.concatenate(wh), np.concatenate(ah))


# (arch, heads at hidden 128: 2 = 64-wide, 4 = 32-wide, long lengths, pooling, head, normalize, output dtype)
CASES = [("bert", 2, (513, 8192), "first", True, True, torch.float32),
         ("bert", 4, (640, 2048), "mean", False, False, torch.bfloat16),
         ("bert", 4, (4097, 1025), "first", False, True, torch.float32),
         ("roberta", 2, (1025, 4097), "mean", False, True, torch.float16),
         ("roberta", 4, (8192, 513), "first", True, False, torch.float32),
         ("roberta", 2, (2048, 640), "mean", True, False, torch.bfloat16)]


@pytest.mark.parametrize("arch,heads,longs,pooling,has_head,normalize,dtype", CASES)
def test_mixed_batch_vs_float64_oracle(enc_mod, arch, heads, longs, pooling, has_head, normalize, dtype):
    gen = torch.Generator().manual_seed(9000 + CASES.index((arch, heads, longs, pooling, has_head, normalize, dtype)))
    max_pos = 8192 if arch == "bert" else 8194
    spec, sd = _model(gen, arch, heads, max_pos)
    head = torch.randn(48, 128, generator=gen) * 128 ** -0.5 if has_head else None
    lens = [SHORT[0], longs[0], SHORT[1], SHORT[4], longs[1], SHORT[2], SHORT[3], SHORT[5]]
    seqs = [_seq(gen, arch, n, 1000) for n in lens]
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize, max_batch_tokens=16384)
    got_h, got = _packed(enc, seqs, return_hidden=True)
    what = "%s dh=%d %s%s%s" % (arch, 128 // heads, pooling, " head" if has_head else "", " norm" if normalize else "")
    _vs_oracle(what, arch, sd, spec, seqs, got_h, got, head, pooling, normalize)
    if dtype != torch.float32:  # bf16 / fp16 reps are the rounding of the fp32 reps of the same batch
        low = _packed(enc, seqs, out_dtype=dtype)
        assert low.dtype == dtype and torch.equal(low, got.to(dtype)), what + ": %s output" % dtype


# ------------------------------------------------------------------------------------------------------------------
# online softmax over 64 key tiles: the row maxima in the first tile, in the last one, or rising from tile to tile
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["tile0", "last_tile", "moving"])
def test_online_softmax_tile_maxima_8192(enc_mod, where):
    # hidden dim 0 of the position embedding sets a per-key level (+a in the favoured tile, -a elsewhere; or rising
    # linearly from -a to +a over the sequence); the key projection turns it into dimension 0 of every head's key and
    # the query bias puts gamma there, as in test_online_softmax_tile_maxima_bert
    L = 8192
    gen = torch.Generator().manual_seed(9100 + ["tile0", "last_tile", "moving"].index(where))
    H, F, heads = 128, 256, 2
    spec = _spec("bert", H, heads, F, 1000, L, layers=1)
    sd = _rand_bert_sd(gen, 1, H, F, 1000, L)
    a = 0.18
    pos = torch.arange(L)
    if where == "moving":
        level = a * (2.0 * pos / (L - 1) - 1.0)
    else:
        fav = pos < 128 if where == "tile0" else pos >= L - 128
        level = torch.where(fav, a, -a)
    sd["embeddings.position_embeddings.weight"][:, 0] = level
    sd["embeddings.LayerNorm.weight"][0], sd["embeddings.LayerNorm.bias"][0] = 1.0, 0.0
    gamma, beta = (12.0, 16.0) if where == "tile0" else (10.0, 14.0)
    p = "encoder.layer.0.attention.self."
    wk, bq = sd[p + "key.weight"], sd[p + "query.bias"]
    for h in range(heads):
        wk[64 * h] = 0.0
        wk[64 * h, 0] = beta / 5.0
        bq[64 * h] = gamma
    seqs = [_seq(gen, "bert", L, 1000), _seq(gen, "bert", 300, 1000)]
    enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=16384)
    got_h, got = _packed(enc, seqs, return_hidden=True)
    _vs_oracle("bert L=8192 max " + where, "bert", sd, spec, seqs[:1], got_h[:L], got[:1], None, "mean", False)
    probe = _Logits()
    oracle.encode_reps(sd, _ospec(spec, "mean"), seqs[0][None], torch.ones(1, L, dtype=torch.long), dtype=F64,
                       probe=probe)
    s = probe.by_layer[0]
    if where == "moving":  # the running maximum is raised at about half of the 63 tile steps of every row
        tmax = s.view(1, heads, L, L // 128, 128).amax(-1)
        raised = (tmax[..., 1:] > torch.cummax(tmax, -1).values[..., :-1]).double().mean(-1)
        spread = float((tmax[..., -1] - tmax[..., 0]).min())
        print("[numerics] premise: running maximum raised at >= %.3f of the tile steps, last - first tile maximum "
              ">= %.1f nats" % (float(raised.min()), spread))
        assert float(raised.min()) >= 0.4 and spread >= 25.0 and bool((tmax.argmax(-1) == L // 128 - 1).all())
    else:
        gap = _tile_gap(s, torch.ones(1, L, dtype=torch.bool), L // 128, where == "tile0")
        need = 30.0 if where == "tile0" else 20.0
        print("[numerics] premise: min tile gap %.1f nats >= %.0f" % (float(gap.min()), need))
        assert float(gap.min()) >= need


# ------------------------------------------------------------------------------------------------------------------
# bitwise properties
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,heads", [("bert", 2), ("roberta", 4)])
def test_batch_invariance_and_pairs(enc_mod, arch, heads):
    gen = torch.Generator().manual_seed(9200 + heads)
    spec, sd = _model(gen, arch, heads, 8194)
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=torch.randn(1, 128, generator=gen) * 0.1, pooling="first",
                              max_batch_tokens=16384)
    doc = _seq(gen, arch, 3000, 1000)
    alone = _packed(enc, [doc])
    for lens in ([3000, 5, 700], [40, 300, 3000], [513, 128, 3000, 8000, 1]):
        seqs = [_seq(gen, arch, n, 1000) for n in lens]
        k = lens.index(3000)
        seqs[k] = doc
        assert torch.equal(_packed(enc, seqs)[k], alone[0]), "%s: a long sequence depends on its batch" % lens
    short = [_seq(gen, arch, n, 1000) for n in (3, 128, 129, 512, 60, 257)]
    want = _packed(enc, short)
    mixed = short[:3] + [_seq(gen, arch, 2500, 1000)] + short[3:] + [_seq(gen, arch, 1024, 1000)]
    got = _packed(enc, mixed)
    assert torch.equal(torch.cat([got[:3], got[4:7]]), want), "sequences <= 512 tokens change next to longer ones"
    # pairs assembled on the device: the same scores as the assembled sequences packed
    a = [_seq(gen, arch, int(n), 1000)[1:-1] for n in (10, 30, 3, 64)]
    b = [_seq(gen, arch, int(n), 1000)[1:-1] for n in (4000, 700, 100, 2040)]
    a_store, b_store = torch.cat(a).to(torch.int32), torch.cat(b).to(torch.int32)
    a0, b0 = np.cumsum([0] + [len(x) for x in a])[:-1], np.cumsum([0] + [len(x) for x in b])[:-1]
    pairs = [(0, 0), (1, 1), (2, 2), (3, 3), (1, 0), (3, 1)]
    spans = np.array([(a0[i], len(a[i]), b0[j], len(b[j])) for i, j in pairs], dtype=np.int64)
    got = enc.encode_pairs(a_store.cuda(), b_store.cuda(), spans, [0], [2, 2])
    assembled = [torch.cat([torch.tensor([0]), a[i], b[j], torch.tensor([2, 2])]) for i, j in pairs]
    assert torch.equal(got, _packed(enc, assembled)), "encode_pairs differs from encode_packed"


def _hf(arch, seed, heads=2, max_pos=2050, vocab=1000, H=128, layers=2, F=512):
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel, XLMRobertaConfig, XLMRobertaModel
    torch.manual_seed(seed)
    kw = dict(vocab_size=vocab, hidden_size=H, num_hidden_layers=layers, num_attention_heads=heads, intermediate_size=F,
              max_position_embeddings=max_pos)
    if arch == "bert":
        return BertModel(BertConfig(**kw)).eval()
    if arch == "xlm-roberta":
        return XLMRobertaModel(XLMRobertaConfig(type_vocab_size=1, pad_token_id=1, **kw)).eval()
    return RobertaModel(RobertaConfig(type_vocab_size=1, pad_token_id=1, **kw)).eval()


def _right_padded(seqs, L, pad):
    ids = torch.full((len(seqs), L), pad, dtype=torch.long)
    mask = torch.zeros(len(seqs), L, dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = s
        mask[i, :len(s)] = 1
    return ids, mask


@pytest.mark.parametrize("arch", ["bert", "roberta"])
def test_drmodel_padded_long_batch(enc_mod, arch):
    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    lm = _hf(arch, 9300).cuda()
    model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling="mean", normalize=True,
                                model_args=ModelArguments("unused", pooling="mean", normalize=True))
    gen = torch.Generator().manual_seed(9300)
    pad = 0 if arch == "bert" else 1
    seqs = [_seq(gen, arch, n, 1000) for n in (2048, 700, 5, 1300, 2000)]
    ids, mask = _right_padded(seqs, 2048, pad)
    batch = {"input_ids": ids.cuda(), "attention_mask": mask.cuda()}
    out = torch.full((5, 128), 7.0, device="cuda")
    model.encode_into(batch, out)
    enc = model._cuda_encoder(lm, None)
    assert torch.equal(out, _packed(enc, seqs)), "encode_into of a padded L=2048 batch differs from encode_packed"
    hidden, reps = model.encode_passage(batch)
    assert torch.equal(reps, out)
    m = mask.bool().cuda()
    want_h, _ = _packed(enc, seqs, return_hidden=True)
    assert torch.equal(hidden[m], want_h) and (hidden[~m] == 0).all(), "hidden rows: real tokens, zero padding"
    with torch.no_grad():  # and the HF module agrees
        hf = lm(**batch).last_hidden_state.float()
    _check(hidden[m].cpu().numpy(), hf[m].cpu().numpy(), "%s DRModel L=2048 hidden vs HF" % arch)
    left = {"input_ids": ids.flip(1).cuda(), "attention_mask": mask.flip(1).cuda()}
    out.fill_(7.0)
    with pytest.raises(ValueError, match="right padding"):
        model.encode_into(left, out)
    with pytest.raises(ValueError, match="right padding"):
        model.encode_passage(left)
    torch.cuda.synchronize()
    assert (out == 7.0).all()


# ------------------------------------------------------------------------------------------------------------------
# refusals before any write
# ------------------------------------------------------------------------------------------------------------------
def test_limits_refused_before_any_write(enc_mod):
    gen = torch.Generator().manual_seed(9400)
    out = torch.full((2, 128), 7.0, device="cuda")
    spec, sd = _model(gen, "roberta", 2, 1090)
    enc = enc_mod.CudaEncoder(spec, sd, max_batch_tokens=4096)
    assert enc_mod.max_seq_len(enc.spec, enc.max_batch_tokens) == 1088
    _packed(enc, [_seq(gen, "roberta", 1088, 1000), _seq(gen, "roberta", 9, 1000)], out=out)  # at the limit: accepted
    out.fill_(7.0)
    with pytest.raises(RuntimeError, match="max_position_embeddings - 2"):
        _packed(enc, [_seq(gen, "roberta", 1089, 1000), _seq(gen, "roberta", 9, 1000)], out=out)
    store = torch.randint(3, 1000, (2000,), generator=gen).to(torch.int32).cuda()
    with pytest.raises(RuntimeError, match="pair 1"):
        enc.encode_pairs(store, store, np.array([[0, 10, 0, 10], [0, 87, 0, 1000]]), [0], [2], out=out)
    spec, sd = _model(gen, "bert", 4, 16384)
    enc = enc_mod.CudaEncoder(spec, sd, max_batch_tokens=20000)
    assert enc_mod.max_seq_len(enc.spec, enc.max_batch_tokens) == 8192
    with pytest.raises(RuntimeError, match="seqlens"):
        _packed(enc, [_seq(gen, "bert", 8193, 1000), _seq(gen, "bert", 9, 1000)], out=out)
    enc = enc_mod.CudaEncoder(spec, sd, max_batch_tokens=3000)
    with pytest.raises(RuntimeError, match="max_batch_tokens"):
        _packed(enc, [_seq(gen, "bert", 3001, 1000), _seq(gen, "bert", 9, 1000)], out=out)
    from test_encoder_gpu import _rand_t5_sd
    t5 = dict(arch="t5", layers=1, hidden=128, heads=2, ffn=256, vocab=1000, ln_eps=1e-6, rel_buckets=32,
              rel_max_distance=128)
    enc = enc_mod.CudaEncoder(t5, _rand_t5_sd(gen, 1, 128, 2, 256, 1000), max_batch_tokens=4096)
    assert enc_mod.max_seq_len(t5, 4096) == 512
    _packed(enc, [_seq(gen, "bert", 512, 1000), _seq(gen, "bert", 9, 1000)], out=out)
    out.fill_(7.0)
    with pytest.raises(RuntimeError, match="512 tokens"):
        _packed(enc, [_seq(gen, "bert", 513, 1000), _seq(gen, "bert", 9, 1000)], out=out)
    torch.cuda.synchronize()
    assert (out == 7.0).all(), "a refused call wrote to the output"


# ------------------------------------------------------------------------------------------------------------------
# BERT and RoBERTa handles interleaved, side streams, poisoned workspaces
# ------------------------------------------------------------------------------------------------------------------
def _long_batch(enc, arch, seed):
    gen = torch.Generator().manual_seed(seed)
    seqs = [_seq(gen, arch, n, 1000) for n in (2500, 3, 513, 300, 129, 1025, 64)]
    h, r = _packed(enc, seqs, return_hidden=True)
    return h.clone(), r.clone()


def test_interleaved_side_stream_poison(enc_mod):
    gen = torch.Generator().manual_seed(9500)
    models = {"bert": _model(gen, "bert", 2, 4096), "roberta": _model(gen, "roberta", 4, 4098)}

    def make(k):
        return enc_mod.CudaEncoder(*models[k], head_weight=torch.ones(8, 128) / 128, pooling="mean", normalize=True,
                                   max_batch_tokens=8192)

    live = {k: make(k) for k in models}
    want = {k: _long_batch(live[k], k, 9600) for k in models}
    for k in ("roberta", "bert", "roberta", "bert"):
        h, r = _long_batch(live[k], k, 9600)
        assert torch.equal(h, want[k][0]) and torch.equal(r, want[k][1]), k + ": interleaved calls differ"
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = {k: _long_batch(live[k], k, 9600) for k in models}
    side.synchronize()
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        poisoned = {k: make(k) for k in models}
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]
    for k in models:
        assert torch.equal(got[k][0], want[k][0]) and torch.equal(got[k][1], want[k][1]), k + ": side stream differs"
        h, r = _long_batch(poisoned[k], k, 9600)
        assert torch.isfinite(h).all() and torch.isfinite(r).all(), k + ": non-finite output"
        assert torch.equal(h, want[k][0]) and torch.equal(r, want[k][1]), k + ": poisoned workspace changes the result"


# ------------------------------------------------------------------------------------------------------------------
# HF fp32 at bge-m3 width (XLM-RoBERTa large shape, 4 layers, random init)
# ------------------------------------------------------------------------------------------------------------------
def test_hf_parity_bge_m3_width(enc_mod):
    lm = _hf("xlm-roberta", 9700, heads=16, max_pos=8194, vocab=250002, H=1024, layers=4, F=4096).cuda()
    enc = enc_mod.CudaEncoder.from_hf(lm, pooling="first", normalize=True)
    gen = torch.Generator().manual_seed(9700)
    lens = [8192] + torch.randint(1, 8193, (5,), generator=gen).tolist() + [1, 513, 128]
    seqs = [_seq(gen, "roberta", n, 250002) for n in lens]
    got_h, got = _packed(enc, seqs, return_hidden=True)
    offs = np.cumsum([0] + lens)
    torch.backends.cuda.matmul.allow_tf32 = False
    for i, s in enumerate(seqs):
        with torch.no_grad():
            hf = lm(input_ids=s[None].cuda()).last_hidden_state[0].float()
        want = torch.nn.functional.normalize(hf[:1], dim=1)
        _check(got[i:i + 1].cpu().numpy(), want.cpu().numpy(), "bge-m3 width L=%d reps vs HF fp32" % len(s))
        _check(got_h[offs[i]:offs[i + 1]].cpu().numpy(), hf.cpu().numpy(), "bge-m3 width L=%d hidden vs HF fp32" % len(s))


# ------------------------------------------------------------------------------------------------------------------
# drivers end to end at --p_max_len 2048: text, padded store, ragged store; rerank of passages beyond 512 tokens
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


def test_drivers_at_2048_tokens(enc_mod, tmp_path):
    from openmatch.dataset import write_ragged_store
    from openmatch.driver import build_index, rerank, retrieve
    from openmatch.utils import load_from_trec
    from openmatch_b200.modeling import LinearHead, RRModel
    from openmatch_b200.retriever.reranker import encode_pair
    tok = ro.offline_tokenizer(str(tmp_path))
    dr_dir, rr_dir = tmp_path / "dr", tmp_path / "rr"
    dr_lm = _hf("roberta", 9800, vocab=len(tok))
    dr_lm.save_pretrained(str(dr_dir))
    tok.save_pretrained(str(dr_dir))
    os.makedirs(rr_dir)
    rr = RRModel(lm=_hf("roberta", 9801, heads=4, vocab=len(tok)), head=LinearHead(128, 1), pooling="first")
    rr.save(str(rr_dir))
    tok.save_pretrained(str(rr_dir))
    rng = np.random.default_rng(9800)
    # every character is one token: documents of ~100 - 2000 tokens, most of them beyond 512
    corpus = {"d%d" % i: " ".join(rng.choice(WORDS, int(rng.integers(20, 420)))) for i in range(40)}
    queries = {"q%d" % i: " ".join(rng.choice(WORDS, int(rng.integers(1, 4)))) for i in range(5)}
    with open(tmp_path / "corpus.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in corpus.items())
    with open(tmp_path / "queries.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in queries.items())
    q_max, p_max = 24, 2048
    doc_ids = [tok(t, truncation=True, max_length=p_max)["input_ids"] for t in corpus.values()]
    assert max(len(r) for r in doc_ids) > 1500 and sum(len(r) > 512 for r in doc_ids) >= 20

    arr = np.full((len(corpus), p_max), 1, np.int32)
    for i, r in enumerate(doc_ids):
        arr[i, :len(r)] = r
    np.save(tmp_path / "corpus_tok.npy", arr)
    (tmp_path / "corpus_tok.ids.txt").write_text("\n".join(corpus))

    def retrieve_with(tag, corpus_args):
        emb = tmp_path / ("emb_" + tag)
        common = ["--output_dir", emb, "--model_name_or_path", dr_dir, "--per_device_eval_batch_size", 8, "--q_max_len",
                  q_max, "--p_max_len", p_max, "--dataloader_num_workers", 0]
        _run(build_index.main, common + corpus_args)
        out = tmp_path / ("run_%s.trec" % tag)
        _run(retrieve.main, common + ["--query_path", tmp_path / "queries.tsv", "--query_template", "<text>",
                                      "--query_column_names", "id,text", "--trec_save_path", out, "--retrieve_depth",
                                      10, "--use_gpu"])
        return load_from_trec(str(out))

    runs = {"text": retrieve_with("text", ["--corpus_path", tmp_path / "corpus.tsv", "--doc_template", "<text>",
                                           "--doc_column_names", "id,text"]),
            "padded": retrieve_with("padded", ["--corpus_path", tmp_path / "corpus_tok.npy"]),
            "ragged": retrieve_with("ragged", ["--corpus_path", write_ragged_store(str(tmp_path / "corpus_rag"), arr,
                                                                                   list(corpus), pad_id=1)])}
    # oracle: the float32 oracle's reps (first pooling, no normalisation) and exact inner-product search
    sd = {k: v.detach() for k, v in dr_lm.state_dict().items()}
    ospec = _ospec(_spec("bert", 128, 2, 512, len(tok), 2050), "first", False)
    prep = np.concatenate([ro.encode_reps(sd, ospec, torch.tensor([r]), torch.ones(1, len(r), dtype=torch.long))[1].numpy()
                           for r in doc_ids])
    qids = [tok(t, truncation=True, max_length=q_max)["input_ids"] for t in queries.values()]
    qrep = np.concatenate([ro.encode_reps(sd, ospec, torch.tensor([r]), torch.ones(1, len(r), dtype=torch.long))[1].numpy()
                           for r in qids])
    scores = qrep.astype(np.float64) @ prep.astype(np.float64).T
    names = list(corpus)
    eps = 2e-3 * float(np.abs(scores).max())  # the bf16 encoder's score error; ranks compared up to ties within it
    for tag, run in runs.items():
        assert sorted(run) == sorted(queries), tag
        for qi, q in enumerate(queries):
            want = [names[j] for j in np.argsort(-scores[qi], kind="stable")[:10]]
            got = list(run[q])
            assert len(got) == 10
            for r, (dg, dw) in enumerate(zip(got, want)):
                sg, sw = scores[qi][names.index(dg)], scores[qi][names.index(dw)]
                assert dg == dw or abs(sg - sw) <= eps, (tag, q, r, dg, dw, sg, sw)

    depth, rr_p = 8, 2000
    out = tmp_path / "rr.trec"
    _run(rerank.main, ["--output_dir", tmp_path / "rr_out", "--model_name_or_path", rr_dir, "--query_path",
                       tmp_path / "queries.tsv", "--corpus_path", tmp_path / "corpus.tsv", "--query_template", "<text>",
                       "--query_column_names", "id,text", "--doc_template", "<text>", "--doc_column_names", "id,text",
                       "--q_max_len", q_max, "--p_max_len", rr_p, "--per_device_eval_batch_size", 8,
                       "--trec_run_path", tmp_path / "run_text.trec", "--trec_save_path", out, "--reranking_depth",
                       depth, "--dataloader_num_workers", 0])
    got = load_from_trec(str(out))
    run = load_from_trec(str(tmp_path / "run_text.trec"), max_len_per_q=depth)
    assert {q: set(v) for q, v in got.items()} == {q: set(v) for q, v in run.items()}
    pairs = [(q, d) for q, docs in run.items() for d in docs]

    def content(text, n):
        return tok(text, add_special_tokens=False, truncation=True, max_length=n)["input_ids"]

    rows = [encode_pair([0], [2], content(queries[q], q_max), content(corpus[d], rr_p)) for q, d in pairs]
    assert sum(len(r) > 512 for r in rows) >= len(rows) // 2
    lm = rr.lm.cuda()
    hf = []
    with torch.no_grad():
        for r in rows:
            hf.append(float(rr.head(lm(input_ids=torch.tensor([r]).cuda()).last_hidden_state[:, 0].cpu())[0, 0]))
    mine = np.array([got[q][d] for q, d in pairs])
    _check(mine.reshape(1, -1), np.array(hf).reshape(1, -1), "roberta rerank driver at 2000-token passages vs HF fp32")


# ------------------------------------------------------------------------------------------------------------------
# the reference's golden vectors beyond 512 tokens: padded through DRModel, and packed
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["ra", "rb", "ba"])
def test_reference_long_golden(enc_mod, golden_dir, cfg):
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel

    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    from openmatch_b200.modeling.linear import LinearHead
    from test_encode_long_cpu import load_long_golden, long_golden_spec
    z, sd, head_w, ids, mask = load_long_golden(golden_dir, cfg)
    spec = long_golden_spec(cfg)
    kw = dict(vocab_size=128, hidden_size=128, num_hidden_layers=2, num_attention_heads=spec["heads"],
              intermediate_size=64, max_position_embeddings=spec["max_pos"])
    if spec["arch"] == "roberta":
        lm = RobertaModel(RobertaConfig(type_vocab_size=1, pad_token_id=1, **kw))
    else:
        lm = BertModel(BertConfig(**kw))
    missing, unexpected = lm.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("pooler.") for k in missing)
    lm = lm.cuda().eval()
    head = LinearHead(128, 64)
    head.linear.weight.data.copy_(head_w)
    head = head.cuda()
    m = mask.bool()
    lens = m.sum(1).numpy().astype(np.int32)
    rows = z[cfg + ".sample_rows"]
    batch = {"input_ids": ids.cuda(), "attention_mask": mask.cuda()}
    for pooling, normalize, hd, key in (("first", False, head, "reps_first_head"), ("mean", True, None, "reps_mean_norm")):
        what = "long golden %s %s" % (cfg, key)
        model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling=pooling, normalize=normalize, head_q=hd,
                                    head_p=hd, model_args=ModelArguments("unused", pooling=pooling, normalize=normalize))
        hidden, reps = model.encode_passage(batch)
        _check(reps.cpu().numpy(), z["%s.%s" % (cfg, key)], what + " DRModel padded")
        _check(hidden.cpu()[m].numpy()[rows], z[cfg + ".hidden_sample"], what + " DRModel padded hidden")
        enc = enc_mod.CudaEncoder(spec, sd, head_weight=head_w if hd is not None else None, pooling=pooling,
                                  normalize=normalize, max_batch_tokens=8192)
        ph, preps = enc.encode_packed(ids[m].cuda(), lens, return_hidden=True)
        _check(preps.cpu().numpy(), z["%s.%s" % (cfg, key)], what + " packed")
        _check(ph.cpu().numpy()[rows], z[cfg + ".hidden_sample"], what + " packed hidden")
