"""GPU: BERT encoders with 32-wide attention heads (all-MiniLM, bge-small, e5-small, gte-small: hidden 384, 12 heads).

attn_kernel<32> / attn_stream_kernel<32> take one work item per (tile, pair of heads).  Reps and attended hidden rows are
held to the float64-oracle bound of tests/test_encoder_numerics_gpu.py (err_kernel <= 2 err_autocast + 2e-4, plus
rel-L2 <= 1e-2 and cosine >= 0.9999) on the padded and the packed path; the reference's own golden vectors, the HF
module, handles of both widths in one process, side streams, poisoned workspaces, refusals and the drivers end to end."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from oracle.encoder import EncoderSpec
from test_encode_packed_gpu import EDGE_LENS, _oracle_per_seq, _packed, _padded, _seqs
from test_encoder_gpu import _check, _ids, _rand_bert_sd
from test_encoder_hd32_cpu import GOLDEN_SPEC, load_golden
from test_encoder_numerics_gpu import F64, _bert_spec, _compare, _judge, _ospec, _scale_query

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


# (hidden, heads, ffn, layers): bge-small / MiniLM-L12 shape, the golden's, ffn % 128 == 64, the widest hidden
SHAPES = {"bge_small": (384, 12, 1536, 12), "h128": (128, 4, 512, 2), "h256": (256, 8, 832, 2),
          "h1024": (1024, 32, 2048, 2)}


def _model(name, gen):
    H, heads, F, layers = SHAPES[name]
    assert H // heads == 32
    return _bert_spec(layers, H, heads, F), _rand_bert_sd(gen, layers, H, F, 2000, 512)


def _other_dtype(enc, reps, ids, mask, tt, dtype):
    # bf16 / fp16 output into a strided buffer: the round-to-nearest-even of the fp32 reps, neighbours untouched
    B, D = reps.shape
    buf = torch.full((B, D + 16), 7.0, dtype=dtype, device="cuda")
    enc.encode(ids.cuda(), mask.cuda(), tt.cuda() if tt is not None else None, out=buf[:, 8:8 + D])
    assert torch.equal(buf[:, 8:8 + D].cpu(), torch.from_numpy(reps).to(dtype))
    assert (buf[:, :8] == 7).all() and (buf[:, 8 + D:] == 7).all()


# (model, L, B, pooling, head, normalize, out dtype, query scale): every attn_kernel packing (L = 1 .. 128 -> 128 .. 1
# sequences per tile) and attn_stream_kernel at 2, 3 and 4 key tiles
PADDED = [("bge_small", 128, 6, "first", False, True, torch.float32, 1), ("bge_small", 512, 2, "mean", False, True,
                                                                          torch.bfloat16, 1),
          ("bge_small", 37, 9, "mean", True, False, torch.float16, 1),
          ("h128", 1, 40, "first", False, False, torch.float32, 1), ("h128", 17, 24, "mean", True, True, torch.float16, 1),
          ("h128", 64, 8, "first", True, False, torch.bfloat16, 15), ("h128", 100, 5, "mean", False, False, torch.float32, 15),
          ("h128", 256, 3, "first", False, True, torch.float16, 15), ("h128", 384, 2, "mean", True, True, torch.float32, 1),
          ("h256", 32, 12, "mean", False, False, torch.bfloat16, 1), ("h256", 384, 2, "first", True, True, torch.float16, 10),
          ("h1024", 100, 4, "first", False, False, torch.float32, 10), ("h1024", 512, 1, "mean", True, True, torch.bfloat16, 1)]


@pytest.mark.parametrize("name,L,B,pooling,has_head,normalize,dtype,alpha", PADDED)
def test_padded_vs_float64_oracle(enc_mod, name, L, B, pooling, has_head, normalize, dtype, alpha):
    gen = torch.Generator().manual_seed(6000 + PADDED.index((name, L, B, pooling, has_head, normalize, dtype, alpha)))
    spec, sd = _model(name, gen)
    sd = _scale_query(sd, spec["layers"], alpha)  # alpha > 1: peaked rows, where a key or head mix-up shows
    H = spec["hidden"]
    head = torch.randn(96, H, generator=gen) * H ** -0.5 if has_head else None
    ids, mask = _ids(gen, B, L, 2000)
    tt = torch.randint(0, 2, ids.shape, generator=gen)
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                              max_batch_tokens=ids.numel())
    what = "hd32 %s L=%d %s%s%s" % (name, L, pooling, " head" if has_head else "", " norm" if normalize else "")
    _, (_, reps), _ = _compare(enc_mod, what, spec, sd, ids, mask, tt, head=head, pooling=pooling, normalize=normalize,
                               enc=enc)
    if dtype != torch.float32:
        _other_dtype(enc, reps, ids, mask, tt, dtype)


PACKED = [("bge_small", "first", False, True, torch.float32), ("h128", "mean", True, True, torch.bfloat16),
          ("h256", "first", True, False, torch.float16), ("h1024", "mean", False, False, torch.float32)]


@pytest.mark.parametrize("name,pooling,has_head,normalize,dtype", PACKED)
def test_packed_vs_float64_oracle_and_padded(enc_mod, name, pooling, has_head, normalize, dtype):
    gen = torch.Generator().manual_seed(6100 + PACKED.index((name, pooling, has_head, normalize, dtype)))
    spec, sd = _model(name, gen)
    H = spec["hidden"]
    head = torch.randn(64, H, generator=gen) * H ** -0.5 if has_head else None
    lens = EDGE_LENS + torch.randint(1, 513, (4,), generator=gen).tolist() + torch.randint(1, 60, (8,), generator=gen).tolist()
    lens = [lens[i] for i in torch.randperm(len(lens), generator=gen).tolist()]
    seqs = _seqs(gen, lens)
    tts = [torch.randint(0, 2, (l,), generator=gen) for l in lens]
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                              max_batch_tokens=len(seqs) * 512)
    hidden, reps = _packed(enc, seqs, tts, return_hidden=True)
    hidden, reps = hidden.cpu().numpy(), reps.cpu().numpy()
    assert hidden.shape == (sum(lens), H)
    ospec = _ospec(spec, pooling, normalize)
    oh, oreps = _oracle_per_seq(sd, ospec, seqs, tts, head, False)
    ah, areps = _oracle_per_seq(sd, ospec, seqs, tts, head, True)
    what = "hd32 %s %s%s%s" % (name, pooling, " head" if has_head else "", " norm" if normalize else "")
    _judge(what + " packed reps", reps, oreps, areps)
    _judge(what + " packed hidden", hidden, oh, ah)
    ids, mask = _padded(seqs, 512)
    ph, preps = enc.encode(ids.cuda(), mask.cuda(), _padded(tts, 512)[0].cuda(), return_hidden=True)
    _check(reps, preps.cpu().numpy(), what + " packed vs padded reps", rel_tol=2e-3, cos_tol=0.99999)
    _check(hidden, ph.cpu().numpy()[mask.numpy().astype(bool)], what + " packed vs padded hidden", rel_tol=2e-3,
           cos_tol=0.99999)
    if dtype != torch.float32:
        buf = torch.full((len(seqs), enc.rep_dim + 16), 7.0, dtype=dtype, device="cuda")
        _packed(enc, seqs, tts, out=buf[:, 8:8 + enc.rep_dim])
        assert torch.equal(buf[:, 8:8 + enc.rep_dim].cpu(), torch.from_numpy(reps).to(dtype))
        assert (buf[:, :8] == 7).all() and (buf[:, 8 + enc.rep_dim:] == 7).all()


def test_reference_golden(enc_mod, golden_dir):
    # the reference's own DRModelForInference.encode_passage on a 4 x 32-wide-head BERT with peaked attention
    # (tests/golden/make_golden_hd32.py), padded and packed
    z, sd, ids, mask, tt = load_golden(golden_dir)
    enc = enc_mod.CudaEncoder(GOLDEN_SPEC, sd, pooling="mean", normalize=True, max_batch_tokens=1024)
    ids, mask, tt = ids.cuda(), mask.cuda(), tt.cuda()
    hidden, reps = enc.encode(ids, mask, tt, return_hidden=True)
    m = mask.bool()
    _check(reps.cpu().numpy(), z["reps"], "hd32 reps vs reference")
    _check(hidden[m].cpu().numpy(), z["hidden_attended"], "hd32 hidden vs reference")
    assert np.abs(reps.cpu().numpy() - z["reps"]).max() <= 2e-3  # normalised reps: max-abs bound (SURVEY 8c)
    lens = m.sum(1).cpu().numpy().astype(np.int32)
    ph, preps = enc.encode_packed(ids[m], lens, token_type_ids=tt[m], return_hidden=True)
    _check(preps.cpu().numpy(), z["reps"], "hd32 packed reps vs reference")
    _check(ph.cpu().numpy(), z["hidden_attended"], "hd32 packed hidden vs reference")


def _hf_bert_hd32(seed=7, max_pos=512):
    from transformers import BertConfig, BertModel
    torch.manual_seed(seed)
    cfg = BertConfig(vocab_size=1000, hidden_size=128, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=512, max_position_embeddings=max_pos)
    return BertModel(cfg).cuda().eval()


@pytest.mark.parametrize("pooling,normalize", [("first", False), ("mean", True)])
def test_hf_parity_through_drmodel(enc_mod, pooling, normalize):
    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    lm = _hf_bert_hd32()
    model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling=pooling, normalize=normalize,
                                model_args=ModelArguments("unused", pooling=pooling, normalize=normalize))
    gen = torch.Generator().manual_seed(6200)
    for L, B in ((96, 7), (384, 2)):
        ids, mask = _ids(gen, B, L, 1000)
        tt = torch.randint(0, 2, ids.shape, generator=gen)
        batch = {"input_ids": ids.cuda(), "attention_mask": mask.cuda(), "token_type_ids": tt.cuda()}
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
        _check(reps.cpu().numpy(), want.cpu().numpy(), "hd32 DRModel vs HF reps L=%d" % L)
        _check(hidden.float().cpu()[m].numpy(), want_h.cpu()[m].numpy(), "hd32 DRModel vs HF hidden L=%d" % L)


# ------------------------------------------------------------------------------------------------------------------
# handles of both widths in one process, side streams, poisoned workspaces
# ------------------------------------------------------------------------------------------------------------------
GEOMS = [(32, 11), (100, 7), (256, 3)]  # attn_kernel with 4 and 1 sequences per tile, attn_stream_kernel


def _inputs(gen):
    out = []
    for L, B in GEOMS:
        ids, mask = _ids(gen, B, L, 1000)
        out.append((ids.cuda(), mask.cuda(), torch.randint(0, 2, ids.shape, generator=gen).cuda()))
    return out


def _run_all(enc, inputs, packed_seqs):
    res = [enc.encode(*x, return_hidden=True) for x in inputs]
    res.append(_packed(enc, packed_seqs, return_hidden=True))
    return [(h.clone(), r.clone()) for h, r in res]


def _same(got, want, what):
    for (gh, gr), (wh, wr) in zip(got, want):
        assert torch.isfinite(gr).all() and torch.isfinite(gh).all(), what + ": non-finite output"
        assert torch.equal(gr, wr) and torch.equal(gh, wh), what


def test_both_head_widths_interleaved_and_side_stream(enc_mod):
    gen = torch.Generator().manual_seed(6300)
    specs = {32: (_bert_spec(2, 256, 8, 512, vocab=1000), _rand_bert_sd(gen, 2, 256, 512, 1000, 512)),
             64: (_bert_spec(2, 256, 4, 512, vocab=1000), _rand_bert_sd(gen, 2, 256, 512, 1000, 512))}
    inputs = _inputs(gen)
    seqs = _seqs(gen, [3, 512, 40, 129, 77, 1, 128, 300, 64, 65], vocab=1000)

    def make(w):
        return enc_mod.CudaEncoder(specs[w][0], specs[w][1], pooling="mean", max_batch_tokens=4096)

    live = {w: make(w) for w in (32, 64)}
    for rnd in range(2):  # calls alternate between the two handles, each call against a fresh handle of its kind
        for w in (32, 64, 32):
            got = _run_all(live[w], inputs, seqs)
            fresh = make(w)
            _same(got, _run_all(fresh, inputs, seqs), "width %d round %d: live handle differs from a fresh one" % (w, rnd))
            del fresh
    want = _run_all(live[32], inputs, seqs)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = _run_all(live[32], inputs, seqs)
    side.synchronize()
    _same(got, want, "side stream differs from the default stream")


def test_poisoned_workspace(enc_mod):
    gen = torch.Generator().manual_seed(6400)
    spec, sd = _bert_spec(2, 384, 12, 1536, vocab=1000), _rand_bert_sd(gen, 2, 384, 1536, 1000, 512)
    inputs = _inputs(gen)
    seqs = _seqs(gen, [5, 384, 128, 1, 200, 64], vocab=1000)
    want = _run_all(enc_mod.CudaEncoder(spec, sd, pooling="first", max_batch_tokens=4096), inputs, seqs)
    torch.cuda.synchronize()
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        enc = enc_mod.CudaEncoder(spec, sd, pooling="first", max_batch_tokens=4096)
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]
    _same(_run_all(enc, inputs, seqs), want, "poisoned workspace changes the result")


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden,heads", [(256, 16), (384, 4), (256, 2), (384, 5)])  # widths 16, 96, 128, 76.8
def test_other_head_widths_are_refused(enc_mod, hidden, heads):
    from openmatch_b200 import _lib
    lib = _lib.load()
    desc = _lib.EncoderDesc(arch=_lib.OM_ARCH_BERT, layers=1, hidden=hidden, heads=heads, ffn=512, vocab=100, max_pos=64,
                            type_vocab=2, ln_eps=1e-12, pooling=_lib.OM_POOL_FIRST, has_head=0, head_out=0, normalize=0,
                            rel_buckets=32, rel_max_distance=128, max_batch_tokens=1024)
    h = ctypes.c_void_p()
    assert lib.om_encoder_create(ctypes.byref(desc), ctypes.byref(h)) == -1  # OM_EINVAL
    assert not h.value
    msg = lib.om_last_error().decode()
    assert ("head width hidden/heads=%d" % (hidden // heads) in msg) if hidden % heads == 0 else ("multiple of heads" in msg)
    with pytest.raises(ValueError, match="32- or 64-wide"):
        enc_mod.CudaEncoder(_bert_spec(1, hidden, heads, 512, vocab=100, max_pos=64), {})


# ------------------------------------------------------------------------------------------------------------------
# drivers end to end: a 32-wide-head checkpoint through build_index -> retrieve
# ------------------------------------------------------------------------------------------------------------------
def _run(main, argv):
    old = sys.argv
    sys.argv = ["prog"] + [str(a) for a in argv]
    try:
        main()
    finally:
        sys.argv = old


@pytest.mark.parametrize("store", ["padded", "ragged"])
def test_build_index_and_retrieve(enc_mod, tmp_path, store):
    from transformers import BertTokenizer

    from openmatch.dataset import write_ragged_store
    from openmatch.driver import build_index, retrieve
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + ["w%d" % i for i in range(995)]
    (tmp_path / "vocab.txt").write_text("\n".join(vocab))
    lm = _hf_bert_hd32(seed=8).cpu()
    lm.save_pretrained(str(tmp_path / "model"))
    BertTokenizer(str(tmp_path / "vocab.txt")).save_pretrained(str(tmp_path / "model"))
    # pretokenised corpus and queries (0 = padding): the encoder's input is known exactly, so the oracle can follow it
    rng = np.random.default_rng(6500)
    n, L, nq, Lq, k = 400, 256, 12, 24, 20
    corpus = rng.integers(5, 1000, (n, L)).astype(np.int32)
    for r in range(n):
        corpus[r, rng.integers(1, L + 1):] = 0
    queries = rng.integers(5, 1000, (nq, Lq)).astype(np.int32)
    for r in range(nq):
        queries[r, rng.integers(2, Lq + 1):] = 0
    names = ["d%d" % i for i in range(n)]
    if store == "padded":
        np.save(tmp_path / "corpus.npy", corpus)
        (tmp_path / "corpus.ids.txt").write_text("\n".join(names))
        cpath = tmp_path / "corpus.npy"
    else:
        cpath = write_ragged_store(str(tmp_path / "corpus"), corpus, names)
    np.save(tmp_path / "queries.npy", queries)
    (tmp_path / "queries.ids.txt").write_text("\n".join("q%d" % i for i in range(nq)))
    common = ["--output_dir", tmp_path / "emb", "--model_name_or_path", tmp_path / "model", "--per_device_eval_batch_size",
              64, "--q_max_len", Lq, "--p_max_len", L, "--dataloader_num_workers", 0, "--pooling", "mean", "--normalize"]
    _run(build_index.main, common + ["--corpus_path", cpath])
    _run(retrieve.main, common + ["--query_path", tmp_path / "queries.npy", "--retrieve_depth", k, "--trec_save_path",
                                  tmp_path / "run.trec"])
    run = {}
    for line in (tmp_path / "run.trec").read_text().splitlines():
        qid, _, did, rank, _, _ = line.split()
        run.setdefault(qid, []).append((int(rank), int(did[1:])))
    # oracle: float64 encoding of the same ids, exact inner-product search
    sd = lm.state_dict()
    ospec = EncoderSpec("bert", 2, 128, 4, 512, lm.config.layer_norm_eps, pooling="mean", normalize=True)

    def enc(x):
        ids = torch.from_numpy(x.astype(np.int64))
        return oracle.encode_reps(sd, ospec, ids, (ids != 0).long(), dtype=F64)[1].numpy()

    S = enc(queries) @ enc(corpus).T
    eps = 2e-3  # the bf16 encoder's score error on normalised reps; ranks are compared up to ties within it
    assert sorted(run) == sorted("q%d" % i for i in range(nq))
    for qi in range(nq):
        got = [d for _, d in sorted(run["q%d" % qi])]
        assert len(got) == k
        want = np.lexsort((np.arange(n), -S[qi]))[:k]
        for r, (g, w) in enumerate(zip(got, want)):
            assert g == w or abs(S[qi, g] - S[qi, w]) <= eps, "q%d rank %d: doc %d (%.5f) vs oracle doc %d (%.5f)" % (
                qi, r, g, S[qi, g], w, S[qi, w])
