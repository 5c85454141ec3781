"""GPU: variable-length encoding without padding (om_encode_packed / CudaEncoder.encode_packed /
DRModel.encode_packed_into / ragged pretokenised stores).

Packed reps and hidden rows are held to the float64-oracle bound of tests/test_encoder_numerics_gpu.py, with the oracle
run per sequence without padding, and to the padded path (om_encode) of the same sequences; placement, determinism,
row groups beyond max_batch_tokens, poisoned workspaces, side streams, invalid input and the retriever end to end."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

import oracle
from test_encoder_gpu import _check, _golden, _rand_bert_sd, _rand_t5_sd
from test_encoder_numerics_gpu import F64, _bert_spec, _judge, _ospec, _t5_spec

pytestmark = pytest.mark.gpu

EDGE_LENS = [1, 31, 64, 65, 127, 128, 129, 255, 256, 257, 384, 512]


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


def _model(name, gen):
    if name == "bert":
        spec, sd = _bert_spec(2, 128, 2, 512), _rand_bert_sd(gen, 2, 128, 512, 2000, 512)
    elif name == "bert_base":
        spec, sd = _bert_spec(2, 768, 12, 3072), _rand_bert_sd(gen, 2, 768, 3072, 2000, 512)
    else:
        spec, sd = _t5_spec(2, 128, 2, 512), _rand_t5_sd(gen, 2, 128, 2, 512, 2000)
    return spec, sd


def _seqs(gen, lens, vocab=2000):
    return [torch.randint(5, vocab, (int(l),), generator=gen) for l in lens]


def _padded(seqs, L):
    ids = torch.zeros(len(seqs), L, dtype=torch.long)
    mask = torch.zeros(len(seqs), L, dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, :len(s)], mask[i, :len(s)] = s, 1
    return ids, mask


def _packed(enc, seqs, tts=None, **kw):
    lens = np.array([len(s) for s in seqs], dtype=np.int32)
    tt = torch.cat(tts).cuda() if tts is not None else None
    return enc.encode_packed(torch.cat(seqs).cuda(), lens, token_type_ids=tt, **kw)


def _oracle_per_seq(sd, ospec, seqs, tts, head, emulate):
    hs, rs = [], []
    for i, s in enumerate(seqs):
        h, r = oracle.encode_reps(sd, ospec, s[None], torch.ones(1, len(s), dtype=torch.long),
                                  tts[i][None] if tts is not None else None, head, dtype=F64, emulate_bf16=emulate)
        hs.append(h[0].numpy())
        rs.append(r[0].numpy())
    return np.concatenate(hs), np.stack(rs)


# (model, pooling, head, normalize, out dtype)
CONFIGS = [("bert", "first", False, False, torch.float32), ("bert", "mean", True, True, torch.bfloat16),
           ("bert", "first", True, False, torch.float16), ("t5", "mean", True, True, torch.float16),
           ("t5", "first", False, False, torch.bfloat16), ("t5", "mean", False, False, torch.float32),
           ("bert_base", "mean", False, True, torch.float32)]


@pytest.mark.parametrize("name,pooling,has_head,normalize,dtype", CONFIGS)
def test_packed_vs_oracle_and_padded(enc_mod, name, pooling, has_head, normalize, dtype):
    gen = torch.Generator().manual_seed(3000 + CONFIGS.index((name, pooling, has_head, normalize, dtype)))
    spec, sd = _model(name, gen)
    H = spec["hidden"]
    head = torch.randn(96, H, generator=gen) * H ** -0.5 if has_head else None
    lens = EDGE_LENS + torch.randint(1, 513, (10,), generator=gen).tolist() + torch.randint(1, 60, (10,), generator=gen).tolist()
    lens = [lens[i] for i in torch.randperm(len(lens), generator=gen).tolist()]
    seqs = _seqs(gen, lens)
    tts = [torch.randint(0, 2, (l,), generator=gen) for l in lens] if spec["arch"] == "bert" else None
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                              max_batch_tokens=len(seqs) * 512)
    hidden, reps = _packed(enc, seqs, tts, return_hidden=True)
    hidden, reps = hidden.cpu().numpy(), reps.cpu().numpy()
    assert hidden.shape == (sum(lens), H)
    ospec = _ospec(spec, pooling, normalize)
    oh, oreps = _oracle_per_seq(sd, ospec, seqs, tts, head, False)
    ah, areps = _oracle_per_seq(sd, ospec, seqs, tts, head, True)
    what = "%s %s%s%s" % (name, pooling, " head" if has_head else "", " norm" if normalize else "")
    _judge(what + " packed reps", reps, oreps, areps)
    _judge(what + " packed hidden", hidden, oh, ah)
    # the padded path on the same sequences (L = 512): same values up to the order of sums
    ids, mask = _padded(seqs, 512)
    tt_pad = _padded(tts, 512)[0].cuda() if tts is not None else None
    ph, preps = enc.encode(ids.cuda(), mask.cuda(), tt_pad, return_hidden=True)
    _check(reps, preps.cpu().numpy(), what + " packed vs padded reps", rel_tol=2e-3, cos_tol=0.99999)
    _check(hidden, ph.cpu().numpy()[mask.numpy().astype(bool)], what + " packed vs padded hidden", rel_tol=2e-3,
           cos_tol=0.99999)
    # other output dtypes: the round-to-nearest-even of the fp32 output, row i = sequence i, into a strided buffer
    if dtype != torch.float32:
        buf = torch.full((len(seqs), enc.rep_dim + 16), 7.0, dtype=dtype, device="cuda")
        _packed(enc, seqs, tts, out=buf[:, 8:8 + enc.rep_dim])
        assert torch.equal(buf[:, 8:8 + enc.rep_dim].cpu(), torch.from_numpy(reps).to(dtype))
        assert (buf[:, :8] == 7).all() and (buf[:, 8 + enc.rep_dim:] == 7).all()


@pytest.mark.parametrize("which", ["bert", "t5"])
def test_reference_goldens_packed(enc_mod, golden_dir, which):
    # the ragged batches the reference's own DRModelForInference encoded (prefix masks), fed without their padding
    z, sd = _golden(golden_dir, "%s_small.npz" % which)
    m = z["attention_mask"].astype(bool)
    lens = m.sum(1)
    assert all(m[i, :lens[i]].all() for i in range(len(lens))), "premise: prefix masks"
    if which == "bert":
        spec = dict(arch="bert", layers=2, hidden=128, heads=2, ffn=512, vocab=512, max_pos=128, type_vocab=2,
                    ln_eps=1e-12)
        enc = enc_mod.CudaEncoder(spec, sd, pooling="first", max_batch_tokens=1024)
        tt = torch.from_numpy(z["token_type_ids"][m])
    else:
        spec = dict(arch="t5", layers=2, hidden=128, heads=2, ffn=512, vocab=512, ln_eps=1e-6, rel_buckets=32,
                    rel_max_distance=128)
        enc = enc_mod.CudaEncoder(spec, sd, head_weight=torch.from_numpy(z["head_weight"]), pooling="mean",
                                  normalize=True, max_batch_tokens=1024)
        tt = None
    ids = torch.from_numpy(z["input_ids"][m]).cuda()
    hidden, reps = enc.encode_packed(ids, lens.astype(np.int32), token_type_ids=tt.cuda() if tt is not None else None,
                                     return_hidden=True)
    ph, preps = enc.encode(torch.from_numpy(z["input_ids"]).cuda(), torch.from_numpy(z["attention_mask"]).cuda(),
                           torch.from_numpy(z["token_type_ids"]).cuda() if which == "bert" else None, return_hidden=True)
    for what, got, pad, want in (("reps", reps.cpu().numpy(), preps.cpu().numpy(), z["reps"]),
                                 ("hidden", hidden.cpu().numpy(), ph.cpu().numpy()[m], z["hidden"][m])):
        rel_packed, _ = _check(got, want, "%s packed %s vs reference" % (which, what))
        rel_padded, _ = _check(pad, want, "%s padded %s vs reference" % (which, what))
        assert rel_packed <= rel_padded + 2e-4, "%s: packed %.3e vs padded %.3e" % (what, rel_packed, rel_padded)


def test_determinism_and_placement(enc_mod):
    gen = torch.Generator().manual_seed(3100)
    spec, sd = _model("bert", gen)
    enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=64 * 512)
    lens = torch.randint(1, 129, (40,), generator=gen).tolist() + [200, 300, 512, 129]
    seqs = _seqs(gen, lens)
    h1, r1 = (x.clone() for x in _packed(enc, seqs, return_hidden=True))
    h2, r2 = _packed(enc, seqs, return_hidden=True)
    assert torch.equal(h1, h2) and torch.equal(r1, r2), "run-to-run difference"
    # a permuted batch: another placement (bins are filled in another order), the same reps within tolerance
    perm = torch.randperm(len(seqs), generator=gen).tolist()
    rp = _packed(enc, [seqs[i] for i in perm])
    _check(rp.cpu().numpy(), r1.cpu().numpy()[perm], "permuted batch", rel_tol=2e-3, cos_tol=0.99999)


def test_layout_beyond_max_batch_tokens(enc_mod):
    gen = torch.Generator().manual_seed(3200)
    spec, sd = _model("t5", gen)
    head = torch.randn(64, 128, generator=gen) * 128 ** -0.5
    small = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling="mean", max_batch_tokens=1024)
    big = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling="mean", max_batch_tokens=1 << 16)
    # whole-tile sequences place identically whatever the group: 20 x 128 tokens + 6 x 256 = 4 row groups of 1024 rows;
    # the same call on an encoder that holds the whole layout, and separate calls on consecutive parts, agree bitwise
    seqs = _seqs(gen, [256] * 6 + [128] * 20)
    h, r = _packed(small, seqs, return_hidden=True)
    hb, rb = _packed(big, seqs, return_hidden=True)
    assert torch.equal(r, rb) and torch.equal(h, hb)
    parts = [seqs[:4], seqs[4:6], seqs[6:14], seqs[14:]]
    rp = torch.cat([_packed(small, p) for p in parts])
    assert torch.equal(rp, r)
    # mixed lengths: several row groups, checked against the single-group encoder and separate calls
    seqs = _seqs(gen, torch.randint(1, 513, (30,), generator=gen).tolist())
    r = _packed(small, seqs).cpu().numpy()
    _check(r, _packed(big, seqs).cpu().numpy(), "row groups vs one group", rel_tol=2e-3, cos_tol=0.99999)
    _check(r, torch.cat([_packed(small, seqs[i:i + 3]) for i in range(0, 30, 3)]).cpu().numpy(), "row groups vs parts",
           rel_tol=2e-3, cos_tol=0.99999)
    # more sequences than max_batch_tokens: encoded in chunks of sequences
    tiny = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling="mean", max_batch_tokens=64)
    seqs = _seqs(gen, torch.randint(1, 9, (150,), generator=gen).tolist())
    _check(_packed(tiny, seqs).cpu().numpy(), _packed(big, seqs).cpu().numpy(), "chunks of sequences", rel_tol=2e-3,
           cos_tol=0.99999)


def test_poisoned_workspace_and_side_stream(enc_mod):
    gen = torch.Generator().manual_seed(3300)
    for name in ("bert", "t5"):
        spec, sd = _model(name, gen)
        seqs = _seqs(gen, [3, 512, 40, 129, 77, 1, 128, 300, 64, 65])
        want_h, want = _packed(enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=4096), seqs,
                               return_hidden=True)
        torch.cuda.synchronize()
        os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
        try:
            enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=4096)
        finally:
            del os.environ["OPENMATCH_B200_POISON_ALLOC"]
        got_h, got = _packed(enc, seqs, return_hidden=True)
        assert torch.isfinite(got).all() and torch.isfinite(got_h).all(), name + ": non-finite output"
        assert torch.equal(got, want) and torch.equal(got_h, want_h), name + ": poisoned workspace changes the result"
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            sh, sr = _packed(enc, seqs, return_hidden=True)
        side.synchronize()
        assert torch.equal(sr, want) and torch.equal(sh, want_h), name + ": side stream differs"


def test_invalid_input(enc_mod):
    from openmatch_b200 import _lib
    gen = torch.Generator().manual_seed(3400)
    spec = _bert_spec(1, 128, 2, 256, vocab=100, max_pos=200)
    enc = enc_mod.CudaEncoder(spec, _rand_bert_sd(gen, 1, 128, 256, 100, 200), max_batch_tokens=4096)
    out = torch.full((3, 128), 7.0, device="cuda")
    toks = torch.randint(5, 100, (600,), device="cuda")
    for lens in ([4, 0, 5], [4, 513, 5], [4, 201, 5], [-1, 2, 3]):  # 201 > max_position_embeddings
        with pytest.raises(RuntimeError, match="seqlens"):
            enc.encode_packed(toks[:max(sum(lens), 0)], np.array(lens), out=out)
    lib, lens = _lib.load(), (ctypes.c_int32 * 3)(4, 5, 6)
    stream = _lib.current_stream_ptr()
    args = [enc._h, toks.data_ptr(), None, lens, 3, out.data_ptr(), _lib.OM_F32, 128, None, stream]
    for slot, bad in ((1, None), (3, None), (4, -1), (5, None), (0, None)):
        a = list(args)
        a[slot] = bad
        assert lib.om_encode_packed(*a) == -1  # OM_EINVAL
    torch.cuda.synchronize()
    assert (out == 7).all(), "a refused call wrote to the output"
    assert lib.om_encode_packed(enc._h, toks.data_ptr(), None, lens, 0, out.data_ptr(), _lib.OM_F32, 128, None,
                                stream) == 0  # empty batch: nothing to do
    assert (out == 7).all()


def _eps_same_ranking(Dw, Iw, Dg, Ig, eps):
    """the two rankings agree up to eps-ties: scores rank by rank within eps, and a differing id only where the wanted
    ranking has another score within 2 eps of that rank's"""
    assert Dw.shape == Dg.shape
    assert (np.abs(Dw - Dg) <= eps).all(), "scores differ by more than eps"
    for q, r in zip(*np.nonzero(Iw != Ig)):
        assert np.sort(np.abs(Dw[q] - Dw[q, r]))[1] <= 2 * eps, "query %d rank %d: not an eps-tie" % (q, r)


@pytest.mark.parametrize("index_dtype", ["float32", "float16"])
def test_retriever_ragged_store_end_to_end(enc_mod, tmp_path, index_dtype):
    from openmatch.arguments import DataArguments, ModelArguments
    from openmatch.dataset import InferenceDataset, write_ragged_store
    from openmatch.modeling import DRModelForInference
    from openmatch.retriever import Retriever
    from transformers import BertConfig, BertModel
    torch.manual_seed(3500)
    lm = BertModel(BertConfig(vocab_size=500, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                              intermediate_size=512, max_position_embeddings=512)).eval()
    rng = np.random.default_rng(3500)
    n, L = 300, 300
    ids = rng.integers(5, 500, (n, L)).astype(np.int32)
    for r in range(n):
        ids[r, rng.integers(1, L + 1):] = 0
    names = ["p%d" % i for i in range(n)]
    np.save(tmp_path / "pad.npy", ids)
    (tmp_path / "pad.ids.txt").write_text("\n".join(names))
    ragged = write_ragged_store(str(tmp_path / "rag"), ids, names)
    queries = rng.integers(5, 500, (20, 32)).astype(np.int64)
    queries[:, 20:] = 0
    margs = ModelArguments(model_name_or_path="unused", pooling="mean", normalize=True)

    class Queries(torch.utils.data.IterableDataset):
        def __iter__(self):
            for i, q in enumerate(queries):
                yield {"text_id": "q%d" % i, "input_ids": q.tolist(), "attention_mask": (q != 0).astype(np.int64).tolist(),
                       "token_type_ids": [0] * len(q)}

    results = {}
    for kind, path in (("padded", str(tmp_path / "pad.npy")), ("ragged", ragged)):
        ds = InferenceDataset.load(None, DataArguments(corpus_path=path, p_max_len=256), is_query=False, batch_size=64)
        assert getattr(ds, "is_ragged", False) == (kind == "ragged")
        args = types.SimpleNamespace(device=torch.device("cuda"), fp16=False, bf16=False, per_device_eval_batch_size=8,
                                     dataloader_num_workers=0, dataloader_pin_memory=False,
                                     output_dir=str(tmp_path / kind), process_index=0, local_process_index=0,
                                     world_size=1, use_gpu=True, index_dtype=index_dtype)
        model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling="mean", normalize=True, model_args=margs)
        r = Retriever.build_all(model, ds, args)
        assert r.index.ntotal == n
        results[kind] = (list(r.doc_lookup), r.retrieve(Queries(), topk=20, as_arrays=True))
    (lw, want), (lg, got) = results["padded"], results["ragged"]
    assert lw == lg == names
    _eps_same_ranking(want.D, want.I, got.D, got.I, eps=2e-3)
    lm.cpu()
