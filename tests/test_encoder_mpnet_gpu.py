"""GPU: MPNet (all-mpnet-base-v2, multi-qa-mpnet) and DistilBERT (TAS-B, msmarco-distilbert) on the sm_90a encoder.

MPNet is BERT's post-LN encoder with RoBERTa's position ids, no token types and a relative position bias shared by all
layers, which attn_kernel and attn_stream_kernel<64, true> add to the logits at BERT's 1/sqrt(64) scale.  DistilBERT
is BERT's encoder under other parameter names, with no token types.  Reps and attended hidden rows are held to the
float64-oracle bound of tests/test_encoder_numerics_gpu.py (err_kernel <= 2 err_autocast + 2e-4, plus rel-L2 <= 1e-2
and cosine >= 0.9999) on the padded and the packed path; then the reference's golden vectors, an adversarial case in
which the bias moves the favoured key of attention rows, the HF modules, device pair assembly, the library's and
Python's refusals, handles of three families in one process, side streams, poisoned workspaces and the drivers end to
end."""
import ctypes
import os

import numpy as np
import pytest
import torch

import mpnet_oracle as mo
from test_encode_packed_gpu import EDGE_LENS
from test_encoder_gpu import _check, _rand_bert_sd
from test_encoder_mpnet_cpu import ARCHS, golden_spec, load_golden
from test_encoder_numerics_gpu import F64, _judge, _ospec
from test_encoder_roberta_gpu import WORDS, _eps_equal_runs, _run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def enc_mod():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import encoder
    return encoder


# (arch, hidden, heads, ffn, vocab, max_pos): all-mpnet-base-v2, TAS-B / msmarco-distilbert, and a small MPNet; 2 layers
SHAPES = {"all_mpnet_base": ("mpnet", 768, 12, 3072, 30527, 514), "tas_b": ("distilbert", 768, 12, 3072, 30522, 512),
          "small_mpnet": ("mpnet", 256, 4, 512, 1000, 514)}
PAD = {"mpnet": 1, "distilbert": 0}
_TO_MPNET = {"attention.self.query": "attention.attn.q", "attention.self.key": "attention.attn.k",
             "attention.self.value": "attention.attn.v", "attention.output.dense": "attention.attn.o",
             "attention.output.LayerNorm": "attention.LayerNorm"}
_TO_DISTIL = {v: k for k, v in mo._DISTIL_LAYER.items()}


def _spec(arch, H, heads, F, vocab, max_pos, layers=2):
    spec = dict(arch=arch, layers=layers, hidden=H, heads=heads, ffn=F, vocab=vocab, max_pos=max_pos, type_vocab=0,
                ln_eps=1e-12)
    if arch == "mpnet":
        spec.update(rel_buckets=32, rel_max_distance=128)
    return spec


def _rand_sd(arch, gen, layers, H, F, vocab, max_pos, heads, rel_std=1.0):
    """a BERT-statistics state dict under ``arch``'s names (MPNet: relative bias of std ``rel_std`` nats)"""
    bert = _rand_bert_sd(gen, layers, H, F, 8, max_pos)
    bert["embeddings.word_embeddings.weight"] = torch.randn(vocab, H, generator=gen) * 0.02
    del bert["embeddings.token_type_embeddings.weight"]
    sd = {}
    for k, v in bert.items():
        if k.startswith("encoder.layer."):
            i, rest = k[len("encoder.layer."):].split(".", 1)
            mod, leaf = rest.rsplit(".", 1)
            if arch == "mpnet":
                k = "encoder.layer.%s.%s.%s" % (i, _TO_MPNET.get(mod, mod), leaf)
            else:
                k = "transformer.layer.%s.%s.%s" % (i, _TO_DISTIL[mod], leaf)
        sd[k] = v
    if arch == "mpnet":
        sd[mo.REL_KEY] = torch.randn(32, heads, generator=gen) * rel_std
    return sd


def _model(name, gen, layers=2):
    arch, H, heads, F, vocab, max_pos = SHAPES[name]
    return _spec(arch, H, heads, F, vocab, max_pos, layers), _rand_sd(arch, gen, layers, H, F, vocab, max_pos, heads)


def _seq(gen, n, vocab, arch):
    """<s> content </s> (MPNet, with a few content ids replaced by the pad id 1) / [CLS] content [SEP] (DistilBERT)"""
    s = torch.randint(4, vocab, (n,), generator=gen)
    s[0] = 0 if arch == "mpnet" else 2
    if n > 1:
        s[-1] = 2 if arch == "mpnet" else 3
    if arch == "mpnet" and n > 4:
        s[torch.randint(1, n - 1, (max(1, n // 50),), generator=gen)] = 1
    return s


def _padded(seqs, L, pad):
    ids = torch.full((len(seqs), L), pad, dtype=torch.long)
    mask = torch.zeros(len(seqs), L, dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = s
        mask[i, :len(s)] = 1
    return ids, mask


def _packed(enc, seqs, **kw):
    lens = np.array([len(s) for s in seqs], dtype=np.int32)
    return enc.encode_packed(torch.cat(seqs).cuda(), lens, **kw)


def _oracles(arch, sd, ospec, ids, mask, head, probe=None):
    return (mo.encode_reps(arch, sd, ospec, ids, mask, head, dtype=F64, probe=probe),
            mo.encode_reps(arch, sd, ospec, ids, mask, head, dtype=F64, emulate_bf16=True))


# ------------------------------------------------------------------------------------------------------------------
# the reference's golden vectors
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ARCHS)
def test_reference_golden(enc_mod, golden_dir, cfg):
    z, sd, head, ids, mask = load_golden(golden_dir, cfg)
    m = mask.bool()
    lens = m.sum(1).numpy().astype(np.int32)
    ids, mask = ids.cuda(), mask.cuda()
    L = ids.shape[1]
    Lpad = L if L <= 128 else 256  # om_encode takes 256 / 384 / 512 above one tile
    ids_p = torch.nn.functional.pad(ids, (0, Lpad - L), value=PAD[cfg])
    mask_p = torch.nn.functional.pad(mask, (0, Lpad - L))
    for pooling, normalize, hw, key in (("first", False, head, "reps_first_head"), ("mean", True, None, "reps_mean_norm")):
        enc = enc_mod.CudaEncoder(golden_spec(cfg), sd, head_weight=hw, pooling=pooling, normalize=normalize,
                                  max_batch_tokens=1024)
        hidden, reps = enc.encode(ids_p, mask_p, return_hidden=True)
        what = "%s %s" % (cfg, key)
        _check(reps.cpu().numpy(), z["%s.%s" % (cfg, key)], what)
        _check(hidden[mask_p.bool()].cpu().numpy(), z[cfg + ".hidden_attended"], what + " hidden")
        ph, preps = enc.encode_packed(ids[m.cuda()], lens, return_hidden=True)
        _check(preps.cpu().numpy(), z["%s.%s" % (cfg, key)], what + " packed")
        _check(ph.cpu().numpy(), z[cfg + ".hidden_attended"], what + " packed hidden")


# ------------------------------------------------------------------------------------------------------------------
# float64 oracle at all-mpnet-base-v2 and TAS-B width and at a small MPNet
# ------------------------------------------------------------------------------------------------------------------
PADDED = [("all_mpnet_base", 1, 16, "first", False, False), ("all_mpnet_base", 33, 12, "mean", True, True),
          ("all_mpnet_base", 128, 6, "mean", False, True), ("all_mpnet_base", 256, 3, "first", True, False),
          ("all_mpnet_base", 384, 2, "mean", False, True), ("all_mpnet_base", 512, 2, "first", False, False),
          ("tas_b", 1, 16, "first", True, False), ("tas_b", 64, 12, "first", False, False),
          ("tas_b", 128, 6, "mean", False, True), ("tas_b", 512, 2, "mean", True, True),
          ("small_mpnet", 100, 9, "mean", False, True), ("small_mpnet", 384, 3, "first", False, False)]


@pytest.mark.parametrize("name,L,B,pooling,has_head,normalize", PADDED)
def test_padded_vs_float64_oracle(enc_mod, name, L, B, pooling, has_head, normalize):
    gen = torch.Generator().manual_seed(9000 + PADDED.index((name, L, B, pooling, has_head, normalize)))
    spec, sd = _model(name, gen)
    arch, H = spec["arch"], spec["hidden"]
    head = torch.randn(96, H, generator=gen) * H ** -0.5 if has_head else None
    lens = [L] + torch.randint(1, L + 1, (B - 1,), generator=gen).tolist()
    ids, mask = _padded([_seq(gen, n, spec["vocab"], arch) for n in lens], L, PAD[arch])
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize, max_batch_tokens=B * L)
    tt = torch.randint(0, 2, ids.shape, generator=gen).cuda()  # ignored: neither model has token types
    hidden, reps = enc.encode(ids.cuda(), mask.cuda(), tt, return_hidden=True)
    (oh, oreps), (ah, areps) = _oracles(arch, sd, _ospec(dict(spec, arch="bert"), pooling, normalize), ids, mask, head)
    m = mask.numpy().astype(bool)
    what = "%s L=%d %s" % (name, L, pooling)
    _judge(what + " reps", reps.cpu().numpy(), oreps.numpy(), areps.numpy())
    _judge(what + " hidden", hidden.cpu().numpy()[m], oh.numpy()[m], ah.numpy()[m])
    for dt in (torch.bfloat16, torch.float16):  # the round-to-nearest-even of the fp32 reps of the same call
        assert torch.equal(enc.encode(ids.cuda(), mask.cuda(), out_dtype=dt), reps.to(dt))


@pytest.mark.parametrize("name,pooling,has_head,normalize", [("all_mpnet_base", "mean", False, True),
                                                             ("tas_b", "first", True, False),
                                                             ("small_mpnet", "first", False, False)])
def test_packed_vs_float64_oracle(enc_mod, name, pooling, has_head, normalize):
    gen = torch.Generator().manual_seed(9100 + len(name))
    spec, sd = _model(name, gen)
    arch, H = spec["arch"], spec["hidden"]
    head = torch.randn(64, H, generator=gen) * H ** -0.5 if has_head else None
    lens = EDGE_LENS + torch.randint(1, 513, (3,), generator=gen).tolist() + torch.randint(1, 60, (8,), generator=gen).tolist()
    lens = [lens[i] for i in torch.randperm(len(lens), generator=gen).tolist()]
    seqs = [_seq(gen, n, spec["vocab"], arch) for n in lens]
    enc = enc_mod.CudaEncoder(spec, sd, head_weight=head, pooling=pooling, normalize=normalize,
                              max_batch_tokens=len(seqs) * 512)
    hidden, reps = _packed(enc, seqs, return_hidden=True)
    ids, mask = _padded(seqs, 512, PAD[arch])
    (oh, oreps), (ah, areps) = _oracles(arch, sd, _ospec(dict(spec, arch="bert"), pooling, normalize), ids, mask, head)
    m = mask.numpy().astype(bool)
    what = "%s packed %s" % (name, pooling)
    _judge(what + " reps", reps.cpu().numpy(), oreps.numpy(), areps.numpy())
    _judge(what + " hidden", hidden.cpu().numpy(), oh.numpy()[m], ah.numpy()[m])


# ------------------------------------------------------------------------------------------------------------------
# attention statistics: the bias decides which key a row favours
# ------------------------------------------------------------------------------------------------------------------
MOVED_SHARE = 0.5  # at least this share of the attended (query, head) rows changes its arg-max key under the bias


@pytest.mark.parametrize("layout,L", [("padded", 64), ("padded", 512), ("packed", 0)])
def test_relative_bias_moves_attention(enc_mod, layout, L):
    """Peaked query weights (x30) and a bias of std 4 nats: the bias moves the favoured key of a stated share of the
    rows (probed on the float64 oracle), and the kernels follow the oracle within the whole-call bound."""
    gen = torch.Generator().manual_seed(9200 + L)
    H, heads, F, vocab = 256, 4, 512, 1000
    spec = _spec("mpnet", H, heads, F, vocab, 514)
    sd = _rand_sd("mpnet", gen, 2, H, F, vocab, 514, heads, rel_std=4.0)
    for i in range(2):
        sd["encoder.layer.%d.attention.attn.q.weight" % i] *= 30.0
    if layout == "padded":
        seqs = [_seq(gen, n, vocab, "mpnet") for n in [L] + torch.randint(L // 2, L + 1, (3,), generator=gen).tolist()]
    else:  # attn_kernel bins and attn_stream_kernel<64, true> tiles in one call
        seqs = [_seq(gen, n, vocab, "mpnet") for n in (300, 17, 129, 90, 512, 40, 256, 3)]
    ids, mask = _padded(seqs, L or 512, 1)
    bias = mo.mpnet_bias(sd, ids.shape[1])[None]
    moved, rows = [0], [0]

    def probe(layer, s):
        ok = torch.isfinite(s).any(-1) & mask.bool()[:, None, :]
        moved[0] += int(((s.argmax(-1) != (s - bias).argmax(-1)) & ok).sum())
        rows[0] += int(ok.sum())

    ospec = _ospec(dict(spec, arch="bert"), "mean", False)
    (oh, oreps), (ah, areps) = _oracles("mpnet", sd, ospec, ids, mask, None, probe=probe)
    share = moved[0] / rows[0]
    print("[mpnet bias] %s L=%d: arg-max key moved in %.1f %% of %d rows" % (layout, L, 100 * share, rows[0]))
    assert share >= MOVED_SHARE
    enc = enc_mod.CudaEncoder(spec, sd, pooling="mean", max_batch_tokens=4096)
    if layout == "padded":
        hidden, reps = enc.encode(ids.cuda(), mask.cuda(), return_hidden=True)
        hidden = hidden.cpu().numpy()[mask.numpy().astype(bool)]
    else:
        hidden, reps = _packed(enc, seqs, return_hidden=True)
        hidden = hidden.cpu().numpy()
    m = mask.numpy().astype(bool)
    what = "mpnet bias %s L=%d" % (layout, L)
    _judge(what + " reps", reps.cpu().numpy(), oreps.numpy(), areps.numpy(), fixed=False)
    _judge(what + " hidden", hidden, oh.numpy()[m], ah.numpy()[m], fixed=False)


# ------------------------------------------------------------------------------------------------------------------
# HF parity through DRModelForInference, device pair assembly
# ------------------------------------------------------------------------------------------------------------------
def _hf(arch, seed=9, heads=2, max_pos=514, vocab=1000):
    torch.manual_seed(seed)
    if arch == "mpnet":
        from transformers import MPNetConfig, MPNetModel
        cfg = MPNetConfig(vocab_size=vocab, hidden_size=128, num_hidden_layers=2, num_attention_heads=heads,
                          intermediate_size=512, max_position_embeddings=max_pos)
        lm = MPNetModel(cfg).eval()
        with torch.no_grad():  # HF initialises the bias at std 0.02: make it matter
            lm.encoder.relative_attention_bias.weight.normal_(0.0, 1.0)
        return lm
    from transformers import DistilBertConfig, DistilBertModel
    cfg = DistilBertConfig(vocab_size=vocab, dim=128, n_layers=2, n_heads=heads, hidden_dim=512,
                           max_position_embeddings=max_pos)
    return DistilBertModel(cfg).eval()


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("pooling,normalize", [("first", False), ("mean", True)])
def test_hf_parity_through_drmodel(enc_mod, arch, pooling, normalize):
    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    lm = _hf(arch).cuda()
    model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling=pooling, normalize=normalize,
                                model_args=ModelArguments("unused", pooling=pooling, normalize=normalize))
    gen = torch.Generator().manual_seed(9300)
    for L, B in ((96, 7), (512, 2)):
        lens = [L] + torch.randint(1, L, (B - 1,), generator=gen).tolist()
        ids, mask = _padded([_seq(gen, n, 1000, arch) for n in lens], L, PAD[arch])
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
        _check(reps.cpu().numpy(), want.cpu().numpy(), "%s DRModel vs HF reps L=%d" % (arch, L))
        _check(hidden.float().cpu()[m].numpy(), want_h.cpu()[m].numpy(), "%s DRModel vs HF hidden L=%d" % (arch, L))


@pytest.mark.parametrize("arch", ARCHS)
def test_pairs_bitwise_equal_packed(enc_mod, arch):
    gen = torch.Generator().manual_seed(9400)
    H, F, vocab = 256, 512, 1000
    head = torch.randn(1, H, generator=gen) * H ** -0.5
    pre, suf = ([0], [2, 2]) if arch == "mpnet" else ([2], [3])
    for heads in ((4,) if arch == "mpnet" else (4, 8)):  # DistilBERT: 64- and 32-wide heads
        sd = _rand_sd(arch, gen, 2, H, F, vocab, 514, heads)
        enc = enc_mod.CudaEncoder(_spec(arch, H, heads, F, vocab, 514), sd, head_weight=head, pooling="first",
                                  max_batch_tokens=2048)
        a = [_seq(gen, int(n), vocab, arch)[1:-1] for n in torch.randint(2, 40, (9,), generator=gen)]
        b = [_seq(gen, int(n), vocab, arch)[1:-1] for n in torch.randint(2, 470, (9,), generator=gen)]
        a[3] = torch.ones(0, dtype=torch.long)  # an empty query side
        b[5][:3] = 1  # pad ids (MPNet) at the start of the passage content
        a_store, b_store = torch.cat(a).to(torch.int32), torch.cat(b).to(torch.int32)
        a0 = np.cumsum([0] + [len(x) for x in a])[:-1]
        b0 = np.cumsum([0] + [len(x) for x in b])[:-1]
        pairs = [(i, j) for i in range(9) for j in range(9) if (i + j) % 4 == 0]
        spans = np.array([(a0[i], len(a[i]), b0[j], len(b[j])) for i, j in pairs], dtype=np.int64)
        got = enc.encode_pairs(a_store.cuda(), b_store.cuda(), spans, pre, suf)
        seqs = [torch.cat([torch.tensor(pre), a[i], b[j], torch.tensor(suf)]) for i, j in pairs]
        want = _packed(enc, seqs)
        assert torch.equal(got, want), "%s heads=%d: encode_pairs differs from encode_packed" % (arch, heads)


# ------------------------------------------------------------------------------------------------------------------
# refusals: the library's and Python's
# ------------------------------------------------------------------------------------------------------------------
def _create(lib, _lib, arch, **kw):
    f = dict(arch=arch, layers=1, hidden=128, heads=2, ffn=256, vocab=100, max_pos=66, type_vocab=0, ln_eps=1e-12,
             pooling=_lib.OM_POOL_FIRST, has_head=0, head_out=0, normalize=0, rel_buckets=32, rel_max_distance=128,
             max_batch_tokens=1024)
    f.update(kw)
    desc = _lib.EncoderDesc(**f)
    h = ctypes.c_void_p()
    rc = lib.om_encoder_create(ctypes.byref(desc), ctypes.byref(h))
    if rc == 0:
        lib.om_encoder_destroy(h)
    return rc, (lib.om_last_error().decode() if rc else "")


def test_library_refuses_unsupported_mpnet(enc_mod):
    from openmatch_b200 import _lib
    lib = _lib.load()
    assert _create(lib, _lib, _lib.OM_ARCH_MPNET)[0] == 0
    assert _create(lib, _lib, _lib.OM_ARCH_DISTILBERT, heads=4)[0] == 0  # DistilBERT takes 32-wide heads
    for kw, msg in ((dict(heads=4), "MPNet head width"), (dict(rel_buckets=64), "rel_buckets=32"),
                    (dict(rel_max_distance=256), "rel_max_distance=128"),
                    (dict(max_pos=2), "MPNet max_position_embeddings=2")):
        rc, err = _create(lib, _lib, _lib.OM_ARCH_MPNET, **kw)
        assert rc == -1 and msg in err, (kw, err)


@pytest.mark.parametrize("arch,max_pos,limit,name", [("mpnet", 66, 64, "max_position_embeddings - 2 (MPNet)"),
                                                     ("mpnet", 1026, 512, "512 tokens"),
                                                     ("distilbert", 64, 64, "8192 tokens, max_position_embeddings")])
def test_length_limit_refused_before_any_write(enc_mod, arch, max_pos, limit, name):
    gen = torch.Generator().manual_seed(9500 + max_pos)
    H, F, vocab = 128, 256, 500
    enc = enc_mod.CudaEncoder(_spec(arch, H, 2, F, vocab, max_pos, layers=1),
                              _rand_sd(arch, gen, 1, H, F, vocab, max_pos, 2), pooling="mean", max_batch_tokens=4096)
    assert enc_mod.max_seq_len(enc.spec, 4096) == limit
    out = torch.full((2, H), 7.0, device="cuda")
    ok = [_seq(gen, limit, vocab, arch), _seq(gen, 10, vocab, arch)]
    _packed(enc, ok, out=out)  # the limit itself: accepted
    if limit <= 128:
        ids, mask = _padded(ok, limit, PAD[arch])
        enc.encode(ids.cuda(), mask.cuda(), out=out)
    out.fill_(7.0)
    long = [_seq(gen, limit + 1, vocab, arch), _seq(gen, 10, vocab, arch)]
    if limit < 128:
        ids, mask = _padded(long, limit + 1, PAD[arch])
        with pytest.raises(RuntimeError, match=name.replace("(", r"\(").replace(")", r"\)")):
            enc.encode(ids.cuda(), mask.cuda(), out=out)
    with pytest.raises(RuntimeError, match=name.replace("(", r"\(").replace(")", r"\)")):
        _packed(enc, long, out=out)
    store = torch.cat(long).to(torch.int32).cuda()
    with pytest.raises(RuntimeError, match=name.replace("(", r"\(").replace(")", r"\)")):
        enc.encode_pairs(store, store, np.array([[0, limit - 1, 0, 1], [0, 2, 0, 2]]), [0], [2], out=out)
    torch.cuda.synchronize()
    assert (out == 7.0).all()


def test_python_refuses_before_the_library(enc_mod):
    from transformers import DistilBertConfig, MPNetConfig

    from openmatch_b200.encoder import CudaEncoder, spec_from_hf_config
    with pytest.raises(ValueError, match="64-wide"):
        spec_from_hf_config(MPNetConfig(hidden_size=384, num_attention_heads=12))
    with pytest.raises(ValueError, match="activation"):
        spec_from_hf_config(DistilBertConfig(activation="relu"))
    with pytest.raises(ValueError, match="32- or 64-wide"):
        CudaEncoder(_spec("distilbert", 384, 3, 256, 100, 64), {})


# ------------------------------------------------------------------------------------------------------------------
# BERT, MPNet and DistilBERT handles in one process, side streams, poisoned workspaces
# ------------------------------------------------------------------------------------------------------------------
def _run_all(enc, gen_seed, arch, vocab=1000):
    gen = torch.Generator().manual_seed(gen_seed)
    res = []
    for L, B in ((32, 11), (100, 7), (256, 3)):
        lens = [L] + torch.randint(1, L, (B - 1,), generator=gen).tolist()
        ids, mask = _padded([_seq(gen, int(n), vocab, arch) for n in lens], L, PAD.get(arch, 0))
        tt = torch.randint(0, 2, ids.shape, generator=gen).cuda()
        res.append(enc.encode(ids.cuda(), mask.cuda(), tt, return_hidden=True))
    seqs = [_seq(gen, n, vocab, arch) for n in (3, 512, 40, 129, 77, 1, 128, 300, 64, 65)]
    res.append(_packed(enc, seqs, return_hidden=True))
    a = torch.randint(4, vocab, (300,), generator=gen).to(torch.int32).cuda()
    a[::7] = 1
    spans = np.array([[0, 20, 20, 200], [5, 0, 40, 3], [100, 30, 0, 90]], dtype=np.int64)
    res.append((enc.encode_pairs(a, a, spans, [0], [2]), torch.zeros(1, device="cuda")))
    return [(h.clone(), r.clone()) for h, r in res]


def _same(got, want, what):
    for (gh, gr), (wh, wr) in zip(got, want):
        assert torch.isfinite(gr).all() and torch.isfinite(gh).all(), what + ": non-finite output"
        assert torch.equal(gr, wr) and torch.equal(gh, wh), what


def test_three_families_interleaved_side_stream_poison(enc_mod):
    gen = torch.Generator().manual_seed(9600)
    H, F, vocab = 256, 512, 1000
    bert_sd = _rand_bert_sd(gen, 2, H, F, vocab, 514)
    specs = {"mpnet": (_spec("mpnet", H, 4, F, vocab, 514), _rand_sd("mpnet", gen, 2, H, F, vocab, 514, 4)),
             "distilbert": (_spec("distilbert", H, 8, F, vocab, 514),
                            _rand_sd("distilbert", gen, 2, H, F, vocab, 514, 8)),
             "bert": (dict(_spec("bert", H, 4, F, vocab, 514), type_vocab=2), bert_sd)}

    def make(k):
        return enc_mod.CudaEncoder(specs[k][0], specs[k][1], head_weight=torch.ones(1, H) / H, pooling="mean",
                                   max_batch_tokens=4096)

    live = {k: make(k) for k in specs}
    for rnd in range(2):  # calls alternate between the handles, each against a fresh handle of its kind
        for k in ("mpnet", "bert", "distilbert", "mpnet"):
            got = _run_all(live[k], 9700 + rnd, k)
            fresh = make(k)
            _same(got, _run_all(fresh, 9700 + rnd, k), "%s round %d: live handle differs from a fresh one" % (k, rnd))
            del fresh
    for k in ("mpnet", "distilbert"):
        want = _run_all(live[k], 9800, k)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            got = _run_all(live[k], 9800, k)
        side.synchronize()
        _same(got, want, "%s: side stream differs from the default stream" % k)
        os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
        try:
            enc = make(k)
        finally:
            del os.environ["OPENMATCH_B200_POISON_ALLOC"]
        _same(_run_all(enc, 9800, k), want, "%s: poisoned workspace changes the result" % k)


# ------------------------------------------------------------------------------------------------------------------
# drivers end to end: saved MPNet and DistilBERT checkpoints with offline WordPiece tokenizers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ARCHS)
def test_build_index_retrieve_and_rerank(enc_mod, tmp_path, arch):
    import oracle
    from oracle.encoder import EncoderSpec
    from openmatch.arguments import ModelArguments
    from openmatch.dataset import write_ragged_store
    from openmatch.driver import build_index, rerank, retrieve
    from openmatch.utils import load_from_trec
    from openmatch_b200.modeling import LinearHead, RRModel
    from openmatch_b200.retriever.reranker import encode_pair, special_tokens
    tok = mo.offline_bert_vocab_tokenizer(str(tmp_path), arch)
    pad = PAD[arch]
    prefix, suffix = special_tokens(tok)
    assert tok.pad_token_id == pad and (prefix, suffix) == (([0], [2]) if arch == "mpnet" else ([2], [3]))
    dr_dir, rr_dir = tmp_path / "dr", tmp_path / "rr"
    dr_lm = _hf(arch, seed=10, vocab=len(tok), max_pos=130)
    dr_lm.save_pretrained(str(dr_dir))
    tok.save_pretrained(str(dr_dir))
    os.makedirs(rr_dir)
    rr = RRModel(lm=_hf(arch, seed=11, heads=2, vocab=len(tok), max_pos=130), head=LinearHead(128, 1), pooling="first")
    rr.save(str(rr_dir))
    tok.save_pretrained(str(rr_dir))
    rng = np.random.default_rng(9900)
    corpus = {"d%d" % i: " ".join(rng.choice(WORDS, int(rng.integers(1, 14)))) for i in range(60)}
    queries = {"q%d" % i: " ".join(rng.choice(WORDS, int(rng.integers(1, 4)))) for i in range(7)}
    with open(tmp_path / "corpus.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in corpus.items())
    with open(tmp_path / "queries.tsv", "w") as f:
        f.writelines("%s\t%s\n" % kv for kv in queries.items())
    q_max, p_max = 24, 96
    assert max(len(tok(t)["input_ids"]) for t in corpus.values()) <= p_max

    def padded_store(stem, texts, width):
        arr = np.full((len(texts), width), pad, np.int32)
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
    ragged_path = write_ragged_store(str(tmp_path / "corpus_rag"), arr, list(corpus), pad_id=pad)
    assert np.load(ragged_path)[0] == prefix[0]  # <s> / [CLS] kept
    ragged_run = retrieve_with("ragged", ["--corpus_path", ragged_path])
    assert len(text_run) == 7 and all(len(v) == 20 for v in text_run.values())
    # oracle encoding (float64) plus exact search: the ranking every run must reproduce up to ties within eps, 1e-2 of
    # the largest score (the bf16 encoder's score error is a few 1e-3 of it)
    sd = {k: v.detach().float() for k, v in dr_lm.state_dict().items()}
    ospec = EncoderSpec("bert", 2, 128, 2, 512, 1e-12, pooling="first")

    def oracle_reps(texts, width):
        rows = [tok(t, truncation=True, max_length=width)["input_ids"] for t in texts]
        ids, mask = _padded([torch.tensor(r) for r in rows], max(len(r) for r in rows), pad)
        return mo.encode_reps(arch, sd, ospec, ids, mask, dtype=F64)[1].numpy()

    P, Q = oracle_reps(corpus.values(), p_max), oracle_reps(queries.values(), q_max)
    D, I = oracle.flat_ip_search(Q, P, 20)
    eps = 1e-2 * float(np.abs(D).max())
    pids, qids = list(corpus), list(queries)
    want = {qids[i]: {pids[j]: float(d) for j, d in zip(I[i], D[i])} for i in range(len(qids))}
    want_sorted = {q: sorted(v, key=lambda d: -v[d]) for q, v in want.items()}
    all_scores = {q: {pids[j]: float(Q[i] @ P[j]) for j in range(len(pids))} for i, q in enumerate(qids)}
    for run in (text_run, padded_run, ragged_run):
        _eps_equal_runs({q: sorted(v, key=lambda d: -v[d]) for q, v in run.items()}, want_sorted, all_scores, eps)
        for q in run:
            for d, s in run[q].items():
                assert abs(s - all_scores[q][d]) <= eps

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
    # HF fp32 RRModel.encode on the reference's pairs, padded with the tokenizer's pad id
    model = RRModel.build(ModelArguments(model_name_or_path=str(rr_dir))).cuda().eval()
    pairs = [(q, d) for q, docs in run.items() for d in docs]

    def content(text, n):
        return tok(text, add_special_tokens=False, truncation=True, max_length=n)["input_ids"]

    rows = [encode_pair(prefix, suffix, content(queries[q], q_max), content(corpus[d], p_max)) for q, d in pairs]
    ids = torch.full((len(rows), q_max + p_max + 2), pad, dtype=torch.long)
    mask = torch.zeros_like(ids)
    for i, r in enumerate(rows):
        ids[i, :len(r)] = torch.tensor(r)
        mask[i, :len(r)] = 1
    with torch.no_grad():
        hf = model.head(model.lm(input_ids=ids.cuda(), attention_mask=mask.cuda()).last_hidden_state[:, 0])[:, 0]
    mine = np.array([got[q][d] for q, d in pairs])
    _check(mine.reshape(1, -1), hf.cpu().numpy().reshape(1, -1), "%s rerank driver vs HF fp32" % arch)
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
