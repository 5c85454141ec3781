"""CPU: MPNet and DistilBERT in the oracle and in the Python front end of the CUDA encoder.

The oracle restatements (tests/mpnet_oracle.py) must reproduce the reference's own encoding of an MPNet and a DistilBERT
model (tests/golden/mpnet_small.npz, made by tests/golden/make_golden_mpnet.py) before the GPU tests may judge the
kernels by them, and the fixture must tell each architecture from the mistakes a wrong parameter table or a missing
bias would make.  ``spec_from_hf_config`` maps both configs and refuses what the encoder cannot compute.
"""
import os

import numpy as np
import pytest
import torch

import mpnet_oracle as mo
import oracle
from oracle.encoder import EncoderSpec

ARCHS = ("mpnet", "distilbert")


def golden_spec(cfg, **kw):
    """the library spec of golden config ``cfg`` (``kw`` overrides)"""
    base = dict(arch=cfg, layers=2, hidden=128, heads=2, ffn=64, vocab=128, type_vocab=0, ln_eps=1e-12)
    if cfg == "mpnet":
        base.update(max_pos=260, rel_buckets=32, rel_max_distance=128)
    else:
        base.update(max_pos=66)
    return dict(base, **kw)


def load_golden(golden_dir, cfg):
    """(fixture, state dict, head weight, input_ids, attention_mask) of config ``cfg``: int8 codes times one fp32 scale
    per tensor, exactly the values the reference ran on"""
    z = np.load(os.path.join(golden_dir, "mpnet_small.npz"))
    pre = "q.%s." % cfg
    sd = {k[len(pre):]: torch.from_numpy(z[k].astype(np.float32) * z["s.%s.%s" % (cfg, k[len(pre):])])
          for k in z.files if k.startswith(pre)}
    head = sd.pop("head.linear.weight")
    ids, mask = (torch.from_numpy(z["%s.%s" % (cfg, k)].astype(np.int64)) for k in ("input_ids", "attention_mask"))
    return z, sd, head, ids, mask


def _ospec(pooling="first", normalize=False):
    return EncoderSpec("bert", 2, 128, 2, 64, 1e-12, pooling=pooling, normalize=normalize)


def _miss(got, want):
    """per-row relative L2 distance"""
    return np.linalg.norm(got - want, axis=-1) / np.linalg.norm(want, axis=-1)


def test_mpnet_bucket_is_t5_bucket():
    from transformers.models.mpnet.modeling_mpnet import MPNetEncoder
    rel = torch.arange(-1023, 1024)
    got = MPNetEncoder.relative_position_bucket(rel)  # num_buckets 32, max_distance 128: the defaults HF calls with
    assert torch.equal(got, oracle.t5_relative_position_bucket(rel, 32, 128))


@pytest.mark.parametrize("cfg", ARCHS)
def test_oracle_reproduces_the_reference_golden(golden_dir, cfg):
    z, sd, head, ids, mask = load_golden(golden_dir, cfg)
    m = mask.bool()
    if cfg == "mpnet":  # a 200-token row (distances past 128, position row 201), a pad id inside content
        assert int(m.sum(1).max()) == 200 and bool(((ids == 1) & m).any()) and bool((ids[~m] == 1).all())
    hidden, reps = mo.encode_reps(cfg, sd, _ospec(), ids, mask, head, dtype=torch.float64)
    assert np.abs(reps.numpy() - z[cfg + ".reps_first_head"]).max() <= 1e-5
    assert np.abs(hidden[m].numpy() - z[cfg + ".hidden_attended"]).max() <= 1e-4
    _, reps = mo.encode_reps(cfg, sd, _ospec("mean", True), ids, mask, dtype=torch.float64)
    assert np.abs(reps.numpy() - z[cfg + ".reps_mean_norm"]).max() <= 1e-5


@pytest.mark.parametrize("control", ["no_bias", "arange_positions"])
def test_mpnet_golden_rejects_bias_and_position_mistakes(golden_dir, control):
    """MPNet without its relative bias, or with BERT's positions 0 .. L-1, misses every row by more than 2e-2"""
    z, sd, _, ids, mask = load_golden(golden_dir, "mpnet")
    kw = dict(use_bias=False) if control == "no_bias" else dict(positions="arange")
    _, reps = mo.mpnet_reps(sd, _ospec("mean", True), ids, mask, dtype=torch.float64, **kw)
    err = _miss(reps.numpy(), z["mpnet.reps_mean_norm"])
    assert (err > 2e-2).all(), err


def test_distilbert_golden_rejects_swapped_layer_norms(golden_dir):
    """sa_layer_norm and output_layer_norm swapped, the mistake a wrong parameter table would make"""
    z, sd, _, ids, mask = load_golden(golden_dir, "distilbert")
    swapped = {}
    for k, v in sd.items():
        k2 = k.replace("sa_layer_norm", "@").replace("output_layer_norm", "sa_layer_norm").replace("@", "output_layer_norm")
        swapped[k2] = v
    _, reps = mo.distilbert_reps(swapped, _ospec("mean", True), ids, mask, dtype=torch.float64)
    err = _miss(reps.numpy(), z["distilbert.reps_mean_norm"])
    assert (err > 2e-2).all(), err


def test_mpnet_golden_bias_moves_attention_arg_max(golden_dir):
    """the fixture's relative bias changes which key a share of the attention rows favours"""
    _, sd, _, ids, mask = load_golden(golden_dir, "mpnet")
    L = ids.shape[1]
    bias = mo.mpnet_bias(sd, L)[None]
    moved, rows = 0, 0

    def probe(layer, s):
        nonlocal moved, rows
        ok = torch.isfinite(s).any(-1) & mask.bool()[:, None, :]
        a, b = s.argmax(-1), (s - bias).argmax(-1)
        moved += int(((a != b) & ok).sum())
        rows += int(ok.sum())

    mo.mpnet_reps(sd, _ospec(), ids, mask, dtype=torch.float64, probe=probe)
    print("bias moves the arg-max key of %d / %d attention rows" % (moved, rows))
    assert moved >= 0.1 * rows


# ------------------------------------------------------------------------------------------------------------------
# spec_from_hf_config
# ------------------------------------------------------------------------------------------------------------------
def test_spec_maps_all_mpnet_base_v2():
    from transformers import MPNetConfig

    from openmatch_b200.encoder import max_seq_len, spec_from_hf_config
    cfg = MPNetConfig(vocab_size=30527, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                      intermediate_size=3072, max_position_embeddings=514, layer_norm_eps=1e-5)
    spec = spec_from_hf_config(cfg)
    assert spec == dict(arch="mpnet", layers=12, hidden=768, heads=12, ffn=3072, vocab=30527, max_pos=514, type_vocab=0,
                        ln_eps=1e-5, rel_buckets=32, rel_max_distance=128)
    assert max_seq_len(spec) == 512
    assert max_seq_len(dict(spec, max_pos=130)) == 128
    assert max_seq_len(dict(spec, max_pos=4098)) == 512  # the relative-bias tables cover 512 tokens
    assert max_seq_len(spec, max_batch_tokens=300) == 300


@pytest.mark.parametrize("dim,heads", [(768, 12), (384, 12), (128, 2)])
def test_spec_maps_distilbert(dim, heads):
    from transformers import DistilBertConfig

    from openmatch_b200.encoder import max_seq_len, spec_from_hf_config
    cfg = DistilBertConfig(dim=dim, n_heads=heads, n_layers=6, hidden_dim=4 * dim, max_position_embeddings=512)
    spec = spec_from_hf_config(cfg)
    assert spec == dict(arch="distilbert", layers=6, hidden=dim, heads=heads, ffn=4 * dim, vocab=30522, max_pos=512,
                        type_vocab=0, ln_eps=1e-12)
    assert max_seq_len(spec) == 512
    assert max_seq_len(dict(spec, max_pos=8194)) == 8192


@pytest.mark.parametrize("kw,match", [
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(relative_attention_num_buckets=64), "relative_attention_num_buckets"),
    (dict(hidden_size=384, num_attention_heads=12), "64-wide"),
    (dict(hidden_size=768, num_attention_heads=8), "64-wide"),
    (dict(max_position_embeddings=2), "max_position_embeddings=2"),
])
def test_spec_refuses_mpnet(kw, match):
    from transformers import MPNetConfig

    from openmatch_b200.encoder import spec_from_hf_config
    base = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, max_position_embeddings=514)
    with pytest.raises(ValueError, match=match):
        spec_from_hf_config(MPNetConfig(**dict(base, **kw)))


@pytest.mark.parametrize("kw,match", [
    (dict(activation="relu"), "activation"),
    (dict(dim=768, n_heads=8), "32- or 64-wide"),
    (dict(dim=768, n_heads=48), "32- or 64-wide"),
])
def test_spec_refuses_distilbert(kw, match):
    from transformers import DistilBertConfig

    from openmatch_b200.encoder import spec_from_hf_config
    with pytest.raises(ValueError, match=match):
        spec_from_hf_config(DistilBertConfig(**dict(dict(dim=768, n_heads=12), **kw)))


def test_unknown_model_type_names_the_supported_backbones():
    from transformers import ElectraConfig

    from openmatch_b200.encoder import spec_from_hf_config
    with pytest.raises(ValueError, match="MPNet, DistilBERT"):
        spec_from_hf_config(ElectraConfig())


@pytest.mark.parametrize("arch", ARCHS)
def test_offline_tokenizers_special_tokens_and_pad_id(tmp_path, arch):
    from openmatch_b200.retriever.reranker import special_tokens
    tok = mo.offline_bert_vocab_tokenizer(str(tmp_path), arch)
    if arch == "mpnet":
        assert tok.pad_token_id == 1 and special_tokens(tok) == ([0], [2])
    else:
        assert tok.pad_token_id == 0 and special_tokens(tok) == ([2], [3])
