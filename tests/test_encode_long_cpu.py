"""CPU: the length limit of the packed encoder calls beyond 512 tokens, as the Python front end computes it.

``encoder.max_seq_len`` mirrors the library's rule (8192 tokens and max_position_embeddings for BERT, minus RoBERTa's
position offset of 2; 512 for T5; never more than max_batch_tokens); ``RRModel.max_pair_len`` and the re-ranker's
refusal follow it."""
import types

import pytest
import torch


def _bert(**kw):
    return dict(dict(arch="bert", layers=1, hidden=128, heads=2, ffn=256, vocab=64, max_pos=512, type_vocab=2,
                     ln_eps=1e-12), **kw)


def test_max_seq_len_rule():
    from openmatch_b200.encoder import max_seq_len
    assert max_seq_len(_bert(max_pos=512)) == 512
    assert max_seq_len(_bert(max_pos=8192)) == 8192
    assert max_seq_len(_bert(max_pos=20000)) == 8192
    assert max_seq_len(_bert(max_pos=1000)) == 1000
    assert max_seq_len(_bert(arch="roberta", max_pos=8194)) == 8192  # bge-m3, bge-reranker-v2-m3
    assert max_seq_len(_bert(arch="roberta", max_pos=514)) == 512
    assert max_seq_len(_bert(arch="roberta", max_pos=1090)) == 1088
    t5 = dict(arch="t5", layers=1, hidden=128, heads=2, ffn=256, vocab=64, ln_eps=1e-6, rel_buckets=32,
              rel_max_distance=128)
    assert max_seq_len(t5) == 512
    assert max_seq_len(t5, max_batch_tokens=300) == 300
    # max_batch_tokens below the position limit bounds it
    assert max_seq_len(_bert(arch="roberta", max_pos=8194), max_batch_tokens=4096) == 4096
    assert max_seq_len(_bert(max_pos=8192), max_batch_tokens=8191) == 8191
    assert max_seq_len(_bert(max_pos=8192)) == 8192  # the default handle size (32768 tokens) holds 8192


def _small(**kw):
    return dict(dict(hidden_size=128, num_attention_heads=2, intermediate_size=128, num_hidden_layers=1, vocab_size=64),
                **kw)


def test_max_pair_len_of_an_xlm_roberta_8194_config(monkeypatch):
    from transformers import XLMRobertaConfig, XLMRobertaModel

    from openmatch_b200.modeling import RRModel
    from openmatch_b200.modeling.linear import LinearHead
    monkeypatch.delenv("OPENMATCH_B200_MAX_BATCH_TOKENS", raising=False)
    rr = RRModel(XLMRobertaModel(XLMRobertaConfig(max_position_embeddings=8194, pad_token_id=1, **_small())),
                 LinearHead(128, 1))
    assert rr.max_pair_len() == 8192
    monkeypatch.setenv("OPENMATCH_B200_MAX_BATCH_TOKENS", "6000")
    assert rr.max_pair_len() == 6000


def test_reranker_refuses_pairs_beyond_the_new_limit(golden_dir, tmp_path):
    from test_rerank_cpu import _data_args, _datasets, _fake_reranker, _fixture
    z, tok, run = _fixture(golden_dir, tmp_path)
    qds, cds = _datasets(tok, _data_args(tmp_path, z))
    qds.max_len, cds.max_len = 24, 8170  # 24 + 8170 + [CLS] + [SEP] = 8196 tokens
    with pytest.raises(ValueError, match="exceed"):
        _fake_reranker(tok, cds, limit=8192).rerank(qds, run)
    cds.max_len = 8166  # 8192 tokens: accepted
    assert len(_fake_reranker(tok, cds, limit=8192).rerank(qds, run)) == 4


# ------------------------------------------------------------------------------------------------------------------
# the reference's golden vectors beyond 512 tokens (tests/golden/long_small.npz, made by make_golden_long.py)
# ------------------------------------------------------------------------------------------------------------------
GOLDEN = {"ra": ("roberta", 2), "rb": ("roberta", 4), "ba": ("bert", 2)}  # config -> (arch, heads of the 128-wide model)


def load_long_golden(golden_dir, cfg):
    """(fixture, state dict, head weight, input_ids, attention_mask) of config ``cfg``: int8 codes times one fp32 scale
    per tensor, exactly the values the reference ran on"""
    import os

    import numpy as np
    z = np.load(os.path.join(golden_dir, "long_small.npz"))
    pre = "q.%s." % cfg
    sd = {k[len(pre):]: torch.from_numpy(z[k].astype(np.float32) * z["s.%s.%s" % (cfg, k[len(pre):])])
          for k in z.files if k.startswith(pre)}
    head = sd.pop("head.linear.weight")
    ids, mask = (torch.from_numpy(z["%s.%s" % (cfg, k)].astype(np.int64)) for k in ("input_ids", "attention_mask"))
    return z, sd, head, ids, mask


def long_golden_spec(cfg):
    arch, heads = GOLDEN[cfg]
    return dict(arch=arch, layers=2, hidden=128, heads=heads, ffn=64, vocab=128, max_pos=1090 if arch == "roberta" else 1024,
                type_vocab=1 if arch == "roberta" else 2, ln_eps=1e-12)


@pytest.mark.parametrize("cfg", list(GOLDEN))
def test_oracle_reproduces_the_long_golden(golden_dir, cfg):
    import numpy as np

    import oracle
    import roberta_oracle as ro
    from oracle.encoder import EncoderSpec
    z, sd, head, ids, mask = load_long_golden(golden_dir, cfg)
    arch, heads = GOLDEN[cfg]
    m = mask.bool()
    lens = m.sum(1)
    assert int(lens.min()) == 513 and int(lens.max()) == (1088 if arch == "roberta" else 1024)
    if arch == "roberta":
        assert bool(((ids == 1) & m).any())

    def encode(spec, hw):
        if arch == "roberta":
            return ro.encode_reps(sd, spec, ids, mask, hw, dtype=torch.float64)
        return oracle.encode_reps(sd, spec, ids, mask, None, hw, dtype=torch.float64)

    hidden, reps = encode(EncoderSpec("bert", 2, 128, heads, 64, 1e-12, pooling="first"), head)
    assert np.abs(reps.numpy() - z[cfg + ".reps_first_head"]).max() <= 1e-5
    assert np.abs(hidden[m].numpy()[z[cfg + ".sample_rows"]] - z[cfg + ".hidden_sample"]).max() <= 1e-4
    _, reps = encode(EncoderSpec("bert", 2, 128, heads, 64, 1e-12, pooling="mean", normalize=True), None)
    assert np.abs(reps.numpy() - z[cfg + ".reps_mean_norm"]).max() <= 1e-5
