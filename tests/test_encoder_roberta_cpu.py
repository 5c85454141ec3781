"""CPU: RoBERTa / XLM-RoBERTa in the oracle, in the Python front end of the CUDA encoder and in the pretokenised stores.

The oracle with RoBERTa's position ids (tests/roberta_oracle.py) must reproduce the reference's own encoding of two
RoBERTa models (tests/golden/roberta_small.npz, made by tests/golden/make_golden_roberta.py) before the GPU tests may
judge the kernels by it.  ``spec_from_hf_config`` accepts RoBERTa and XLM-RoBERTa configs and refuses what the encoder
cannot compute; the pretokenised stores pad and mask with the tokenizer's pad id (1 for RoBERTa, 0 for BERT, as before).
"""
import os

import numpy as np
import pytest
import torch

import roberta_oracle as ro
from oracle.encoder import EncoderSpec

GOLDEN_HEADS = {"a": 2, "b": 4}  # hidden 128: 2 x 64-wide or 4 x 32-wide heads


def golden_spec(cfg, **kw):
    """the library spec of golden config ``cfg`` (``kw`` overrides)"""
    return dict(dict(arch="roberta", layers=2, hidden=128, heads=GOLDEN_HEADS[cfg], ffn=64, vocab=128, max_pos=66,
                     type_vocab=1, ln_eps=1e-12), **kw)


def load_golden(golden_dir, cfg):
    """(fixture, state dict, head weight, input_ids, attention_mask) of config ``cfg``: int8 codes times one fp32 scale
    per tensor, exactly the values the reference ran on"""
    z = np.load(os.path.join(golden_dir, "roberta_small.npz"))
    pre = "q.%s." % cfg
    sd = {k[len(pre):]: torch.from_numpy(z[k].astype(np.float32) * z["s.%s.%s" % (cfg, k[len(pre):])])
          for k in z.files if k.startswith(pre)}
    head = sd.pop("head.linear.weight")
    ids, mask = (torch.from_numpy(z[k].astype(np.int64)) for k in ("input_ids", "attention_mask"))
    return z, sd, head, ids, mask


def test_position_ids_are_hf_roberta_position_ids():
    from transformers.models.roberta.modeling_roberta import RobertaEmbeddings
    ids = torch.tensor([[0, 5, 1, 7, 2, 1, 1]])
    assert ro.position_ids(ids).tolist() == [[2, 3, 1, 4, 5, 1, 1]]
    ids = torch.randint(0, 4, (6, 70), generator=torch.Generator().manual_seed(0))
    assert torch.equal(ro.position_ids(ids), RobertaEmbeddings.create_position_ids_from_input_ids(ids, 1))


@pytest.mark.parametrize("cfg", ["a", "b"])
def test_oracle_reproduces_the_reference_golden(golden_dir, cfg):
    z, sd, head, ids, mask = load_golden(golden_dir, cfg)
    m = mask.bool()
    # the fixture's cases: a 64-token row reaching position row 65, a pad id inside attended content, right padding
    pos = ro.position_ids(ids)
    assert int(pos.max()) == 65 and bool(((ids == 1) & m).any()) and bool((ids[~m] == 1).all())
    spec_first = EncoderSpec("bert", 2, 128, GOLDEN_HEADS[cfg], 64, 1e-12, pooling="first")
    spec_mean = EncoderSpec("bert", 2, 128, GOLDEN_HEADS[cfg], 64, 1e-12, pooling="mean", normalize=True)
    hidden, reps = ro.encode_reps(sd, spec_first, ids, mask, head, dtype=torch.float64)
    assert np.abs(reps.numpy() - z[cfg + ".reps_first_head"]).max() <= 1e-5
    assert np.abs(hidden[m].numpy() - z[cfg + ".hidden_attended"]).max() <= 1e-4
    _, reps = ro.encode_reps(sd, spec_mean, ids, mask, dtype=torch.float64)
    assert np.abs(reps.numpy() - z[cfg + ".reps_mean_norm"]).max() <= 1e-5
    # the fixture tells RoBERTa's positions from BERT-style ones, by more than the kernels' 1e-2 rel-L2 bound: positions
    # 0, 1, ... (no offset) miss every row, and positions 2, 3, ... (the id-1 token counted) miss the row holding it
    import oracle
    want = z[cfg + ".reps_mean_norm"]
    for offset, rows in ((0, slice(None)), (2, slice(2, 3))):
        sd_bert = dict(sd, **{ro.POS_KEY: sd[ro.POS_KEY][offset:]})
        _, reps_b = oracle.encode_reps(sd_bert, spec_mean, ids, mask, dtype=torch.float64)
        err = np.linalg.norm(reps_b.numpy()[rows] - want[rows], axis=-1)
        assert (err > 2e-2 * np.linalg.norm(want[rows], axis=-1)).all(), (offset, err)


@pytest.mark.parametrize("kind", ["roberta", "xlm-roberta"])
@pytest.mark.parametrize("hidden,heads", [(768, 12), (384, 12), (1024, 16)])
def test_spec_accepts_roberta_and_xlm_roberta(kind, hidden, heads):
    from transformers import RobertaConfig, XLMRobertaConfig

    from openmatch_b200.encoder import spec_from_hf_config
    cls = RobertaConfig if kind == "roberta" else XLMRobertaConfig
    cfg = cls(hidden_size=hidden, num_attention_heads=heads, intermediate_size=4 * hidden, max_position_embeddings=514,
              type_vocab_size=1, pad_token_id=1, vocab_size=250002 if kind == "xlm-roberta" else 50265)
    spec = spec_from_hf_config(cfg)
    assert spec["arch"] == "roberta"
    assert (spec["hidden"], spec["heads"], spec["max_pos"], spec["type_vocab"]) == (hidden, heads, 514, 1)
    assert spec["vocab"] == cfg.vocab_size and spec["ln_eps"] == cfg.layer_norm_eps


@pytest.mark.parametrize("override,match", [
    (dict(pad_token_id=0), "pad_token_id"),
    (dict(position_embedding_type="relative_key"), "absolute"),
    (dict(hidden_act="gelu_new"), "gelu"),
    (dict(hidden_size=256, num_attention_heads=16), "32- or 64-wide"),
    (dict(max_position_embeddings=2), "max_position_embeddings"),
])
def test_spec_refuses_what_the_encoder_cannot_compute(override, match):
    from transformers import RobertaConfig

    from openmatch_b200.encoder import spec_from_hf_config
    base = dict(hidden_size=128, num_attention_heads=2, intermediate_size=256, max_position_embeddings=66,
                type_vocab_size=1, pad_token_id=1)
    with pytest.raises(ValueError, match=match):
        spec_from_hf_config(RobertaConfig(**dict(base, **override)))


def test_cuda_encoder_refuses_other_head_widths_before_the_library():
    from openmatch_b200.encoder import CudaEncoder
    with pytest.raises(ValueError, match="32- or 64-wide"):
        CudaEncoder(golden_spec("a", hidden=256, heads=16), {})


def test_max_pair_len_leaves_out_the_position_offset():
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel

    from openmatch_b200.modeling import RRModel
    from openmatch_b200.modeling.linear import LinearHead
    small = dict(hidden_size=128, num_attention_heads=2, intermediate_size=128, num_hidden_layers=1, vocab_size=64)
    rr = RRModel(RobertaModel(RobertaConfig(max_position_embeddings=66, **small)), LinearHead(128, 1))
    assert rr.max_pair_len() == 64
    rr = RRModel(RobertaModel(RobertaConfig(max_position_embeddings=514, **small)), LinearHead(128, 1))
    assert rr.max_pair_len() == 512
    rr = RRModel(BertModel(BertConfig(max_position_embeddings=64, **small)), LinearHead(128, 1))
    assert rr.max_pair_len() == 64


def _store(tmp_path, tok, texts, width):
    """a padded int32 store of ``tok(text)`` rows (with special tokens), padded with the tokenizer's pad id"""
    rows = [tok(t)["input_ids"] for t in texts]
    arr = np.full((len(rows), width), tok.pad_token_id, np.int32)
    for i, r in enumerate(rows):
        arr[i, :len(r)] = r
    path = str(tmp_path / "store.npy")
    np.save(path, arr)
    return path, rows


def _dataset(tok, path, max_len):
    from openmatch_b200.arguments import DataArguments
    from openmatch_b200.dataset import InferenceDataset
    return InferenceDataset.load(tok, DataArguments(corpus_path=path, p_max_len=max_len), is_query=False, final=False)


@pytest.mark.parametrize("family", ["roberta", "bert"])
def test_padded_store_masks_the_tokenizers_pad_id(tmp_path, family):
    from transformers import BertTokenizer

    from openmatch_b200.retriever.reranker import _content, special_tokens, token_store
    if family == "roberta":
        tok = ro.offline_tokenizer(str(tmp_path))
        prefix, suffix, pad = [0], [2], 1
    else:
        (tmp_path / "vocab.txt").write_text("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + list("abcdehlorw")))
        tok = BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)
        prefix, suffix, pad = [2], [3], 0
    assert special_tokens(tok) == (prefix, suffix) and tok.pad_token_id == pad
    path, rows = _store(tmp_path, tok, ["hello", "a", "world hello"], 14)
    ds = _dataset(tok, path, 16)  # wider than the store: padded to 16 with the pad id
    assert ds.pad_id == pad
    ex = [ds.process_one(r) for r in ds._records()]
    for e, r in zip(ex, rows):
        assert e["input_ids"] == r + [pad] * (16 - len(r))
        assert e["attention_mask"] == [1] * len(r) + [0] * (16 - len(r))  # the prefix (<s> = 0 for RoBERTa) is kept
    names, block = next(iter(ds.iter_batches()))
    assert block.shape == (1, 16) and block[0].tolist() == ex[0]["input_ids"]
    # pair content: padding dropped, [prefix] ... [suffix] stripped
    store, where = token_store(ds, ["0", "2"], prefix, suffix)
    assert store[where["0"][0]:sum(where["0"])].tolist() == rows[0][1:-1]
    assert store[where["2"][0]:sum(where["2"])].tolist() == rows[2][1:-1]
    row = np.array(rows[1] + [pad] * 4, np.int32)
    assert _content(row, prefix, suffix, 16, pad).tolist() == rows[1][1:-1]


def test_pretokenized_store_without_tokenizer_pads_with_zero(tmp_path):
    path = str(tmp_path / "s.npy")
    np.save(path, np.array([[5, 6, 0, 0]], np.int32))
    ds = _dataset(None, path, 6)
    assert ds.pad_id == 0
    ex = ds.process_one(next(iter(ds._records())))
    assert ex["input_ids"] == [5, 6, 0, 0, 0, 0] and ex["attention_mask"] == [1, 1, 0, 0, 0, 0]


def test_ragged_store_drops_the_given_pad_id(tmp_path):
    from openmatch_b200.dataset.inference_dataset import write_ragged_store
    p = write_ragged_store(str(tmp_path / "r"), np.array([[0, 5, 2, 1, 1], [0, 1, 7, 2, 1]]), pad_id=1)
    assert np.load(p).tolist() == [0, 5, 2, 0, 7, 2]
    assert np.load(str(tmp_path / "r.offsets.npy")).tolist() == [0, 3, 6]
