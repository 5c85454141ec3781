"""MPNet and DistilBERT restated for the float64 oracle (oracle/encoder.py), shared by their tests and the probe.

Restated from transformers 5.5:
  MPNet      : transformers/models/mpnet/modeling_mpnet.py  (embeddings :57-95 with padding_idx 1 hard-coded at :60
               and create_position_ids_from_input_ids :889-897; self-attention :136-186, scores / sqrt(d) + bias at
               :163-167; attention LayerNorm :210; intermediate / output :216-243; the bias is computed once per
               forward in MPNetEncoder :293 from arange(L) (compute_position_bias :324-340, 32 buckets, max distance
               128 by default) with T5's bidirectional relative_position_bucket :343-361)
  DistilBERT : transformers/models/distilbert/modeling_distilbert.py  (embeddings :83-122: word + position rows
               arange(L), LayerNorm eps 1e-12; eager attention :126-151 (q k^T * d^-0.5); q/k/v/out_lin :169-206;
               ffn lin1 / lin2 :210-228; sa_layer_norm / output_layer_norm, eps 1e-12 :240-262)
MPNet has BERT's post-LN layer with a shared relative position bias added after the 1/sqrt(d) scaling; its position ids
are RoBERTa's (tests/roberta_oracle.py).  DistilBERT is BERT's arithmetic under other names with no token-type
embeddings: ``distilbert_as_bert`` renames its state dict and adds one zero token-type row, which adds exactly zero.
Both take ``probe`` like ``oracle.encode_reps``: every layer's masked logits, bias included (natural-log units).
"""
import torch
import torch.nn.functional as F

import oracle
import roberta_oracle as ro
from oracle import encoder as oe

MPNET_BUCKETS, MPNET_MAX_DISTANCE = 32, 128
REL_KEY = "encoder.relative_attention_bias.weight"


def mpnet_bias(sd, L, dtype=torch.float64):
    """[heads, L, L] relative position bias of an L-token row: bucket of (key index - query index)"""
    pos = torch.arange(L)
    bucket = oracle.t5_relative_position_bucket(pos[None, :] - pos[:, None], MPNET_BUCKETS, MPNET_MAX_DISTANCE)
    return sd[REL_KEY].to(dtype)[bucket].permute(2, 0, 1)


def mpnet_encode(sd, spec, input_ids, attention_mask, nm, use_bias=True, positions="ids"):
    """``MPNetModel.forward`` -> last_hidden_state [B, L, H].  ``use_bias=False`` / ``positions="arange"`` are the
    negative controls the tests use (MPNet without its bias, BERT-style positions 0 .. L-1)."""
    B, L = input_ids.shape
    H, nh = spec.hidden, spec.heads
    dh = H // nh
    pos = ro.position_ids(input_ids) if positions == "ids" else torch.arange(L)[None].expand(B, L)
    emb = nm.t(sd["embeddings.word_embeddings.weight"])[input_ids] + nm.t(sd["embeddings.position_embeddings.weight"])[pos]
    h = F.layer_norm(emb, (H,), nm.t(sd["embeddings.LayerNorm.weight"]), nm.t(sd["embeddings.LayerNorm.bias"]),
                     spec.ln_eps)
    bias = mpnet_bias(sd, L, nm.dtype)[None] if use_bias else 0.0
    mask = oe._key_mask(attention_mask, nm.dtype)
    for i in range(spec.layers):
        p = f"encoder.layer.{i}."

        def lin(x, name):
            return nm.lin(x, sd[p + name + ".weight"], sd[p + name + ".bias"])

        def heads(x):
            return x.view(B, L, nh, dh).permute(0, 2, 1, 3)

        q, k, v = (heads(lin(h, "attention.attn." + n)) for n in ("q", "k", "v"))
        s = nm.mm(q, k.transpose(-1, -2)) * (dh ** -0.5) + bias + mask
        nm.look(i, s)
        ctx = nm.mm(oe._softmax_rows(s), v).permute(0, 2, 1, 3).reshape(B, L, H)
        h = F.layer_norm(lin(ctx, "attention.attn.o") + h, (H,), nm.t(sd[p + "attention.LayerNorm.weight"]),
                         nm.t(sd[p + "attention.LayerNorm.bias"]), spec.ln_eps)
        inter = F.gelu(lin(h, "intermediate.dense"))
        h = F.layer_norm(lin(inter, "output.dense") + h, (H,), nm.t(sd[p + "output.LayerNorm.weight"]),
                         nm.t(sd[p + "output.LayerNorm.bias"]), spec.ln_eps)
    return h


def mpnet_reps(sd, spec, input_ids, attention_mask, head_weight=None, dtype=torch.float32, emulate_bf16=False,
               probe=None, use_bias=True, positions="ids"):
    """(hidden, reps) of an MPNet model, as ``oracle.encode_reps`` returns them for BERT"""
    nm = oe._Num(dtype, emulate_bf16, probe)
    with torch.no_grad():
        hidden = mpnet_encode(sd, spec, input_ids, attention_mask, nm, use_bias, positions)
        reps = oe.pool_head_normalize(hidden, attention_mask, spec.pooling, head_weight, spec.normalize, nm)
    return hidden, reps


_DISTIL_LAYER = {"attention.q_lin": "attention.self.query", "attention.k_lin": "attention.self.key",
                 "attention.v_lin": "attention.self.value", "attention.out_lin": "attention.output.dense",
                 "sa_layer_norm": "attention.output.LayerNorm", "ffn.lin1": "intermediate.dense",
                 "ffn.lin2": "output.dense", "output_layer_norm": "output.LayerNorm"}


def distilbert_as_bert(sd):
    """A DistilBERT state dict under BERT's names, with one zero token-type row"""
    out = {}
    for k, v in sd.items():
        if k.startswith("transformer.layer."):
            i, rest = k[len("transformer.layer."):].split(".", 1)
            mod, leaf = rest.rsplit(".", 1)
            k = "encoder.layer.%s.%s.%s" % (i, _DISTIL_LAYER[mod], leaf)
        out[k] = v
    H = sd["embeddings.word_embeddings.weight"].shape[1]
    out["embeddings.token_type_embeddings.weight"] = torch.zeros(1, H, dtype=sd["embeddings.word_embeddings.weight"].dtype)
    return out


def distilbert_reps(sd, spec, input_ids, attention_mask, head_weight=None, dtype=torch.float32, emulate_bf16=False,
                    probe=None):
    """(hidden, reps) of a DistilBERT model (``spec.arch == 'bert'``, ``spec.ln_eps == 1e-12``)"""
    return oracle.encode_reps(distilbert_as_bert(sd), spec, input_ids, attention_mask, None, head_weight, dtype,
                              emulate_bf16, probe)


def encode_reps(arch, sd, spec, input_ids, attention_mask, head_weight=None, dtype=torch.float32, emulate_bf16=False,
                probe=None):
    """the oracle of ``arch`` ("mpnet" | "distilbert")"""
    f = mpnet_reps if arch == "mpnet" else distilbert_reps
    return f(sd, spec, input_ids, attention_mask, head_weight, dtype, emulate_bf16, probe)


def offline_bert_vocab_tokenizer(directory, arch):
    """An ``MPNetTokenizer`` (``<s>`` 0, ``<pad>`` 1, ``</s>`` 2, ``<unk>`` 3) or ``DistilBertTokenizer`` (``[PAD]`` 0,
    ``[UNK]`` 1, ``[CLS]`` 2, ``[SEP]`` 3) over a locally written WordPiece ``vocab.txt`` of lower-case letters, digits
    and a few words, with no download."""
    from transformers import DistilBertTokenizer, MPNetTokenizer
    words = ["the", "a", "of", "river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky",
             "rain", "city", "road", "car", "train", "music", "piano"]
    chars = list("abcdefghijklmnopqrstuvwxyz0123456789")
    if arch == "mpnet":
        special = ["<s>", "<pad>", "</s>", "<unk>"]
        tail = ["<mask>"]
    else:
        special = ["[PAD]", "[UNK]", "[CLS]", "[SEP]"]
        tail = ["[MASK]"]
    vocab = list(dict.fromkeys(special + words + chars + ["##" + c for c in chars] + tail))  # "a" is both
    path = f"{directory}/vocab.txt"
    with open(path, "w") as f:
        f.write("\n".join(vocab) + "\n")
    if arch == "mpnet":
        return MPNetTokenizer(path, do_lower_case=True)
    return DistilBertTokenizer(path, do_lower_case=True)
