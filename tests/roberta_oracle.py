"""RoBERTa on top of the BERT oracle (oracle/encoder.py), shared by the RoBERTa tests and the probe.

RoBERTa is BERT's encoder with position ids computed from the token ids (HF ``create_position_ids_from_input_ids``,
padding_idx = pad_token_id = 1).  ``bert_encode`` reads ``position_embeddings[arange(L)]``; handing it, row by row, the
table ``position_embeddings[position_ids[b]]`` gives exactly RoBERTa's embedding sum, and every later step is per row,
so ``encode_reps`` below is the oracle's arithmetic unchanged.  ``offline_tokenizer`` builds a byte-level
``RobertaTokenizer`` without a download.
"""
import json

import torch

import oracle

PAD = 1
POS_KEY = "embeddings.position_embeddings.weight"


def position_ids(input_ids: torch.Tensor, pad: int = PAD) -> torch.Tensor:
    """``pad + cumsum(ids != pad) * (ids != pad)`` per row: HF's RoBERTa position ids"""
    m = (input_ids != pad).long()
    return torch.cumsum(m, dim=1) * m + pad


def encode_reps(sd, spec, input_ids, attention_mask, head_weight=None, dtype=torch.float32, emulate_bf16=False):
    """(hidden [B, L, H], reps) of a RoBERTa model with state dict ``sd`` (BERT names, ``spec.arch == 'bert'``)"""
    pos = position_ids(input_ids)
    # only the word rows the batch uses (a 250k-row table is not converted to float64 once per row)
    used, ids = torch.unique(input_ids, return_inverse=True)
    sd = dict(sd, **{"embeddings.word_embeddings.weight": sd["embeddings.word_embeddings.weight"][used]})
    hidden, reps = [], []
    for b in range(input_ids.shape[0]):
        sd_b = dict(sd)
        sd_b[POS_KEY] = sd[POS_KEY][pos[b]]
        h, r = oracle.encode_reps(sd_b, spec, ids[b:b + 1], attention_mask[b:b + 1], None, head_weight, dtype,
                                  emulate_bf16)
        hidden.append(h)
        reps.append(r)
    return torch.cat(hidden), torch.cat(reps)


def _bytes_to_unicode():
    """GPT-2's byte-level alphabet: 256 printable characters, one per byte"""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return [chr(c) for c in cs]


def offline_tokenizer(directory):
    """A ``RobertaTokenizer`` over ``<s> <pad> </s> <unk>``, the 256 byte-level characters and ``<mask>``, with no
    merges: pad 1, prefix [0], suffix [2]; every character is one token."""
    from transformers import RobertaTokenizer
    vocab = ["<s>", "<pad>", "</s>", "<unk>"] + _bytes_to_unicode() + ["<mask>"]
    with open(f"{directory}/vocab.json", "w") as f:
        json.dump({t: i for i, t in enumerate(vocab)}, f)
    with open(f"{directory}/merges.txt", "w") as f:
        f.write("#version: 0.2\n")
    return RobertaTokenizer(f"{directory}/vocab.json", f"{directory}/merges.txt")
