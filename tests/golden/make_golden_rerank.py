"""Generates tests/golden/rerank_small.npz by executing the REFERENCE's own Python code in the build container:

    PYTHONPATH=/root/reference/src python tests/golden/make_golden_rerank.py

Cross-encoder re-ranking of a TREC run over TSV queries and passages.  What is executed unmodified from the reference:
  * openmatch.modeling.RRModel.encode (reranking_model.py:106-125): BERT, 'first' pooling, LinearHead(128, 1)
  * openmatch.modeling.linear.LinearHead (linear.py)
  * openmatch.utils.fill_template / find_all_markers (the query / doc templates)
The reference's pair builder ``encode_pair`` (retriever/reranker.py:23-29) calls ``tokenizer.encode_plus`` on id lists,
which transformers 5 no longer has; it is restated below (``encode_pair``) and pinned by a hand-checked case.  Query
and passage contents are what its ``InferenceDataset(final=False)`` gives: the text through the template, tokenised
without special tokens, truncated to q_max_len / p_max_len.

The model is a seeded random tiny BERT (hidden 128, 2 layers, 2 heads, max_position_embeddings 256) with a local-vocab
BertTokenizer (no download).  As in make_golden_hd32.py, every parameter is put on a 7-level grid per tensor (int8 code
times one fp32 scale) and the reference runs on exactly those values, so the fixture stays small; it stores the codes
("q.<name>") and scales ("s.<name>"), the vocabulary, the TSV lines, the run, the padded pair input_ids /
attention_mask and the reference's fp32 scores.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = 3
Q_MAX, P_MAX = 16, 64
WORDS = ["the", "a", "of", "river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky", "rain",
         "city", "road", "car", "train", "music", "piano", "guitar", "stone", "bread", "cheese", "wine", "house",
         "garden", "winter", "summer", "light"]
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS


def encode_pair(tokenizer, item1, item2, max_len_1=32, max_len_2=128):
    """The reference's encode_pair: encode_plus(item1 + item2, truncation='longest_first', padding='max_length',
    max_length=max_len_1 + max_len_2 + 2) for a single sequence of ids, i.e. [CLS] item1 item2 [SEP] (the tokenizer's
    single-sequence special tokens), token types 0, right-padded with the pad id.  Truncation never fires here."""
    L = max_len_1 + max_len_2 + 2
    ids = [tokenizer.cls_token_id] + list(item1) + list(item2) + [tokenizer.sep_token_id]
    assert len(ids) <= L
    n = len(ids)
    return {"input_ids": ids + [tokenizer.pad_token_id] * (L - n), "attention_mask": [1] * n + [0] * (L - n),
            "token_type_ids": [0] * L}


def dequantize(z):
    return {k[2:]: z[k].astype(np.float32) * z["s." + k[2:]] for k in z.keys() if k.startswith("q.")}


def main():
    REF_SRC = "/root/reference/src"
    if not os.path.isdir(REF_SRC):
        sys.exit("reference tree not available; golden vectors can only be regenerated in the build container")
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF_SRC)
    import tempfile

    import torch

    import make_golden  # noqa: F401  (installs the faiss shim the reference's package imports need)
    from transformers import BertConfig, BertModel, BertTokenizer

    from openmatch.arguments import ModelArguments
    from openmatch.modeling import RRModel
    from openmatch.modeling.linear import LinearHead
    from openmatch.utils import fill_template, find_all_markers

    tmp = tempfile.mkdtemp()
    with open(os.path.join(tmp, "vocab.txt"), "w") as f:
        f.write("\n".join(VOCAB))
    tok = BertTokenizer(os.path.join(tmp, "vocab.txt"), do_lower_case=True)

    # the restated encode_pair, checked by hand: [CLS]=2 river=8 bank=9 | money=10 [SEP]=3, padded to 3 + 4 + 2
    v = {w: i for i, w in enumerate(VOCAB)}
    assert (v["river"], v["bank"], v["money"]) == (8, 9, 10)
    q = tok("river bank", add_special_tokens=False)["input_ids"]
    d = tok("money", add_special_tokens=False)["input_ids"]
    assert encode_pair(tok, q, d, 3, 4) == {"input_ids": [2, 8, 9, 10, 3, 0, 0, 0, 0],
                                            "attention_mask": [1] * 5 + [0] * 4, "token_type_ids": [0] * 9}
    assert tok("river bank money")["input_ids"] == [2, 8, 9, 10, 3]  # the tokenizer's own single-sequence template

    torch.manual_seed(77)
    gen = torch.Generator().manual_seed(7777)
    cfg = BertConfig(vocab_size=len(VOCAB), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                     intermediate_size=256, max_position_embeddings=256)
    bert = BertModel(cfg).eval()
    head = LinearHead(128, 1)
    arrays = {}
    with torch.no_grad():
        named = [(n, p) for n, p in bert.named_parameters() if not n.startswith("pooler.")]
        named.append(("head.linear.weight", head.linear.weight))
        for name, p in named:
            w = p.detach().numpy().astype(np.float32)
            if name.endswith("LayerNorm.weight"):
                w = w + 0.1 * torch.randn(w.shape, generator=gen).numpy()
            elif name.endswith(".bias"):
                w = 0.02 * torch.randn(w.shape, generator=gen).numpy()
            scale = np.float32(max(float(np.abs(w).max()), 1e-6) / LEVELS)
            arrays["q." + name] = np.clip(np.round(w / scale), -LEVELS, LEVELS).astype(np.int8)
            arrays["s." + name] = scale
            p.copy_(torch.from_numpy(arrays["q." + name].astype(np.float32) * scale))

    rng = np.random.default_rng(7)

    def sent(n):
        return " ".join(rng.choice(WORDS, n))

    # queries up to 20 words (q_max_len 16 truncates some), passages up to 90 (p_max_len 64 truncates some)
    queries = ["q%d\t%s" % (i, sent(int(n))) for i, n in enumerate([3, 20, 7, 12])]
    corpus = ["d%d\t%s\t%s" % (i, sent(2), sent(int(n))) for i, n in enumerate([5, 88, 30, 61, 12, 1, 40, 70, 9])]
    q_template, d_template = "<text>", "<title> <text>"

    def content(line, cols, template, max_len):
        rec = dict(zip(cols, line.split("\t")))
        text = fill_template(template, rec, find_all_markers(template), allow_not_found=True)
        return rec["id"], tok(text, add_special_tokens=False, truncation=True, max_length=max_len)["input_ids"]

    qtok = dict(content(x, ["id", "text"], q_template, Q_MAX) for x in queries)
    dtok = dict(content(x, ["id", "title", "text"], d_template, P_MAX) for x in corpus)
    run = []  # (qid, did, score): 6 documents per query, in a retrieval-like order
    for qi in range(len(queries)):
        docs = rng.choice(len(corpus), 6, replace=False)
        run += [("q%d" % qi, "d%d" % d, float(10 - r)) for r, d in enumerate(docs)]
    pairs = [encode_pair(tok, qtok[q], dtok[d], Q_MAX, P_MAX) for q, d, _ in run]
    items = {k: torch.tensor([p[k] for p in pairs]) for k in ("input_ids", "attention_mask", "token_type_ids")}
    margs = ModelArguments(model_name_or_path="unused", pooling="first")
    model = RRModel(lm=bert, head=head, pooling="first", tokenizer=tok, model_args=margs).eval()
    with torch.no_grad():
        scores = model.encode(items)
    assert scores.shape == (len(run), 1)
    path = os.path.join(HERE, "rerank_small.npz")
    np.savez_compressed(path, vocab=np.array(VOCAB), queries=np.array(queries), corpus=np.array(corpus),
                        run_qid=np.array([r[0] for r in run]), run_did=np.array([r[1] for r in run]),
                        run_score=np.array([r[2] for r in run], np.float32), q_max_len=Q_MAX, p_max_len=P_MAX,
                        input_ids=items["input_ids"].numpy().astype(np.int16),
                        attention_mask=items["attention_mask"].numpy().astype(np.int8),
                        scores=scores[:, 0].numpy().astype(np.float32), **arrays)
    print("golden vectors written to", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
