"""Generates tests/golden/bert_hd32_small.npz by executing the REFERENCE's own Python code in the build container:

    PYTHONPATH=/root/reference/src python tests/golden/make_golden_hd32.py

A BERT encoder with 32-wide attention heads (hidden 128, 4 heads: the head width of all-MiniLM, bge-small, e5-small
and gte-small), randomly initialised, encoded by the reference's unmodified
openmatch.modeling.DRModelForInference.encode_passage (dense_retrieval_model.py:133-161,261-282) with mean pooling and
normalisation.  Writes that one file only; the other fixtures come from make_golden.py.

To keep the fixture small, every parameter is first replaced by a coarse grid value, code * scale with an int8 code in
[-3, 3] and one fp32 scale per tensor, and the reference runs on exactly those values.  The query weights are scaled
up 60x so that attention rows are peaked rather than nearly uniform: a head that attends with another head's keys or
values then changes the output visibly.  The file stores the codes
("q.<name>") and scales ("s.<name>"); ``dequantize`` rebuilds the fp32 tensors bit for bit (the tests do the same,
tests/test_encoder_hd32_cpu.py::load_golden).
The pooler, which OpenMatch never reads, is not stored.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = 3


def dequantize(z):
    """{name: fp32 array} from the codes and scales of a fixture written by this script"""
    return {k[2:]: z[k].astype(np.float32) * z["s." + k[2:]] for k in z.keys() if k.startswith("q.")}


def main():
    REF_SRC = "/root/reference/src"
    if not os.path.isdir(REF_SRC):
        sys.exit("reference tree not available; golden vectors can only be regenerated in the build container")
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF_SRC)
    import torch

    from make_golden import synth_ids  # installs the faiss shim the reference imports need
    from transformers import BertConfig, BertModel

    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference

    torch.manual_seed(32)
    gen = torch.Generator().manual_seed(3232)
    cfg = BertConfig(vocab_size=128, hidden_size=128, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=64, max_position_embeddings=64)
    bert = BertModel(cfg).eval()
    assert cfg.hidden_size // cfg.num_attention_heads == 32
    arrays = {}
    with torch.no_grad():
        for name, p in bert.named_parameters():
            w = p.detach().numpy().astype(np.float32)
            if name.startswith("pooler."):
                continue
            if name.endswith("LayerNorm.weight"):  # keep LayerNorm gains near 1 and varied
                w = w + 0.1 * torch.randn(w.shape, generator=gen).numpy()
            elif name.endswith(".bias"):  # HF initialises biases to zero: give them values to check
                w = 0.02 * torch.randn(w.shape, generator=gen).numpy()
            if name.endswith("attention.self.query.weight"):  # peaked attention rows: each head's own keys matter
                w = 60.0 * w
            scale = np.float32(max(float(np.abs(w).max()), 1e-6) / LEVELS)
            arrays["q." + name] = np.clip(np.round(w / scale), -LEVELS, LEVELS).astype(np.int8)
            arrays["s." + name] = scale
        params = dict(bert.named_parameters())
        for name, w in dequantize(arrays).items():
            params[name].copy_(torch.from_numpy(w))
    margs = ModelArguments(model_name_or_path="unused", pooling="mean", normalize=True)
    model = DRModelForInference(lm_q=bert, lm_p=bert, tied=True, pooling="mean", normalize=True, model_args=margs)
    ids, mask = synth_ids(gen, 4, 20, cfg.vocab_size, 101, 102, ragged=True)
    tt = torch.zeros_like(ids)
    tt[:, 10:] = 1
    with torch.no_grad():
        hidden, reps = model.encode_passage({"input_ids": ids, "attention_mask": mask, "token_type_ids": tt})
    m = mask.numpy().astype(bool)
    path = os.path.join(HERE, "bert_hd32_small.npz")
    np.savez_compressed(path, input_ids=ids.numpy().astype(np.int16), attention_mask=mask.numpy().astype(np.int8),
                        token_type_ids=tt.numpy().astype(np.int8), hidden_attended=hidden.numpy()[m],
                        reps=reps.numpy(), **arrays)
    print("golden vectors written to", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
