"""Generates tests/golden/mpnet_small.npz by executing the REFERENCE's own Python code in the build container:

    PYTHONPATH=/root/reference/src python tests/golden/make_golden_mpnet.py

Two randomly initialised 2-layer encoders of hidden 128 (2 heads x 64, FFN 64): an MPNet (config "mpnet",
max_position_embeddings 260, pad_token_id 1) and a DistilBERT (config "distilbert", max_position_embeddings 66), each
encoded by the reference's unmodified openmatch.modeling.DRModelForInference.encode_passage
(dense_retrieval_model.py:133-161,261-282) twice: first-token pooling with a LinearHead(128, 64), and mean pooling with
normalisation.

MPNet's batch holds four rows right-padded with id 1: one of 200 tokens (key distances beyond 128, where the bias
buckets saturate; its last token takes position row 201), one with id 1 inside its attended content (position 1, the
count does not advance), and two shorter ones.  DistilBERT's batch holds four rows of at most 64 tokens right-padded
with id 0 (its last position row is 63).

As in make_golden_roberta.py, every parameter is first replaced by a coarse grid value, code * scale with an int8 code
in [-3, 3] and one fp32 scale per tensor, and the reference runs on exactly those values; the query weights are scaled
60x so attention rows are peaked, and MPNet's relative_attention_bias is scaled so that its 7 levels span +-6 nats,
enough to move the arg-max key of attention rows.  The file stores config c's codes as "q.<c>.<name>" and scales as
"s.<c>.<name>" (the LinearHead as "<c>.head.linear.weight"), each config's inputs ("<c>.input_ids",
"<c>.attention_mask"), the attended rows of the last hidden state ("<c>.hidden_attended") and the representations
("<c>.reps_first_head", "<c>.reps_mean_norm").  The pooler, which OpenMatch never reads, is not stored.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = 3
REL_SPAN = 6.0  # nats: the largest |relative bias| after quantisation


def synth_rows(gen, vocab, lens, L, pad, first, last):
    """int64 [len(lens), L] ids right-padded with ``pad``, ``first`` / ``last`` around content ids >= 4, and the mask"""
    import torch
    ids = torch.randint(4, vocab, (len(lens), L), generator=gen)
    mask = torch.zeros(len(lens), L, dtype=torch.long)
    for b, n in enumerate(lens):
        ids[b, 0], ids[b, n - 1] = first, last
        ids[b, n:] = pad
        mask[b, :n] = 1
    return ids, mask


def main():
    REF_SRC = "/root/reference/src"
    if not os.path.isdir(REF_SRC):
        sys.exit("reference tree not available; golden vectors can only be regenerated in the build container")
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF_SRC)
    import torch

    import make_golden  # noqa: F401  installs the faiss shim the reference imports need
    from transformers import DistilBertConfig, DistilBertModel, MPNetConfig, MPNetModel

    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    from openmatch.modeling.linear import LinearHead

    torch.manual_seed(77)
    gen = torch.Generator().manual_seed(7777)
    arrays = {}
    for cfg_name in ("mpnet", "distilbert"):
        if cfg_name == "mpnet":
            cfg = MPNetConfig(vocab_size=128, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                              intermediate_size=64, max_position_embeddings=260, pad_token_id=1, bos_token_id=0,
                              eos_token_id=2)
            model = MPNetModel(cfg).eval()
            ids, mask = synth_rows(gen, 128, (200, 20, 40, 5), 200, pad=1, first=0, last=2)
            ids[2, 7] = 1  # a pad id inside attended content
            query_suffix = "attention.attn.q.weight"
        else:
            cfg = DistilBertConfig(vocab_size=128, dim=128, n_layers=2, n_heads=2, hidden_dim=64,
                                   max_position_embeddings=66, pad_token_id=0)
            model = DistilBertModel(cfg).eval()
            ids, mask = synth_rows(gen, 128, (64, 20, 40, 5), 64, pad=0, first=2, last=3)
            query_suffix = "attention.q_lin.weight"
        head = LinearHead(128, 64)
        params = dict(model.named_parameters())
        params["head.linear.weight"] = head.linear.weight
        with torch.no_grad():
            for name, p in params.items():
                if name.startswith("pooler."):
                    continue
                w = p.detach().numpy().astype(np.float32)
                if name.endswith("LayerNorm.weight") or name.endswith("layer_norm.weight"):  # gains near 1, varied
                    w = w + 0.1 * torch.randn(w.shape, generator=gen).numpy()
                elif name.endswith(".bias"):  # HF initialises biases to zero: give them values to check
                    w = 0.02 * torch.randn(w.shape, generator=gen).numpy()
                if name.endswith(query_suffix):  # peaked attention rows: each head's own keys matter
                    w = 60.0 * w
                if name == "encoder.relative_attention_bias.weight":
                    w = torch.randn(w.shape, generator=gen).numpy()
                    w = w * (REL_SPAN / np.abs(w).max())
                scale = np.float32(max(float(np.abs(w).max()), 1e-6) / LEVELS)
                arrays["q.%s.%s" % (cfg_name, name)] = np.clip(np.round(w / scale), -LEVELS, LEVELS).astype(np.int8)
                arrays["s.%s.%s" % (cfg_name, name)] = scale
                params[name].copy_(torch.from_numpy(arrays["q.%s.%s" % (cfg_name, name)].astype(np.float32) * scale))
        items = {"input_ids": ids, "attention_mask": mask}
        with torch.no_grad():
            margs = ModelArguments(model_name_or_path="unused", pooling="first", normalize=False)
            dr = DRModelForInference(lm_q=model, lm_p=model, tied=True, pooling="first", normalize=False, head_q=head,
                                     head_p=head, model_args=margs)
            hidden, reps_first = dr.encode_passage(items)
            margs = ModelArguments(model_name_or_path="unused", pooling="mean", normalize=True)
            dr = DRModelForInference(lm_q=model, lm_p=model, tied=True, pooling="mean", normalize=True,
                                     model_args=margs)
            hidden2, reps_mean = dr.encode_passage(items)
        assert torch.equal(hidden, hidden2)
        m = mask.numpy().astype(bool)
        arrays[cfg_name + ".input_ids"] = ids.numpy().astype(np.int16)
        arrays[cfg_name + ".attention_mask"] = mask.numpy().astype(np.int8)
        arrays[cfg_name + ".hidden_attended"] = hidden.numpy()[m]
        arrays[cfg_name + ".reps_first_head"] = reps_first.numpy()
        arrays[cfg_name + ".reps_mean_norm"] = reps_mean.numpy()
    path = os.path.join(HERE, "mpnet_small.npz")
    np.savez_compressed(path, **arrays)
    print("golden vectors written to", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
