"""Generates tests/golden/roberta_small.npz by executing the REFERENCE's own Python code in the build container:

    PYTHONPATH=/root/reference/src python tests/golden/make_golden_roberta.py

Two randomly initialised 2-layer RoBERTa encoders (hidden 128 as 2 heads x 64 = config "a", and as 4 heads x 32 = config
"b"; max_position_embeddings 66, type_vocab_size 1, pad_token_id 1), each encoded by the reference's unmodified
openmatch.modeling.DRModelForInference.encode_passage (dense_retrieval_model.py:133-161,261-282) twice: first-token
pooling with a LinearHead(128, 64), and mean pooling with normalisation.  The batch holds four rows right-padded with id
1: one of exactly 64 tokens (its last token takes position row 65, the table's last), one with id 1 inside its
attended content (position 1, and the count does not advance), and two shorter ones.  Writes that one file only.

As in make_golden_hd32.py, every parameter is first replaced by a coarse grid value, code * scale with an int8 code in
[-3, 3] and one fp32 scale per tensor, and the reference runs on exactly those values; the query weights are scaled 60x
so attention rows are peaked.  The file stores config c's codes as "q.<c>.<name>" and scales as "s.<c>.<name>" (the
LinearHead as "<c>.head.linear.weight"), the inputs, the attended rows of the last hidden state ("<c>.hidden_attended")
and the representations ("<c>.reps_first_head", "<c>.reps_mean_norm").  The pooler, which OpenMatch never reads, is not
stored.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = 3
CONFIGS = {"a": 2, "b": 4}  # config -> attention heads of the 128-wide model (head width 64 / 32)


def dequantize(z, cfg):
    """{name: fp32 array} of config ``cfg`` from the codes and scales of a fixture written by this script"""
    pre = "q.%s." % cfg
    return {k[len(pre):]: z[k].astype(np.float32) * z["s.%s.%s" % (cfg, k[len(pre):])] for k in z.keys()
            if k.startswith(pre)}


def synth_rows(gen, vocab):
    """int64 [4, 64] ids right-padded with 1, <s> = 0 first and </s> = 2 last, and the attention mask"""
    import torch
    L, lens = 64, (64, 20, 40, 5)
    ids = torch.randint(3, vocab, (len(lens), L), generator=gen)
    mask = torch.zeros(len(lens), L, dtype=torch.long)
    for b, n in enumerate(lens):
        ids[b, 0], ids[b, n - 1] = 0, 2
        ids[b, n:] = 1
        mask[b, :n] = 1
    ids[2, 7] = 1  # a pad id inside attended content
    return ids, mask


def main():
    REF_SRC = "/root/reference/src"
    if not os.path.isdir(REF_SRC):
        sys.exit("reference tree not available; golden vectors can only be regenerated in the build container")
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF_SRC)
    import torch

    import make_golden  # noqa: F401  installs the faiss shim the reference imports need
    from transformers import RobertaConfig, RobertaModel

    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    from openmatch.modeling.linear import LinearHead

    torch.manual_seed(66)
    gen = torch.Generator().manual_seed(6666)
    arrays = {}
    ids, mask = None, None
    for cfg_name, heads in CONFIGS.items():
        cfg = RobertaConfig(vocab_size=128, hidden_size=128, num_hidden_layers=2, num_attention_heads=heads,
                            intermediate_size=64, max_position_embeddings=66, type_vocab_size=1, pad_token_id=1,
                            bos_token_id=0, eos_token_id=2)
        model = RobertaModel(cfg).eval()
        head = LinearHead(128, 64)
        params = dict(model.named_parameters())
        params["head.linear.weight"] = head.linear.weight
        with torch.no_grad():
            for name, p in params.items():
                if name.startswith("pooler."):
                    continue
                w = p.detach().numpy().astype(np.float32)
                if name.endswith("LayerNorm.weight"):  # keep LayerNorm gains near 1 and varied
                    w = w + 0.1 * torch.randn(w.shape, generator=gen).numpy()
                elif name.endswith(".bias"):  # HF initialises biases to zero: give them values to check
                    w = 0.02 * torch.randn(w.shape, generator=gen).numpy()
                if name.endswith("attention.self.query.weight"):  # peaked attention rows: each head's own keys matter
                    w = 60.0 * w
                scale = np.float32(max(float(np.abs(w).max()), 1e-6) / LEVELS)
                arrays["q.%s.%s" % (cfg_name, name)] = np.clip(np.round(w / scale), -LEVELS, LEVELS).astype(np.int8)
                arrays["s.%s.%s" % (cfg_name, name)] = scale
            for name, w in dequantize(arrays, cfg_name).items():
                params[name].copy_(torch.from_numpy(w))
        if ids is None:
            ids, mask = synth_rows(gen, cfg.vocab_size)
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
        arrays[cfg_name + ".hidden_attended"] = hidden.numpy()[m]
        arrays[cfg_name + ".reps_first_head"] = reps_first.numpy()
        arrays[cfg_name + ".reps_mean_norm"] = reps_mean.numpy()
    path = os.path.join(HERE, "roberta_small.npz")
    np.savez_compressed(path, input_ids=ids.numpy().astype(np.int16), attention_mask=mask.numpy().astype(np.int8),
                        **arrays)
    print("golden vectors written to", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
