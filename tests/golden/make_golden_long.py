"""Generates tests/golden/long_small.npz by executing the REFERENCE's own Python code in the build container:

    PYTHONPATH=/root/reference/src python tests/golden/make_golden_long.py

Three randomly initialised 2-layer encoders of hidden 128 whose sequences go beyond 512 tokens: RoBERTa with
max_position_embeddings 1090 as 2 heads x 64 (config "ra") and as 4 heads x 32 (config "rb"), and BERT with 1024 positions
and 2 heads x 64 (config "ba").  Each is encoded by the reference's unmodified
openmatch.modeling.DRModelForInference.encode_passage (dense_retrieval_model.py:133-161,261-282) twice: first-token
pooling with a LinearHead(128, 64), and mean pooling with normalisation.  The batch holds rows of 513, 640, 1000, 1025
and 1088 tokens (BERT: 513, 640, 1000 and 1024), right-padded (RoBERTa with id 1, BERT with id 0); one RoBERTa row has
id 1 inside its content.

As in make_golden_roberta.py, every parameter is first replaced by a coarse grid value, code * scale with an int8 code
in [-3, 3] and one fp32 scale per tensor, and the reference runs on exactly those values; the query weights are scaled
60x so attention rows are peaked.  The file stores config c's codes as "q.<c>.<name>", scales as "s.<c>.<name>", the
inputs as "<c>.input_ids" / "<c>.attention_mask", the representations ("<c>.reps_first_head", "<c>.reps_mean_norm")
and, to stay small, the last hidden state at the rows "<c>.sample_rows" of the attended tokens ("<c>.hidden_sample":
the first two and the last two tokens of each row and every 128th position).  Writes that one file only.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = 3
# config -> (model type, heads, max_position_embeddings, row lengths)
CONFIGS = {"ra": ("roberta", 2, 1090, (513, 640, 1000, 1025, 1088)),
           "rb": ("roberta", 4, 1090, (513, 640, 1000, 1025, 1088)),
           "ba": ("bert", 2, 1024, (513, 640, 1000, 1024))}


def sample_rows(lens):
    """indices into the attended rows (row-major over the batch) of the hidden states the fixture keeps"""
    out, off = [], 0
    for n in lens:
        pos = sorted(set([0, 1, n - 2, n - 1] + list(range(127, n, 128))))
        out += [off + p for p in pos]
        off += n
    return np.array(out, dtype=np.int64)


def synth_rows(gen, kind, lens, vocab):
    """int64 [B, max(lens)] right-padded ids and the attention mask; RoBERTa rows are <s> content </s>"""
    import torch
    L, pad = max(lens), 1 if kind == "roberta" else 0
    ids = torch.randint(5, vocab, (len(lens), L), generator=gen)
    mask = torch.zeros(len(lens), L, dtype=torch.long)
    for b, n in enumerate(lens):
        if kind == "roberta":
            ids[b, 0], ids[b, n - 1] = 0, 2
        ids[b, n:] = pad
        mask[b, :n] = 1
    if kind == "roberta":
        ids[2, 300] = 1  # a pad id inside attended content
    return ids, mask


def main():
    REF_SRC = "/root/reference/src"
    if not os.path.isdir(REF_SRC):
        sys.exit("reference tree not available; golden vectors can only be regenerated in the build container")
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF_SRC)
    import torch

    import make_golden  # noqa: F401  installs the faiss shim the reference imports need
    from make_golden_roberta import dequantize
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel

    from openmatch.arguments import ModelArguments
    from openmatch.modeling import DRModelForInference
    from openmatch.modeling.linear import LinearHead

    torch.manual_seed(1090)
    gen = torch.Generator().manual_seed(10900)
    arrays = {}
    for cfg_name, (kind, heads, max_pos, lens) in CONFIGS.items():
        kw = dict(vocab_size=128, hidden_size=128, num_hidden_layers=2, num_attention_heads=heads,
                  intermediate_size=64, max_position_embeddings=max_pos)
        if kind == "roberta":
            model = RobertaModel(RobertaConfig(type_vocab_size=1, pad_token_id=1, bos_token_id=0, eos_token_id=2,
                                               **kw)).eval()
        else:
            model = BertModel(BertConfig(**kw)).eval()
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
                if name.endswith("attention.self.query.weight"):  # peaked attention rows
                    w = 60.0 * w
                scale = np.float32(max(float(np.abs(w).max()), 1e-6) / LEVELS)
                arrays["q.%s.%s" % (cfg_name, name)] = np.clip(np.round(w / scale), -LEVELS, LEVELS).astype(np.int8)
                arrays["s.%s.%s" % (cfg_name, name)] = scale
            for name, w in dequantize(arrays, cfg_name).items():
                params[name].copy_(torch.from_numpy(w))
        ids, mask = synth_rows(gen, kind, lens, 128)
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
        rows = sample_rows(lens)
        arrays[cfg_name + ".input_ids"] = ids.numpy().astype(np.int16)
        arrays[cfg_name + ".attention_mask"] = mask.numpy().astype(np.int8)
        arrays[cfg_name + ".sample_rows"] = rows
        arrays[cfg_name + ".hidden_sample"] = hidden.numpy()[mask.numpy().astype(bool)][rows]
        arrays[cfg_name + ".reps_first_head"] = reps_first.numpy()
        arrays[cfg_name + ".reps_mean_norm"] = reps_mean.numpy()
    path = os.path.join(HERE, "long_small.npz")
    np.savez_compressed(path, **arrays)
    print("golden vectors written to", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
