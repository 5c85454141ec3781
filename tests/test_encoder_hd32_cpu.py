"""CPU: 32-wide attention heads in the oracle and in the Python front end of the CUDA encoder.

The float64 oracle must reproduce the reference's own encoding of a 32-wide-head BERT (tests/golden/bert_hd32_small.npz,
made by tests/golden/make_golden_hd32.py) before the GPU tests may judge the kernels by it; head widths other than 32 and
64 are refused with ValueError before the library is called."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle.encoder import EncoderSpec


GOLDEN_SPEC = dict(arch="bert", layers=2, hidden=128, heads=4, ffn=64, vocab=128, max_pos=64, type_vocab=2, ln_eps=1e-12)


def load_golden(golden_dir):
    """(fixture, state dict, input_ids, attention_mask, token_type_ids): the weights are int8 codes times one fp32 scale
    per tensor, exactly the values the reference ran on (tests/golden/make_golden_hd32.py)"""
    z = np.load(os.path.join(golden_dir, "bert_hd32_small.npz"))
    sd = {k[2:]: torch.from_numpy(z[k].astype(np.float32) * z["s." + k[2:]]) for k in z.files if k.startswith("q.")}
    ids, mask, tt = (torch.from_numpy(z[k].astype(np.int64)) for k in ("input_ids", "attention_mask", "token_type_ids"))
    return z, sd, ids, mask, tt


def test_oracle_reproduces_the_reference_golden(golden_dir):
    z, sd, ids, mask, tt = load_golden(golden_dir)
    assert sd["encoder.layer.0.attention.self.query.weight"].shape == (128, 128)
    spec = EncoderSpec("bert", 2, 128, 4, 64, 1e-12, pooling="mean", normalize=True)
    probe = []
    hidden, reps = oracle.encode_reps(sd, spec, ids, mask, tt, dtype=torch.float64,
                                      probe=lambda layer, s: probe.append(torch.softmax(s, -1).amax(-1)))
    m = mask.bool()
    assert np.abs(reps.numpy() - z["reps"]).max() <= 1e-5
    assert np.abs(hidden[m].numpy() - z["hidden_attended"]).max() <= 1e-4
    # premise: peaked attention rows (median row-max probability > 0.5), so each head's own keys and values matter: the
    # same weights split into two 64-wide heads miss the reference by more than twice the kernels' rel-L2 bound of 1e-2
    for p in probe:
        assert float(p[m[:, None, :].expand_as(p)].median()) > 0.5
    _, reps64 = oracle.encode_reps(sd, EncoderSpec("bert", 2, 128, 2, 64, 1e-12, pooling="mean", normalize=True), ids,
                                   mask, tt, dtype=torch.float64)
    assert np.linalg.norm(reps64.numpy() - z["reps"]) > 2e-2 * np.linalg.norm(z["reps"])


@pytest.mark.parametrize("hidden,heads", [(384, 12), (128, 4), (1024, 32), (768, 12), (1024, 16)])
def test_spec_accepts_32_and_64_wide_heads(hidden, heads):
    from transformers import BertConfig

    from openmatch_b200.encoder import spec_from_hf_config
    spec = spec_from_hf_config(BertConfig(hidden_size=hidden, num_attention_heads=heads, intermediate_size=4 * hidden))
    assert (spec["hidden"], spec["heads"]) == (hidden, heads)


@pytest.mark.parametrize("hidden,heads", [(256, 16), (384, 4), (256, 2), (384, 5)])  # widths 16, 96, 128, 76.8
def test_other_head_widths_raise_before_the_library(hidden, heads):
    from transformers import BertConfig

    from openmatch_b200.encoder import CudaEncoder, spec_from_hf_config
    with pytest.raises(ValueError, match="32- or 64-wide"):
        spec_from_hf_config(BertConfig(hidden_size=hidden, num_attention_heads=heads, intermediate_size=4 * hidden))
    spec = dict(arch="bert", layers=1, hidden=hidden, heads=heads, ffn=512, vocab=100, max_pos=64, type_vocab=2,
                ln_eps=1e-12)
    with pytest.raises(ValueError, match="32- or 64-wide"):
        CudaEncoder(spec, {})
