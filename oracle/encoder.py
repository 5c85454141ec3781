"""Oracle: fp32 CPU restatement of the encoder arithmetic behind ``DRModel.encode``
(``src/openmatch/modeling/dense_retrieval_model.py:133-155``): HF encoder forward -> ``first`` / ``mean``
pooling (``:145-150``, ``src/openmatch/utils.py:233-235``) -> optional bias-free ``LinearHead``
(``src/openmatch/modeling/linear.py:19,22-23``) -> optional ``F.normalize(dim=1)`` (``:153-154``).

The encoder maths lives in an un-vendored dependency, HuggingFace ``transformers`` (setup.py:24 pins only
``>=4.10.0``; 5.5.0 is installed here).  Restated from
  BERT : transformers/models/bert/modeling_bert.py  (embeddings :53-112, self-attention :115-207,
         self-output :287-298, intermediate/output :339-356, layer :359-421)
  T5   : transformers/models/t5/modeling_t5.py      (T5LayerNorm :46-69, T5DenseActDense :84-104,
         relative buckets :188-234, attention :153-345, stack :637-790)
Explicit matmuls on plain tensors keyed by the HF ``state_dict`` names; no HF module is executed here.
tests/test_oracle_pinning.py checks this file against the reference's own ``DRModelForInference`` (golden
vectors in tests/golden/, made by tests/golden/make_golden.py inside the build container).

``encode_reps`` computes in float32 by default.  ``dtype=torch.float64`` gives the high-precision yardstick the GPU
numerics tests compare against; ``emulate_bf16=True`` additionally rounds to bf16 what the reference rounds under
bf16 autocast (SURVEY section 8(d)): both operands of every matmul (activations, weights and biases), the output of
every Linear and the probabilities P before P V.  Softmax, LayerNorm / RMSNorm, the residual stream and pooling stay in
``dtype``.  ``probe(layer, logits)`` receives every layer's masked attention logits [B, heads, L, L] (float64, -inf at
masked keys, natural-log units) so a test can check the attention statistics it claims to exercise.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F


@dataclass
class EncoderSpec:
    arch: str  # "bert" | "t5"
    layers: int
    hidden: int
    heads: int
    ffn: int
    ln_eps: float
    pooling: str = "first"  # "first" | "mean"
    normalize: bool = False
    rel_buckets: int = 32  # T5 only
    rel_max_distance: int = 128  # T5 only


class _Num:
    """Arithmetic of one oracle run: the compute dtype and whether matmuls see bf16-rounded operands (autocast)."""

    def __init__(self, dtype=torch.float32, emulate_bf16=False, probe=None):
        self.dtype, self.bf16, self.probe = dtype, emulate_bf16, probe

    def t(self, t):
        return t.detach().to(self.dtype)

    def r(self, t):  # bf16 rounding of a matmul operand / Linear output (identity without emulation)
        return t.to(torch.bfloat16).to(self.dtype) if self.bf16 else t

    def mm(self, a, b):
        return self.r(a) @ self.r(b)

    def lin(self, x, w, b=None):  # F.linear under autocast: bf16 x, W, b; bf16 output
        y = self.mm(x, self.t(w).T)
        return self.r(y + self.r(self.t(b)) if b is not None else y)

    def look(self, layer, logits):
        if self.probe is not None:
            self.probe(layer, logits.detach().to(torch.float64))


_F32 = _Num()


def _key_mask(attention_mask: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    # additive key-padding mask [B, 1, 1, L]: 0 where attended, -inf where padded
    m = torch.zeros(attention_mask.shape, dtype=dtype)
    m = m.masked_fill(attention_mask == 0, float("-inf"))
    return m[:, None, None, :]


def _softmax_rows(s: torch.Tensor) -> torch.Tensor:
    # rows whose keys are all masked never reach pooling; define them as zeros instead of NaN
    mx = s.max(dim=-1, keepdim=True).values
    mx = torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)
    e = torch.exp(s - mx)
    z = e.sum(dim=-1, keepdim=True)
    return e / torch.where(z == 0, torch.ones_like(z), z)


def bert_encode(sd: Dict[str, torch.Tensor], spec: EncoderSpec, input_ids, attention_mask, token_type_ids=None,
                nm: _Num = _F32):
    """``BertModel.forward`` -> last_hidden_state [B, L, H] (pooler skipped: OpenMatch ignores it)."""
    B, L = input_ids.shape
    H, nh = spec.hidden, spec.heads
    dh = H // nh
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    emb = (nm.t(sd["embeddings.word_embeddings.weight"])[input_ids]
           + nm.t(sd["embeddings.token_type_embeddings.weight"])[token_type_ids]
           + nm.t(sd["embeddings.position_embeddings.weight"])[torch.arange(L)][None])
    h = F.layer_norm(emb, (H,), nm.t(sd["embeddings.LayerNorm.weight"]), nm.t(sd["embeddings.LayerNorm.bias"]),
                     spec.ln_eps)
    mask = _key_mask(attention_mask, nm.dtype)
    for i in range(spec.layers):
        p = f"encoder.layer.{i}."

        def lin(x, name):
            return nm.lin(x, sd[p + name + ".weight"], sd[p + name + ".bias"])

        def heads(x):
            return x.view(B, L, nh, dh).permute(0, 2, 1, 3)

        q, k, v = (heads(lin(h, "attention.self." + n)) for n in ("query", "key", "value"))
        s = nm.mm(q, k.transpose(-1, -2)) * (dh ** -0.5) + mask
        nm.look(i, s)
        ctx = nm.mm(_softmax_rows(s), v).permute(0, 2, 1, 3).reshape(B, L, H)
        h = F.layer_norm(lin(ctx, "attention.output.dense") + h, (H,),
                         nm.t(sd[p + "attention.output.LayerNorm.weight"]),
                         nm.t(sd[p + "attention.output.LayerNorm.bias"]), spec.ln_eps)
        inter = F.gelu(lin(h, "intermediate.dense"))  # exact erf GELU (hidden_act="gelu")
        h = F.layer_norm(lin(inter, "output.dense") + h, (H,), nm.t(sd[p + "output.LayerNorm.weight"]),
                         nm.t(sd[p + "output.LayerNorm.bias"]), spec.ln_eps)
    return h


def t5_relative_position_bucket(rel: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bidirectional bucket of rel = key_pos - query_pos (modeling_t5.py:188-234), same fp32 arithmetic."""
    nb = num_buckets // 2
    out = (rel > 0).to(torch.long) * nb
    n = rel.abs()
    max_exact = nb // 2
    is_small = n < max_exact
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact)
                         * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return out + torch.where(is_small, n, large)


def _rms(x, w, eps):
    var = x.pow(2).mean(-1, keepdim=True)
    return w * (x * torch.rsqrt(var + eps))


def t5_encode(sd: Dict[str, torch.Tensor], spec: EncoderSpec, input_ids, attention_mask, nm: _Num = _F32):
    """``T5EncoderModel.forward`` -> last_hidden_state [B, L, H] (after final_layer_norm)."""
    B, L = input_ids.shape
    H, nh = spec.hidden, spec.heads
    emb_key = "shared.weight" if "shared.weight" in sd else "encoder.embed_tokens.weight"
    h = nm.t(sd[emb_key])[input_ids]
    dh = sd["encoder.block.0.layer.0.SelfAttention.q.weight"].shape[0] // nh
    pos = torch.arange(L)
    bucket = t5_relative_position_bucket(pos[None, :] - pos[:, None], spec.rel_buckets, spec.rel_max_distance)
    rel = nm.t(sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"])  # [buckets, heads]
    bias = rel[bucket].permute(2, 0, 1)[None]  # [1, heads, L, L], shared by all layers
    mask = _key_mask(attention_mask, nm.dtype)
    for i in range(spec.layers):
        p = f"encoder.block.{i}.layer."
        x = _rms(h, nm.t(sd[p + "0.layer_norm.weight"]), spec.ln_eps)

        def heads(t):
            return t.view(B, L, nh, dh).permute(0, 2, 1, 3)

        q, k, v = (heads(nm.lin(x, sd[p + f"0.SelfAttention.{n}.weight"])) for n in ("q", "k", "v"))
        s = nm.mm(q, k.transpose(-1, -2)) + bias + mask  # no 1/sqrt(d) scaling in T5
        nm.look(i, s)
        ctx = nm.mm(_softmax_rows(s), v).permute(0, 2, 1, 3).reshape(B, L, nh * dh)
        h = h + nm.lin(ctx, sd[p + "0.SelfAttention.o.weight"])
        x = _rms(h, nm.t(sd[p + "1.layer_norm.weight"]), spec.ln_eps)
        if p + "1.DenseReluDense.wi.weight" in sd:
            inter = torch.relu(nm.lin(x, sd[p + "1.DenseReluDense.wi.weight"]))
        else:  # gated-GELU variant (t5 v1.1): gelu_new(wi_0 x) * (wi_1 x)
            g = nm.lin(x, sd[p + "1.DenseReluDense.wi_0.weight"])
            inter = nm.r(F.gelu(g, approximate="tanh") * nm.lin(x, sd[p + "1.DenseReluDense.wi_1.weight"]))
        h = h + nm.lin(inter, sd[p + "1.DenseReluDense.wo.weight"])
    return _rms(h, nm.t(sd["encoder.final_layer_norm.weight"]), spec.ln_eps)


def pool_head_normalize(hidden, attention_mask, pooling: str, head_weight: Optional[torch.Tensor], normalize: bool,
                        nm: _Num = _F32):
    """dense_retrieval_model.py:145-154 + utils.py:233-235 + linear.py:22-23."""
    if pooling == "first":
        reps = hidden[:, 0, :]
    elif pooling == "mean":
        m = attention_mask.unsqueeze(-1).expand(hidden.size()).to(hidden.dtype)
        reps = torch.sum(hidden * m, 1) / torch.clamp(m.sum(1), min=1e-9)
    else:
        raise ValueError("Unknown pooling type: {}".format(pooling))
    if head_weight is not None:
        reps = nm.lin(reps, head_weight)
    if normalize:
        reps = F.normalize(reps, dim=1)
    return reps


def encode_reps(sd, spec: EncoderSpec, input_ids, attention_mask, token_type_ids=None, head_weight=None,
                dtype=torch.float32, emulate_bf16=False, probe=None):
    """(hidden, reps) exactly as ``DRModel.encode`` returns them, in ``dtype`` on CPU (see the module docstring for
    ``emulate_bf16`` and ``probe``)."""
    nm = _Num(dtype, emulate_bf16, probe)
    with torch.no_grad():
        if spec.arch == "bert":
            hidden = bert_encode(sd, spec, input_ids, attention_mask, token_type_ids, nm)
        elif spec.arch == "t5":
            hidden = t5_encode(sd, spec, input_ids, attention_mask, nm)
        else:
            raise ValueError(spec.arch)
        reps = pool_head_normalize(hidden, attention_mask, spec.pooling, head_weight, spec.normalize, nm)
    return hidden, reps
