"""CUDA encoder handle: host-side marshalling for ``om_encoder_*`` / ``om_encode`` (csrc/encoder.cu).

Replaces the HF forward + pooling + head + normalise sequence of ``DRModel.encode``
(``src/openmatch/modeling/dense_retrieval_model.py:133-155``) for inference.  Weights are handed over by
their HuggingFace ``state_dict`` names; the library keeps packed bf16 / fp32 copies in HBM.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib

_OUT_DTYPES = {torch.float32: _lib.OM_F32, torch.bfloat16: _lib.OM_BF16, torch.float16: _lib.OM_F16,
               torch.int8: _lib.OM_I8}

_HEAD_WIDTHS = (32, 64)  # BERT head widths hidden / heads the CUDA attention kernels implement (T5: d_kv 64)

_BERT_KEYS = ("num_hidden_layers", "hidden_size", "num_attention_heads", "intermediate_size", "vocab_size",
              "max_position_embeddings", "type_vocab_size", "layer_norm_eps")


def _check_bert_heads(hidden: int, heads: int):
    if heads <= 0 or hidden % heads != 0 or hidden // heads not in _HEAD_WIDTHS:
        raise ValueError("CUDA encoder needs 32- or 64-wide attention heads, got hidden_size=%d / num_attention_heads=%d"
                         % (hidden, heads))


ROBERTA_PAD_ID = 1  # padding_idx of RoBERTa's and MPNet's position ids, fixed in the library (include/openmatch_b200.h)

_ARCHS = {"bert": _lib.OM_ARCH_BERT, "t5": _lib.OM_ARCH_T5ENC, "roberta": _lib.OM_ARCH_ROBERTA,
          "mpnet": _lib.OM_ARCH_MPNET, "distilbert": _lib.OM_ARCH_DISTILBERT}
_BERT_LIKE = ("bert", "roberta", "mpnet", "distilbert")

# MPNetEncoder.compute_position_bias buckets with num_buckets = 32 and max_distance = 128 whatever the config says
MPNET_REL_BUCKETS, MPNET_REL_MAX_DISTANCE = 32, 128


def spec_from_hf_config(config) -> Dict:
    """Translate a HF ``BertConfig`` / ``RobertaConfig`` / ``XLMRobertaConfig`` / ``MPNetConfig`` /
    ``DistilBertConfig`` / ``T5Config`` into the plain dict ``CudaEncoder`` consumes."""
    mt = getattr(config, "model_type", "")
    if mt in ("bert", "roberta", "xlm-roberta"):
        roberta = mt != "bert"
        _check_bert_heads(config.hidden_size, config.num_attention_heads)
        if getattr(config, "hidden_act", "gelu") != "gelu":
            raise ValueError("CUDA encoder supports hidden_act='gelu' (erf) only, got %r" % config.hidden_act)
        if getattr(config, "position_embedding_type", "absolute") not in (None, "absolute"):
            raise ValueError("CUDA encoder supports absolute position embeddings only")
        if roberta and config.pad_token_id != ROBERTA_PAD_ID:
            raise ValueError("CUDA encoder computes RoBERTa position ids with padding_idx %d, got pad_token_id=%r"
                             % (ROBERTA_PAD_ID, config.pad_token_id))
        if roberta and config.max_position_embeddings < 3:
            raise ValueError("RoBERTa max_position_embeddings=%d leaves no position (positions start at 2)"
                             % config.max_position_embeddings)
        return dict(arch="roberta" if roberta else "bert", layers=config.num_hidden_layers,
                    hidden=config.hidden_size, heads=config.num_attention_heads, ffn=config.intermediate_size,
                    vocab=config.vocab_size, max_pos=config.max_position_embeddings, type_vocab=config.type_vocab_size,
                    ln_eps=config.layer_norm_eps)
    if mt == "mpnet":
        if config.num_attention_heads <= 0 or config.hidden_size != 64 * config.num_attention_heads:
            raise ValueError("CUDA encoder needs 64-wide MPNet attention heads, got hidden_size=%d / "
                             "num_attention_heads=%d" % (config.hidden_size, config.num_attention_heads))
        if getattr(config, "hidden_act", "gelu") != "gelu":
            raise ValueError("CUDA encoder supports hidden_act='gelu' (erf) only, got %r" % config.hidden_act)
        if config.relative_attention_num_buckets != MPNET_REL_BUCKETS:
            raise ValueError("CUDA encoder needs MPNet relative_attention_num_buckets=%d (the buckets HF computes), got %r"
                             % (MPNET_REL_BUCKETS, config.relative_attention_num_buckets))
        if config.max_position_embeddings < 3:
            raise ValueError("MPNet max_position_embeddings=%d leaves no position (positions start at 2)"
                             % config.max_position_embeddings)
        return dict(arch="mpnet", layers=config.num_hidden_layers, hidden=config.hidden_size,
                    heads=config.num_attention_heads, ffn=config.intermediate_size, vocab=config.vocab_size,
                    max_pos=config.max_position_embeddings, type_vocab=0, ln_eps=config.layer_norm_eps,
                    rel_buckets=MPNET_REL_BUCKETS, rel_max_distance=MPNET_REL_MAX_DISTANCE)
    if mt == "distilbert":
        _check_bert_heads(config.dim, config.n_heads)
        if getattr(config, "activation", "gelu") != "gelu":
            raise ValueError("CUDA encoder supports activation='gelu' (erf) only, got %r" % config.activation)
        return dict(arch="distilbert", layers=config.n_layers, hidden=config.dim, heads=config.n_heads,
                    ffn=config.hidden_dim, vocab=config.vocab_size, max_pos=config.max_position_embeddings,
                    type_vocab=0, ln_eps=1e-12)  # every DistilBERT LayerNorm has eps 1e-12 (modeling_distilbert.py)
    if mt == "t5":
        if config.d_kv != 64:
            raise ValueError("CUDA encoder supports d_kv == 64 only")
        if getattr(config, "feed_forward_proj", "relu") != "relu":
            raise ValueError("CUDA encoder supports the non-gated ReLU T5 feed-forward only")
        return dict(arch="t5", layers=config.num_layers, hidden=config.d_model, heads=config.num_heads,
                    ffn=config.d_ff, vocab=config.vocab_size, max_pos=0, type_vocab=0,
                    ln_eps=config.layer_norm_epsilon, rel_buckets=config.relative_attention_num_buckets,
                    rel_max_distance=getattr(config, "relative_attention_max_distance", 128))
    raise ValueError("CUDA encoder supports BERT, RoBERTa / XLM-RoBERTa, MPNet, DistilBERT and T5-encoder backbones, "
                     "got model_type=%r" % mt)


MAX_SEQ_LEN = 8192     # longest sequence of a packed call for BERT / RoBERTa / DistilBERT (include/openmatch_b200.h)
MAX_T5_SEQ_LEN = 512   # T5 and MPNet: their relative-bias tables cover 512 tokens


def max_seq_len(spec: Dict, max_batch_tokens: int = 256 * 128) -> int:
    """Longest sequence ``encode_packed`` / ``encode_pairs`` take for ``spec`` (a ``spec_from_hf_config`` dict) on a
    handle of ``max_batch_tokens``: 8192 tokens and ``max_position_embeddings`` (BERT, DistilBERT) /
    ``max_position_embeddings - 2`` (RoBERTa, whose positions start at 2); 512 tokens for T5, and for MPNet within
    ``max_position_embeddings - 2``; never more than ``max_batch_tokens``."""
    if spec["arch"] == "t5":
        limit = MAX_T5_SEQ_LEN
    elif spec["arch"] == "mpnet":
        limit = min(MAX_T5_SEQ_LEN, spec["max_pos"] - 2)
    else:
        limit = min(MAX_SEQ_LEN, spec["max_pos"] - (2 if spec["arch"] == "roberta" else 0))
    return min(limit, int(max_batch_tokens))


class CudaEncoder:
    def __init__(self, spec: Dict, state_dict: Dict[str, torch.Tensor], head_weight: Optional[torch.Tensor] = None,
                 pooling: str = "first", normalize: bool = False, max_batch_tokens: int = 256 * 128):
        if pooling not in ("first", "mean"):
            raise ValueError("Unknown pooling type: {}".format(pooling))
        if spec["arch"] not in _ARCHS:
            raise ValueError("Unknown encoder arch %r" % spec["arch"])
        if spec["arch"] in _BERT_LIKE:
            _check_bert_heads(spec["hidden"], spec["heads"])
        self._lib = _lib.load()
        head_head_out = int(head_weight.shape[0]) if head_weight is not None else 0
        desc = _lib.EncoderDesc(
            arch=_ARCHS[spec["arch"]], layers=spec["layers"],
            hidden=spec["hidden"], heads=spec["heads"], ffn=spec["ffn"], vocab=spec["vocab"],
            max_pos=spec.get("max_pos", 0), type_vocab=spec.get("type_vocab", 0), ln_eps=float(spec["ln_eps"]),
            pooling=_lib.OM_POOL_MEAN if pooling == "mean" else _lib.OM_POOL_FIRST,
            has_head=1 if head_weight is not None else 0, head_out=head_head_out, normalize=1 if normalize else 0,
            rel_buckets=spec.get("rel_buckets", 32), rel_max_distance=spec.get("rel_max_distance", 128),
            max_batch_tokens=int(max_batch_tokens))
        h = ctypes.c_void_p()
        _lib.check(self._lib.om_encoder_create(ctypes.byref(desc), ctypes.byref(h)))
        self._h = h
        self.spec = dict(spec)
        self.hidden = spec["hidden"]
        self.max_batch_tokens = int(max_batch_tokens)
        self.ignored = []
        for name, t in state_dict.items():
            self._set(name, t)
        if head_weight is not None:
            self._set("head.linear.weight", head_weight)
        _lib.check(self._lib.om_encoder_finalize(self._h))
        self.rep_dim = int(self._lib.om_encoder_rep_dim(self._h))

    @classmethod
    def from_hf(cls, lm, head=None, pooling="first", normalize=False, max_batch_tokens=256 * 128):
        head_w = head.linear.weight if head is not None else None
        return cls(spec_from_hf_config(lm.config), lm.state_dict(), head_w, pooling, normalize, max_batch_tokens)

    def _set(self, name: str, t: torch.Tensor):
        t = t.detach()
        if not t.is_floating_point():
            return
        t = t.to(torch.float32).contiguous()
        kind = _lib.OM_DEVICE if t.is_cuda else _lib.OM_HOST
        shape = (ctypes.c_int64 * t.dim())(*t.shape)
        rc = _lib.check(self._lib.om_encoder_set_weight(self._h, name.encode(), t.data_ptr(), kind, shape, t.dim()))
        if rc == 1:
            self.ignored.append(name)

    def _out(self, out: Optional[torch.Tensor], out_dtype: torch.dtype, B: int, device):
        """``out`` of the encode methods, checked, or a new ``[B, rep_dim]`` tensor of ``out_dtype``"""
        if out is None:
            if out_dtype == torch.int8:
                raise ValueError("int8 output goes into the rows of an int8 index (FlatIPIndex.reserve_rows): pass out")
            out = torch.empty((B, self.rep_dim), dtype=out_dtype, device=device)
        if out.dtype not in _OUT_DTYPES or out.stride(1) != 1:
            raise ValueError("out must be a row-major fp32 / bf16 / fp16 CUDA tensor or int8 index rows")
        if out.shape[0] != B or out.shape[1] != self.rep_dim:
            raise ValueError("out must be [%d, %d], got %s" % (B, self.rep_dim, tuple(out.shape)))
        return out

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.om_encoder_destroy(h)

    @torch.no_grad()
    def encode(self, input_ids: torch.Tensor, attention_mask: torch.Tensor,
               token_type_ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
               out_dtype: torch.dtype = torch.float32, return_hidden: bool = False):
        """int64 [B, L] CUDA tensors in -> reps [B, rep_dim] (and last_hidden_state fp32 [B, L, H]).  ``out`` / ``out_dtype``:
        fp32, bf16 or fp16 (fp16 and bf16 are the round-to-nearest-even of the fp32 reps of the same call); ``out`` may
        have any row stride (e.g. the rows ``FlatIPIndex.reserve_rows`` hands out).  An int8 ``out`` must be the rows of
        an int8 index: the fp32 reps of the same call are quantised by the index's rule, scales included."""
        if not input_ids.is_cuda:
            raise RuntimeError("openmatch_b200 encoder runs on CUDA tensors only (no CPU path)")
        B, L = input_ids.shape
        ids = input_ids.to(torch.int64).contiguous()
        mask = attention_mask.to(torch.int64).contiguous()
        tt = token_type_ids.to(torch.int64).contiguous() if token_type_ids is not None else None
        out = self._out(out, out_dtype, B, ids.device)
        hidden = torch.empty((B, L, self.hidden), dtype=torch.float32, device=ids.device) if return_hidden else None
        _lib.check(self._lib.om_encode(
            self._h, ids.data_ptr(), mask.data_ptr(), tt.data_ptr() if tt is not None else None, B, L,
            out.data_ptr(), _OUT_DTYPES[out.dtype], out.stride(0),
            hidden.data_ptr() if hidden is not None else None, _lib.current_stream_ptr()))
        return (hidden, out) if return_hidden else out

    @torch.no_grad()
    def encode_packed(self, tokens: torch.Tensor, seqlens, token_type_ids: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.float32,
                      return_hidden: bool = False):
        """Variable-length batch without padding: ``tokens`` int64 ``[T]`` CUDA tensor holding the sequences back to
        back, ``seqlens`` their lengths (host int32 array / list / CPU tensor, each in [1, ``max_seq_len(spec,
        max_batch_tokens)``]: up to 8192 tokens for BERT / RoBERTa within the position table, 512 for T5; sum = T) ->
        reps ``[B, rep_dim]`` (and last_hidden_state fp32 ``[T, H]``, packed like ``tokens``).  The same representations
        ``encode`` gives the sequences padded, up to the order of floating-point sums; ``out`` / ``out_dtype`` as there."""
        if not tokens.is_cuda:
            raise RuntimeError("openmatch_b200 encoder runs on CUDA tensors only (no CPU path)")
        if isinstance(seqlens, torch.Tensor):
            seqlens = seqlens.detach().cpu().numpy()
        lens = np.ascontiguousarray(np.asarray(seqlens).reshape(-1), dtype=np.int32)
        B, T = int(lens.shape[0]), int(lens.sum(dtype=np.int64))
        ids = tokens.reshape(-1).to(torch.int64).contiguous()
        if ids.numel() != T:
            raise ValueError("tokens holds %d ids, seqlens sum to %d" % (ids.numel(), T))
        tt = token_type_ids.reshape(-1).to(torch.int64).contiguous() if token_type_ids is not None else None
        out = self._out(out, out_dtype, B, ids.device)
        hidden = torch.empty((T, self.hidden), dtype=torch.float32, device=ids.device) if return_hidden else None
        _lib.check(self._lib.om_encode_packed(
            self._h, ids.data_ptr(), tt.data_ptr() if tt is not None else None, lens.ctypes.data, B,
            out.data_ptr(), _OUT_DTYPES[out.dtype], out.stride(0),
            hidden.data_ptr() if hidden is not None else None, _lib.current_stream_ptr()))
        return (hidden, out) if return_hidden else out

    @torch.no_grad()
    def encode_pairs(self, a_tokens: torch.Tensor, b_tokens: torch.Tensor, spans, prefix=(), suffix=(),
                     out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.float32):
        """Cross-encoder pairs assembled on the device: sequence i = ``prefix ++ a_tokens[a_start : a_start + a_len] ++
        b_tokens[b_start : b_start + b_len] ++ suffix`` with ``spans[i] = (a_start, a_len, b_start, b_len)`` (host int64
        ``[B, 4]``), token types 0; ``a_tokens`` / ``b_tokens``: int32 CUDA token stores; ``prefix`` / ``suffix``: up to
        4 ids each; an assembled pair is at most ``max_seq_len(spec, max_batch_tokens)`` tokens long (as in
        ``encode_packed``).  -> reps ``[B, rep_dim]``, bitwise what ``encode_packed`` returns for the assembled
        sequences; ``out`` / ``out_dtype`` as there."""
        if not a_tokens.is_cuda or not b_tokens.is_cuda:
            raise RuntimeError("openmatch_b200 encoder runs on CUDA tensors only (no CPU path)")
        if isinstance(spans, torch.Tensor):
            spans = spans.detach().cpu().numpy()
        sp = np.ascontiguousarray(np.asarray(spans, dtype=np.int64).reshape(-1, 4))
        pre = np.ascontiguousarray(np.asarray(prefix, dtype=np.int32).reshape(-1))
        suf = np.ascontiguousarray(np.asarray(suffix, dtype=np.int32).reshape(-1))
        B = int(sp.shape[0])
        a, b = (t.reshape(-1).to(torch.int32).contiguous() for t in (a_tokens, b_tokens))
        na, nb = a.numel(), b.numel()
        # an empty store has no address; any valid one does (every span of it is then empty)
        a = a if na else torch.zeros(1, dtype=torch.int32, device=a.device)
        b = b if nb else torch.zeros(1, dtype=torch.int32, device=b.device)
        out = self._out(out, out_dtype, B, a.device)
        _lib.check(self._lib.om_encode_pairs(
            self._h, a.data_ptr(), na, b.data_ptr(), nb, sp.ctypes.data, B, pre.ctypes.data if pre.size else None,
            int(pre.size), suf.ctypes.data if suf.size else None, int(suf.size), out.data_ptr(), _OUT_DTYPES[out.dtype],
            out.stride(0), _lib.current_stream_ptr()))
        return out
