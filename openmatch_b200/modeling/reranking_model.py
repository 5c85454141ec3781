"""Cross-encoder re-ranker with the reference's public surface (``src/openmatch/modeling/reranking_model.py``):
``RROutput`` and ``RRModel`` (``encode``, ``build``, ``save``).

A pair's score is ``head(pool(last_hidden_state))[:, 0]``: the backbone, ``first`` / ``mean`` pooling and a bias-free
``LinearHead(H, 1)``.  Two execution paths, chosen per call as in ``DRModel``:
  * inference (no autograd): the sm_90a encoder computes the whole score (``CudaEncoder``, head_out 1, no
    normalisation).  ``encode`` takes the reference's padded batches and encodes them packed; ``encode_pairs`` scores
    pairs assembled on the device from token stores (``om_encode_pairs``), the ``Reranker`` hot path.
  * training mode under autograd: the HF module, pooling and head under PyTorch autograd.
Re-ranker training (``forward``, the rr losses) and the T5 encoder-decoder scoring (``pos_token`` / ``neg_token``
logits) are not implemented: they raise ``NotImplementedError``.
"""
from __future__ import annotations

import json
import logging
import os
from dataclasses import dataclass, fields
from typing import Dict

import torch
import torch.nn as nn
from torch import Tensor

from ..arguments import DataArguments, ModelArguments
from ..utils import mean_pooling
from .linear import LinearHead

logger = logging.getLogger(__name__)


@dataclass
class RROutput:
    """Same three fields as the reference's ``ModelOutput`` subclass; supports attribute and key access."""
    pos_pair_scores: Tensor = None
    neg_pair_scores: Tensor = None
    loss: Tensor = None

    def __getitem__(self, key):
        if isinstance(key, str):
            return getattr(self, key)
        return self.to_tuple()[key]

    def to_tuple(self):
        return tuple(getattr(self, f.name) for f in fields(self) if getattr(self, f.name) is not None)

    def keys(self):
        return [f.name for f in fields(self) if getattr(self, f.name) is not None]


def _decoder_mode(lm, model_args) -> bool:
    return "T5" in type(lm).__name__ and not (model_args is not None and model_args.encoder_only)


_DECODER_MSG = ("RRModel: T5 encoder-decoder scoring (pos_token / neg_token logits) is not implemented; "
                "pass --encoder_only to score with the T5 encoder, pooling and a linear head")


class RRModel(nn.Module):
    def __init__(self, lm, head: nn.Module, feature: str = "last_hidden_state", pooling: str = "first",
                 pos_token: str = None, neg_token: str = None, tokenizer=None, model_args: ModelArguments = None,
                 data_args: DataArguments = None, train_args=None):
        super().__init__()
        if _decoder_mode(lm, model_args):
            raise NotImplementedError(_DECODER_MSG)
        if pooling not in ("first", "mean"):
            raise ValueError("Unknown pooling type: {}".format(pooling))
        self.lm, self.head = lm, head
        self.feature, self.pooling = feature, pooling
        self.pos_token, self.neg_token, self.tokenizer = pos_token, neg_token, tokenizer
        self.model_args, self.data_args, self.train_args = model_args, data_args, train_args
        self._cuda_encoder_cache = None  # (weights version, CudaEncoder)

    def _get_config_dict(self):
        return {"plm_backbone": {"type": type(self.lm).__name__, "feature": self.feature}, "pooling": self.pooling,
                "pos_token": self.pos_token, "neg_token": self.neg_token}

    def forward(self, pos_pairs: Dict[str, Tensor] = None, neg_pairs: Dict[str, Tensor] = None):
        raise NotImplementedError("RRModel.forward: re-ranker training (train_rr, the mr / smr / bce / ce losses) is not "
                                  "implemented; RRModel scores pairs for inference (encode, encode_pairs)")

    # ------------------------------------------------------------------ scoring
    def max_pair_len(self) -> int:
        """longest assembled pair the model takes (``encoder.max_seq_len``): 8192 tokens and max_position_embeddings for
        BERT / DistilBERT (minus RoBERTa's position offset of 2), 512 for T5 and MPNet, at most
        OPENMATCH_B200_MAX_BATCH_TOKENS"""
        from ..encoder import max_seq_len, spec_from_hf_config
        max_tokens = int(os.environ.get("OPENMATCH_B200_MAX_BATCH_TOKENS", 256 * 128))
        return max_seq_len(spec_from_hf_config(self.lm.config), max_tokens)

    def _cuda_encoder(self):
        from ..encoder import CudaEncoder
        version = sum(int(p._version) for p in self.parameters())
        hit = self._cuda_encoder_cache
        if hit is None or hit[0] != version:
            max_tokens = int(os.environ.get("OPENMATCH_B200_MAX_BATCH_TOKENS", 256 * 128))
            enc = CudaEncoder.from_hf(self.lm, self.head, self.pooling, normalize=False, max_batch_tokens=max_tokens)
            self._cuda_encoder_cache = hit = (version, enc)
        return hit[1]

    def encode(self, items):
        """Scores ``[B, 1]`` of right-padded pair batches (``input_ids`` / ``attention_mask`` / optional
        ``token_type_ids``, ``[B, L]``, each row's tokens at most ``max_pair_len()``: up to 8192 for BERT / RoBERTa),
        as the reference's ``RRModel.encode`` (:106-125)."""
        if items is None:
            return None, None
        if self.feature != "last_hidden_state":
            raise NotImplementedError("only feature='last_hidden_state' is supported")
        input_ids, mask = items["input_ids"], items["attention_mask"]
        tt = items.get("token_type_ids", None)
        if torch.is_grad_enabled() and self.training:
            out = self.lm(**{k: v for k, v in items.items()}, return_dict=True)
            hidden = out.last_hidden_state
            reps = hidden[:, 0, :] if self.pooling == "first" else mean_pooling(hidden, mask)
            return self.head(reps)
        if not input_ids.is_cuda:
            raise RuntimeError("openmatch_b200 encodes on a CUDA device only (no CPU path): move the batch to GPU")
        # om_encode takes L <= 128 or a multiple of 128; the reference's pairs are q_max + p_max + 2 tokens (162 by
        # default): encode the rows packed, without their padding
        m = mask.bool()
        lens = m.sum(1)
        L = m.shape[1]
        if not torch.equal(m, torch.arange(L, device=m.device)[None, :] < lens[:, None]):
            raise ValueError("RRModel.encode: attention_mask must be right padding (each row's tokens first)")
        tokens = input_ids[m]
        return self._cuda_encoder().encode_packed(tokens, lens.to(torch.int32).cpu(),
                                                  token_type_ids=tt[m] if tt is not None else None)

    @torch.no_grad()
    def encode_pairs(self, a_tokens: Tensor, b_tokens: Tensor, spans, prefix=(), suffix=(), out: Tensor = None) -> Tensor:
        """Scores ``[B, 1]`` fp32 of the pairs ``prefix ++ a_tokens[a_start : a_start + a_len] ++ b_tokens[b_start :
        b_start + b_len] ++ suffix`` (``spans`` host int64 ``[B, 4]``), assembled on the device (``om_encode_pairs``).
        ``out`` may be a slice of a larger buffer."""
        return self._cuda_encoder().encode_pairs(a_tokens, b_tokens, spans, prefix, suffix, out=out)

    # ------------------------------------------------------------------ build / save
    @classmethod
    def build(cls, model_args: ModelArguments, data_args: DataArguments = None, train_args=None, tokenizer=None,
              **hf_kwargs):
        from transformers import AutoConfig, AutoModel, T5EncoderModel
        path = model_args.model_name_or_path
        hf_config = hf_kwargs.get("config") or AutoConfig.from_pretrained(path, cache_dir=hf_kwargs.get("cache_dir"))
        if model_args.encoder_only:
            model_class = T5EncoderModel
        elif "T5" in ((hf_config.architectures or [""])[0] or type(hf_config).__name__):
            raise NotImplementedError(_DECODER_MSG)
        else:
            model_class = AutoModel
        om_config = None
        cfg_file = os.path.join(path, "openmatch_config.json")
        if os.path.exists(cfg_file):
            with open(cfg_file) as f:
                om_config = json.load(f)
        lm = model_class.from_pretrained(path, **hf_kwargs)
        if os.path.isdir(path) and om_config is not None:  # an OpenMatch checkpoint directory
            logger.info("loading reranking model weight from %s", path)
            head = LinearHead.load(ckpt_dir=path)
        else:  # a plain HuggingFace model
            head = LinearHead(model_args.projection_in_dim, 1)
        pick = (lambda key, default: default) if om_config is None else (lambda key, default: om_config[key])
        return cls(lm=lm, head=head,
                   feature=model_args.feature if om_config is None else om_config["plm_backbone"]["feature"],
                   pooling=pick("pooling", model_args.pooling), pos_token=pick("pos_token", model_args.pos_token),
                   neg_token=pick("neg_token", model_args.neg_token), tokenizer=tokenizer, model_args=model_args,
                   data_args=data_args, train_args=train_args)

    def save(self, output_dir: str):
        self.lm.save_pretrained(output_dir)
        self.head.save(output_dir)
        with open(os.path.join(output_dir, "openmatch_config.json"), "w") as f:
            json.dump(self._get_config_dict(), f, indent=4)
