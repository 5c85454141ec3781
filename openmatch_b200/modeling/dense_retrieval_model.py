"""Bi-encoder wrapper with the reference's public surface
(``src/openmatch/modeling/dense_retrieval_model.py``): ``DROutput``, ``DRModel`` (``encode``,
``encode_passage``, ``encode_query``, ``forward``, ``build``, ``save``, ``dist_gather_tensor``) and
``DRModelForInference``.

Two execution paths, chosen per call:
  * inference (no autograd: ``DRModelForInference``, or ``DRModel`` in eval mode under ``torch.no_grad``):
    the whole encode -> pool -> head -> normalise sequence runs in the hand-written sm_90a encoder
    (``openmatch_b200.encoder.CudaEncoder`` -> csrc/encoder.cu).  CUDA tensors only, no fallback.
  * training (autograd needed): the HF module runs under PyTorch autograd (the CUDA encoder is
    forward-only); scores, log-softmax, loss and the rep gradients come from the fused loss kernel
    (``openmatch_b200.loss``), preceded by the NCCL all-gather when ``negatives_x_device`` is set.
"""
from __future__ import annotations

import copy
import json
import logging
import os
from dataclasses import dataclass, fields
from typing import Dict, Optional

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor

from ..arguments import DataArguments, DRTrainingArguments as TrainingArguments, ModelArguments
from ..loss import fused_contrastive_loss
from ..utils import mean_pooling
from .linear import LinearHead

logger = logging.getLogger(__name__)

# widest padded batch om_encode takes (L <= 128, or 256 / 384 / 512); wider batches are encoded packed
PADDED_MAX_LEN = 512


@dataclass
class DROutput:
    """Same four fields as the reference's ``ModelOutput`` subclass; supports attribute and key access."""
    q_reps: Tensor = None
    p_reps: Tensor = None
    loss: Tensor = None
    scores: Tensor = None

    def __getitem__(self, key):
        if isinstance(key, str):
            return getattr(self, key)
        return self.to_tuple()[key]

    def to_tuple(self):
        return tuple(getattr(self, f.name) for f in fields(self) if getattr(self, f.name) is not None)

    def keys(self):
        return [f.name for f in fields(self) if getattr(self, f.name) is not None]


class DRModel(nn.Module):
    def __init__(self, lm_q, lm_p, tied: bool = True, feature: str = "last_hidden_state", pooling: str = "first",
                 head_q: nn.Module = None, head_p: nn.Module = None, normalize: bool = False,
                 model_args: ModelArguments = None, data_args: DataArguments = None,
                 train_args: TrainingArguments = None):
        super().__init__()
        self.tied = tied
        self.lm_q, self.lm_p = lm_q, lm_p
        self.head_q, self.head_p = head_q, head_p
        self.feature, self.pooling, self.normalize = feature, pooling, normalize
        self.model_args, self.train_args, self.data_args = model_args, train_args, data_args
        self._cuda_encoders = {}  # (id(lm), id(head)) -> (weights version, CudaEncoder)
        self.force_torch_path = False  # GradCache's no-grad representation pass must match its autograd pass
        if train_args is not None and train_args.negatives_x_device:
            if not dist.is_initialized():
                raise ValueError('Distributed training has not been initialized for representation all gather.')
            self.process_rank = dist.get_rank()
            self.world_size = dist.get_world_size()

    # ------------------------------------------------------------------ config / checkpoints
    def _get_config_dict(self):
        return {"tied": self.tied,
                "plm_backbone": {"type": type(self.lm_q).__name__, "feature": self.feature},
                "pooling": self.pooling, "linear_head": bool(self.head_q), "normalize": self.normalize}

    # ------------------------------------------------------------------ training forward
    def forward(self, query: Dict[str, Tensor] = None, passage: Dict[str, Tensor] = None):
        _, q_reps = self.encode_query(query)
        _, p_reps = self.encode_passage(passage)
        if q_reps is None or p_reps is None:
            return DROutput(q_reps=q_reps, p_reps=p_reps)
        if self.train_args.negatives_x_device:
            q_reps = self.dist_gather_tensor(q_reps)
            p_reps = self.dist_gather_tensor(p_reps)
        # target_i = i * train_n_passages: the positive of query i leads its passage group
        target = torch.arange(q_reps.size(0), device=q_reps.device, dtype=torch.long) * self.data_args.train_n_passages
        loss, scores = fused_contrastive_loss(q_reps, p_reps, target, "mean", return_scores=True)
        if self.training and self.train_args.negatives_x_device:
            loss = loss * self.world_size  # undo DDP's gradient averaging
        return DROutput(loss=loss, scores=scores, q_reps=q_reps, p_reps=p_reps)

    # ------------------------------------------------------------------ encode
    def _needs_autograd(self) -> bool:
        return self.force_torch_path or (torch.is_grad_enabled() and self.training)

    def _cuda_encoder(self, model, head):
        from ..encoder import CudaEncoder
        key = (id(model), id(head))
        version = sum(int(p._version) for p in model.parameters()) + (sum(int(p._version) for p in head.parameters())
                                                                      if head is not None else 0)
        hit = self._cuda_encoders.get(key)
        if hit is None or hit[0] != version:
            max_tokens = int(os.environ.get("OPENMATCH_B200_MAX_BATCH_TOKENS", 256 * 128))
            enc = CudaEncoder.from_hf(model, head, self.pooling, self.normalize, max_batch_tokens=max_tokens)
            self._cuda_encoders[key] = hit = (version, enc)
        return hit[1]

    def encode(self, items, model, head, need_hidden: bool = True):
        if items is None:
            return None, None
        decoder_path = "T5" in type(model).__name__ and not (self.model_args is not None and self.model_args.encoder_only)
        if decoder_path:
            # The reference's default T5 mode (:137-141): the full encoder-decoder with a single zero decoder token, reps =
            # decoder last_hidden_state[:, 0].  The decoder is outside the CUDA encoder (GTR / --encoder_only is the hot
            # path, SURVEY 8(a4)), so this mode runs the HF module on the GPU — for training and for inference alike.
            if not getattr(self, "_warned_decoder_path", False):
                logger.warning("encoder-decoder T5 pooling runs the HuggingFace module (not the sm_90a encoder); "
                               "use --encoder_only for the accelerated path")
                self._warned_decoder_path = True
            dec = torch.zeros((items["input_ids"].shape[0], 1), dtype=torch.long, device=items["input_ids"].device)
            out = model(**{k: v for k, v in items.items()}, decoder_input_ids=dec, return_dict=True)
            hidden = out.last_hidden_state
            reps = hidden[:, 0, :]
            if head is not None:
                reps = head(reps)
            if self.normalize:
                reps = F.normalize(reps, dim=1)
            return hidden, reps
        if self.feature != "last_hidden_state":
            raise NotImplementedError("only feature='last_hidden_state' is supported")
        input_ids = items["input_ids"]
        if not self._needs_autograd():
            if not input_ids.is_cuda:
                raise RuntimeError("openmatch_b200 encodes on a CUDA device only (no CPU path): move the batch to GPU")
            enc = self._cuda_encoder(model, head)
            B, L = input_ids.shape
            if L > PADDED_MAX_LEN:
                return self._encode_long(enc, items, need_hidden)
            max_b = max(1, enc.max_batch_tokens // L)
            hiddens, reps = [], []
            for lo in range(0, B, max_b):
                sl = slice(lo, lo + max_b)
                tt = items.get("token_type_ids", None)
                r = enc.encode(input_ids[sl], items["attention_mask"][sl], tt[sl] if tt is not None else None,
                               return_hidden=need_hidden)
                if need_hidden:
                    hiddens.append(r[0])
                    r = r[1]
                reps.append(r)
            hidden = (torch.cat(hiddens) if len(hiddens) > 1 else hiddens[0]) if need_hidden else None
            return hidden, (torch.cat(reps) if len(reps) > 1 else reps[0])
        # training: HF module under autograd (bf16/fp16 autocast is applied by the trainer)
        out = model(**{k: v for k, v in items.items()}, return_dict=True)
        hidden = getattr(out, self.feature)
        if self.pooling == "first":
            reps = hidden[:, 0, :]
        elif self.pooling == "mean":
            reps = mean_pooling(hidden, items["attention_mask"])
        else:
            raise ValueError("Unknown pooling type: {}".format(self.pooling))
        if head is not None:
            reps = head(reps)
        if self.normalize:
            reps = F.normalize(reps, dim=1)
        return hidden, reps

    @staticmethod
    def _encode_long(enc, items, need_hidden: bool, out: Tensor = None):
        """A padded batch wider than ``PADDED_MAX_LEN`` tokens (each row up to ``encoder.max_seq_len``: 8192 for BERT /
        RoBERTa) is encoded packed, without its padding.  The rows must be right-padded.  ``need_hidden``: the hidden
        states come back ``[B, L, H]`` with the real tokens' rows filled and the padding rows zero (HF computes values
        there that no pooling reads)."""
        input_ids, mask = items["input_ids"], items["attention_mask"]
        m = mask.bool()
        lens = m.sum(1)
        B, L = m.shape
        if not torch.equal(m, torch.arange(L, device=m.device)[None, :] < lens[:, None]):
            raise ValueError("DRModel.encode: attention_mask must be right padding (each row's tokens first)")
        from ..encoder import max_seq_len
        limit = max_seq_len(enc.spec, enc.max_batch_tokens)
        if int(lens.max()) > limit:
            raise ValueError("DRModel.encode: a row of %d tokens exceeds the model's %d" % (int(lens.max()), limit))
        tt = items.get("token_type_ids", None)
        r = enc.encode_packed(input_ids[m], lens.to(torch.int32).cpu(), token_type_ids=tt[m] if tt is not None else None,
                              out=out, return_hidden=need_hidden)
        if not need_hidden:
            return None, r
        hidden = torch.zeros((B, L, enc.hidden), dtype=torch.float32, device=input_ids.device)
        hidden[m] = r[0]
        return hidden, r[1]

    @torch.no_grad()
    def encode_into(self, items, out: Tensor, is_query: bool = False) -> Tensor:
        """Inference only: representations of ``items`` written IN PLACE into ``out`` (fp32 / bf16 / fp16 ``[B, rep_dim]``
        CUDA tensor with unit column stride — e.g. the rows ``FlatIPIndex.reserve_rows`` handed out, int8 rows of an
        int8 index included, which the encoder quantises), no
        intermediate ``[B, d]`` tensor and no copy.  Same arithmetic as ``encode`` (:133-155)."""
        model, head = (self.lm_q, self.head_q) if is_query else (self.lm_p, self.head_p)
        input_ids = items["input_ids"]
        if "T5" in type(model).__name__ and not (self.model_args is not None and self.model_args.encoder_only):
            if out.dtype == torch.int8:
                raise NotImplementedError("encode_into: int8 index rows need the CUDA encoder; encoder-decoder T5 pooling "
                                          "is not on it (use --encoder_only, or an fp32 / fp16 index)")
            out.copy_(self.encode(items, model, head, need_hidden=False)[1])  # encoder-decoder pooling: HF module
            return out
        if not input_ids.is_cuda:
            raise RuntimeError("openmatch_b200 encodes on a CUDA device only (no CPU path): move the batch to GPU")
        enc = self._cuda_encoder(model, head)
        B, L = input_ids.shape
        if out.shape[0] != B or out.shape[1] != enc.rep_dim:
            raise ValueError("out must be [%d, %d], got %s" % (B, enc.rep_dim, tuple(out.shape)))
        if L > PADDED_MAX_LEN:
            self._encode_long(enc, items, False, out=out)
            return out
        max_b = max(1, enc.max_batch_tokens // L)
        tt = items.get("token_type_ids", None)
        for lo in range(0, B, max_b):
            sl = slice(lo, lo + max_b)
            enc.encode(input_ids[sl], items["attention_mask"][sl], tt[sl] if tt is not None else None, out=out[sl])
        return out

    @torch.no_grad()
    def encode_packed_into(self, tokens: Tensor, seqlens, out: Tensor, is_query: bool = False) -> Tensor:
        """Inference only, like ``encode_into``, for a variable-length batch without padding: ``tokens`` int CUDA tensor
        ``[sum(seqlens)]`` (the sequences back to back), ``seqlens`` host lengths (each in [1, ``encoder.max_seq_len``]:
        up to 8192 tokens for BERT / RoBERTa, 512 for T5); the representations
        go IN PLACE into ``out`` ``[len(seqlens), rep_dim]``.  Equal to ``encode_into`` of the same sequences padded, up
        to the order of floating-point sums."""
        model, head = (self.lm_q, self.head_q) if is_query else (self.lm_p, self.head_p)
        if "T5" in type(model).__name__ and not (self.model_args is not None and self.model_args.encoder_only):
            raise NotImplementedError("encode_packed_into: encoder-decoder T5 pooling is not on the CUDA encoder; "
                                      "use --encoder_only or pad the batch")
        if not tokens.is_cuda:
            raise RuntimeError("openmatch_b200 encodes on a CUDA device only (no CPU path): move the batch to GPU")
        self._cuda_encoder(model, head).encode_packed(tokens, seqlens, out=out)
        return out

    def rep_dim(self, is_query: bool = False) -> int:
        """width of the representations ``encode`` produces (head output, else the backbone's hidden size)"""
        head = self.head_q if is_query else self.head_p
        if head is not None:
            return int(head.linear.weight.shape[0])
        lm = self.lm_q if is_query else self.lm_p
        return int(getattr(lm.config, "hidden_size", None) or lm.config.d_model)

    def encode_passage(self, psg):
        return self.encode(psg, self.lm_p, self.head_p)

    def encode_query(self, qry):
        return self.encode(qry, self.lm_q, self.head_q)

    # ------------------------------------------------------------------ build / save
    @classmethod
    def build(cls, model_args: ModelArguments, data_args: DataArguments = None, train_args: TrainingArguments = None,
              **hf_kwargs):
        from transformers import AutoModel, T5EncoderModel
        path = model_args.model_name_or_path
        model_class = T5EncoderModel if model_args.encoder_only else AutoModel
        om_config = None
        cfg_file = os.path.join(path, "openmatch_config.json")
        if os.path.isdir(path) and os.path.exists(cfg_file):
            with open(cfg_file) as f:
                om_config = json.load(f)
        head_q = head_p = None
        if om_config is not None:  # an OpenMatch checkpoint directory
            tied = om_config["tied"]
            if tied:
                lm_q = lm_p = model_class.from_pretrained(path, **hf_kwargs)
                if om_config["linear_head"]:
                    head_q = head_p = LinearHead.load(path)
            else:
                lm_q = model_class.from_pretrained(os.path.join(path, "query_model"), **hf_kwargs)
                lm_p = model_class.from_pretrained(os.path.join(path, "passage_model"), **hf_kwargs)
                if om_config["linear_head"]:
                    head_q = LinearHead.load(os.path.join(path, "query_head"))
                    head_p = LinearHead.load(os.path.join(path, "passage_head"))
        else:  # a plain HuggingFace model
            tied = not model_args.untie_encoder
            lm_q = model_class.from_pretrained(path, **hf_kwargs)
            lm_p = lm_q if tied else copy.deepcopy(lm_q)
            if model_args.add_linear_head:
                head_q = LinearHead(model_args.projection_in_dim, model_args.projection_out_dim)
                head_p = head_q if tied else copy.deepcopy(head_q)
        return cls(lm_q=lm_q, lm_p=lm_p, tied=tied,
                   feature=model_args.feature if om_config is None else om_config["plm_backbone"]["feature"],
                   pooling=model_args.pooling if om_config is None else om_config["pooling"],
                   head_q=head_q, head_p=head_p,
                   normalize=model_args.normalize if om_config is None else om_config["normalize"],
                   model_args=model_args, data_args=data_args, train_args=train_args)

    def save(self, output_dir: str):
        if self.tied:
            self.lm_q.save_pretrained(output_dir)
            if self.head_q is not None:
                self.head_q.save(output_dir)
        else:
            for sub, lm, head in (("query", self.lm_q, self.head_q), ("passage", self.lm_p, self.head_p)):
                os.makedirs(os.path.join(output_dir, sub + "_model"))
                lm.save_pretrained(os.path.join(output_dir, sub + "_model"))
                if head is not None:
                    os.makedirs(os.path.join(output_dir, sub + "_head"))
                    head.save(os.path.join(output_dir, sub + "_head"))
        with open(os.path.join(output_dir, "openmatch_config.json"), "w") as f:
            json.dump(self._get_config_dict(), f, indent=4)

    def dist_gather_tensor(self, t: Optional[torch.Tensor]):
        """All-gather along dim 0 in rank order; the local slice keeps its autograd history so gradients
        flow only to this rank's rows (dense_retrieval_model.py:247-258)."""
        if t is None:
            return None
        t = t.contiguous()
        parts = [torch.empty_like(t) for _ in range(self.world_size)]
        dist.all_gather(parts, t.detach())
        parts[self.process_rank] = t
        return torch.cat(parts, dim=0)


class DRModelForInference(DRModel):
    @torch.no_grad()
    def encode_passage(self, psg):
        return super().encode_passage(psg)

    @torch.no_grad()
    def encode_query(self, qry):
        return super().encode_query(qry)

    @torch.no_grad()
    def forward(self, query: Dict[str, Tensor] = None, passage: Dict[str, Tensor] = None):
        # the retriever only consumes the representations: skip the [B, L, H] last_hidden_state copy
        _, q_reps = self.encode(query, self.lm_q, self.head_q, need_hidden=False)
        _, p_reps = self.encode(passage, self.lm_p, self.head_p, need_hidden=False)
        return DROutput(q_reps=q_reps, p_reps=p_reps)
