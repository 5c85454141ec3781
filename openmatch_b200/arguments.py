"""Argument dataclasses with the reference's flag names and defaults (``src/openmatch/arguments.py``).

The reference derives its runtime arguments from HF ``TrainingArguments``; that class cannot even be
constructed on this image (it hard-requires ``accelerate``), and the hot path only reads a dozen of its
attributes.  ``RuntimeArguments`` is a standalone dataclass exposing exactly those attributes
(``device, world_size, process_index, local_process_index, fp16, bf16, per_device_*_batch_size,
dataloader_*, output_dir, seed, learning_rate, warmup_ratio, num_train_epochs, save_steps, logging_dir``
...), parsed by ``HfArgumentParser`` like the original, and it initialises ``torch.distributed`` (NCCL, one
process per GPU) when launched under ``torchrun``.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import List, Optional

import torch


@dataclass
class ModelArguments:
    model_name_or_path: str = field(metadata={"help": "HF model id or local (HF / OpenMatch) checkpoint dir"})
    target_model_path: str = field(default=None, metadata={"help": "re-ranker target model (unused by DR)"})
    config_name: Optional[str] = field(default=None, metadata={"help": "config name/path if different"})
    tokenizer_name: Optional[str] = field(default=None, metadata={"help": "tokenizer name/path if different"})
    cache_dir: Optional[str] = field(default=None, metadata={"help": "HF cache directory"})
    untie_encoder: bool = field(default=False, metadata={"help": "separate query / passage encoders"})
    feature: str = field(default="last_hidden_state", metadata={"help": "HF output field to pool"})
    pooling: str = field(default="first", metadata={"help": "'first' (CLS) or 'mean'"})
    add_linear_head: bool = field(default=False)
    projection_in_dim: int = field(default=768)
    projection_out_dim: int = field(default=768)
    dtype: Optional[str] = field(default="float32", metadata={"help": "kept for CLI compatibility"})
    encoder_only: bool = field(default=False, metadata={"help": "use only the encoder of a T5 checkpoint"})
    pos_token: Optional[str] = field(default=None)
    neg_token: Optional[str] = field(default=None)
    normalize: bool = field(default=False, metadata={"help": "L2-normalise the embeddings"})


@dataclass
class DataArguments:
    train_dir: str = field(default=None)
    train_path: str = field(default=None)
    eval_path: str = field(default=None)
    query_path: str = field(default=None)
    corpus_path: str = field(default=None)
    data_dir: str = field(default=None)
    data_path: str = field(default=None)
    processed_data_path: str = field(default=None)
    dataset_name: str = field(default=None)
    passage_field_separator: str = field(default=' ')
    dataset_proc_num: int = field(default=12)
    train_n_passages: int = field(default=8)
    positive_passage_no_shuffle: bool = field(default=False)
    negative_passage_no_shuffle: bool = field(default=False)
    encode_in_path: List[str] = field(default=None)
    encode_is_qry: bool = field(default=False)
    encode_num_shard: int = field(default=1)
    encode_shard_index: int = field(default=0)
    q_max_len: int = field(default=32, metadata={"help": "query length after tokenisation (pad / truncate)"})
    p_max_len: int = field(default=128, metadata={"help": "passage length after tokenisation (pad / truncate)"})
    data_cache_dir: Optional[str] = field(default=None)
    query_template: str = field(default="<text>")
    query_column_names: str = field(default="id,text")
    doc_template: str = field(default="Title: <title> Text: <text>")
    doc_column_names: str = field(default="id,title,text")


@dataclass
class RuntimeArguments:
    """The subset of HF ``TrainingArguments`` the dense-retrieval path reads, same names and defaults."""
    output_dir: str = field(default=None, metadata={"help": "where embeddings / checkpoints are written"})
    overwrite_output_dir: bool = field(default=False)
    do_train: bool = field(default=False)
    do_eval: bool = field(default=False)
    per_device_train_batch_size: int = field(default=8)
    per_device_eval_batch_size: int = field(default=8)
    gradient_accumulation_steps: int = field(default=1)
    learning_rate: float = field(default=5e-5)
    weight_decay: float = field(default=0.0)
    adam_beta1: float = field(default=0.9)
    adam_beta2: float = field(default=0.999)
    adam_epsilon: float = field(default=1e-8)
    max_grad_norm: float = field(default=1.0)
    num_train_epochs: float = field(default=3.0)
    max_steps: int = field(default=-1)
    warmup_ratio: float = field(default=0.0)
    warmup_steps: int = field(default=0)
    logging_dir: Optional[str] = field(default=None)
    logging_steps: int = field(default=500)
    save_steps: int = field(default=500)
    seed: int = field(default=42)
    fp16: bool = field(default=False)
    bf16: bool = field(default=False)
    local_rank: int = field(default=-1)
    dataloader_num_workers: int = field(default=0)
    dataloader_pin_memory: bool = field(default=True)
    dataloader_drop_last: bool = field(default=False)
    remove_unused_columns: Optional[bool] = field(default=False)
    no_cuda: bool = field(default=False)

    def __post_init__(self):
        env_rank = int(os.environ.get("LOCAL_RANK", -1))
        if env_rank != -1 and self.local_rank == -1:
            self.local_rank = env_rank
        self._dist_ready = False

    # ---- distributed state (NCCL, one process per GPU) ----
    def _setup(self):
        if self._dist_ready:
            return
        self._dist_ready = True
        if int(os.environ.get("WORLD_SIZE", "1")) > 1 and not torch.distributed.is_initialized():
            if torch.cuda.is_available():
                torch.cuda.set_device(max(self.local_rank, 0))
            torch.distributed.init_process_group(backend="nccl" if torch.cuda.is_available() else "gloo")

    @property
    def device(self) -> torch.device:
        self._setup()
        if torch.cuda.is_available() and not self.no_cuda:
            return torch.device("cuda", max(self.local_rank, 0) if self.local_rank != -1 else torch.cuda.current_device())
        return torch.device("cpu")

    @property
    def world_size(self) -> int:
        self._setup()
        return torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1

    @property
    def process_index(self) -> int:
        self._setup()
        return torch.distributed.get_rank() if torch.distributed.is_initialized() else 0

    @property
    def local_process_index(self) -> int:
        return max(self.local_rank, 0)

    @property
    def n_gpu(self) -> int:
        return 1 if torch.cuda.is_available() and not self.no_cuda else 0

    @property
    def should_save(self) -> bool:
        return self.process_index == 0


@dataclass
class DRTrainingArguments(RuntimeArguments):
    warmup_ratio: float = field(default=0.1)
    negatives_x_device: bool = field(default=False, metadata={"help": "share negatives across devices"})
    do_encode: bool = field(default=False)
    grad_cache: bool = field(default=False, metadata={"help": "gradient-cache update (not available: needs grad_cache)"})
    gc_q_chunk_size: int = field(default=4)
    gc_p_chunk_size: int = field(default=32)


@dataclass
class InferenceArguments(RuntimeArguments):
    use_gpu: bool = field(default=False, metadata={"help": "kept for CLI compatibility: the index always lives in HBM"})
    encoded_save_path: str = field(default=None)
    trec_save_path: str = field(default=None)
    trec_run_path: str = field(default=None)
    id_key_name: str = field(default="id")
    retrieve_depth: int = field(default=100, metadata={"help": "top-k for driver.retrieve (reference hard-codes 100)"})
    reranking_depth: int = field(default=None, metadata={"help": "driver.rerank: documents per query of the run to "
                                                                   "re-rank (default: all)"})
    index_dtype: str = field(default="float32", metadata={
        "help": "row storage of the search index: 'float32' (fp32 rows + fp16 scan copy, 6 bytes per element), "
                "'float16' (fp16 rows only, 2 bytes per element; search is exact over the fp16-rounded rows) or 'int8' "
                "(one byte per element + a per-row scale; search is exact over the dequantised rows)"})
    index_memory: str = field(default="device", metadata={
        "help": "where the search index keeps its rows: 'device' (GPU memory) or 'host' (pinned host memory, streamed "
                "through the GPU by every search, for corpora larger than the GPU's memory; one process, built from "
                "embedding files by driver.retrieve; results are bitwise those of 'device')"})
