"""Build-index throughput through the public API (SURVEY 8(f1)): a synthetic PRE-TOKENISED corpus (int32 .npy memory map,
`PretokenizedDataset`) -> `Retriever.build_all` (block ingest: pinned staging, async H2D, sm_90a encoder writing straight
into the HBM index shard) -> reference-format embedding file.  Prints one JSON line.
  python tools/ingest_bench.py [n_passages=1000000] [batch=256] [L=128]
"""
import json
import os
import sys
import tempfile
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transformers import BertConfig, BertModel  # noqa: E402

from openmatch_b200.arguments import DataArguments, ModelArguments  # noqa: E402
from openmatch_b200.dataset import InferenceDataset  # noqa: E402
from openmatch_b200.modeling import DRModelForInference  # noqa: E402
from openmatch_b200.retriever import Retriever  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
bs = int(sys.argv[2]) if len(sys.argv) > 2 else 256
L = int(sys.argv[3]) if len(sys.argv) > 3 else 128
tmp = tempfile.mkdtemp(prefix="om_ingest_")
rng = np.random.default_rng(0)
ids = rng.integers(1000, 30000, (n, L), dtype=np.int32)
ids[:, 0] = 101
ids[:, -1] = 102
np.save(os.path.join(tmp, "corpus.npy"), ids)
del ids
torch.manual_seed(0)
lm = BertModel(BertConfig(), add_pooling_layer=False)
model = DRModelForInference(lm_q=lm, lm_p=lm, tied=True, pooling="first", model_args=ModelArguments(model_name_or_path="unused"))
dargs = DataArguments(corpus_path=os.path.join(tmp, "corpus.npy"), p_max_len=L)
args = types.SimpleNamespace(device=torch.device("cuda"), fp16=False, bf16=False, per_device_eval_batch_size=bs,
                             dataloader_num_workers=0, dataloader_pin_memory=False, output_dir=os.path.join(tmp, "emb"),
                             process_index=0, local_process_index=1, world_size=1, use_gpu=True)  # local_process_index 1: no tqdm
ds = InferenceDataset.load(None, dargs, is_query=False, batch_size=bs)
ret = Retriever(model, ds, args)
# warm-up: weights hand-over + first launches
w = InferenceDataset.load(None, DataArguments(corpus_path=os.path.join(tmp, "corpus.npy"), p_max_len=L), batch_size=bs)
w.iter_batches = lambda it=w.iter_batches: (b for i, b in enumerate(it()) if i < 4)
ret._encode_dataset(w, is_query=False, into_index=True)
ret.reset_index()
torch.cuda.synchronize()
t0 = time.perf_counter()
names, _ = ret._encode_dataset(ds, is_query=False, into_index=True)
torch.cuda.synchronize()
t1 = time.perf_counter()
assert ret.index.ntotal == n == len(names)
ret.doc_lookup = list(names)
from openmatch_b200.embedding_store import write_embedding_file  # noqa: E402
os.makedirs(args.output_dir, exist_ok=True)
write_embedding_file(os.path.join(args.output_dir, "embeddings.corpus.rank.0"), ret.index.master_rows(), names)
t2 = time.perf_counter()
print(json.dumps({"what": "Retriever block ingest: int32 memmap -> pinned -> H2D -> bert-base encoder -> index rows in place",
                  "passages": n, "batch": bs, "L": L, "encode_into_index_s": t1 - t0,
                  "passages_per_s": n / (t1 - t0), "embedding_file_write_s": t2 - t1,
                  "embedding_file_gb": n * 768 * 4 / 1e9}))
