"""Probe (not part of the product): MPNet and DistilBERT encoders on the CUDA encoder against eager HF.

  python tools/encode_mpnet_probe.py [rounds] [out.json]

Randomly initialised HF models, each used by both sides, with the pooling their retrievers use:
  all-mpnet-base-v2  MPNet, 12 layers, hidden 768, 12 x 64-wide heads, FFN 3072, vocab 30 527, 514 positions;
                     mean pooling + normalise
  tas-b              DistilBERT, 6 layers of the same width, vocab 30 522, 512 positions; first-token pooling
  bert-base          BERT, 12 layers of the same width, vocab 30 522; mean pooling + normalise (the yardstick: the
                     GEMMs are MPNet's, attention has no bias)
B = 256, two regimes:
  full128    every sequence 128 tokens: om_encode (CudaEncoder.encode) vs HF on [B, 128]
  ragged128  lengths ~ clip(N(0.55 L, 0.2 L), 8, L) at L = 128, right-padded with the model's pad id: om_encode_packed
             (CudaEncoder.encode_packed) and om_encode on the padded batch vs HF on the padded batch
Ids are <s> / [CLS] first, then ids >= 4.  HF is the eager module in bf16 autocast (MPNet's attention is an explicit
matmul because of its bias; DistilBERT and BERT use SDPA), followed by the same pooling and normalisation.  After a
warm-up, every round times each contender once (CUDA events, the order rotating from round to round); reported are the
medians as passages/s and the max rel-L2 of each CUDA path's reps against HF's.  The card's name and power limit are
read in the same process (read-only query)."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.encoder import CudaEncoder  # noqa: E402

B, L = 256, 128


def make_model(name):
    """(HF module, pooling, normalize, first id, pad id) of probe model ``name``"""
    torch.manual_seed(0)
    if name == "all-mpnet-base-v2":
        from transformers import MPNetConfig, MPNetModel
        cfg = MPNetConfig(vocab_size=30527, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                          intermediate_size=3072, max_position_embeddings=514, layer_norm_eps=1e-5)
        return MPNetModel(cfg), "mean", True, 0, 1
    if name == "tas-b":
        from transformers import DistilBertConfig, DistilBertModel
        cfg = DistilBertConfig(vocab_size=30522, dim=768, n_layers=6, n_heads=12, hidden_dim=3072,
                               max_position_embeddings=512, attn_implementation="sdpa")
        return DistilBertModel(cfg), "first", False, 101, 0
    from transformers import BertConfig, BertModel
    cfg = BertConfig(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                     intermediate_size=3072, max_position_embeddings=512, attn_implementation="sdpa")
    return BertModel(cfg), "mean", True, 101, 0


MODELS = ("all-mpnet-base-v2", "tas-b", "bert-base")


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        smi = r.stdout.strip().splitlines()[:1]
    except (OSError, subprocess.SubprocessError):
        smi = []
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": smi}


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    out_path = sys.argv[2] if len(sys.argv) > 2 else None
    info = gpu_info()
    records = []
    for model_name in MODELS:
        lm, pooling, normalize, first, pad = make_model(model_name)
        lm = lm.cuda().eval()
        enc = CudaEncoder.from_hf(lm, pooling=pooling, normalize=normalize, max_batch_tokens=B * L)
        vocab, layers = lm.config.vocab_size, enc.spec["layers"]

        def hf(ids, mask):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                h = lm(input_ids=ids, attention_mask=mask).last_hidden_state.float()
            if pooling == "first":
                r = h[:, 0]
            else:
                m = mask.unsqueeze(-1).float()
                r = (h * m).sum(1) / m.sum(1).clamp(min=1e-9)
            return torch.nn.functional.normalize(r, dim=1) if normalize else r

        rng = np.random.default_rng(7)
        for regime in ("full128", "ragged128"):
            if regime == "full128":
                lens = np.full(B, L, dtype=np.int32)
            else:
                lens = np.clip(np.round(rng.standard_normal(B) * 0.2 * L + 0.55 * L), 8, L).astype(np.int32)
            ids = torch.randint(4, vocab, (B, L), generator=torch.Generator().manual_seed(1))
            ids[:, 0] = first
            mask = (torch.arange(L)[None] < torch.from_numpy(lens).long()[:, None]).long()
            ids = torch.where(mask.bool(), ids, torch.full_like(ids, pad)).cuda()
            mask = mask.cuda()
            tokens = ids[mask.bool()]
            outs = {}
            runs = {"hf_bf16": lambda: outs.__setitem__("hf_bf16", hf(ids, mask)),
                    "om_encode": lambda: outs.__setitem__("om_encode", enc.encode(ids, mask))}
            if regime == "ragged128":
                runs["om_encode_packed"] = lambda: outs.__setitem__("om_encode_packed", enc.encode_packed(tokens, lens))
            names = list(runs)
            for _ in range(3):
                for n in names:
                    runs[n]()
            torch.cuda.synchronize()
            times = {n: [] for n in names}
            for r in range(rounds):
                order = names[r % len(names):] + names[:r % len(names)]
                ev = {n: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for n in names}
                for n in order:
                    ev[n][0].record()
                    runs[n]()
                    ev[n][1].record()
                torch.cuda.synchronize()
                for n in names:
                    times[n].append(ev[n][0].elapsed_time(ev[n][1]))
            ref = outs["hf_bf16"].double()
            rec = dict(model="%s shape (H 768, 12 x 64-wide heads, F 3072, %d layers, vocab %d, %s pooling%s)"
                       % (model_name, layers, vocab, pooling, " + normalise" if normalize else ""),
                       regime=regime, B=B, L=L, real_tokens=int(lens.sum()), rounds=rounds)
            for n in names:
                ms = float(np.median(times[n]))
                rec["ms_" + n] = ms
                rec["passages_per_s_" + n] = B / ms * 1e3
                rec["ms_minmax_" + n] = [min(times[n]), max(times[n])]
                if n != "hf_bf16":
                    d = outs[n].double()
                    rec["reps_max_rel_l2_vs_hf_" + n] = float(((d - ref).norm(dim=1) / ref.norm(dim=1)).max())
                    rec["speedup_vs_hf_" + n] = rec["ms_hf_bf16"] / ms
            records.append(rec)
        del enc, lm
        torch.cuda.empty_cache()
    result = {"gpu": info, "records": records}
    print(json.dumps(result))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
