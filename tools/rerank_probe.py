"""Probe (not part of the product): cross-encoder scoring of re-ranking batches, three ways, on two backbones.

  python tools/rerank_probe.py [rounds] [out.json]

Backbones (randomly initialised HF BertModel, 'first' pooling, LinearHead(H, 1); both sides use the same weights):
  bert-base  H 768, 12 layers, 12 x 64-wide heads, F 3072
  MiniLM-L6  H 384, 6 layers, 12 x 32-wide heads, F 1536
Batches: B = 256 pairs (8 queries x 32 passages), query lengths uniform in [4, 32], passage lengths clip(N(0.55 L,
0.2 L), 8, L) at L = 128, [CLS] q p [SEP]; fixed seeds.  Contenders, per batch:
  hf_bf16_sdpa     eager HF in bf16 autocast with SDPA attention on the reference's padded pairs (encode_pair:
                   q_max_len + p_max_len + 2 = 162 tokens), already on the device, then pooling and head
  host_packed      the pairs assembled on the host from the token stores, copied to the device, om_encode_packed
  om_encode_pairs  the pairs assembled on the device from the token stores (uploaded once per re-rank call, outside
                   the timed region) by om_encode_pairs
Each round times every contender once (host clock around a device synchronise, the order rotating from round to
round) after a warm-up; reported are medians of the rounds as pairs/s, whether host_packed and om_encode_pairs give
byte-identical scores, and the deviation of HF's scores from om_encode_pairs'.  The card's name, power limit and max SM
clock are read in the same process (read-only query)."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.encoder import CudaEncoder  # noqa: E402
from openmatch_b200.retriever.reranker import assemble_pairs  # noqa: E402

NQ, NP, Q_MAX, P_MAX = 8, 32, 32, 128
B = NQ * NP
CLS, SEP = 101, 102
BACKBONES = {"bert-base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072),
             "MiniLM-L6": dict(hidden_size=384, num_hidden_layers=6, num_attention_heads=12, intermediate_size=1536)}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip().splitlines()[:1]
    except (OSError, subprocess.SubprocessError):
        smi = []
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": smi}


def make_batch(seed):
    rng = np.random.default_rng(seed)
    qlens = rng.integers(4, Q_MAX + 1, NQ)
    plens = np.clip(np.round(rng.standard_normal(NP) * 0.2 * P_MAX + 0.55 * P_MAX), 8, P_MAX).astype(np.int64)
    a = rng.integers(1000, 30000, int(qlens.sum())).astype(np.int32)
    b = rng.integers(1000, 30000, int(plens.sum())).astype(np.int32)
    qoff = np.concatenate([[0], np.cumsum(qlens)[:-1]])
    poff = np.concatenate([[0], np.cumsum(plens)[:-1]])
    spans = np.array([(qoff[i], qlens[i], poff[j], plens[j]) for i in range(NQ) for j in range(NP)], dtype=np.int64)
    return a, b, spans


def main():
    from transformers import BertConfig, BertModel

    from openmatch_b200.modeling.linear import LinearHead
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    out_path = sys.argv[2] if len(sys.argv) > 2 else None
    info = gpu_info()
    a, b, spans = make_batch(7)
    tokens, lens = assemble_pairs(a, b, spans, [CLS], [SEP])
    L = Q_MAX + P_MAX + 2
    ids = torch.zeros(B, L, dtype=torch.long)
    for i, row in enumerate(np.split(tokens, np.cumsum(lens)[:-1])):
        ids[i, :len(row)] = torch.from_numpy(row)
    ids = ids.cuda()
    mask = (ids != 0).long()
    tt = torch.zeros_like(ids)
    records = []
    for name, shape in BACKBONES.items():
        torch.manual_seed(0)
        cfg = BertConfig(vocab_size=30522, max_position_embeddings=512, attn_implementation="sdpa", **shape)
        lm = BertModel(cfg).cuda().eval()
        head = LinearHead(cfg.hidden_size, 1).cuda()
        enc = CudaEncoder.from_hf(lm, head, pooling="first", normalize=False, max_batch_tokens=256 * 256)
        ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()

        def hf():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                h = lm(input_ids=ids, attention_mask=mask, token_type_ids=tt).last_hidden_state
                return head(h[:, 0].float())[:, 0].float()

        def host_packed():
            t, ln = assemble_pairs(a, b, spans, [CLS], [SEP])
            return enc.encode_packed(torch.from_numpy(t).cuda(), ln)[:, 0]

        def pairs():
            return enc.encode_pairs(ad, bd, spans, [CLS], [SEP])[:, 0]

        runs = {"hf_bf16_sdpa": hf, "host_packed": host_packed, "om_encode_pairs": pairs}
        names, outs = list(runs), {}
        for _ in range(3):
            for n in names:
                outs[n] = runs[n]()
        torch.cuda.synchronize()
        times = {n: [] for n in names}
        for r in range(rounds):
            for n in names[r % len(names):] + names[:r % len(names)]:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[n] = runs[n]()
                torch.cuda.synchronize()
                times[n].append((time.perf_counter() - t0) * 1e3)
        c = outs["om_encode_pairs"].double()
        h = outs["hf_bf16_sdpa"].double()
        rec = dict(backbone=name, shape=shape, B=B, assembled_tokens=int(lens.sum()), padded_tokens=B * L, rounds=rounds,
                   packed_vs_pairs_byte_identical=bool(torch.equal(outs["host_packed"], outs["om_encode_pairs"])),
                   hf_max_abs_dev_over_max_abs=float((h - c).abs().max() / c.abs().max()),
                   hf_rel_l2=float((h - c).norm() / c.norm()))
        for n in names:
            ms = float(np.median(times[n]))
            rec["ms_" + n] = ms
            rec["pairs_per_s_" + n] = B / ms * 1e3
            rec["ms_minmax_" + n] = [min(times[n]), max(times[n])]
        for n in ("host_packed", "om_encode_pairs"):
            rec["speedup_vs_hf_" + n] = rec["ms_hf_bf16_sdpa"] / rec["ms_" + n]
        records.append(rec)
        del lm, head, enc
        torch.cuda.empty_cache()
    result = {"gpu": info, "records": records}
    print(json.dumps(result))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
