"""Probe (not part of the product): padded om_encode vs packed om_encode_packed on the same sequences.

  python tools/encode_packed_probe.py [rounds] [out.json]

bert-base and t5-base (GTR: mean pooling, head, normalise), B = 256, synthetic weights, three length regimes:
  ragged128  the ragged regime of synthetic.token_batch(ragged=True) at L = 128 (lengths ~ clip(N(0.55 L, 0.2 L), 8, L))
  doc512     a document-like mix up to 512: lengths ~ clip(lognormal around 180, 16, 512), padded to L = 512
  full128    every sequence 128 tokens (the worst case: packing can only add its overhead)
After a warm-up, each round times one padded call and one packed call (CUDA events, alternating order), several rounds;
reported are the median times as passages/s and real tokens/s, layout rows per real token of both paths, and the max
rel-L2 between the two paths' reps.  The card's name and power limit are read in the same process (read-only query)."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200 import synthetic  # noqa: E402
from openmatch_b200.encoder import CudaEncoder  # noqa: E402

B = 256


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        smi = r.stdout.strip().splitlines()[:1]
    except (OSError, subprocess.SubprocessError):
        smi = []
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": smi}


def lengths(regime, rng):
    if regime == "ragged128":
        return 128, np.clip(np.round(rng.standard_normal(B) * 0.2 * 128 + 0.55 * 128), 8, 128).astype(np.int32)
    if regime == "doc512":
        return 512, np.clip(np.round(rng.lognormal(np.log(180), 0.6, B)), 16, 512).astype(np.int32)
    return 128, np.full(B, 128, dtype=np.int32)


def layout_rows(lens):
    """rows of the packed layout (the same placement rule as csrc/encoder.cu: first-fit decreasing into 128-row tiles,
    longer sequences on whole tiles)"""
    long_rows = int(sum(-(-l // 128) * 128 for l in lens if l > 128))
    fill = []
    for l in sorted((int(l) for l in lens if l <= 128), reverse=True):
        for i, f in enumerate(fill):
            if f + l <= 128:
                fill[i] += l
                break
        else:
            fill.append(l)
    return long_rows + 128 * len(fill)


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    out_path = sys.argv[2] if len(sys.argv) > 2 else None
    info = gpu_info()
    print("GPU:", info, flush=True)
    rng = np.random.default_rng(7)
    records = []
    for arch in ("bert", "t5"):
        if arch == "t5":
            spec = dict(synthetic.T5_BASE)
            enc = CudaEncoder(spec, synthetic.t5_state_dict(spec, seed=0), head_weight=torch.randn(768, 768) * 0.03,
                              pooling="mean", normalize=True, max_batch_tokens=B * 512)
        else:
            spec = dict(synthetic.BERT_BASE)
            if spec.get("max_pos", 512) < 512:
                spec["max_pos"] = 512
            enc = CudaEncoder(spec, synthetic.bert_state_dict(spec, seed=0), pooling="first", max_batch_tokens=B * 512)
        for regime in ("ragged128", "doc512", "full128"):
            L, lens = lengths(regime, rng)
            ids = torch.randint(1000, spec["vocab"], (B, L), generator=torch.Generator().manual_seed(1))
            mask = (torch.arange(L)[None] < torch.from_numpy(lens).long()[:, None]).long()
            ids = ids * mask
            d_ids, d_mask = ids.cuda(), mask.cuda()
            tokens = ids[mask.bool()].cuda()
            out_pad = torch.empty(B, enc.rep_dim, device="cuda")
            out_pk = torch.empty(B, enc.rep_dim, device="cuda")
            for _ in range(3):
                enc.encode(d_ids, d_mask, out=out_pad)
                enc.encode_packed(tokens, lens, out=out_pk)
            torch.cuda.synchronize()
            t_pad, t_pk = [], []
            for r in range(rounds):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                order = (0, 1) if r % 2 == 0 else (1, 0)
                for which in order:
                    e0, e1 = ev[2 * which], ev[2 * which + 1]
                    e0.record()
                    if which == 0:
                        enc.encode(d_ids, d_mask, out=out_pad)
                    else:
                        enc.encode_packed(tokens, lens, out=out_pk)
                    e1.record()
                torch.cuda.synchronize()
                t_pad.append(ev[0].elapsed_time(ev[1]))
                t_pk.append(ev[2].elapsed_time(ev[3]))
            a, b = out_pad.double(), out_pk.double()
            rel = float(((a - b).norm(dim=1) / a.norm(dim=1).clamp_min(1e-30)).max())
            real = int(lens.sum())
            ms_pad, ms_pk = float(np.median(t_pad)), float(np.median(t_pk))
            rec = dict(arch=arch, regime=regime, B=B, L=L, real_tokens=real, rows_per_token_padded=B * L / real,
                       rows_per_token_packed=layout_rows(lens) / real, ms_padded=ms_pad, ms_packed=ms_pk,
                       passages_per_s_padded=B / ms_pad * 1e3, passages_per_s_packed=B / ms_pk * 1e3,
                       tokens_per_s_padded=real / ms_pad * 1e3, tokens_per_s_packed=real / ms_pk * 1e3,
                       speedup=ms_pad / ms_pk, reps_max_rel_l2=rel, rounds=rounds,
                       ms_padded_minmax=[min(t_pad), max(t_pad)], ms_packed_minmax=[min(t_pk), max(t_pk)])
            records.append(rec)
            print(json.dumps(rec), flush=True)
    result = {"gpu": info, "records": records}
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
