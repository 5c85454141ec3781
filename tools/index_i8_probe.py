"""int8 row storage against fp16 row storage, on one GPU.

  python tools/index_i8_probe.py [--steps 5] [--out PATH]

1. C2 shape (8.8 M x 768 corpus, 6 980 queries, k = 1000) on rows that both storages hold exactly (per row: integer
   codes in [-127, 127] with one of them +-127, times 2^-7, so the int8 quantiser and fp16 both reproduce them): an fp16
   index and an int8 index, searched alternately in one process.  Per storage: step ms (host clock around a synchronous
   search, profile off), finalize_ns of one extra profiled step, row bytes (drop of free device memory around the row
   allocation), uncertified queries, and whether D / I are byte-identical between the two.
2. The HBM-bound regime over the same corpora: nq = 1 and nq = 64 at k = 100, alternated, median ms.
3. Synthetic, informational: recall@10 / @1000 of an int8 index against a float32 index of the same anisotropic,
   L2-normalised embeddings (what quantisation costs in ranking, not a speed).
The card's name, power limit and maximum SM clock are read in the same call and reported beside the numbers.  The
whole record is printed as one JSON line at the end, and also written to PATH with --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.index import FlatIPIndex  # noqa: E402

CHUNK = 1 << 20


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": r.stdout.strip().splitlines()[:1]}


def exact_rows(n, d, g):
    """rows both storages hold exactly: codes round(N(0, 1) * 36) clamped to [-127, 127], the row's largest set to
    +-127, times 2^-7"""
    c = torch.clamp(torch.round(torch.randn((n, d), generator=g, device="cuda") * 36), -127, 127)
    j = c.abs().argmax(dim=1)
    sign = torch.where(c[torch.arange(n, device="cuda"), j] < 0, -1.0, 1.0)
    c[torch.arange(n, device="cuda"), j] = 127 * sign
    return (c * 2.0 ** -7).half()


def build(n, d, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = FlatIPIndex(d, dtype=dtype)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    idx.reserve_rows(n)
    torch.cuda.synchronize()
    nbytes = free0 - torch.cuda.mem_get_info()[0]
    for lo in range(0, n, CHUNK):
        idx.add(exact_rows(min(CHUNK, n - lo), d, g))
    torch.cuda.synchronize()
    return idx, nbytes


def queries(nq, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((nq, d), generator=g, device="cuda")


def step(idx, q, k):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    D, I = idx.search_device(q, k)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, D, I


def profiled_finalize_ns(idx, q, k):
    idx.set_param("profile", 1)
    idx.search_device(q, k)
    ns = idx.stat("finalize_ns")
    idx.set_param("profile", 0)
    return ns


def recall_row(n=200_000, d=768, nq=200, seed=3):
    """synthetic anisotropic, normalised embeddings: a few strong directions plus noise"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    scales = torch.exp(-torch.arange(d, device="cuda", dtype=torch.float32) / 64)
    x = torch.nn.functional.normalize(torch.randn((n, d), generator=g, device="cuda") * scales + 0.05, dim=1)
    q = torch.nn.functional.normalize(torch.randn((nq, d), generator=g, device="cuda") * scales + 0.05, dim=1)
    f, i8 = FlatIPIndex(d), FlatIPIndex(d, dtype=torch.int8)
    f.add(x)
    i8.add(x)
    out = {"synthetic": True, "rows": n, "dim": d, "nq": nq}
    for k in (10, 1000):
        If = f.search_device(q, k)[1].cpu()
        Iq = i8.search_device(q, k)[1].cpu()
        hit = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(If, Iq))
        out["recall@%d" % k] = round(hit / (nq * k), 5)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON record to this file")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--c2-rows", type=int, default=8_800_000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    out = {"card": card()}
    n, d, nq, k = a.c2_rows, 768, 6980, 1000
    q = queries(nq, d, 1)
    idx, res = {}, {}
    for name, dt in (("fp16", torch.float16), ("int8", torch.int8)):
        idx[name], nbytes = build(n, d, dt, seed=7)
        res[name] = {"row_bytes": nbytes, "ms": []}
    for name in idx:  # warm-up
        step(idx[name], q, k)
    last = {}
    for _ in range(a.steps):
        for name in idx:
            ms, D, I = step(idx[name], q, k)
            res[name]["ms"].append(round(ms, 2))
            res[name]["uncertified"] = idx[name].stat("uncertified")
            res[name]["exact_queries"] = idx[name].stat("exact_queries")
            last[name] = (D, I)
    for name in idx:
        res[name]["median_ms"] = statistics.median(res[name]["ms"])
        res[name]["finalize_ns"] = profiled_finalize_ns(idx[name], q, k)
    out["c2"] = {"rows": n, "dim": d, "nq": nq, "k": k, "storage": res,
                 "D_identical": torch.equal(last["fp16"][0].view(torch.int32), last["int8"][0].view(torch.int32)),
                 "I_identical": torch.equal(last["fp16"][1], last["int8"][1]),
                 "int8_over_fp16": round(res["int8"]["median_ms"] / res["fp16"]["median_ms"], 3)}
    print(json.dumps(out["c2"]), flush=True)
    del last

    small = {}
    for nqs in (1, 64):
        qs = q[:nqs].contiguous()
        r = {name: [] for name in idx}
        for name in idx:
            step(idx[name], qs, 100)
        for _ in range(max(10, 4 * a.steps)):
            for name in idx:
                r[name].append(step(idx[name], qs, 100)[0])
        small["nq%d" % nqs] = {name: {"median_ms": round(statistics.median(v), 3),
                                      "uncertified": idx[name].stat("uncertified")} for name, v in r.items()}
        small["nq%d" % nqs]["int8_over_fp16"] = round(small["nq%d" % nqs]["int8"]["median_ms"] /
                                                      small["nq%d" % nqs]["fp16"]["median_ms"], 3)
    out["hbm_bound_k100"] = small
    print(json.dumps(small), flush=True)
    del idx
    torch.cuda.empty_cache()
    out["recall_int8_vs_fp32"] = recall_row()
    print(json.dumps(out["recall_int8_vs_fp32"]), flush=True)
    out["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
