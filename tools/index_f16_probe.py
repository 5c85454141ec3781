"""fp16 row storage against the default fp32-mastered index, on one GPU.

  python tools/index_f16_probe.py [--steps 3] [--out PATH]

1. C2 shape (8.8 M x 768 corpus, 6 980 queries, k = 1000) on a Gaussian corpus rounded to fp16, so that both storages
   hold the same values: an fp32 index and an fp16 index, searched alternately in one process.  Per storage: step ms
   (host clock around a synchronous search, profile off), finalize_ns of one extra profiled step, index bytes
   (drop of free device memory around the row allocation), and whether D / I are byte-identical between the two.
2. One fp16 index of 21 M x 1024 (43 GB; the fp32 storage would need 129 GB): step ms and the uncertified count.
The card's name and power limit are read in the same call and reported beside the numbers.  The whole record is printed
as one JSON line at the end, and also written to PATH with --out."""
import argparse
import json
import os
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


def build(n, d, dtype, seed):
    """index of n fp16-rounded Gaussian rows (generated on the device in chunks); returns (index, bytes its rows took:
    the drop of free device memory around the one allocation reserve_rows(n) makes)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = FlatIPIndex(d, dtype=dtype)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    idx.reserve_rows(n)
    torch.cuda.synchronize()
    nbytes = free0 - torch.cuda.mem_get_info()[0]
    for lo in range(0, n, CHUNK):
        idx.add(torch.randn((min(CHUNK, n - lo), d), generator=g, device="cuda").half())
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON record to this file")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--c2-rows", type=int, default=8_800_000)
    ap.add_argument("--big-rows", type=int, default=21_000_000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    out = {"card": card()}
    n, d, nq, k = a.c2_rows, 768, 6980, 1000
    q = queries(nq, d, 1)
    idx = {}
    res = {}
    for name, dt in (("fp32", torch.float32), ("fp16", torch.float16)):
        idx[name], nbytes = build(n, d, dt, seed=7)
        res[name] = {"index_bytes": nbytes, "ms": []}
    for name in idx:  # warm-up
        step(idx[name], q, k)
    last = {}
    for _ in range(a.steps):
        for name in idx:
            ms, D, I = step(idx[name], q, k)
            res[name]["ms"].append(round(ms, 2))
            res[name]["uncertified"] = idx[name].stat("uncertified")
            last[name] = (D, I)
    for name in idx:
        res[name]["finalize_ns"] = profiled_finalize_ns(idx[name], q, k)
    same_D = torch.equal(last["fp32"][0].view(torch.int32), last["fp16"][0].view(torch.int32))
    same_I = torch.equal(last["fp32"][1], last["fp16"][1])
    out["c2"] = {"rows": n, "dim": d, "nq": nq, "k": k, "storage": res, "D_identical": same_D, "I_identical": same_I}
    print(json.dumps(out["c2"]), flush=True)
    del idx, last
    torch.cuda.empty_cache()

    n, d = a.big_rows, 1024
    q = queries(nq, d, 2)
    big, nbytes = build(n, d, torch.float16, seed=8)
    step(big, q, k)
    ms = []
    for _ in range(a.steps):
        ms.append(round(step(big, q, k)[0], 2))
    out["fp16_21m_1024"] = {"rows": n, "dim": d, "nq": nq, "k": k, "index_bytes": nbytes, "ms": ms,
                            "uncertified": big.stat("uncertified"), "exact_queries": big.stat("exact_queries")}
    print(json.dumps(out["fp16_21m_1024"]), flush=True)
    out["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
