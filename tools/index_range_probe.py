"""Range search against search(k), on one GPU.

  python tools/index_range_probe.py [--steps 3] [--rows 8800000] [--out PATH]

The corpus is the C2 shape (8.8 M x 768 rows, float32 index, N(0, 1) elements) and 6 980 N(0, 1) queries.  For k =
100, 1 000 and 10 000 the radius of query i is the k-th score of a prior search(q, k) (k = 10 000: the 10 000-th score
of a range search at 0.9 x the 4 096-th, compared with search(q, 4096), since search takes k <= 4 096), so range search
returns k rows per query.  In one process, alternating range_search and search(k) step by step (host clock around a synchronous call,
profile off), median and range of ms per call.  Long lists: nq = 1 and 8 at radius -inf (every row of the
corpus per query).  Streaming: nq = 1 and 64 with the radius at the 100th score.  The
card's name, power limit and maximum SM clock are read in the same call and reported beside the numbers.  The record is
printed as one JSON line, and also written to PATH with --out."""
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": r.stdout.strip().splitlines()[:1]}


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rows", type=int, default=8_800_000)
    ap.add_argument("--nq", type=int, default=6980)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    g = torch.Generator(device="cuda").manual_seed(0)
    idx = FlatIPIndex(a.dim)
    idx.reserve_rows(a.rows)  # capacity only: no re-allocation while adding
    for lo in range(0, a.rows, 1 << 20):
        idx.add(torch.randn(min(1 << 20, a.rows - lo), a.dim, device="cuda", generator=g))
    q = torch.randn(a.nq, a.dim, device="cuda", generator=g)
    rec = {"card": card(), "rows": a.rows, "dim": a.dim, "cases": []}
    cases = [(a.nq, 100), (a.nq, 1000), (a.nq, 10000), (1, 100), (64, 100)]
    for nq, k in cases:
        qq = q[:nq].contiguous()
        ks = min(k, 4096)
        D, _ = idx.search_device(qq, ks)
        rho = D[:, ks - 1].contiguous()
        if k > ks:  # the k-th score, from a range search below the 4096-th (top scores are positive)
            lims, Dr, _ = idx.range_search_device(qq, 0.9 * rho)
            assert bool((lims[1:] - lims[:-1] >= k).all()), "0.9 x the 4096-th score holds fewer than k rows"
            rho = Dr[lims[:-1] + (k - 1)].contiguous()
        idx.range_search_device(qq, rho)  # warm-up of both calls
        idx.search_device(qq, ks)
        tr, ts = [], []
        for _ in range(a.steps):
            tr.append(timed(lambda: idx.range_search_device(qq, rho)))
            ts.append(timed(lambda: idx.search_device(qq, ks)))
        lims, _, _ = idx.range_search_device(qq, rho)
        rec["cases"].append({
            "nq": nq, "k": k, "search_k": ks, "results": int(lims[-1]),
            "range_ms_median": statistics.median(tr), "range_ms": [min(tr), max(tr)],
            "search_ms_median": statistics.median(ts), "search_ms": [min(ts), max(ts)],
            "range_candidates": idx.stat("range_candidates"), "range_resweeps": idx.stat("range_resweeps"),
            "exact_queries": idx.stat("exact_queries")})
    # a few queries with very long lists (every row passes): the re-score, sort and gather of a handful of queries
    for nq in (1, 8):
        qq = q[:nq].contiguous()
        rho = torch.full((nq,), float("-inf"), device="cuda")
        idx.range_search_device(qq, rho)
        tr = [timed(lambda: idx.range_search_device(qq, rho)) for _ in range(a.steps)]
        rec["cases"].append({"nq": nq, "radius": "-inf", "results": nq * a.rows, "range_ms_median": statistics.median(tr),
                             "range_ms": [min(tr), max(tr)], "range_resweeps": idx.stat("range_resweeps")})
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
