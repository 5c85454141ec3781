"""Filtered range search against the unfiltered range search, on one GPU.

  python tools/index_range_filter_probe.py [--steps 3] [--rows 8800000] [--out PATH]

The corpus is the C2 shape (8.8 M x 768 rows, float32 index, N(0, 1) elements) and 6 980 N(0, 1) queries; the radius
of each query is its 1 000th unfiltered score.  In one process, alternating the variants step by step (host clock
around the synchronous call, profile off), median and range of ms per call:
  unfiltered; allow-all bitmap; 50 % and 1 % random bitmaps; 1 % as one contiguous range; 2 excluded ids per query (two
  of its unfiltered top 10).
Bitmaps are packed once, before the timed calls, so the times are the library's.  The same at nq = 1 and 64 with the
radius at the 100th score.  For each variant: the results, the rows re-scored (``range_candidates``), the queries swept
again and those on the exact scan, of its last step.  The card's name, power limit and maximum SM clock are read in the
same call and reported beside the numbers.  The record is printed as one JSON line, and also written to PATH with
--out."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmatch_b200.index import FlatIPIndex, pack_allow  # noqa: E402


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


def variants(n, top, seed):
    """name -> range_search keyword arguments; bitmaps as packed words, exclusions as a device CSR pair"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand(n, device="cuda", generator=g)
    contiguous = torch.zeros(n, dtype=torch.bool, device="cuda")
    contiguous[n // 3:n // 3 + n // 100] = True
    nq = top.shape[0]
    exclude = (torch.arange(0, 2 * nq + 1, 2, device="cuda"), top[:, 3:5].reshape(-1).contiguous())
    return {"unfiltered": {}, "allow_all": {"allow": pack_allow(torch.ones(n, dtype=torch.bool, device="cuda"), n)},
            "random_50pct": {"allow": pack_allow(u < 0.5, n)}, "random_1pct": {"allow": pack_allow(u < 0.01, n)},
            "range_1pct": {"allow": pack_allow(contiguous, n)}, "exclude_2": {"exclude": exclude}}


def measure(idx, q, rho, var, steps):
    for kw in var.values():  # warm-up of every variant
        idx.range_search_device(q, rho, **kw)
    times = {name: [] for name in var}
    for _ in range(steps):
        for name, kw in var.items():
            times[name].append(timed(lambda: idx.range_search_device(q, rho, **kw)))
    out = {}
    for name, kw in var.items():
        lims, _, _ = idx.range_search_device(q, rho, **kw)
        t = times[name]
        out[name] = {"ms_median": statistics.median(t), "ms": [min(t), max(t)], "results": int(lims[-1]),
                     "range_candidates": idx.stat("range_candidates"), "range_resweeps": idx.stat("range_resweeps"),
                     "exact_queries": idx.stat("exact_queries")}
    return out


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
    rec = {"card": card(), "rows": a.rows, "dim": a.dim, "steps": a.steps, "cases": []}
    for nq, k in ((a.nq, 1000), (1, 100), (64, 100)):
        qq = q[:nq].contiguous()
        D, I = idx.search_device(qq, k)
        rho = D[:, k - 1].contiguous()
        var = variants(a.rows, I[:, :10], seed=nq)
        rec["cases"].append({"nq": nq, "radius_at": k, "variants": measure(idx, qq, rho, var, a.steps)})
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
