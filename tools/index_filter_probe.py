"""Filtered search against the unfiltered search, on one GPU.

  python tools/index_filter_probe.py [--steps 3] [--out PATH]

The corpus is the C2 shape (8.8 M x 768 rows, float32 index, N(0, 1) elements) with 8 near-duplicates of each of the
6 980 queries (the query scaled by 4 plus noise of 1e-3) written at random rows: 55 840 rows, 0.63 % of the corpus,
that are the top scorers of their query.  In one process, alternating the variants step by step (host clock around a
synchronous search, profile off), median ms per variant:
  unfiltered; allow-all bitmap; 50 % and 1 % random bitmaps; 1 % as one contiguous range; 2 excluded ids per query (two
  of its unfiltered top 10); adversarial: a bitmap that disallows exactly the near-duplicates.
At nq = 6 980 / k = 1 000 and at nq = 1 and 64 with k = 100.  For each variant the uncertified and exact-scan query
counts of its last step are reported.  The card's name, power limit and maximum SM clock are read in the same call and
reported beside the numbers.  The record is printed as one JSON line, and also written to PATH with --out."""
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
DUPS = 8


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": r.stdout.strip().splitlines()[:1]}


def build(n, d, q, seed):
    """the index, and the rows holding near-duplicates of the queries (bool [n] on the device)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    nq = q.shape[0]
    dup_rows = torch.randperm(n, generator=g, device="cuda")[:DUPS * nq]
    dup_of = torch.arange(DUPS * nq, device="cuda") % nq
    is_dup = torch.zeros(n, dtype=torch.bool, device="cuda")
    is_dup[dup_rows] = True
    idx = FlatIPIndex(d)
    idx.reserve_rows(n)
    for lo in range(0, n, CHUNK):
        hi = min(n, lo + CHUNK)
        x = torch.randn((hi - lo, d), generator=g, device="cuda")
        sel = (dup_rows >= lo) & (dup_rows < hi)
        x[dup_rows[sel] - lo] = 4 * q[dup_of[sel]] + 1e-3 * torch.randn((int(sel.sum()), d), generator=g, device="cuda")
        idx.add(x)
    torch.cuda.synchronize()
    return idx, is_dup


def step(idx, q, k, kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx.search_device(q, k, **kw)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def variants(n, q, idx, is_dup, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    top = idx.search_device(q, 10)[1]
    rng = torch.rand(n, generator=g, device="cuda")
    rng_range = torch.zeros(n, dtype=torch.bool, device="cuda")
    rng_range[n // 3:n // 3 + n // 100] = True
    exclude = (torch.arange(0, 2 * q.shape[0] + 1, 2, device="cuda"), top[:, 3:5].reshape(-1).contiguous())
    return {"unfiltered": {}, "allow_all": {"allow": torch.ones(n, dtype=torch.bool, device="cuda")},
            "random_50pct": {"allow": rng < 0.5}, "random_1pct": {"allow": rng < 0.01},
            "range_1pct": {"allow": rng_range}, "exclude_2": {"exclude": exclude},
            "adversarial_dups_disallowed": {"allow": ~is_dup}}


def measure(idx, q, k, var, steps):
    res = {name: [] for name in var}
    for name, kw in var.items():  # warm-up
        step(idx, q, k, kw)
    for _ in range(steps):
        for name, kw in var.items():
            res[name].append(round(step(idx, q, k, kw), 3))
    out = {}
    for name, kw in var.items():
        idx.search_device(q, k, **kw)
        out[name] = {"median_ms": statistics.median(res[name]), "ms": res[name], "uncertified": idx.stat("uncertified"),
                     "exact_queries": idx.stat("exact_queries")}
    base = out["unfiltered"]["median_ms"]
    for name in out:
        out[name]["over_unfiltered"] = round(out[name]["median_ms"] / base, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON record to this file")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rows", type=int, default=8_800_000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    out = {"card": card()}
    n, d, nq = a.rows, 768, 6980
    q = torch.randn((nq, d), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    idx, is_dup = build(n, d, q, seed=7)
    var = variants(n, q, idx, is_dup, seed=5)
    out["c2"] = {"rows": n, "dim": d, "nq": nq, "k": 1000, "variants": measure(idx, q, 1000, var, a.steps)}
    print(json.dumps(out["c2"]), flush=True)
    for nqs in (1, 64):
        qs = q[:nqs].contiguous()
        vs = dict(var)
        vs["exclude_2"] = {"exclude": (var["exclude_2"]["exclude"][0][:nqs + 1].contiguous(), var["exclude_2"]["exclude"][1])}
        out["nq%d_k100" % nqs] = measure(idx, qs, 100, vs, max(10, 4 * a.steps))
        print(json.dumps(out["nq%d_k100" % nqs]), flush=True)
    out["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
