"""Probe (not a test): the wide search scan on each cluster shape at C2 (8.8 M x 768) and one C5 shard (2.625 M x 1024),
6 980 queries, k = 1000.  Shapes alternate over several rounds in one process; per shape it prints the step time, the
scan time per step, the scan's TFLOP/s, the L2 -> SM bytes per step derived from the shapes, the co-resident clusters,
the rounds, the uncertified queries, and whether D and I are byte-identical to the 2 x 1 result.

    python tools/scan_probe.py [--rounds 2] [--steps 3] [--workloads c2,c5]

Reads the card name, power limit and maximum SM clock with a read-only nvidia-smi query and samples the SM clock during
the timed steps (bench.ClockSampler); it changes no device setting."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from openmatch_b200.index import FlatIPIndex  # noqa: E402

SHAPES = [(2, 1), (4, 1), (2, 2), (4, 2), None]  # None: the automatic choice
WORKLOADS = {"c2": (8_800_000, 768), "c5": (2_625_000, 1024)}


def l2_bytes_per_step(n, d, nq, C, cq, cx):
    """L2 -> SM operand bytes of the cluster-scan rounds of one search (the doubling schedule without overflow retries):
    per CTA and 64-wide k block, a 128/cx-row query slice and a 256/cq-row corpus slice of 128 B rows."""
    qctas = -(-nq // (128 * cq)) * cq
    kb = -(-d // 64)
    per_cta = (128 // cx + 256 // cq) * 128
    pos, total = min(n, C), 0
    while pos < n:
        step = min(n - pos, pos)
        xctas = -(-step // (256 * cx)) * cx
        total += qctas * xctas * kb * per_cta
        pos += step
    return total


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def fill(n, d):
    idx = FlatIPIndex(d)
    idx.reserve_rows(n)
    chunk = 550_000
    for c0 in range(0, n, chunk):
        m = min(chunk, n - c0)
        rows = idx.reserve_rows(m)
        rows.normal_(generator=torch.Generator(device="cuda").manual_seed(1234 + c0 // chunk))
        idx.commit_rows(m)
    return idx


def probe(name, n, d, nq, k, rounds, steps):
    idx = fill(n, d)
    q = torch.randn(nq, d, generator=torch.Generator(device="cuda").manual_seed(99), device="cuda")
    D = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    I = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    res = {s: {"ms": [], "scan_ms": [], "mhz": []} for s in SHAPES}
    ref = None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(rounds):
        for s in SHAPES:
            idx.set_param("scan_cluster_q", s[0] if s else 0)
            idx.set_param("scan_cluster_x", s[1] if s else 0)
            idx.search_device(q, k, out=(D, I))  # warm-up (first launch of the shape: module load, occupancy query)
            torch.cuda.synchronize()
            idx.set_param("profile", 1)
            scan_ns = unc = 0
            with ClockSampler(0) as clk:
                e0.record()
                for _ in range(steps):
                    idx.search_device(q, k, out=(D, I))
                    scan_ns += idx.stat("scan_ns")
                    unc += idx.stat("uncertified")
                e1.record()
                torch.cuda.synchronize()
            idx.set_param("profile", 0)
            o = res[s]
            o["ms"].append(e0.elapsed_time(e1) / steps)
            o["scan_ms"].append(scan_ns / 1e6 / steps)
            o["mhz"].append(clk.summary()["sm_mhz"])
            o.update(rounds=idx.stat("rounds"), unc=unc, used=idx.stat("scan_cluster"), clusters=idx.stat("scan_max_clusters"),
                     C=idx.stat("candidates"))
            if s == (2, 1) and ref is None:
                ref = (D.clone(), I.clone())
            o.setdefault("same", True)
            o["same"] = o["same"] and torch.equal(D.view(torch.int32), ref[0].view(torch.int32)) and torch.equal(I, ref[1])
    flop = 2.0 * nq * n * d
    print("%s: %d x %d, %d queries, k = %d (medians over %d rounds of %d steps)" % (name, n, d, nq, k, rounds, steps))
    print("  shape      used  step ms  scan ms  scan TFLOP/s  L2->SM TB/step  clusters  rounds  uncert  SM MHz  D,I == 2x1")
    for s in SHAPES:
        o = res[s]
        used = o["used"]
        cq, cx = used // 10, used % 10
        med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
        mhz = [m for m in o["mhz"] if m]
        print("  %-9s  %4d  %7.1f  %7.1f  %12.0f  %14.3f  %8d  %6d  %6d  %6s  %s" % (
            "%dx%d" % s if s else "auto", used, med(o["ms"]), med(o["scan_ms"]), flop / (med(o["scan_ms"]) * 1e-3) / 1e12,
            l2_bytes_per_step(n, d, nq, o["C"], cq, cx) / 1e12 if used else float("nan"), o["clusters"], o["rounds"],
            o["unc"], med(mhz) if mhz else "-", "yes" if o["same"] else "NO"), flush=True)
    del idx
    torch.cuda.empty_cache()
    return all(res[s]["same"] for s in SHAPES)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--nq", type=int, default=6980)
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--workloads", default="c2,c5")
    args = ap.parse_args()
    print("GPU (name, power limit, max SM clock): %s" % gpu_info(), flush=True)
    ok = True
    for w in args.workloads.split(","):
        n, d = WORKLOADS[w]
        ok = probe(w, n, d, args.nq, args.k, args.rounds, args.steps) and ok
    print("PROBE OK" if ok else "PROBE FAILED: results differ between shapes")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
