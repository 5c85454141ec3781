"""The host-resident index against the device index, on one GPU.

  python tools/index_host_probe.py [--steps 3] [--rows 8800000] [--small-window 1048576] [--out PATH]

The corpus is the C2 shape (8.8 M x 768 rows, N(0, 1) elements) and 6 980 N(0, 1) queries at k = 1 000, on fp16 and int8
storage.  Per storage, in one process: the host -> device copy rate of one pinned window (CUDA events); the device index
step T_dev alternated with the host index step T_host at the automatic window and at --small-window rows (host clock
around a synchronous call, profile off; median and range of ms); one profiled call per window for "partitions" and
"upload_wait_ns"; streaming nq = 1 and 64 at k = 100; and whether D and I are byte-identical between host and device.
The two host indexes pin the rows twice over: MemAvailable must hold them three times (the GPU machines are shared),
otherwise N is shrunk and the record says so.  The card's name, power limit and maximum SM clock are
read in the same call.  The record is printed as one JSON line, and also written to PATH with --out."""
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


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def row_bytes(dtype, d):
    return (d + 7) // 8 * 8 * 2 if dtype == torch.float16 else (d + 15) // 16 * 16 + 16


def copy_rate(nbytes, reps=5):
    """GB/s of one pinned host buffer -> device buffer copy of nbytes (CUDA events, median of reps)."""
    src = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    rates = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src, non_blocking=True)
        b.record()
        b.synchronize()
        rates.append(nbytes / (a.elapsed_time(b) * 1e-3) / 1e9)
    return statistics.median(rates)


def stats(idx):
    return {s: idx.stat(s) for s in ("partitions", "uncertified", "uncertified_wide", "exact_queries", "rounds")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rows", type=int, default=8_800_000)
    ap.add_argument("--nq", type=int, default=6980)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--small-window", type=int, default=1 << 20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"card": card(), "dim": a.dim, "nq": a.nq, "k": a.k, "storages": []}
    for dtype in (torch.float16, torch.int8):
        rb = row_bytes(dtype, a.dim)
        avail = mem_available()
        n = a.rows
        if 3 * n * rb > avail:  # two host indexes pin the rows twice; the shared host keeps their size again free
            n = max(1 << 20, int(avail / (3 * rb)) // 256 * 256)
        r = {"storage": str(dtype), "rows": n, "rows_shrunk_from": a.rows if n != a.rows else None,
             "mem_available_gb": avail / 1e9, "row_bytes": rb}
        g = torch.Generator(device="cuda").manual_seed(0)
        dev = FlatIPIndex(a.dim, dtype)
        hosts = {"auto": FlatIPIndex(a.dim, dtype, memory="host"),
                 "small": FlatIPIndex(a.dim, dtype, memory="host", window_rows=a.small_window)}
        t_add = {"device": 0.0, "auto": 0.0, "small": 0.0}
        for lo in range(0, n, 1 << 20):
            x = torch.randn(min(1 << 20, n - lo), a.dim, device="cuda", generator=g)
            t_add["device"] += timed(lambda: dev.add(x))
            for name, h in hosts.items():
                t_add[name] += timed(lambda: h.add(x))
            del x
        r["add_s"] = {key: v / 1e3 for key, v in t_add.items()}
        q = torch.randn(a.nq, a.dim, device="cuda", generator=g)
        r["copy_gb_s"] = copy_rate(min(n, a.small_window) * rb)
        r["row_gb"] = n * rb / 1e9
        want = dev.search_device(q, a.k)
        r["cases"] = []
        for name, h in hosts.items():
            got = h.search_device(q, a.k)  # warm-up of both, and the byte comparison
            same = bool(torch.equal(got[0].view(torch.int32), want[0].view(torch.int32)) and torch.equal(got[1], want[1]))
            dev.search_device(q, a.k)
            td, th = [], []
            for _ in range(a.steps):
                td.append(timed(lambda: dev.search_device(q, a.k)))
                th.append(timed(lambda: h.search_device(q, a.k)))
            h.set_param("profile", 1)
            h.search_device(q, a.k)
            h.set_param("profile", 0)
            prof = {s: h.stat(s) for s in ("upload_wait_ns", "scan_ns", "select_ns", "finalize_ns", "other_ns")}
            case = {"window": name, "identical": same, "T_dev_ms_median": statistics.median(td), "T_dev_ms": [min(td), max(td)],
                    "T_host_ms_median": statistics.median(th), "T_host_ms": [min(th), max(th)],
                    "stats": stats(h), "profile": prof}
            bound = max(case["T_dev_ms_median"], r["row_gb"] / r["copy_gb_s"] * 1e3)
            case["aim_ms"] = 1.2 * bound
            case["aim_met"] = case["T_host_ms_median"] <= case["aim_ms"]
            stream = []
            for nq in (1, 64):
                qq = q[:nq].contiguous()
                want_s = dev.search_device(qq, 100)
                got_s = h.search_device(qq, 100)
                sd, sh = [], []
                for _ in range(a.steps):
                    sd.append(timed(lambda: dev.search_device(qq, 100)))
                    sh.append(timed(lambda: h.search_device(qq, 100)))
                stream.append({"nq": nq, "k": 100, "T_dev_ms_median": statistics.median(sd),
                               "T_host_ms_median": statistics.median(sh), "T_host_ms": [min(sh), max(sh)],
                               "identical": bool(torch.equal(got_s[0], want_s[0]) and torch.equal(got_s[1], want_s[1]))})
            case["streaming"] = stream
            r["cases"].append(case)
            print(json.dumps({"storage": r["storage"], **case}), flush=True)
        rec["storages"].append(r)
        del dev, hosts, want, q
        torch.cuda.empty_cache()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
