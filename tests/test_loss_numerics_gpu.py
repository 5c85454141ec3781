"""GPU numerics of the fused contrastive loss (csrc/loss.cu) against a float64 oracle with an elementwise error bound.

Every element of S, the loss, dX and dY must lie within the bound of ``oracle/loss_bound.py`` (derived term by term in
its docstring) around ``loss_bound.loss64``: F.cross_entropy and autograd in float64 on the bf16-rounded inputs, on the
GPU (cuBLAS DGEMM) for large shapes and on the CPU for small ones.  The file covers
  * the input regimes of real training (random, cosine / flat, temperature-scaled / peaked with hard negatives,
    un-normalised reps with logits in the hundreds, exact ties, a NaN), each asserting its premise on the oracle's
    logits and that the bound rejects five modelled kernel bugs;
  * a shape matrix that reaches every host-side path of om_contrastive_loss_fwd_bwd (split-K of dQ into 3 or 4
    slices, odd d, more LOGITS tiles than CTAs, several softmax rows per warp (pair), d > 1024, np < nq, np = 1,
    nq = 1, target columns at the chunk edges, the vector bf16 copy), each asserting that the path is taken, each
    repeated once for bitwise determinism;
  * one-sided gradients through the C ABI, bitwise equal to the two-sided call;
  * call sequences at fixed shapes that alternate scores / grads / targets / dtypes and grow the workspace: every call
    must match its own oracle and be bitwise equal to the same call made after a call at an unrelated shape;
  * the measurement switches OM_LOSS_SPLITK / OM_LOSS_LOOPED_SOFTMAX / OM_LOSS_COPY_INPUTS, one subprocess each.
Each judged call prints one "[loss-numerics]" line with max(err / bound) per output; run with -s to see them."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import loss_bound as lb

pytestmark = pytest.mark.gpu

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KNOB_VARS = ("OM_LOSS_SPLITK", "OM_LOSS_LOOPED_SOFTMAX", "OM_LOSS_COPY_INPUTS")


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import loss
    return loss


def _cdiv(a, b):
    return -(-a // b)


def plan(nq, n_p, d, *, bf16=False, aligned=True, dq=True, dp=True, knobs=None):
    """The host decisions of om_contrastive_loss_fwd_bwd for this device (restated from csrc/loss.cu)."""
    knobs = os.environ if knobs is None else knobs
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    splitk = max(1, int(knobs["OM_LOSS_SPLITK"])) if knobs.get("OM_LOSS_SPLITK") else 0
    num_k = _cdiv(n_p, 64)
    tiles = lambda m, n: _cdiv(m, 128) * _cdiv(n, 128)  # noqa: E731
    dq_tiles = tiles(nq, d)
    split, kper = 1, num_k
    if dq:
        want = min(sms // dq_tiles, num_k // 8, 4)
        if splitk:
            want = min(splitk, num_k, 4, sms // dq_tiles)
        if dq_tiles * 8 > (65536 - 256 - 64) // 4:
            want = 1
        if want > 1:
            kper = _cdiv(num_k, want)
            split = _cdiv(num_k, kper)
    direct = bf16 and d % 8 == 0 and aligned and not knobs.get("OM_LOSS_COPY_INPUTS")
    gemm_tiles = max(tiles(nq, n_p), (dq_tiles * split if dq else 0) + (tiles(n_p, d) if dp else 0))
    prep = 0 if direct else min(sms, _cdiv((nq + n_p) * _cdiv(d, 8), 256))
    grid = max(1, min(max(gemm_tiles, _cdiv(nq, 8), prep), sms))
    sm_fast = n_p % 4 == 0 and n_p <= 4096 and not knobs.get("OM_LOSS_LOOPED_SOFTMAX")
    return dict(sms=sms, split=split, kper=kper, direct=direct, grid=grid, sm_fast=sm_fast,
                logit_tiles=tiles(nq, n_p), grad_items=gemm_tiles if dq or dp else 0,
                rows_per_unit=_cdiv(nq, (4 if sm_fast else 8) * grid),
                vec_store=d % 2 == 0, vec_reduce=d % 4 == 0)


def _call(L, x, y, target=None, reduction="mean", scores=True, grads=True):
    """One call of the public API on x, y (device tensors; leaves sharing their storage, so the pointers the kernel
    sees are those of x and y).  Returns the outputs, detached."""
    xg = x.detach().requires_grad_(grads)
    yg = y.detach().requires_grad_(grads)
    out = L.fused_contrastive_loss(xg, yg, target, reduction, return_scores=scores)
    loss, S = out if scores else (out, None)
    res = {"loss": loss.detach().clone(), "S": S}
    if grads:
        loss.backward()
        res["dX"], res["dY"] = xg.grad, yg.grad
    torch.cuda.synchronize()
    return res


def _dev(nq, n_p, d):
    return "cuda" if nq * n_p * d >= (1 << 22) else "cpu"


def judge(what, x, y, got, target=None, reduction="mean", split=1):
    """Checks every output in got against the oracle's bound; returns (oracle, bounds, ratios)."""
    nq, d = x.shape
    dev = _dev(nq, y.shape[0], d)
    xb, yb = lb.bf16_round(x.to(dev)), lb.bf16_round(y.to(dev))
    o = lb.loss64(xb, yb, None if target is None else target.to(dev), reduction)
    b = lb.bounds(xb, yb, o, split, bf16_grads=x.dtype == BF16)
    r = lb.ratios(got, o, b)
    print("[loss-numerics] %-58s %s" % (what, "  ".join("%s %.3g" % kv for kv in r.items())))
    for k, v in r.items():
        assert v <= 1.0, "%s: %s max(err / bound) = %.4g" % (what, k, v)
    return o, b, r


def _same(a, b):
    return all((a[k] is None and b[k] is None) or torch.equal(a[k], b[k]) for k in a)


# ------------------------------------------------------------------------------------------------------------------
# regimes: the statistics of real training, and the five modelled bugs each must expose
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nq,n_p,d,dtype", [(256, 2048, 200, F32), (512, 4096, 768, BF16)])
@pytest.mark.parametrize("regime", lb.REGIMES)
def test_regime(L, regime, nq, n_p, d, dtype):
    x, y, info = lb.make_regime(regime, nq, n_p, d, seed=nq + d)
    x, y = x.cuda().to(dtype), y.cuda().to(dtype)
    p = plan(nq, n_p, d, bf16=dtype == BF16)
    got = _call(L, x, y)
    o, b, _ = judge("%s %dx%dx%d %s" % (regime, nq, n_p, d, str(dtype)[6:]), x, y, got, split=p["split"])
    lb.premise(regime, o, info)
    if regime == "nan":
        assert torch.isnan(got["loss"]), "a NaN input must give a NaN loss, as in PyTorch"
    if regime == "ties":
        assert torch.equal(got["S"].to(F64), o["S"].to("cuda")), "integer logits must be exact"
        a, c = info["dups"]
        assert torch.equal(got["dY"][a.cuda()], got["dY"][c.cuda()]), "tied columns must get identical gradients"
    for name, mut in lb.mutants(lb.bf16_round(x.to(o["S"].device)), lb.bf16_round(y.to(o["S"].device)), o,
                                dq_split=p["split"]).items():
        r = lb.ratios(mut, o, b)
        assert max(r.values()) > 1.0, "%s: the bound accepts the modelled bug %s (%s)" % (regime, name, r)


# ------------------------------------------------------------------------------------------------------------------
# shape / path matrix
# ------------------------------------------------------------------------------------------------------------------
MATRIX = {
    # id: (nq, np, d, dtype, target, reduction, premise on the plan)
    "split3_vector_reduce": (256, 1600, 768, F32, None, "mean", lambda p: p["split"] == 3 and p["vec_reduce"]),
    "split3_odd_d": (130, 1600, 37, F32, None, "mean",
                     lambda p: p["split"] == 3 and not p["vec_store"] and not p["vec_reduce"]),
    "split4_d_mod4_2": (40, 2048, 30, F32, None, "sum", lambda p: p["split"] == 4 and p["vec_store"] and not p["vec_reduce"]),
    "bf16_direct_2rows_per_pair": (1024, 4096, 768, BF16, None, "mean",
                                   lambda p: p["direct"] and p["logit_tiles"] == 256 > p["grid"] and p["sm_fast"]
                                   and p["rows_per_unit"] >= 2 and p["grad_items"] > p["grid"]),
    "looped_512_tiles": (1024, 8192, 768, F32, None, "mean",
                         lambda p: p["logit_tiles"] == 512 > p["grid"] and not p["sm_fast"]),
    "looped_2rows_per_warp": (1536, 6144, 768, F32, None, "mean", lambda p: not p["sm_fast"] and p["rows_per_unit"] >= 2),
    "bf16_direct_d4096": (64, 512, 4096, BF16, None, "mean", lambda p: p["direct"] and p["sm_fast"]),
    "np_lt_nq_random_targets": (300, 64, 128, F32, "random", "sum", lambda p: True),
    "np1": (256, 1, 64, F32, "zeros", "mean", lambda p: not p["sm_fast"]),
    "nq1": (1, 8, 768, F32, None, "mean", lambda p: p["sm_fast"]),
    "nq1_last_target": (1, 4096, 768, F32, "last", "mean", lambda p: p["sm_fast"]),
    "target_chunk_edges": (6, 4096, 128, F32, "edges", "sum", lambda p: p["sm_fast"]),
    "bf16_copy_vector": (128, 1024, 256, BF16, None, "mean", lambda p: not p["direct"]),
}


def _matrix_inputs(case):
    nq, n_p, d, dtype, tkind, reduction, _ = MATRIX[case]
    g = torch.Generator().manual_seed(nq * 7 + n_p + d)
    x = torch.randn(nq, d, generator=g) * 0.5
    y = torch.randn(n_p, d, generator=g) * 0.5
    target = {None: None, "random": torch.randint(0, n_p, (nq,), generator=g), "zeros": torch.zeros(nq, dtype=torch.int64),
              "last": torch.tensor([n_p - 1]),
              # both warp halves of sm_fast (128-column chunks) and the last float4 of the row
              "edges": torch.tensor([0, 127, 128, 255, 256, n_p - 1])}[tkind]
    if case == "bf16_copy_vector":
        # Q one element into its allocation (not 16-byte aligned: copied, scalar), P aligned and d % 8 == 0 (copied
        # with 16-byte vectors)
        buf = torch.empty(nq * d + 1, dtype=dtype, device="cuda")
        buf[1:].copy_(x.reshape(-1))
        xd = buf[1:].view(nq, d)
    else:
        xd = x.cuda().to(dtype)
    return xd, y.cuda().to(dtype), None if target is None else target.cuda(), reduction


@pytest.mark.parametrize("case", list(MATRIX))
def test_matrix(L, case):
    nq, n_p, d, dtype, tkind, _, premise = MATRIX[case]
    x, y, target, reduction = _matrix_inputs(case)
    aligned = (x.data_ptr() | y.data_ptr()) % 16 == 0
    p = plan(nq, n_p, d, bf16=dtype == BF16, aligned=aligned)
    assert premise(p), "%s: the shape does not take the intended path: %s" % (case, p)
    if case == "np_lt_nq_random_targets":
        assert n_p < nq and len(set(target.tolist())) < nq
    if case == "bf16_copy_vector":
        assert x.data_ptr() % 16 != 0 and y.data_ptr() % 32 == 0 and d % 8 == 0
    got = _call(L, x, y, target, reduction)
    judge("%s %dx%dx%d %s %s" % (case, nq, n_p, d, str(dtype)[6:], reduction), x, y, got, target, reduction,
          p["split"])
    if case == "np1":
        assert got["loss"].item() == 0.0 and not got["dX"].any() and not got["dY"].any()
    again = _call(L, x, y, target, reduction)
    assert _same(got, again), "%s: run-to-run difference" % case


# ------------------------------------------------------------------------------------------------------------------
# gradient wiring: one-sided calls through the C ABI
# ------------------------------------------------------------------------------------------------------------------
def _abi(x, y, dq, dp, scores):
    from openmatch_b200 import _lib
    lib = _lib.load()
    nq, d = x.shape
    n_p = y.shape[0]
    out = {"loss": torch.empty((), device="cuda"),
           "dX": torch.empty(nq, d, device="cuda") if dq else None,
           "dY": torch.empty(n_p, d, device="cuda") if dp else None,
           "S": torch.empty(nq, n_p, device="cuda") if scores else None}
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _lib.check(lib.om_contrastive_loss_fwd_bwd(
        x.data_ptr(), y.data_ptr(), _lib.OM_BF16 if x.dtype == BF16 else _lib.OM_F32, nq, n_p, d, None,
        _lib.OM_REDUCE_MEAN, 1.0, out["loss"].data_ptr(), ptr(out["dX"]), ptr(out["dY"]), ptr(out["S"]),
        _lib.current_stream_ptr()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("nq,n_p,d,dtype", [(256, 1600, 768, F32), (64, 512, 768, BF16)])
def test_one_sided_gradients_match_two_sided(L, nq, n_p, d, dtype):
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(nq, d, generator=g) * 0.5).cuda().to(dtype)
    y = (torch.randn(n_p, d, generator=g) * 0.5).cuda().to(dtype)
    both = _abi(x, y, True, True, True)
    judge("two-sided %dx%dx%d" % (nq, n_p, d), x, y, {k: both[k] for k in ("S", "loss", "dX", "dY")},
          split=plan(nq, n_p, d, bf16=dtype == BF16)["split"])
    for dq, dp in ((True, False), (False, True), (False, False)):
        one = _abi(x, y, dq, dp, True)
        for k in ("S", "loss") + (("dX",) if dq else ()) + (("dY",) if dp else ()):
            assert torch.equal(one[k], both[k]), "dQ=%s dP=%s: %s differs from the two-sided call" % (dq, dp, k)
    # through autograd: only x requires grad
    xg = x.detach().requires_grad_()
    L.fused_contrastive_loss(xg, y).backward()
    assert y.grad is None and torch.equal(xg.grad.float(), both["dX"].to(dtype).float())


# ------------------------------------------------------------------------------------------------------------------
# call sequences at fixed shapes (the tensor maps are cached across calls)
# ------------------------------------------------------------------------------------------------------------------
STEPS = [dict(scores=True, grads=True, target=False), dict(scores=False, grads=True, target=False),
         dict(scores=True, grads=True, target=True), dict(scores=False, grads=False, target=True),
         dict(scores=False, grads=True, target=False), "grow", dict(scores=True, grads=True, target=False),
         dict(scores=False, grads=True, target=True, other_dtype=True), dict(scores=True, grads=True, target=False),
         dict(scores=False, grads=True, target=False)]


@pytest.mark.parametrize("nq,n_p,d,dtype", [(64, 512, 768, F32), (130, 1040, 200, F32), (64, 512, 768, BF16)])
def test_call_sequence(L, nq, n_p, d, dtype):
    other = F32 if dtype == BF16 else BF16
    # persistent inputs, refilled before every call as a training loop does: the pointers repeat
    bufs = {dt: (torch.empty(nq, d, dtype=dt, device="cuda"), torch.empty(n_p, d, dtype=dt, device="cuda"))
            for dt in (dtype, other)}
    tbuf = torch.empty(nq, dtype=torch.int64, device="cuda")
    g = torch.Generator().manual_seed(nq + d)
    calls = []
    for i, st in enumerate(STEPS):
        if st == "grow":  # a larger problem in between: the workspace is reallocated
            xg, yg = torch.randn(4 * nq, d, generator=g) * 0.5, torch.randn(8 * n_p, d, generator=g) * 0.5
            got = _call(L, xg.cuda(), yg.cuda())
            judge("seq step %d: grow %dx%dx%d" % (i, 4 * nq, 8 * n_p, d), xg.cuda(), yg.cuda(), got,
                  split=plan(4 * nq, 8 * n_p, d)["split"])
            continue
        dt = other if st.get("other_dtype") else dtype
        x, y = torch.randn(nq, d, generator=g) * 0.5, torch.randn(n_p, d, generator=g) * 0.5
        t = torch.randint(0, n_p, (nq,), generator=g) if st["target"] else None
        xb, yb = bufs[dt]
        xb.copy_(x)
        yb.copy_(y)
        if t is not None:
            tbuf.copy_(t)
        got = _call(L, xb, yb, tbuf if t is not None else None, scores=st["scores"], grads=st["grads"])
        calls.append((i, st, dt, x, y, t, {k: (v.clone() if v is not None else None) for k, v in got.items()}))
    failures = []  # every failing step is reported, not only the first
    for i, st, dt, x, y, t, got in calls:
        what = "seq step %d: %dx%dx%d %s scores=%s grads=%s target=%s" % (
            i, nq, n_p, d, str(dt)[6:], st["scores"], st["grads"], st["target"])
        try:
            judge(what, x.cuda().to(dt), y.cuda().to(dt), got, None if t is None else t.cuda(),
                  split=plan(nq, n_p, d, bf16=dt == BF16)["split"] if st["grads"] else 1)
        except AssertionError as e:
            failures.append(str(e).splitlines()[0])
        # the same call after an unrelated shape (which rebuilds every cached tensor map)
        _call(L, torch.randn(8, 32, device="cuda"), torch.randn(72, 32, device="cuda"))
        xb, yb = bufs[dt]
        xb.copy_(x)
        yb.copy_(y)
        if t is not None:
            tbuf.copy_(t)
        fresh = _call(L, xb, yb, tbuf if t is not None else None, scores=st["scores"], grads=st["grads"])
        if not _same(got, fresh):
            failures.append("%s: differs from the same call made after a rebuild" % what)
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------------------------
# measurement switches: read once per process, so one subprocess per setting
# ------------------------------------------------------------------------------------------------------------------
KNOB_SHAPES = {"130x1040x200_f32": (130, 1040, 200, F32), "40x2048x30_f32": (40, 2048, 30, F32),
               "64x512x768_bf16": (64, 512, 768, BF16)}
KNOB_SETTINGS = {"auto": {}, "splitk1": {"OM_LOSS_SPLITK": "1"}, "splitk2": {"OM_LOSS_SPLITK": "2"},
                 "splitk3": {"OM_LOSS_SPLITK": "3"}, "splitk4": {"OM_LOSS_SPLITK": "4"},
                 "looped": {"OM_LOSS_LOOPED_SOFTMAX": "1"}, "copy": {"OM_LOSS_COPY_INPUTS": "1"}}


def knob_child(out_path):
    """Runs in a fresh process with one switch set: checks the three shapes against the oracle, saves the outputs."""
    from openmatch_b200 import loss as L
    res = {}
    for name, (nq, n_p, d, dtype) in KNOB_SHAPES.items():
        g = torch.Generator().manual_seed(nq + n_p + d)
        x = (torch.randn(nq, d, generator=g) * 0.5).cuda().to(dtype)
        y = (torch.randn(n_p, d, generator=g) * 0.5).cuda().to(dtype)
        p = plan(nq, n_p, d, bf16=dtype == BF16)
        got = _call(L, x, y)
        judge("knobs %s %s" % (",".join("%s=%s" % kv for kv in os.environ.items() if kv[0] in KNOB_VARS) or "auto",
                               name), x, y, got, split=p["split"])
        res[name] = ({k: v.cpu() for k, v in got.items()}, p)
    torch.save(res, out_path)


def test_measurement_switches(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    env0 = {k: v for k, v in os.environ.items() if k not in KNOB_VARS}
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_loss_numerics_gpu as t; t.knob_child(sys.argv[1])"
            % (ROOT, os.path.join(ROOT, "tests")))
    flags = ["-s"] if sys.flags.no_user_site else []
    out = {}
    for name, knobs in KNOB_SETTINGS.items():
        path = str(tmp_path / (name + ".pt"))
        r = subprocess.run([sys.executable] + flags + ["-c", code, path], env={**env0, **knobs}, cwd=ROOT,
                           capture_output=True, text=True, timeout=300)
        print(r.stdout, end="")
        assert r.returncode == 0, "%s: child failed (rc %d)\n%s" % (name, r.returncode, r.stderr[-3000:])
        out[name] = torch.load(path)
    for n in (1, 2, 3, 4):
        assert out["splitk%d" % n]["130x1040x200_f32"][1]["split"] == n
    for shape in KNOB_SHAPES:
        ref = out["auto"][shape][0]
        for name in ("splitk1", "splitk2", "splitk3", "splitk4"):
            got = out[name][shape][0]
            for k in ("S", "loss", "dY"):
                assert torch.equal(got[k], ref[k]), "%s %s: %s differs across OM_LOSS_SPLITK" % (shape, name, k)
    assert out["copy"]["64x512x768_bf16"][1]["direct"] is False and out["auto"]["64x512x768_bf16"][1]["direct"]
    assert _same(out["copy"]["64x512x768_bf16"][0], out["auto"]["64x512x768_bf16"][0]), \
        "OM_LOSS_COPY_INPUTS: the copied bf16 inputs must give the in-place result bit for bit"
    assert not out["looped"]["40x2048x30_f32"][1]["sm_fast"]
