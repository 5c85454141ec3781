"""GPU: the index with int8 row storage (``FlatIPIndex(d, dtype=torch.int8)``, ``om_index_create_typed(d, OM_I8)``).

Contract under test: an int8 index stores each row as codes and a per-row scale (tests/index_i8_oracle.py, bit for bit)
and its search is the exact top-k by fp32 inner product of the fp32 query with the dequantised rows fp32(s * c), ties
by ascending id.  So an int8 index built from X must answer bit for bit like a default (fp32) index built from
dequantize(quantize(X)), and the answer must pass the float64 oracle's check on those rows."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import index_i8_oracle as io
from oracle import search_bound as sb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS = ("uncertified", "uncertified_wide", "exact_queries")
DEFAULTS = {"round_growth": 0, "certify": 1, "exact_only": 0, "debug_stage_scores": 0, "force_safe_rounds": 0}


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _np(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _same(a, b, what):
    a, b = _np(a), _np(b)
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    if a.dtype.kind == "f":
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32), err_msg=what)
    else:
        np.testing.assert_array_equal(a, b, err_msg=what)


def _search(idx, q, k, **params):
    for name, v in {**DEFAULTS, **params}.items():
        idx.set_param(name, v)
    D, I = idx.search(q, k)
    return D, I, tuple(idx.stat(s) for s in STATS)


def _stored(idx):
    """(codes int8 [n, d], scales float32 [n], padding bytes) as the index holds them"""
    from openmatch_b200.index import _wrap_device
    n, d = idx.ntotal, idx.d
    p, pitch = idx._rows_at(0)
    full = _wrap_device(p - n * pitch, (n, pitch), pitch, torch.int8).cpu().numpy()
    dpad = (d + 15) // 16 * 16
    assert pitch == dpad + 16
    scale = np.ascontiguousarray(full[:, dpad:dpad + 4]).view(np.float32)[:, 0]
    pad = np.concatenate([full[:, d:dpad], full[:, dpad + 4:]], axis=1)
    return full[:, :d], scale, pad


def _check_stored(idx, x, what):
    c, s, pad = _stored(idx)
    c0, s0 = io.quantize_i8(x)
    _same(c, c0, "%s: codes" % what)
    _same(s, s0, "%s: scales" % what)
    assert (pad == 0).all(), "%s: padding bytes must be zero" % what


# ---------------------------------------------------------------------------------------------------------------------
# bitwise equivalence: int8 index of X == fp32 index of dequantize(quantize(X))
# ---------------------------------------------------------------------------------------------------------------------
N_EQ = 12000
_PAIRS = {}


def _pair(om, d, n=N_EQ):
    if (d, n) not in _PAIRS:
        rng = np.random.default_rng(d + n)
        x = rng.standard_normal((n, d), dtype=np.float32)
        x[:40] = x[40:80]  # exact duplicates: ties broken by id
        q8 = om.FlatIPIndex(d, dtype=torch.int8)
        q8.add(x)
        f = om.FlatIPIndex(d)
        f.add(io.stored_i8(x))
        _PAIRS[(d, n)] = (q8, f, rng)
    return _PAIRS[(d, n)]


CONFIGS = [dict(), dict(force_safe_rounds=1), dict(round_growth=8), dict(round_growth=2), dict(exact_only=1)]
# (nq, k, d): every nq of {1, 7, 128, 129, 1500}, every k of {1, 10, 1000, 4096, > n}, every d of {64, 384, 768, 1000, 4096}
EQ_CASES = [(1, 1, 64), (7, 10, 384), (128, 1000, 768), (129, 4096, 1000), (1500, 10, 4096), (1500, 1000, 64),
            (129, 10, 768), (1, 4096, 384), (7, 1000, 1000), (128, 100, 4096)]


@pytest.mark.parametrize("nq,k,d", EQ_CASES, ids=["nq%d-k%d-d%d" % c for c in EQ_CASES])
def test_int8_index_equals_fp32_index_of_dequantised_rows(om, nq, k, d):
    q8, f, rng = _pair(om, d)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    q[0] = np.arange(d, dtype=np.float32) % 7  # a query with many tied scores
    for cfg in CONFIGS:
        Dq, Iq, st = _search(q8, q, k, **cfg)
        Df, If, _ = _search(f, q, k, **cfg)
        _same(Iq, If, "I %s" % cfg)
        _same(Dq, Df, "D %s" % cfg)
        if k <= 100 and not cfg.get("exact_only"):
            assert q8.stat("rounds") >= 2, "premise: the corpus spans several threshold rounds"


def test_int8_index_with_k_beyond_its_rows(om):
    q8, f, rng = _pair(om, 384, n=3000)
    q = rng.standard_normal((129, 384), dtype=np.float32)
    for nq in (1, 129):
        Dq, Iq, _ = _search(q8, q[:nq], 4096)
        Df, If, _ = _search(f, q[:nq], 4096)
        _same(Iq, If, "I k > n")
        _same(Dq, Df, "D k > n")
        assert (Iq[:, 3000:] == -1).all() and (Iq[:, :3000] >= 0).all()


def _dequantised_pair(om, x):
    q8 = om.FlatIPIndex(x.shape[1], dtype=torch.int8)
    q8.add(x)
    f = om.FlatIPIndex(x.shape[1])
    f.add(torch.cat(list(q8.rows_f32())))
    return q8, f


@pytest.mark.parametrize("nq", [9, 300])
def test_int8_massive_ties(om, nq):
    # 0/1 data: scores take a handful of values, so tie order decides almost every rank and a thread's row of a tile
    # holds more survivors than its stash parks
    rng = np.random.default_rng(7 + nq)
    x = rng.integers(0, 2, (30000, 64)).astype(np.float32)
    q = rng.integers(0, 2, (nq, 64)).astype(np.float32)
    q8, f = _dequantised_pair(om, x)
    for k in (1, 64, 1000):
        Dq, Iq, _ = _search(q8, q, k)
        Df, If, _ = _search(f, q, k)
        _same(Iq, If, "I k=%d" % k)
        _same(Dq, Df, "D k=%d" % k)


@pytest.mark.parametrize("nq", [3, 300])
def test_int8_sorted_corpus_forces_overflow_retry(om, nq):
    # every later row beats every earlier row for every query: each tile's survivors exceed the stash, the doubling
    # schedule overflows its candidate lists and the overflow-proof schedule must take over.  Column 0 at 127 gives
    # every row scale 1, so the codes are the rows and every score m * v is exact
    n, d = 60000, 64
    v = np.arange(n) // 4  # ascending scores with 4-way ties
    x = np.zeros((n, d), np.float32)
    x[:, 0], x[:, 1], x[:, 2] = 127, v // 127, v % 127
    m = np.arange(nq) % 3 + 1
    q = np.zeros((nq, d), np.float32)
    q[:, 1], q[:, 2] = 127 * m, m
    q8, f = _dequantised_pair(om, x)
    _check_stored(q8, x, "sorted corpus")
    Dq, Iq, _ = _search(q8, q, 100)
    assert q8.stat("overflow_retries") >= 1
    Df, If, _ = _search(f, q, 100)
    _same(Iq, If, "I")
    _same(Dq, Df, "D")
    Dq, Iq, _ = _search(q8, q, 100, force_safe_rounds=1)
    _same(Iq, If, "I safe rounds")
    _same(Dq, Df, "D safe rounds")


# ---------------------------------------------------------------------------------------------------------------------
# stored codes and scales == the CPU oracle, every ingest route
# ---------------------------------------------------------------------------------------------------------------------
def _edge_rows(rng, n, d):
    x = rng.standard_normal((n, d), dtype=np.float32) * 3
    x[0] = 0                                        # zero row
    x[1] = 1e-3 * x[1]
    x[1, 7] = 50.0                                  # one dominant element
    x[2] = 1e-30 * x[2]                             # tiny scale
    x[3] = 0
    x[3, :3] = (1e-44, -2e-44, 3e-45)               # subnormal: the scale rounds to 0
    x[4] = np.float32(127) * np.round(x[4])         # exact code halves after the division
    return x


@pytest.mark.parametrize("d", [64, 90, 768])
def test_codes_and_scales_equal_the_oracle_on_every_route(om, d):
    rng = np.random.default_rng(d)
    n = 2500
    x = _edge_rows(rng, n, d)
    xb = torch.from_numpy(x).bfloat16()
    xh = torch.from_numpy(x).half()
    routes = {"host f32": (x, x), "host f32 tensor": (torch.from_numpy(x), x), "host bf16": (xb, xb.float().numpy()),
              "host f16": (xh, xh.float().numpy()), "host f16 numpy": (xh.numpy(), xh.float().numpy()),
              "device f32": (torch.from_numpy(x).cuda(), x), "device bf16": (xb.cuda(), xb.float().numpy()),
              "device f16": (xh.cuda(), xh.float().numpy())}
    for name, (data, want) in routes.items():
        idx = om.FlatIPIndex(d, dtype=torch.int8)
        idx.add(data[:1000])
        idx.add(data[1000:])
        assert idx.ntotal == n
        _check_stored(idx, want, name)
        rows = idx.master_rows()
        assert rows.dtype == torch.int8 and rows.shape == (n, d) and rows.stride() == ((d + 15) // 16 * 16 + 16, 1)
        _same(torch.cat(list(idx.rows_f32(chunk_rows=777))), io.stored_i8(want), "%s: rows_f32" % name)


# ---------------------------------------------------------------------------------------------------------------------
# float64 oracle on the stored values, escalation, certificate
# ---------------------------------------------------------------------------------------------------------------------
K = 10
ORACLE_CASES = [("gaussian", 768, 20000), ("anisotropic", 768, 20000), ("coherent", 768, 20000), ("gaussian", 64, 20000)]


@pytest.mark.parametrize("regime,d,n", ORACLE_CASES, ids=["%s-%d" % (r, d) for r, d, _ in ORACLE_CASES])
def test_oracle_on_stored_rows(om, regime, d, n):
    x, q, _, _ = sb.make_regime(regime, 300, n, d, k=K, seed=d + 1)
    xs = io.stored_i8(x)
    idx = om.FlatIPIndex(d, dtype=torch.int8)
    idx.add(x)
    s, beta = sb.score64(q, xs), sb.rescore_bound(q, xs)
    for params in (dict(), dict(round_growth=8), dict(force_safe_rounds=1)):
        D, I, st = _search(idx, q, K, **params)
        De, Ie, _ = _search(idx, q, K, exact_only=1, **params)
        _same(I, Ie, "%s %s: I vs exact_only" % (regime, params))
        _same(D, De, "%s %s: D vs exact_only" % (regime, params))
        rs = sb.check_topk(q, xs, D, I, K, s=s, beta=beta)
        print("[i8 numerics] regime=%s d=%d %s |D-s64|/beta=%.3f uncertified=%d uncertified_wide=%d exact_queries=%d"
              % (regime, d, params, rs["rescore_ratio"], *st))


def test_quantisation_collisions_force_the_wide_level_and_the_exact_scan(om):
    # 6000 rows that quantise to the same codes (v + 1e-6 noise; their scales differ in the last bits): the k-th score
    # is tied far beyond the widest candidate list, the certificate cannot hold and the exact scan answers
    rng = np.random.default_rng(4097)
    n, d = 20000, 128
    x = rng.standard_normal((n, d), dtype=np.float32)
    v = rng.standard_normal(d, dtype=np.float32)
    dup = rng.choice(n, 6000, replace=False)
    x[dup] = v + 1e-6 * rng.standard_normal((6000, d), dtype=np.float32)
    c, s = io.quantize_i8(x[dup])
    assert (c == c[0]).all() and np.abs(s / s[0] - 1).max() < 1e-5, "premise: the near-duplicates collide after quantisation"
    q = (v + 0.1 * rng.standard_normal((5, d), dtype=np.float32)).astype(np.float32)
    xs = io.stored_i8(x)
    idx = om.FlatIPIndex(d, dtype=torch.int8)
    idx.add(x)
    f = om.FlatIPIndex(d)
    f.add(xs)
    for k in (10, 1000):
        D, I, st = _search(idx, q, k)
        assert st[0] > 0 and st[1] > 0 and st[2] > 0, "premise: the escalation levels must run (stats %s)" % (st,)
        sb.check_topk(q, xs, D, I, k)
        Df, If, _ = _search(f, q, k)
        _same(I, If, "collisions I")
        _same(D, Df, "collisions D")


def _dominant_queries(rng, nq, d):
    q = 0.01 * rng.standard_normal((nq, d), dtype=np.float32)
    q[np.arange(nq), rng.integers(0, d, nq)] = 30.0  # one dominant element: sig_lo carries every other coordinate
    return q


CERT_CASES = [("gaussian", 768), ("anisotropic", 768), ("coherent", 768), ("dominant", 768), ("gaussian", 1000),
              ("dominant", 64)]


@pytest.mark.parametrize("regime,d", CERT_CASES, ids=["%s-%d" % c for c in CERT_CASES])
def test_certificate_measured_on_the_hardware(om, regime, d):
    """|stage score - float64 score of the stored row| / E(q) over the returned stage top-k, E from the oracle"""
    rng = np.random.default_rng(d)
    if regime == "dominant":
        x, _, _, _ = sb.make_regime("anisotropic", 1, 20000, d, k=100, seed=d)
        q = _dominant_queries(rng, 200, d)
    else:
        x, q, _, _ = sb.make_regime(regime, 200, 20000, d, k=100, seed=d)
    xs = io.stored_i8(x)
    idx = om.FlatIPIndex(d, dtype=torch.int8)
    idx.add(x)
    E = io.cert_E_i8(q, xs)
    s = sb.score64(q, xs)
    worst = 0.0
    for nq in (1, 64, 200):
        D, I, _ = _search(idx, q[:nq], 100, debug_stage_scores=1)
        ex = np.take_along_axis(s[:nq], I, axis=1)
        worst = max(worst, float((np.abs(D.astype(np.float64) - ex) / E[:nq, None]).max()))
    Dc, Ic, st = _search(idx, q, 100)
    sb.check_topk(q, xs, Dc, Ic, 100, s=s)
    print("[i8 certificate] regime=%s d=%d worst |stage - exact| / E = %.4f uncertified=%d / %d"
          % (regime, d, worst, st[0], q.shape[0]))
    assert worst < 1.0


# ---------------------------------------------------------------------------------------------------------------------
# encoder writing int8 rows in place
# ---------------------------------------------------------------------------------------------------------------------
def _tiny_bert(hidden=128):
    from openmatch_b200 import synthetic
    from openmatch_b200.encoder import CudaEncoder
    spec = dict(arch="bert", layers=2, hidden=hidden, heads=2, ffn=512, vocab=2000, max_pos=128, type_vocab=2, ln_eps=1e-12)
    sd = synthetic.bert_state_dict(spec, seed=3)
    return CudaEncoder(spec, sd, pooling="first", max_batch_tokens=256 * 32), synthetic


def test_encoder_writes_int8_rows_in_place(om):
    enc, synthetic = _tiny_bert()
    ids, mask = synthetic.token_batch(200, 32, 2000, ragged=True)
    ids, mask = ids.cuda(), mask.cuda()
    r32 = enc.encode(ids, mask)
    lens = mask.sum(1).cpu()
    toks = ids[mask.bool()]
    p32 = enc.encode_packed(toks, lens)
    for name, write, want in (
            ("om_encode", lambda lo, rows: enc.encode(ids[lo:lo + 64], mask[lo:lo + 64], out=rows), r32),
            ("om_encode_packed", lambda lo, rows: enc.encode_packed(toks[int(lens[:lo].sum()):int(lens[:lo + 64].sum())],
                                                                   lens[lo:lo + 64], out=rows), p32)):
        idx = om.FlatIPIndex(enc.rep_dim, dtype=torch.int8)
        for lo in (0, 64):  # two batches: the second lands after the first at the row pitch
            rows = idx.reserve_rows(64)
            write(lo, rows)
            idx.commit_rows(64)
        ref = om.FlatIPIndex(enc.rep_dim, dtype=torch.int8)
        ref.add(want[:128])
        _check_stored(idx, want[:128].cpu().numpy(), name)
        for a, b in zip(_stored(idx), _stored(ref)):
            _same(a, b, "%s: in-place rows vs add of the fp32 output" % name)
        q = want[128:].float().cpu().numpy()
        for nq in (1, 72):
            D, I, _ = _search(idx, q[:nq], 20)
            D0, I0, _ = _search(ref, q[:nq], 20)
            _same(I, I0, "%s in-place I" % name)
            _same(D, D0, "%s in-place D" % name)
    with pytest.raises(RuntimeError, match="int8 rows need"):
        enc.encode(ids[:4], mask[:4], out=torch.empty((4, enc.rep_dim + 8), dtype=torch.int8, device="cuda")[:, :enc.rep_dim])


# ---------------------------------------------------------------------------------------------------------------------
# range rule, ABI, memory
# ---------------------------------------------------------------------------------------------------------------------
def test_nonfinite_input_is_refused(om):
    d = 64
    idx = om.FlatIPIndex(d, dtype=torch.int8)
    idx.add(np.ones((10, d), np.float32))
    for bad_value in (np.inf, -np.inf, np.nan):
        x = np.ones((5, d), np.float32)
        x[3, 7] = bad_value
        for data in (x, torch.from_numpy(x).cuda(), torch.from_numpy(x).half()):
            with pytest.raises(RuntimeError, match="inf or NaN"):
                idx.add(data)
            assert idx.ntotal == 10
    big = np.full((2, d), 3e38, np.float32)  # finite: any fp32 range is stored
    idx.add(big)
    assert idx.ntotal == 12
    D, I = idx.search(np.ones((1, d), np.float32), 3)
    assert list(I[0]) == [10, 11, 0]


def test_nonfinite_in_place_commit_blocks_search_until_reset(om):
    d = 72
    from openmatch_b200.index import _wrap_device
    idx = om.FlatIPIndex(d, dtype=torch.int8)
    rows = idx.reserve_rows(8)
    pitch = rows.stride(0)
    full = _wrap_device(rows.data_ptr(), (8, pitch), pitch, torch.int8)  # whole rows: codes, padding, scale
    full.zero_()
    rows.fill_(1)
    full[:, 80:84] = torch.tensor([1.0], device="cuda").view(torch.int8)  # scale 1.0 on every row
    full[2, 80:84] = torch.tensor([float("inf")], device="cuda").view(torch.int8)
    full[6, 80:84] = torch.tensor([float("nan")], device="cuda").view(torch.int8)
    idx.commit_rows(8)
    q = np.ones((3, d), np.float32)
    with pytest.raises(RuntimeError, match="inf or NaN"):
        idx.search(q, 4)
    assert idx.stat("nonfinite_rows") == 2
    with pytest.raises(RuntimeError, match="inf or NaN"):
        idx.search_device(torch.from_numpy(q).cuda(), 4)
    idx.reset()
    assert idx.stat("nonfinite_rows") == 0
    idx.add(np.eye(8, d, dtype=np.float32))
    D, I = idx.search(q, 4)
    assert idx.stat("nonfinite_rows") == 0 and list(I[0]) == [0, 1, 2, 3]


def test_abi_storage_rules(om):
    import ctypes

    from openmatch_b200 import _lib
    lib = _lib.load()
    h = ctypes.c_void_p()
    _lib.check(lib.om_index_create_typed(100, _lib.OM_I8, ctypes.byref(h)))
    try:
        assert lib.om_index_storage(h) == _lib.OM_I8
        p = ctypes.c_void_p()
        assert lib.om_index_reserve(h, 4, ctypes.byref(p)) == -5  # OM_ESTATE: cannot hand out fp32 rows
        pitch = ctypes.c_int64()
        _lib.check(lib.om_index_reserve_rows(h, 4, ctypes.byref(p), ctypes.byref(pitch)))
        assert pitch.value == 112 + 16 and p.value
    finally:
        lib.om_index_destroy(h)
    with pytest.raises(ValueError, match="int8"):
        from openmatch_b200.encoder import CudaEncoder  # noqa: F401
        enc, _ = _tiny_bert()
        enc.encode(torch.ones((1, 4), dtype=torch.int64, device="cuda"), torch.ones((1, 4), dtype=torch.int64, device="cuda"),
                   out_dtype=torch.int8)


def test_int8_storage_takes_dpad_plus_16_bytes_per_row(om):
    N, d = 1_000_000, 768
    drops = {}
    for dt in (torch.float16, torch.int8):
        idx = om.FlatIPIndex(d, dtype=dt)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        idx.reserve_rows(N)
        torch.cuda.synchronize()
        drops[dt] = free0 - torch.cuda.mem_get_info()[0]
        del idx
    cap = -(-N // 256) * 256  # index_grow: round_up(max(N, 1024), 256)
    print("[i8 memory] reserve_rows(%d) at d=%d: fp16 storage %.1f MiB, int8 storage %.1f MiB" %
          (N, d, drops[torch.float16] / 2 ** 20, drops[torch.int8] / 2 ** 20))
    assert abs(drops[torch.int8] - cap * (768 + 16)) <= 2 * 2 ** 20


# ---------------------------------------------------------------------------------------------------------------------
# streams and state
# ---------------------------------------------------------------------------------------------------------------------
def _busy(stream, seconds=0.2):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(seconds * 1.5e9))


def _i8_sequence(om, x, q, stream=None):
    out = []
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
    with ctx:
        if stream is not None:
            _busy(torch.cuda.default_stream())
        idx = om.FlatIPIndex(x.shape[1], dtype=torch.int8)
        xd = torch.from_numpy(x).cuda()
        idx.add(xd[:2000])
        idx.add(xd[2000:3000])
        qd = torch.from_numpy(q).cuda()
        for nq in (1, 129, 300):
            D, I = idx.search_device(qd[:nq], 20)
            out.append((D.clone(), I.clone(), tuple(idx.stat(s) for s in STATS)))
        idx.reset()
        idx.add(xd[3000:])
        D, I = idx.search_device(qd, 20)
        out.append((D.clone(), I.clone(), tuple(idx.stat(s) for s in STATS)))
    torch.cuda.synchronize()
    return out


def _same_seq(got, want, what):
    for i, ((D, I, st), (D0, I0, st0)) in enumerate(zip(got, want)):
        _same(I, I0, "%s step %d: I" % (what, i))
        _same(D, D0, "%s step %d: D" % (what, i))
        assert st == st0, "%s step %d: stats" % (what, i)


def test_int8_paths_on_a_side_stream_and_on_poisoned_allocations(om):
    x, q, _, _ = sb.make_regime("anisotropic", 300, 6000, 256, k=10, seed=53)
    want = _i8_sequence(om, x, q)
    _same_seq(_i8_sequence(om, x, q, torch.cuda.Stream()), want, "side stream")
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        _same_seq(_i8_sequence(om, x, q), want, "poisoned allocations")
        _same_seq(_i8_sequence(om, x, q, torch.cuda.Stream()), want, "poisoned allocations, side stream")
    finally:
        del os.environ["OPENMATCH_B200_POISON_ALLOC"]


# ---------------------------------------------------------------------------------------------------------------------
# drivers
# ---------------------------------------------------------------------------------------------------------------------
WORDS = ["the", "a", "of", "river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky", "rain",
         "city", "road", "car", "train", "music", "piano", "guitar", "stone", "bread", "cheese", "wine"]


def _run(main, argv):
    old = sys.argv
    sys.argv = ["prog"] + [str(a) for a in argv]
    try:
        main()
    finally:
        sys.argv = old


def test_build_index_and_retrieve_with_int8_index(om, tmp_path):
    import pickle

    from transformers import BertConfig, BertModel, BertTokenizer

    from openmatch.driver import build_index, retrieve
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + sorted(set(WORDS))
    (tmp_path / "vocab.txt").write_text("\n".join(vocab))
    tok = BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                     intermediate_size=256, max_position_embeddings=64)
    BertModel(cfg).save_pretrained(str(tmp_path / "model"))
    tok.save_pretrained(str(tmp_path / "model"))
    rng = np.random.default_rng(0)
    with open(tmp_path / "corpus.tsv", "w") as f:
        for i in range(300):
            f.write("d%d\t%s\t%s\n" % (i, " ".join(rng.choice(WORDS, 2)), " ".join(rng.choice(WORDS, 12))))
    with open(tmp_path / "queries.tsv", "w") as f:
        for i in range(9):
            f.write("q%d\t%s\n" % (i, " ".join(rng.choice(WORDS, 4))))

    def common(out):
        return ["--output_dir", out, "--model_name_or_path", tmp_path / "model", "--per_device_eval_batch_size", 32,
                "--q_max_len", 8, "--p_max_len", 32, "--dataloader_num_workers", 0]

    corpus = ["--corpus_path", tmp_path / "corpus.tsv", "--doc_template", "<title> <text>", "--doc_column_names",
              "id,title,text"]
    queries = ["--query_path", tmp_path / "queries.tsv", "--query_template", "<text>", "--query_column_names", "id,text",
               "--retrieve_depth", 20]
    e8, e32 = tmp_path / "emb8", tmp_path / "emb32"
    _run(build_index.main, common(e8) + corpus + ["--index_dtype", "int8"])
    _run(build_index.main, common(e32) + corpus)
    with open(e8 / "embeddings.corpus.rank.0", "rb") as f:
        enc8, ids8 = pickle.load(f)
    with open(e32 / "embeddings.corpus.rank.0", "rb") as f:
        enc32, ids32 = pickle.load(f)
    assert enc8.dtype == np.float32 and enc8.shape == (300, 128) and ids8 == ids32
    _same(enc8, io.stored_i8(enc32), "int8 index export vs dequantize(quantize(fp32 export))")
    # the int8 index over its own export (re-quantising dequantised rows gives the same rows back), and the fp32 index
    # over the exported (dequantised) embeddings
    _run(retrieve.main, common(e8) + queries + ["--trec_save_path", tmp_path / "run8.trec", "--index_dtype", "int8"])
    _run(retrieve.main, common(e8) + queries + ["--trec_save_path", tmp_path / "run32.trec"])
    run8, run32 = (tmp_path / "run8.trec").read_text(), (tmp_path / "run32.trec").read_text()
    assert len(run8.splitlines()) == 9 * 20
    assert run8 == run32


# ---------------------------------------------------------------------------------------------------------------------
# sharded search over int8 shards (tests/index_i8_dist_worker.py)
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join("tests", "index_i8_dist_worker.py")]
    env = dict(os.environ, NCCL_DEBUG="WARN", OMP_NUM_THREADS="8")
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_sharded_int8_search_equals_unsharded(om):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = _torchrun(2)
    assert r.returncode == 0 and "I8 DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_sharded_int8_entry_point_at_world_size_one(om):
    r = _torchrun(1, timeout=600)
    assert r.returncode == 0 and "I8 DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
