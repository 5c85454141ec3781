"""GPU: the index with fp16 row storage (``FlatIPIndex(d, dtype=torch.float16)``, ``om_index_create_typed(d, OM_F16)``).

Contract under test: search over an fp16 index is the exact top-k by fp32 inner product of the fp32 query with the
STORED fp16 rows, ties by ascending id.  So an fp16 index built from X must answer bit for bit like an fp32 index built
from X16 = fp16(X) (same scan operand, same re-score summation order, and a corpus quantisation term of 0 in both),
and the answer must pass the float64 oracle's check on X16 at the adversarial regimes of oracle/search_bound.py."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import search_bound as sb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS = ("uncertified", "uncertified_wide", "exact_queries")
DEFAULTS = {"round_growth": 0, "pair_scan": 1, "scan_cluster_q": 0, "scan_cluster_x": 0, "certify": 1, "exact_only": 0,
            "debug_stage_scores": 0, "force_safe_rounds": 0}


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def _bits(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _same(a, b, what):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
    if a.dtype.kind == "f":
        np.testing.assert_array_equal(_bits(a), _bits(b), err_msg=what)
    else:
        np.testing.assert_array_equal(a, b, err_msg=what)


def _search(idx, q, k, **params):
    for name, v in {**DEFAULTS, **params}.items():
        idx.set_param(name, v)
    D, I = idx.search(q, k)
    return D, I, tuple(idx.stat(s) for s in STATS)


# ---------------------------------------------------------------------------------------------------------------------
# bitwise equivalence: fp16 index of X == fp32 index of fp16(X)
# ---------------------------------------------------------------------------------------------------------------------
N_EQ = 12000
_PAIRS = {}


def _pair(om, d):
    if d not in _PAIRS:
        rng = np.random.default_rng(d)
        x = rng.standard_normal((N_EQ, d), dtype=np.float32)
        x[:40] = x[40:80]  # exact duplicates: ties broken by id
        h = om.FlatIPIndex(d, dtype=torch.float16)
        h.add(x)
        f = om.FlatIPIndex(d)
        f.add(_f16(x))
        _PAIRS[d] = (h, f, rng)
    return _PAIRS[d]


CONFIGS = [dict(), dict(pair_scan=0), dict(scan_cluster_q=2, scan_cluster_x=1), dict(scan_cluster_q=2, scan_cluster_x=2),
           dict(scan_cluster_q=4, scan_cluster_x=1), dict(scan_cluster_q=4, scan_cluster_x=2), dict(force_safe_rounds=1),
           dict(exact_only=1), dict(certify=0), dict(debug_stage_scores=1)]
# (nq, k, d): every nq of {1, 64, 128, 129, 300, 1000}, every k of {1, 10, 100, 1000, 4096}, every d of {64, 90, 768, 1024}
EQ_CASES = [(1, 1, 64), (64, 10, 90), (128, 100, 768), (129, 1000, 1024), (300, 4096, 90), (1000, 10, 768),
            (300, 100, 64), (129, 10, 90), (1, 4096, 768), (300, 1000, 1024)]


@pytest.mark.parametrize("nq,k,d", EQ_CASES, ids=["nq%d-k%d-d%d" % c for c in EQ_CASES])
def test_fp16_index_equals_fp32_index_of_rounded_rows(om, nq, k, d):
    h, f, rng = _pair(om, d)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    q[0] = _f16(np.arange(d, dtype=np.float32) % 7)  # a query with many tied scores
    for cfg in CONFIGS:
        Dh, Ih, sh = _search(h, q, k, **cfg)
        Df, If, sf = _search(f, q, k, **cfg)
        _same(Ih, If, "I %s" % cfg)
        _same(Dh, Df, "D %s" % cfg)
        assert sh == sf, "stats %s: fp16 index %s, fp32 index %s" % (cfg, sh, sf)


# ---------------------------------------------------------------------------------------------------------------------
# float64 oracle on the stored values
# ---------------------------------------------------------------------------------------------------------------------
K = 10
ORACLE_CASES = [("gaussian", 768, 20000), ("anisotropic", 768, 20000), ("coherent", 768, 20000),
                ("query_quant", 768, 20000), ("corpus_quant", 64, 20000), ("range_edges", 768, 20000)]


def _stored(x):
    """the corpus as fp16 storage holds it: range edges beyond the half range are saturated first (fp16 storage would
    refuse them), then rounded to nearest even"""
    return _f16(np.clip(x, -sb.F16_MAX, sb.F16_MAX))


@pytest.mark.parametrize("regime,d,n", ORACLE_CASES, ids=["%s-%d" % (r, d) for r, d, _ in ORACLE_CASES])
def test_oracle_on_stored_rows(om, regime, d, n):
    x, q, premise, _ = sb.make_regime(regime, 300, n, d, k=K, seed=d + 1)
    x16 = _stored(x)
    idx = om.FlatIPIndex(d, dtype=torch.float16)
    idx.add(x16)
    s, beta = sb.score64(q, x16), sb.rescore_bound(q, x16)
    for params in (dict(), dict(pair_scan=0), dict(round_growth=8)):
        D, I, st = _search(idx, q, K, **params)
        De, Ie, _ = _search(idx, q, K, exact_only=1, **params)
        _same(I, Ie, "%s %s: I vs exact_only" % (regime, params))
        _same(D, De, "%s %s: D vs exact_only" % (regime, params))
        rs = sb.check_topk(q, x16, D, I, K, s=s, beta=beta)
        print("[f16 numerics] regime=%s d=%d %s |D-s64|/beta=%.3f uncertified=%d uncertified_wide=%d exact_queries=%d"
              % (regime, d, params, rs["rescore_ratio"], *st))


def test_oracle_escalation_runs_on_half_precision_collisions(om):
    # 6000 rows that collide in fp16 (v + 1e-4 noise rounds to the same halves): the k-th score is tied far beyond the
    # widest candidate list, the certificate cannot hold and the exact scan answers
    rng = np.random.default_rng(4097)
    n, d = 20000, 128
    x = rng.standard_normal((n, d), dtype=np.float32)
    v = rng.standard_normal(d, dtype=np.float32)
    dup = rng.choice(n, 6000, replace=False)
    x[dup] = v + 1e-4 * rng.standard_normal((6000, d), dtype=np.float32)
    q = (v + 0.1 * rng.standard_normal((5, d), dtype=np.float32)).astype(np.float32)
    x16 = _f16(x)
    idx = om.FlatIPIndex(d, dtype=torch.float16)
    idx.add(x)
    for k in (10, 1000):
        D, I, st = _search(idx, q, k)
        assert st[0] > 0 and st[2] > 0, "premise: the escalation levels must run (stats %s)" % (st,)
        sb.check_topk(q, x16, D, I, k)


# ---------------------------------------------------------------------------------------------------------------------
# ingest routes and the encoder's fp16 output
# ---------------------------------------------------------------------------------------------------------------------
def _tiny_bert():
    from openmatch_b200 import synthetic
    from openmatch_b200.encoder import CudaEncoder
    spec = dict(arch="bert", layers=2, hidden=128, heads=2, ffn=512, vocab=2000, max_pos=128, type_vocab=2, ln_eps=1e-12)
    sd = synthetic.bert_state_dict(spec, seed=3)
    return CudaEncoder(spec, sd, pooling="first", max_batch_tokens=256 * 32), synthetic


def test_ingest_routes_equal_add_of_fp16_values(om):
    rng = np.random.default_rng(11)
    n, d = 3000, 90
    x = rng.standard_normal((n, d), dtype=np.float32) * 3
    x16 = torch.from_numpy(x).half()
    ref = om.FlatIPIndex(d, dtype=torch.float16)
    ref.add(x16.cuda())
    q = rng.standard_normal((129, d), dtype=np.float32)
    D0, I0, st0 = _search(ref, q, 50)
    xb = torch.from_numpy(x).bfloat16()
    routes = {"host f32": x, "host f32 tensor": torch.from_numpy(x), "host bf16": xb, "host f16": x16,
              "host f16 numpy": x16.numpy(), "device f32": torch.from_numpy(x).cuda(), "device bf16": xb.cuda(),
              "device f16": x16.cuda()}
    for name, data in routes.items():
        idx = om.FlatIPIndex(d, dtype=torch.float16)
        idx.add(data[:1000])
        idx.add(data[1000:])
        want = xb.float().half() if "bf16" in name else x16
        rows = idx.master_rows()
        assert rows.dtype == torch.float16 and rows.shape == (n, d) and rows.stride() == (96, 1)
        _same(rows, want, "%s: stored rows" % name)
        if "bf16" not in name:
            D, I, st = _search(idx, q, 50)
            _same(I, I0, name)
            _same(D, D0, name)
            assert st == st0


def test_encoder_writes_fp16_rows_in_place(om):
    enc, synthetic = _tiny_bert()
    ids, mask = synthetic.token_batch(200, 32, 2000, ragged=True)
    ids, mask = ids.cuda(), mask.cuda()
    r32 = enc.encode(ids, mask)
    r16 = enc.encode(ids, mask, out_dtype=torch.float16)
    _same(r16, r32.half(), "fp16 encoder output vs fp16(fp32 output)")
    idx = om.FlatIPIndex(enc.rep_dim, dtype=torch.float16)
    for lo in (0, 64):  # two batches: the second lands after the first at the row pitch
        rows = idx.reserve_rows(64)
        enc.encode(ids[lo:lo + 64], mask[lo:lo + 64], out=rows)
        idx.commit_rows(64)
    ref = om.FlatIPIndex(enc.rep_dim, dtype=torch.float16)
    ref.add(r32[:128].half())
    _same(idx.master_rows(), ref.master_rows(), "in-place rows")
    q = r32[128:].float().cpu().numpy()
    for nq in (1, 72):
        D, I, st = _search(idx, q[:nq], 20)
        D0, I0, st0 = _search(ref, q[:nq], 20)
        _same(I, I0, "in-place I")
        _same(D, D0, "in-place D")
        assert st == st0


# ---------------------------------------------------------------------------------------------------------------------
# range rule
# ---------------------------------------------------------------------------------------------------------------------
def test_out_of_range_input_is_refused(om):
    d = 64
    idx = om.FlatIPIndex(d, dtype=torch.float16)
    good = np.ones((10, d), np.float32)
    idx.add(good)
    for bad_value in (65520.0, -7e4, np.inf, np.nan):
        x = np.ones((5, d), np.float32)
        x[3, 7] = bad_value
        for data in (x, torch.from_numpy(x).cuda()):
            with pytest.raises(RuntimeError, match="fp16"):
                idx.add(data)
            assert idx.ntotal == 10
    edge = np.full((2, d), 65519.0, np.float32)  # rounds down to 65504
    idx.add(edge)
    assert idx.ntotal == 12 and (idx.master_rows()[10:].float() == 65504.0).all()
    D, I = idx.search(np.ones((1, d), np.float32), 3)
    assert list(I[0]) == [10, 11, 0]
    # fp32 indices keep their behaviour: the same input is accepted
    f = om.FlatIPIndex(d)
    f.add(x)
    assert f.ntotal == 5


def test_nonfinite_in_place_commit_blocks_search_until_reset(om):
    d = 72
    idx = om.FlatIPIndex(d, dtype=torch.float16)
    rows = idx.reserve_rows(8)
    rows.copy_(torch.ones(8, d))
    rows[2, 5] = float("inf")
    rows[6, 0] = float("nan")
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
    assert lib.om_index_create_typed(16, _lib.OM_BF16, ctypes.byref(h)) == -1
    _lib.check(lib.om_index_create_typed(16, _lib.OM_F16, ctypes.byref(h)))
    try:
        assert lib.om_index_storage(h) == _lib.OM_F16
        p = ctypes.c_void_p()
        assert lib.om_index_reserve(h, 4, ctypes.byref(p)) == -5  # OM_ESTATE: cannot hand out fp32 rows
        pitch = ctypes.c_int64()
        _lib.check(lib.om_index_reserve_rows(h, 4, ctypes.byref(p), ctypes.byref(pitch)))
        assert pitch.value == 16 and p.value
    finally:
        lib.om_index_destroy(h)
    f = om.FlatIPIndex(20)
    assert lib.om_index_storage(f._h) == _lib.OM_F32
    assert f.reserve_rows(3).dtype == torch.float32


# ---------------------------------------------------------------------------------------------------------------------
# memory
# ---------------------------------------------------------------------------------------------------------------------
def test_fp16_storage_takes_a_third_of_the_memory(om):
    N, d = 1_000_000, 768
    drops = {}
    for dt in (torch.float32, torch.float16):
        idx = om.FlatIPIndex(d, dtype=dt)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        idx.reserve_rows(N)
        torch.cuda.synchronize()
        drops[dt] = free0 - torch.cuda.mem_get_info()[0]
        del idx
    cap = -(-N // 256) * 256  # index_grow: round_up(max(N, 1024), 256)
    print("[f16 memory] reserve_rows(%d) at d=%d: fp32 storage %.1f MiB, fp16 storage %.1f MiB" %
          (N, d, drops[torch.float32] / 2 ** 20, drops[torch.float16] / 2 ** 20))
    assert abs(drops[torch.float16] - cap * 768 * 2) <= 2 * 2 ** 20
    assert abs(drops[torch.float16] / drops[torch.float32] - 1 / 3) < 0.01


# ---------------------------------------------------------------------------------------------------------------------
# streams and state
# ---------------------------------------------------------------------------------------------------------------------
def _busy(stream, seconds=0.2):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(seconds * 1.5e9))


def _f16_sequence(om, x, q, stream=None):
    """add -> reserve / commit -> search (nq = 1, 129, 300) -> reset -> add -> search on `stream` (None: the default
    stream), with a busy default stream in front when a side stream is used"""
    out = []
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
    with ctx:
        if stream is not None:
            _busy(torch.cuda.default_stream())
        idx = om.FlatIPIndex(x.shape[1], dtype=torch.float16)
        xd = torch.from_numpy(x).cuda()
        idx.add(xd[:2000])
        rows = idx.reserve_rows(1000)
        rows.copy_(xd[2000:3000])
        idx.commit_rows(1000)
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


def test_fp16_paths_on_a_side_stream_and_on_poisoned_allocations(om):
    x, q, _, _ = sb.make_regime("anisotropic", 300, 6000, 256, k=10, seed=53)
    want = _f16_sequence(om, x, q)
    _same_seq(_f16_sequence(om, x, q, torch.cuda.Stream()), want, "side stream")
    os.environ["OPENMATCH_B200_POISON_ALLOC"] = "1"
    try:
        probe = om.FlatIPIndex(256, dtype=torch.float16)
        assert torch.isnan(probe.reserve_rows(100)).all(), "premise: fresh rows must hold the NaN poison"
        _same_seq(_f16_sequence(om, x, q), want, "poisoned allocations")
        _same_seq(_f16_sequence(om, x, q, torch.cuda.Stream()), want, "poisoned allocations, side stream")
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


def test_build_index_and_retrieve_with_fp16_index(om, tmp_path):
    import pickle

    from transformers import BertConfig, BertModel, BertTokenizer

    from openmatch.driver import build_index, retrieve
    from openmatch_b200.embedding_store import EmbeddingFile
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
    e16, e32 = tmp_path / "emb16", tmp_path / "emb32"
    _run(build_index.main, common(e16) + corpus + ["--index_dtype", "float16"])
    _run(build_index.main, common(e32) + corpus)
    with open(e16 / "embeddings.corpus.rank.0", "rb") as f:
        enc16, ids16 = pickle.load(f)
    with open(e32 / "embeddings.corpus.rank.0", "rb") as f:
        enc32, ids32 = pickle.load(f)
    assert enc16.dtype == np.float32 and enc16.shape == (300, 128) and ids16 == ids32
    _same(enc16, _f16(enc32), "fp16 index export vs fp16(fp32 export)")
    ef = EmbeddingFile(str(e16 / "embeddings.corpus.rank.0"))
    assert ef.shape == (300, 128) and list(ef.ids) == ids16
    _same(np.concatenate([np.asarray(c) for c in ef.chunks()]), enc16, "EmbeddingFile rows")
    # the fp16 index over its own export, and the fp32 index over the same (fp16-rounded) embeddings
    _run(retrieve.main, common(e16) + queries + ["--trec_save_path", tmp_path / "run16.trec", "--index_dtype", "float16"])
    _run(retrieve.main, common(e16) + queries + ["--trec_save_path", tmp_path / "run32.trec"])
    run16, run32 = (tmp_path / "run16.trec").read_text(), (tmp_path / "run32.trec").read_text()
    assert len(run16.splitlines()) == 9 * 20
    assert run16 == run32


# ---------------------------------------------------------------------------------------------------------------------
# sharded search over fp16 shards (tests/index_f16_dist_worker.py)
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join("tests", "index_f16_dist_worker.py")]
    env = dict(os.environ, NCCL_DEBUG="WARN", OMP_NUM_THREADS="8")
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_sharded_fp16_search_equals_unsharded(om):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = _torchrun(2)
    assert r.returncode == 0 and "F16 DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_sharded_fp16_entry_point_at_world_size_one(om):
    r = _torchrun(1, timeout=600)
    assert r.returncode == 0 and "F16 DIST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
