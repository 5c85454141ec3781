"""GPU: the host-resident index (``om_index_create_host``, ``FlatIPIndex(memory="host")``).

Contract under test: an index whose rows live in pinned host memory and are streamed through the GPU one partition of
``window_rows`` rows at a time returns D and I byte-identical to a device index that received the same adds, for every
storage, k <= 4096, filters, ties across partition boundaries and escalated queries.  The calls it does not offer
return their codes and write nothing."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.float16, torch.int8]


@pytest.fixture(scope="module")
def om():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from openmatch_b200 import index as om_index
    return om_index


def _same(got, want, what):
    Dg, Ig = (t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in got)
    Dw, Iw = (t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in want)
    assert Dg.shape == Dw.shape and Ig.shape == Iw.shape, what
    if Dg.tobytes() != Dw.tobytes() or Ig.tobytes() != Iw.tobytes():
        bad = np.argwhere((Dg.view(np.int32) != Dw.view(np.int32)) | (Ig != Iw))
        r, c = bad[0]
        raise AssertionError("%s: %d slots differ, first (query %d, rank %d): host (%r, %d) device (%r, %d)"
                             % (what, len(bad), r, c, Dg[r, c], Ig[r, c], Dw[r, c], Iw[r, c]))


def _pair(om, dtype, window, d, *adds):
    dev = om.FlatIPIndex(d, dtype)
    host = om.FlatIPIndex(d, dtype, memory="host", window_rows=window)
    for x in adds:
        dev.add(x)
        host.add(x)
    assert host.ntotal == dev.ntotal
    return dev, host


def _data(seed, n, d, nq):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, d), dtype=np.float32), rng.standard_normal((nq, d), dtype=np.float32), rng


# ---------------------------------------------------------------------------------------------------------------------
# the grid: storage x window x nq x k, with a partial last partition, k above a partition and above n
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("window", [256, 4096, 16384])
def test_grid(om, dtype, window):
    n, d = 10077, 64
    x, q, _ = _data(1, n, d, 300)
    dev, host = _pair(om, dtype, window, d, x[:6000], x[6000:])
    for nq in (1, 64, 300):
        for k in (1, 10, 1000, 4096):
            _same(host.search(q[:nq], k), dev.search(q[:nq], k), "%s window %d nq %d k %d" % (dtype, window, nq, k))
    assert host.stat("partitions") == (n + window - 1) // window
    # k above n
    small_dev, small_host = _pair(om, dtype, window, d, x[:3001])
    _same(small_host.search(q[:64], 4096), small_dev.search(q[:64], 4096), "%s window %d k > n" % (dtype, window))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
def test_ties_across_partitions(om, dtype):
    """Integer rows repeated every 37 rows: each score is shared by rows in many partitions, so the merge must order the
    equal scores by id across partition boundaries."""
    rng = np.random.default_rng(2)
    base = rng.integers(-2, 3, (37, 32)).astype(np.float32)
    x = base[np.arange(5000) % 37]
    q = rng.integers(-2, 3, (70, 32)).astype(np.float32)
    dev, host = _pair(om, dtype, 256, 32, x)
    for k in (10, 200, 1000):
        D, I = host.search(q, k)
        _same((D, I), dev.search(q, k), "%s ties k %d" % (dtype, k))
        assert (np.diff(D, axis=1) <= 0).all()


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
def test_escalation_inside_partitions(om, dtype):
    """6000 near-duplicate rows inside one 8192-row partition: the queries that meet them fail the certificate at level 0
    and at the 4096-wide level and are answered by the exact scan, inside the partition."""
    n, d, nq, k = 20000, 64, 40, 50
    x, q, rng = _data(3, n, d, nq)
    v = rng.standard_normal(d, dtype=np.float32)
    x[1000:7000] = v + 1e-6 * rng.standard_normal((6000, d), dtype=np.float32)
    q[1::2] = v + 0.05 * rng.standard_normal((nq // 2, d), dtype=np.float32)
    dev, host = _pair(om, dtype, 8192, d, x)
    _same(host.search(q, k), dev.search(q, k), "%s escalated" % dtype)
    stats = {s: host.stat(s) for s in ("uncertified", "uncertified_wide", "exact_queries", "partitions")}
    print("[host escalated] %s: %s" % (dtype, stats))
    assert stats["uncertified"] > 0 and stats["exact_queries"] > 0 and stats["partitions"] == 3


# ---------------------------------------------------------------------------------------------------------------------
# filters
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
@pytest.mark.parametrize("nq", [8, 300])
def test_filters(om, dtype, nq):
    n, d, k = 9000, 64, 100
    x, q, rng = _data(4, n, d, nq)
    dev, host = _pair(om, dtype, 1024, d, x)
    sparse = torch.from_numpy(rng.random(n) < 0.01)
    span = torch.zeros(n, dtype=torch.bool)
    span[700:3300] = True  # crosses partitions 0 .. 3
    hole = torch.ones(n, dtype=torch.bool)
    hole[2048:3072] = False  # partition 2 has no allowed row
    for name, allow in (("1 %", sparse), ("span", span), ("empty partition", hole)):
        _same(host.search(q, k, allow=allow), dev.search(q, k, allow=allow), "%s %s" % (dtype, name))
    top = dev.search(q, 300)[1]
    excl = [list(rng.choice(top[i], 60, replace=False)) + [1, 2049, 8999] for i in range(nq)]
    _same(host.search(q, k, exclude=excl), dev.search(q, k, exclude=excl), "%s exclusions" % dtype)
    _same(host.search(q, k, allow=span, exclude=excl), dev.search(q, k, allow=span, exclude=excl), "%s both" % dtype)


# ---------------------------------------------------------------------------------------------------------------------
# adds
# ---------------------------------------------------------------------------------------------------------------------
def _add_abi(idx, x: torch.Tensor):
    """om_index_add of a host or CUDA tensor in its own dtype (fp32, bf16 or fp16), straight through the C ABI."""
    from openmatch_b200 import _lib
    x = x.contiguous()
    kind = _lib.OM_DEVICE if x.is_cuda else _lib.OM_HOST
    dt = {torch.float32: _lib.OM_F32, torch.bfloat16: _lib.OM_BF16, torch.float16: _lib.OM_F16}[x.dtype]
    _lib.check(idx._lib.om_index_add(idx._h, x.data_ptr(), kind, dt, x.shape[0], torch.cuda.current_stream().cuda_stream))
    torch.cuda.current_stream().synchronize()


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "i8"])
def test_adds(om, dtype):
    """Adds of sizes that straddle chunk boundaries, host and device inputs in fp32, bf16 and fp16, then reset and re-add."""
    d = 48
    x, q, _ = _data(5, 5000, d, 50)
    t = torch.from_numpy(x)
    inputs = [t[:100], t[100:700].cuda(), t[700:2000].to(torch.bfloat16), t[2000:2001].half().cuda(),
              t[2001:3500].half(), t[3500:4100].to(torch.bfloat16).cuda(), t[4100:5000]]
    dev = om.FlatIPIndex(d, dtype)
    host = om.FlatIPIndex(d, dtype, memory="host", window_rows=512)
    for xi in inputs:
        _add_abi(dev, xi)
        _add_abi(host, xi)
    assert host.ntotal == dev.ntotal == 5000
    _same(host.search(q, 64), dev.search(q, 64), "%s mixed adds" % dtype)
    dev.reset()
    host.reset()
    assert host.ntotal == 0
    dev.add(x[:1500])
    host.add(x[:1500])
    _same(host.search(q, 64), dev.search(q, 64), "%s after reset" % dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.int8], ids=["f16", "i8"])
def test_refused_add_changes_nothing(om, dtype):
    d = 32
    x, q, _ = _data(6, 3000, d, 20)
    dev, host = _pair(om, dtype, 256, d, x[:1000])
    want = host.search(q, 30)
    bad = x[1000:2000].copy()
    bad[900, 3] = 70000.0 if dtype == torch.float16 else np.inf  # in the add's fourth chunk
    with pytest.raises(RuntimeError, match="no row was added"):
        host.add(bad)
    if dtype == torch.float16:
        bad[900, 3] = np.nan
        with pytest.raises(RuntimeError, match="no row was added"):
            host.add(bad)
    assert host.ntotal == 1000
    _same(host.search(q, 30), want, "%s after a refused add" % dtype)
    dev.add(x[1000:2000])
    host.add(x[1000:2000])
    _same(host.search(q, 30), dev.search(q, 30), "%s add after a refused one" % dtype)


# ---------------------------------------------------------------------------------------------------------------------
# memkinds, edges, streams
# ---------------------------------------------------------------------------------------------------------------------
def test_memkinds_and_edges(om):
    d = 64
    x, q, _ = _data(7, 2500, d, 33)
    dev, host = _pair(om, torch.float16, 512, d, x)
    want = dev.search(q, 20)
    qd = torch.from_numpy(q).cuda()
    _same(host.search_device(qd, 20), want, "device in, device out")
    qp = torch.from_numpy(q).pin_memory()
    Dp, Ip = torch.empty((33, 20)).pin_memory(), torch.empty((33, 20), dtype=torch.int64).pin_memory()
    host.search_pinned(qp, 20, Dp, Ip)
    _same((Dp, Ip), want, "host in, host out")
    _same(host.search(qd, 20), want, "device in, host out")
    D0, I0 = host.search(q[:0], 5)
    assert D0.shape == (0, 5) and I0.shape == (0, 5)
    empty = om.FlatIPIndex(d, torch.float16, memory="host", window_rows=256)
    D, I = empty.search(q, 7)
    assert (I == -1).all() and (D == np.float32(-np.finfo(np.float32).max)).all()
    auto = om.FlatIPIndex(d, torch.int8, memory="host")
    auto.add(x)
    dev8 = om.FlatIPIndex(d, torch.int8)
    dev8.add(x)
    _same(auto.search(q, 20), dev8.search(q, 20), "automatic window")
    assert auto.stat("partitions") == 1


def test_side_stream(om):
    """A search on a non-blocking side stream whose earlier work (the query upload) is still running: the uploads of the
    partitions must wait for it, and the result is the default-stream one."""
    d = 64
    x, q, _ = _data(8, 6000, d, 40)
    dev, host = _pair(om, torch.float32, 1024, d, x)
    want = dev.search(q, 25)
    s = torch.cuda.Stream()
    qd = torch.from_numpy(q).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        qs = torch.empty_like(qd)
        cycles = int(0.1 * torch.cuda.get_device_properties(0).clock_rate * 1e3)
        torch.cuda._sleep(cycles)
        qs.copy_(qd)
        assert not s.query(), "premise: the side stream must still be busy"
        host.set_param("profile", 1)
        got = host.search_device(qs, 25)
        host.set_param("profile", 0)
    _same(got, want, "side stream")
    assert host.stat("partitions") == 6 and host.stat("upload_wait_ns") >= 0


def test_poisoned_allocations():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    code = r"""
import numpy as np, torch
from openmatch_b200 import index as om
rng = np.random.default_rng(9)
x = rng.standard_normal((5000, 72), dtype=np.float32); q = rng.standard_normal((70, 72), dtype=np.float32)
for dt in (torch.float32, torch.float16, torch.int8):
    dev = om.FlatIPIndex(72, dt); host = om.FlatIPIndex(72, dt, memory="host", window_rows=768)
    for a, b in ((0, 1700), (1700, 5000)):
        dev.add(x[a:b]); host.add(x[a:b])
    for k in (1, 100, 1500):
        Dd, Id = dev.search(q, k); Dh, Ih = host.search(q, k)
        assert Dd.tobytes() == Dh.tobytes() and Ih.tobytes() == Id.tobytes(), (dt, k)
print("ok")
"""
    env = dict(os.environ, OPENMATCH_B200_POISON_ALLOC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# refused entry points
# ---------------------------------------------------------------------------------------------------------------------
def test_refused_entry_points(om):
    from openmatch_b200 import _lib
    lib = _lib.load()
    d, nq, k = 32, 4, 5
    x, q, _ = _data(10, 600, d, nq)
    host = om.FlatIPIndex(d, torch.float32, memory="host", window_rows=256)
    host.add(x)
    st = torch.cuda.current_stream().cuda_stream
    p, pitch, fp = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
    assert lib.om_index_reserve_rows(host._h, 10, ctypes.byref(p), ctypes.byref(pitch)) == -5
    assert b"host-resident" in lib.om_last_error()
    assert lib.om_index_reserve(host._h, 10, ctypes.byref(fp)) == -5
    assert lib.om_index_commit(host._h, 10, st) == -5
    assert p.value is None and fp.value is None and host.ntotal == 600
    with pytest.raises(RuntimeError, match="host-resident"):
        host.reserve_rows(10)

    qd = torch.from_numpy(q).cuda()
    D = torch.full((nq, k), 7.0, device="cuda")
    I = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    lims = torch.full((nq + 1,), 7, dtype=torch.int64)
    rho = torch.zeros(nq, device="cuda")
    dummy_comm = ctypes.c_void_p(1)  # never dereferenced: the host-resident index is refused first
    rcs = [
        lib.om_index_search_sharded(host._h, dummy_comm, qd.data_ptr(), _lib.OM_DEVICE, nq, k, D.data_ptr(), I.data_ptr(),
                                    _lib.OM_DEVICE, 0, st),
        lib.om_index_search_sharded_filtered(host._h, dummy_comm, qd.data_ptr(), _lib.OM_DEVICE, nq, k, D.data_ptr(),
                                             I.data_ptr(), _lib.OM_DEVICE, 0, None, st),
        lib.om_index_range_search(host._h, qd.data_ptr(), _lib.OM_DEVICE, nq, rho.data_ptr(), lims.data_ptr(), _lib.OM_HOST,
                                  0, st),
        lib.om_index_range_search_sharded(host._h, dummy_comm, qd.data_ptr(), _lib.OM_DEVICE, nq, rho.data_ptr(),
                                          lims.data_ptr(), _lib.OM_HOST, 0, st),
    ]
    assert rcs == [-1, -1, -1, -1]
    assert b"host-resident" in lib.om_last_error()
    torch.cuda.synchronize()
    assert (D == 7.0).all() and (I == 7).all() and (lims == 7).all()
    with pytest.raises(RuntimeError, match="host-resident"):
        host.range_search(q, 0.0)
    h = ctypes.c_void_p()
    assert lib.om_index_create_host(d, _lib.OM_F16, 300, ctypes.byref(h)) == -1 and not h.value
    assert lib.om_index_create_host(d, _lib.OM_F16, -256, ctypes.byref(h)) == -1 and not h.value


# ---------------------------------------------------------------------------------------------------------------------
# retriever and driver
# ---------------------------------------------------------------------------------------------------------------------
def _args(tmp, **kw):
    base = dict(device=torch.device("cuda"), fp16=False, bf16=False, per_device_eval_batch_size=16, dataloader_num_workers=0,
                dataloader_pin_memory=False, output_dir=str(tmp), process_index=0, local_process_index=0, world_size=1,
                use_gpu=True)
    base.update(kw)
    return types.SimpleNamespace(**base)


@pytest.mark.parametrize("index_dtype", ["float32", "int8"])
def test_retriever_from_embeddings(om, tmp_path, index_dtype):
    import pickle
    from openmatch_b200.retriever.dense_retriever import Retriever
    rng = np.random.default_rng(11)
    d, sizes = 40, (700, 1, 1300)
    for r, n in enumerate(sizes):
        with open(tmp_path / f"embeddings.corpus.rank.{r}", "wb") as f:
            pickle.dump((rng.integers(-3, 4, (n, d)).astype(np.float32), [f"d{r}_{i}" for i in range(n)]), f, protocol=4)
    with open(tmp_path / "embeddings.query.rank.0", "wb") as f:
        pickle.dump((rng.integers(-3, 4, (25, d)).astype(np.float32), [f"q{i}" for i in range(25)]), f, protocol=4)

    class NoModel(torch.nn.Module):
        pass

    results = {}
    for memory in ("device", "host"):
        r = Retriever.from_embeddings(NoModel(), _args(tmp_path, index_dtype=index_dtype, index_memory=memory))
        assert r.index.memory == memory and r.index.ntotal == sum(sizes)
        results[memory] = r.search(topk=100, as_arrays=True)
    a, b = results["device"], results["host"]
    assert list(a.query_ids) == list(b.query_ids) and list(a.doc_names) == list(b.doc_names)
    _same((b.D, b.I), (a.D, a.I), "retriever %s" % index_dtype)


def test_retrieve_driver_trec_identical(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from transformers import BertConfig, BertModel, BertTokenizer
    from openmatch.driver import build_index, retrieve
    words = ["river", "bank", "money", "loan", "water", "fish", "tree", "green", "blue", "sky", "rain", "city", "road"]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    (tmp_path / "vocab.txt").write_text("\n".join(vocab))
    tok = BertTokenizer(str(tmp_path / "vocab.txt"), do_lower_case=True)
    torch.manual_seed(0)
    model_dir = tmp_path / "model"
    BertModel(BertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=256, max_position_embeddings=64)).save_pretrained(str(model_dir))
    tok.save_pretrained(str(model_dir))
    rng = np.random.default_rng(12)
    with open(tmp_path / "corpus.tsv", "w") as f:
        for i in range(600):
            f.write("d%d\t%s\n" % (i, " ".join(rng.choice(words, 10))))
    with open(tmp_path / "queries.tsv", "w") as f:
        for i in range(9):
            f.write("q%d\t%s\n" % (i, " ".join(rng.choice(words, 4))))

    def run(main, argv):
        old = sys.argv
        sys.argv = ["prog"] + [str(a) for a in argv]
        try:
            main()
        finally:
            sys.argv = old

    emb = tmp_path / "emb"
    common = ["--output_dir", emb, "--model_name_or_path", model_dir, "--per_device_eval_batch_size", 16, "--q_max_len", 8,
              "--p_max_len", 16, "--dataloader_num_workers", 0]
    run(build_index.main, common + ["--corpus_path", tmp_path / "corpus.tsv", "--doc_template", "<text>",
                                    "--doc_column_names", "id,text"])
    runs = {}
    for memory in ("device", "host"):
        runs[memory] = tmp_path / ("run.%s.trec" % memory)
        run(retrieve.main, common + ["--query_path", tmp_path / "queries.tsv", "--query_template", "<text>",
                                     "--query_column_names", "id,text", "--trec_save_path", runs[memory],
                                     "--retrieve_depth", 50, "--index_memory", memory])
    a, b = runs["device"].read_bytes(), runs["host"].read_bytes()
    assert len(a.splitlines()) == 9 * 50 and a == b
