"""CPU: argument and dtype rules of int8 index storage that hold without a GPU, the int8 oracle's quantiser at its edge
cases, and the int8 terms of the certificate on a CPU model (tests/index_i8_oracle.py)."""
import ctypes
import types

import numpy as np
import pytest
import torch

import index_i8_oracle as io
from oracle import search_bound as sb


def test_storage_and_dtype_rules():
    from openmatch_b200 import _lib
    from openmatch_b200.encoder import _OUT_DTYPES
    from openmatch_b200.index import _STORAGE
    lib = _lib.load()
    assert _lib.OM_I8 == 3 and lib.om_abi_version() == 2
    assert _STORAGE[torch.int8] == _lib.OM_I8 and _OUT_DTYPES[torch.int8] == _lib.OM_I8
    h = ctypes.c_void_p()
    assert lib.om_index_create_typed(16, 9, ctypes.byref(h)) == -1 and b"OM_I8" in lib.om_last_error()
    # the fused loss takes fp32 / bf16 only: int8 is refused before any device work
    assert lib.om_contrastive_loss_fwd_bwd(1, 1, _lib.OM_I8, 1, 1, 8, None, 0, ctypes.c_float(1.0), 1, None, None, None,
                                           None) == -1


def test_index_dtype_argument_takes_int8():
    from openmatch_b200.arguments import InferenceArguments
    from openmatch_b200.retriever.dense_retriever import _index_dtype
    assert "int8" in InferenceArguments.__dataclass_fields__["index_dtype"].metadata["help"]
    assert _index_dtype(types.SimpleNamespace(index_dtype="int8")) == torch.int8
    with pytest.raises(ValueError, match="int8"):
        _index_dtype(types.SimpleNamespace(index_dtype="uint8"))


def test_quantiser_edge_cases():
    d = 40
    x = np.zeros((7, d), np.float32)
    x[1, 3] = 5.0                                  # one dominant element, the rest zero
    x[2] = np.linspace(-1, 1, d, dtype=np.float32)
    x[2, 0] = 1000.0                               # dominant element over small ones: most codes round to 0
    x[3] = 1e-30 * np.arange(d, dtype=np.float32)  # tiny scale (normal)
    x[4, :2] = (1e-44, -3e-44)                     # subnormal values: the scale rounds to 0 -> a zero row
    x[5] = np.float32(127) * np.arange(-20, 20, dtype=np.float32)  # codes with exact halves: ties to even
    x[6] = -2.5
    c, s = io.quantize_i8(x)
    assert s[0] == 0 and (c[0] == 0).all()
    assert s[1] == np.float32(5.0) / np.float32(127) and c[1, 3] == 127 and np.count_nonzero(c[1]) == 1
    assert c[2, 0] == 127 and np.abs(c[2, 1:]).max() <= 1
    assert s[3] > 0 and np.abs(c[3]).max() == 127
    assert s[4] == 0 and (c[4] == 0).all()
    assert np.abs(c).max() <= 127 and c.min() >= -127
    assert (c[6] == -127).all() and s[6] == np.float32(2.5) / np.float32(127)
    # half-to-even: x / s exactly k + 1/2 rounds to the even neighbour
    y = np.array([[127.0, 0.5, 1.5, 2.5, -0.5, -1.5]], np.float32)
    cy, sy = io.quantize_i8(y)
    assert sy[0] == 1.0 and list(cy[0]) == [127, 0, 2, 2, 0, -2]
    # dequantised values: fp32(s * c)
    xs = io.dequantize_i8(c, s)
    assert xs.dtype == np.float32 and np.array_equal(xs[1, 3], np.float32(s[1] * np.float32(127)))
    rel = np.abs(xs[2:4] - x[2:4]).max(axis=1) / s[2:4]
    assert (rel <= 0.5 + 1e-6).all()


def test_query_split_reaches_fifteen_bits():
    rng = np.random.default_rng(0)
    q = rng.standard_normal((64, 768), dtype=np.float32)
    q[0] = 0
    q[1, 5] = 1e4  # one dominant element: the low level carries the rest
    qh, ql, sh, sl = io.query_split_i8(q)
    assert np.abs(qh).max() <= 127 and np.abs(ql).max() <= 127
    a, b = io.query_norms_i8(q)
    assert a[0] == 0 and b[0] == 0
    n = np.linalg.norm(q.astype(np.float64), axis=1)
    # the residual after two levels is below half a step of sig_lo per element
    assert (b[1:] <= 0.5 * sl[1:].astype(np.float64) * np.sqrt(768) * 1.0001).all()
    assert np.median(b[2:] / n[2:]) < 2e-4


@pytest.mark.parametrize("regime", ["gaussian", "anisotropic", "coherent"])
def test_certificate_terms_on_a_cpu_model(regime):
    """E(q) of an int8 index bounds |stage - fp32 re-score| for every row: the accumulation term covers the scan's
    fp32 roundings, the stored-value gap and the re-score; the query term covers |<q - q_h, x^>|."""
    x, q, _, _ = sb.make_regime(regime, 64, 3000, 256, k=10, seed=7)
    c, s = io.quantize_i8(x)
    xs = io.dequantize_i8(c, s)
    t = io.i8_terms(q, xs)
    assert (t["stage_rounding"] + t["stored_vs_real"] + t["rescore"] <= t["accumulation"]).all()
    E = io.cert_E_i8(q, xs)
    exact = sb.score64(q, xs)
    stage = io.stage_i8(q, c, s)  # before its fp32 roundings
    gap = np.abs(stage - exact).max(axis=1)
    qt = io.cert_E_i8(q, xs, terms=True)["query_quant"]
    assert (gap <= qt * (1 + 1e-9) + 2 * t["stored_vs_real"]).all()
    assert (gap + t["stage_rounding"] + t["rescore"] < E).all()
    print("[i8 model] %s: worst (|stage - exact| + roundings) / E = %.3f" %
          (regime, float(((gap + t["stage_rounding"] + t["rescore"]) / E).max())))
