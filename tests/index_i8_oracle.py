"""CPU oracle of int8 index storage (``FlatIPIndex(d, dtype=torch.int8)``, csrc/quant_i8.cuh and csrc/scan_i8.cuh).

TEST INFRASTRUCTURE ONLY (tests/test_index_i8_cpu.py, tests/test_index_i8_gpu.py).  numpy only; shares no code with the
kernels.

Quantisation rule, in IEEE fp32 arithmetic (numpy float32 division rounds to nearest, ``np.rint`` rounds half to even):
    s = amax / 127,  amax = max_j |x_j|;   c_j = clamp(rint(x_j / s), -127, 127);   a zero row: s = 0, codes 0.
The stored value of element j is fp32(s * c_j) (``dequantize_i8``).

Scan operand of a query: the two-level split q ~ q_h = sig_hi q_hi + sig_lo q_lo with sig_hi = amax / 127 and
sig_lo = sig_hi / 254, q_hi by the rule above and q_lo the same rule applied to the residual r = q - sig_hi q_hi at the
fixed scale sig_lo.  The kernel computes r and the final residual with FMAs, i.e. exactly rounded once; float64 holds
x - s c exactly here (a 24-bit value minus a product of 24 and 8 bits, within 2^32 of each other), so rounding the
float64 value to float32 reproduces the FMA.

Certificate of an int8 index: certify_kernel's E(q) (oracle/search_bound.py) with
    a = |sig_hi q_hi| + |sig_lo q_lo| (>= |q_h|),  b = |q - q_h|,  X = max_r |x^_r|,  X_e = 0,
    E = 1.001 (b X + (d + 16) 2^-22 (a + b) X).
What the (d + 16) 2^-22 term must cover for int8 rows (``i8_terms``):
  * stage rounding: the scan's products and sums are exact integers A_hi, A_lo; the stage score
    fp32(s * fp32(sig_hi * fp32(A_hi) + fp32(sig_lo * fp32(A_lo)))) goes through at most 5 roundings (two int -> fp32
    conversions once |A| > 2^24, a product, an FMA, a product), each relative 2^-24 of a magnitude <= a |y| with
    y = s c (Cauchy-Schwarz on each product): <= 5 * 2^-24 * (1 + 2^-22) * a X (1 + 2^-24);
  * stored vs real corpus values: |x^ - s c| <= 2^-24 |x^| per element: <= 2^-24 a X;
  * the re-score: gamma_{m+5} |q| X with |q| <= a + b (finalize_kernel's chain, oracle/search_bound.py).
"""
from __future__ import annotations

import numpy as np

from oracle import search_bound as sb

F32 = np.float32


def quantize_i8(x: np.ndarray):
    """rows [n, d] (float32, or anything exactly representable in it) -> (codes int8 [n, d], scales float32 [n])"""
    x = np.asarray(x, dtype=F32)
    amax = np.max(np.abs(x), axis=1) if x.shape[1] else np.zeros(x.shape[0], F32)
    s = (amax / F32(127)).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.rint(x / s[:, None]).astype(F32)
    c = np.where(s[:, None] > 0, np.clip(c, -127, 127), F32(0))
    return c.astype(np.int8), s


def dequantize_i8(codes: np.ndarray, scales: np.ndarray) -> np.ndarray:
    """fp32(s * c), the values an int8 index stores"""
    return (np.asarray(scales, F32)[:, None] * np.asarray(codes, np.int8).astype(F32)).astype(F32)


def stored_i8(x: np.ndarray) -> np.ndarray:
    return dequantize_i8(*quantize_i8(x))


def query_split_i8(q: np.ndarray):
    """(q_hi int8, q_lo int8, sig_hi float32 [nq], sig_lo float32 [nq]) as queries_to_i8_kernel computes them"""
    q = np.asarray(q, F32)
    sh = (np.max(np.abs(q), axis=1) / F32(127)).astype(F32)
    sl = (sh / F32(254)).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ch = np.where(sh[:, None] > 0, np.clip(np.rint(q / sh[:, None]), -127, 127), 0).astype(F32)
        r = (q.astype(np.float64) - sh[:, None].astype(np.float64) * ch).astype(F32)
        cl = np.where(sl[:, None] > 0, np.clip(np.rint(r / sl[:, None]), -127, 127), 0).astype(F32)
    return ch.astype(np.int8), cl.astype(np.int8), sh, sl


def query_norms_i8(q: np.ndarray):
    """(a, b) per query in float64: |sig_hi q_hi| + |sig_lo q_lo| and |q - q_h|"""
    qh, ql, sh, sl = query_split_i8(q)
    hi = sh[:, None].astype(np.float64) * qh
    lo = sl[:, None].astype(np.float64) * ql
    a = np.linalg.norm(hi, axis=1) + np.linalg.norm(lo, axis=1)
    b = np.linalg.norm(np.asarray(q, np.float64) - hi - lo, axis=1)
    return a, b


def cert_E_i8(q: np.ndarray, xs: np.ndarray, terms: bool = False):
    """certify_kernel's E(q) for an int8 index whose stored (dequantised) rows are xs"""
    d = q.shape[1]
    a, b = query_norms_i8(q)
    X = float(np.linalg.norm(np.asarray(xs, np.float64), axis=1).max()) if xs.shape[0] else 0.0
    t = {"query_quant": b * X, "accumulation": sb.acc_coef(d) * (a + b) * X}
    E = 1.001 * (t["query_quant"] + t["accumulation"])
    if terms:
        t["E"] = E
        return t
    return E


def i8_terms(q: np.ndarray, xs: np.ndarray) -> dict:
    """float64 bounds of what the accumulation term of cert_E_i8 has to cover (module docstring), per query"""
    d = q.shape[1]
    a, b = query_norms_i8(q)
    X = float(np.linalg.norm(np.asarray(xs, np.float64), axis=1).max()) if xs.shape[0] else 0.0
    u = 2.0 ** -24
    return {
        "stage_rounding": 5 * u * (1 + 2.0 ** -22) * a * X * (1 + u),
        "stored_vs_real": u * a * X,
        "rescore": sb._gamma(sb.rescore_chain(d), u) * (a + b) * X,
        "accumulation": sb.acc_coef(d) * (a + b) * X,
    }


def stage_i8(q: np.ndarray, codes: np.ndarray, scales: np.ndarray) -> np.ndarray:
    """float64 exact value s_r * (sig_hi A_hi + sig_lo A_lo) of the scan's combined score [nq, n] (before its fp32
    roundings)"""
    qh, ql, sh, sl = query_split_i8(q)
    c = np.asarray(codes, np.float64)
    Ah, Al = qh.astype(np.float64) @ c.T, ql.astype(np.float64) @ c.T
    return (sh[:, None].astype(np.float64) * Ah + sl[:, None].astype(np.float64) * Al) * np.asarray(scales, np.float64)[None, :]
