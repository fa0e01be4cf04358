"""Operand-exact references for the aggregation kernels: the fanout mean bit for bit, the K3 GEMM (gs_sage_gemm) in each
math mode as the float64 product of the operands that mode actually multiplies, with error bounds that depend only on
the accumulation.

Comparing a kernel with float64 on the UNROUNDED operands needs a tolerance as large as the operand rounding itself
(bf16: ~4e-3 row-relative), which hides a kernel that rounds an operand the wrong way.  Here the operand rounding is
part of the reference, so what is left to bound is the fp32 accumulation:

  fanout mean (gather.cu, layer_small.cu): s = +0; s = s + x_j for j = 0 .. k-1 (fp32); s = s + self when include_self;
      s / fp32(k + include_self) (one IEEE division).  Ids outside [0, n_rows) read row n_rows - 1.  A bf16 table is
      widened exactly.  Reproducible bit for bit (the library is built without fast math).
  K3 operands:  fp32   the fp32 values                 tf32   x & 0xFFFFE000 (tf32_mask, tc_common.cuh)
                bf16   round to nearest even            tf32x3 hi = trunc(x), lo = trunc(x - hi);
                                                               hi*hi + hi*lo + lo*hi (no lo*lo term)
  check_gemm: (a) |out - ref| <= K * 2^-23 * S1 + ulp(|ref|), S1 = sum_k |a_ik b_kj| over the multiplied operands,
                  K the number of products summed (3 K for tf32x3)
                  (the gamma_K bound with u doubled, so a truncating accumulator passes; the ulp covers bias / ReLU);
              (b) sqrt(mean((|out - ref| / S2)^2)) <= RMS_BOUND, S2 = sqrt(sum_k (a_ik b_kj)^2) - the typical error,
                  which (a) alone bounds too loosely to see a dropped partial product.

Test infrastructure - not imported by the product.
"""
import numpy as np

from . import dropout as _dropout

U23 = 2.0 ** -23
# The H100's wgmma accumulates in fp32 with truncation: at K = 640 the tf32x3 statistic (b) is 4.8e-6 (2^-17.7), what a
# numpy emulation of truncating k8 steps gives (5.8e-6; 2.8e-7 when rounding to nearest).  A tf32x3 kernel that drops
# A_lo * B_hi in its last K-block is at ~9e-5, one that rounds a bf16 operand toward zero at ~4e-3.
RMS_BOUND = 2.0 ** -17
MATHS = ("fp32", "tf32x3", "tf32", "bf16")


def _f32(x):
    return np.ascontiguousarray(x, dtype=np.float32)


def tf32_trunc(x):
    """x with the low 13 mantissa bits cleared: the tf32 operand the wgmma kernels multiply (tf32_mask)."""
    x = _f32(x)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32x3_split(x):
    """(hi, lo): hi = trunc(x), lo = trunc(x - hi) with the difference in fp32, as the kernels split A and B."""
    x = _f32(x)
    hi = tf32_trunc(x)
    return hi, tf32_trunc(x - hi)


def bf16_rne(x):
    """fp32 -> bfloat16 (round to nearest, ties to even; NaN stays NaN) -> fp32, as __floats2bfloat162_rn rounds."""
    x = _f32(x)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    r = np.where(nan, (u & 0xFFFF0000) | 0x00400000, r)
    return r.astype(np.uint32).view(np.float32).reshape(x.shape)


def bf16_widen(bits):
    """bfloat16 bit patterns (uint16) -> fp32, exactly."""
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def gather_clamped(table, ids):
    """table[ids] with ids outside [0, n_rows) reading row n_rows - 1 (clamp_row in gather.cu), widened to fp32.
    table: float32 [n_rows, F] or uint16 bf16 bits."""
    table = np.asarray(table)
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    n = table.shape[0]
    rows = table[np.where((ids < 0) | (ids >= n), n - 1, ids)]
    return bf16_widen(rows) if rows.dtype == np.uint16 else _f32(rows)


def mean_f32(rows, k, self_rows=None, include_self=False, neigh_site=None, self_site=None):
    """The kernels' fanout mean in fp32, bit for bit.  rows: neighbour rows [n * k, F] (or [n, k, F]) in j order;
    self_rows: [n, F] (needed when include_self).  neigh_site / self_site: optional dropout sites (seed, call, rate) of
    gs_gather_mean_dropout, applied as oracle.dropout does (neighbour j of row i at position i * k + j, self row i at i;
    kept elements x / fp32(1 - rate), dropped ones +0) before the sum."""
    rows = _f32(rows)
    F = rows.shape[-1]
    rows = rows.reshape(-1, k, F)
    n = rows.shape[0]
    if neigh_site is not None:
        with np.errstate(over="ignore"):
            rows = _dropout.apply(rows.reshape(n * k, F), *neigh_site).reshape(n, k, F)
    acc = np.zeros((n, F), dtype=np.float32)
    with np.errstate(over="ignore"):                      # a sum that overflows is +-inf, as on the device
        for j in range(k):
            acc = acc + rows[:, j]
        if include_self:
            s = _f32(self_rows)
            if self_site is not None:
                s = _dropout.apply(s, *self_site)
            acc = acc + s
    return acc / np.float32(k + (1 if include_self else 0))


def operands(a, math):
    """The (a, b)-side operand terms a mode multiplies: a list of fp32 arrays per side, paired by index in
    gemm_reference (tf32x3: hi*hi, hi*lo, lo*hi)."""
    if math == "fp32":
        return [_f32(a)]
    if math == "tf32":
        return [tf32_trunc(a)]
    if math == "bf16":
        return [bf16_rne(a)]
    if math == "tf32x3":
        return list(tf32x3_split(a))
    raise ValueError("unknown math mode %r" % (math,))


def _terms(A, B, math):
    a, b = operands(A, math), operands(B, math)
    if math == "tf32x3":
        return [(a[0], b[0]), (a[0], b[1]), (a[1], b[0])]
    return [(a[0], b[0])]


def gemm_reference(parts, math, combine="add", bias=None, act=None):
    """float64 act(concat_or_add(A_p @ B_p) + bias) of the operands `math` multiplies.  parts: [(A [M, K_p], B [K_p, N_p])]
    (fp32 values); combine "add" | "concat"; act None | "relu".  Returns (ref, S1, S2, K): [M, ntot] float64 arrays and
    the per-column number of products summed (K_p, 3 K_p for tf32x3; the parts' sum for add)."""
    refs, s1s, s2s, ks = [], [], [], []
    for A, B in parts:
        A, B = _f32(A), _f32(B)
        ref = np.zeros((A.shape[0], B.shape[1]))
        s1 = np.zeros_like(ref)
        s2 = np.zeros_like(ref)
        for a, b in _terms(A, B, math):
            a, b = a.astype(np.float64), b.astype(np.float64)
            ref += a @ b
            s1 += np.abs(a) @ np.abs(b)
            s2 += (a * a) @ (b * b)
        refs.append(ref)
        s1s.append(s1)
        s2s.append(s2)
        ks.append(np.full(B.shape[1], A.shape[1] * len(_terms(A[:0], B[:0], math)), dtype=np.float64))
    if combine == "concat":
        ref, s1, s2, K = (np.concatenate(x, axis=-1) for x in (refs, s1s, s2s, ks))
    elif combine == "add":
        ref, s1, s2, K = sum(refs), sum(s1s), sum(s2s), sum(ks)
    else:
        raise ValueError("combine must be 'add' or 'concat'")
    if bias is not None:
        ref = ref + _f32(bias).astype(np.float64)
    if act == "relu":
        ref = np.maximum(ref, 0.0)
    elif act is not None:
        raise ValueError("act must be None or 'relu'")
    return ref, s1, np.sqrt(s2), K


def _ulp(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def gemm_bound(ref, S1, K):
    """Criterion (a)'s per-element bound: K * 2^-23 * S1 + one ulp of |ref|."""
    return K * U23 * S1 + _ulp(ref)


def _err(out, ref):
    out = np.asarray(out, dtype=np.float64)
    err = np.abs(out - ref)
    return np.where(np.isfinite(out), err, np.inf)


def gemm_errors(out, ref, S1, S2, K):
    """(worst, rms): worst = max |out - ref| / bound (criterion (a) holds iff <= 1), rms = criterion (b)'s statistic."""
    err = _err(out, ref)
    if err.size == 0:
        return 0.0, 0.0
    worst = float((err / gemm_bound(ref, S1, K)).max())
    rel = np.divide(err, S2, out=np.where(err > 0, np.inf, 0.0), where=S2 > 0)
    return worst, float(np.sqrt(np.mean(rel * rel)))


def check_gemm(out, ref, S1, S2, K, rms_bound=RMS_BOUND):
    """(ok, worst, rms): both criteria of the module docstring."""
    worst, rms = gemm_errors(out, ref, S1, S2, K)
    return worst <= 1.0 and rms <= rms_bound, worst, rms


def l2_normalize_reference(ref):
    """float64 x / sqrt(max(sum x^2, fp32(1e-12))) per row: tf.nn.l2_normalize with the kernels' epsilon."""
    ss = np.sum(ref * ref, axis=-1, keepdims=True)
    return ref / np.sqrt(np.maximum(ss, np.float64(np.float32(1e-12))))


def check_l2_normalized(out, ref, bound):
    """(ok, worst) for out = l2_normalize(v) where |v - ref| <= bound elementwise (gemm_bound) and v's row of C values
    is normalised in fp32 (sum of squares, sqrt, divide, scale): |out - ref/N| <= bound/N + |ref/N| (||bound||/N +
    (C + 3) 2^-24) with N = max(row norm of ref, 1e-6).  A NaN or inf in out fails."""
    C = ref.shape[-1]
    nref = l2_normalize_reference(ref)
    N = np.sqrt(np.maximum(np.sum(ref * ref, axis=-1, keepdims=True), np.float64(np.float32(1e-12))))
    bn = np.sqrt(np.sum(bound * bound, axis=-1, keepdims=True))
    lim = bound / N + np.abs(nref) * (bn / N + (C + 3) * 2.0 ** -24)
    err = _err(out, nref)
    worst = float((err / lim).max()) if err.size else 0.0
    return worst <= 1.0, worst


def f32_bits(x):
    return _f32(x).view(np.uint32)


def bits_equal(a, b):
    """fp32 arrays equal bit for bit (so -0 != +0)."""
    a, b = _f32(a), _f32(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
