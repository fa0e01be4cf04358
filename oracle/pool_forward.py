"""Operand-exact reference of K4's forward: gs_maxpool_mlp_fused / gs_meanpool_mlp_fused (csrc/maxpool_tc.cu), the
gather -> Dense(bias, ReLU) -> max or mean over each group's k rows of the bf16 pooling models, in one kernel.

Contract, for group g < n_groups and hidden unit h:

  operands  X[g, j] = the table row row(g, j), columns < K only, as stored in bf16 (widened exactly), with
            row(g, j) = row_ids[g k + j], or row0 + g k + j without ids; a row outside [0, n_rows) reads row n_rows - 1
            (numerics.gather_clamped).  Wm is rounded to bf16 to nearest even, as maxpool_pack_kernel does
            (numerics.bf16_rne).  Columns >= K and rows no group reads are never read: they may hold anything.
  pre_j     the exact product X[g, j] . Wm[:, h]; the kernel accumulates it in fp32 in an order it does not specify.
  b         bias[h], or 0 when the bias is NULL.
  max       out = fmaxf(fl32(max_j pre_j) + b, 0)
  mean      s = +0; s = s + fmaxf(fl32(pre_j + b), 0) for j = 0 .. k-1 in fp32; out = s / fp32(k), one IEEE division.

The sign of a zero output is not part of the contract (fmaxf(-0, +0) may return either), so zeros compare by value
(same_values).  NaN or inf in a row or weight the kernel reads is out of scope: its fmaxf drops a NaN that TensorFlow's
max would propagate.

Grid reference (grid_reference).  Let q(x) be the largest power of two that divides every element of x.  Every product
of X and Wm is a multiple of q_pre = q(X) q(Wm), and every partial sum of pre_j, in any order, is a multiple of q_pre of
magnitude <= S1_j = sum_K |x w|.  So if S1_j < 2^24 q_pre every partial sum is an fp32 value and pre_j is exact whatever
the order (and whatever rounding the accumulator uses).  With q = min(q_pre, q(b)), pre_j + b is exact if
S1_j + |b| < 2^24 q.  The mean's terms fmaxf(pre_j + b, 0) are >= 0, so its partial sums are multiples of q no larger
than s: all exact if s < 2^24 q.  Then the contract gives one answer: max: relu(max_j pre_j + b) exactly; mean:
fl32(s / k) with s exact.  grid_reference asserts these conditions from the operands, and also that fp64 and the fp32
loop in j order agree, before it answers; a test cannot pick ranges that silently round.

Bounded reference (bounded_reference, check_bounded) for operands off the grid.  u = 2^-24, and with
e_j = K 2^-23 S1_j (numerics.gemm_bound's accumulation term: the gamma_K bound with u doubled, so it holds for any order
and for a truncating accumulator) the accumulated p_j is within e_j of pre_j.  E = max_j e_j.
  max:  m = max_j p_j is within E of max_j pre_j (max is 1-Lipschitz in the largest component), so x = m + b (exact)
        is within E of r = max_j pre_j + b, ref = relu(r).  fl32(x) moves x by at most ulp(|x|) / 2.  If r >= 0,
        |x| <= ref + E; if r < 0 the output is nonzero only when 0 < x <= E.  relu is 1-Lipschitz, so
        |out - ref| <= E + ulp(ref + E)  (a whole ulp: the half-ulp of the larger of the two cases).
  mean: t_j = relu(pre_j + b), t'_j = relu(fl32(p_j + b)).  |t'_j - t_j| <= d_j = e_j + u (|pre_j + b| + e_j) + 2^-150
        (one rounding, relative u, absolute 2^-150 when it underflows).  The fp32 sum in j order of k nonnegative terms
        is within gamma_{k-1} sum_j t'_j + (k - 1) 2^-150 of their exact sum (Higham, gamma_n = n u / (1 - n u)), and
        sum_j t'_j <= sum_j t_j + sum_j d_j.  Dividing by k, with ref = T = mean_j t_j and D = mean_j d_j:
        |s / k - T| <= B = D + gamma_{k-1} (T + D) + (k - 1) 2^-150 / k; the division adds u (T + B) + 2^-150:
        |out - ref| <= B + u (T + B) + 2^-150.
  RMS, in the style of numerics' criterion (b): sqrt(mean((max(|out - ref| - R, 0) / S2*)^2)) <= numerics.RMS_BOUND,
        where S2* is S2 = sqrt(sum_K (x w)^2) of the row that attains the max (max), or the mean of the k rows' S2 (mean),
        and R is the bound above with e_j = 0: what the epilogue's own roundings may add with an exact accumulator (max:
        ulp(ref); mean: the sum, the bias adds and the division).  Subtracting it leaves the accumulation's error, which
        S2 scales; without it a bias much larger than a row's products (S2 -> 0) would dominate the statistic.  The
        worst-case bound alone is too loose to see an operand rounded the wrong way on part of the sum.

The references compute in torch float64 on the device of their inputs (numpy inputs: the CPU), so the bench shape
(128,000 rows x 602 x 512, 79 GFLOP) can be checked on the GPU it ran on.

Test infrastructure - not imported by the product.
"""
import math

import numpy as np
import torch

from . import numerics as nu

U = 2.0 ** -24
TINY = 2.0 ** -150                       # the largest absolute error of one rounding that underflows
POOLS = ("max", "mean")


def row_index(n_rows, n_groups, k, row_ids=None, row0=0):
    """The table row each (group, j) reads, int64 [n_groups * k] in (g, j) order: row_ids, or row0 + g k + j, with rows
    outside [0, n_rows) reading row n_rows - 1 (the rule of numerics.gather_clamped)."""
    if row_ids is None:
        ids = row0 + np.arange(n_groups * k, dtype=np.int64)
    else:
        ids = np.asarray(row_ids, dtype=np.int64).reshape(-1)[:n_groups * k]
    return np.where((ids < 0) | (ids >= n_rows), n_rows - 1, ids)


def gather(table, K, n_groups, k, row_ids=None, row0=0):
    """X [n_groups * k, K] fp32: columns < K of the rows the groups read (numerics.gather_clamped).  table: float32 with
    bf16 values, or uint16 bf16 bits, [n_rows, >= K]."""
    table = np.asarray(table)
    if row_ids is None:
        ids = row0 + np.arange(n_groups * k, dtype=np.int64)
    else:
        ids = np.asarray(row_ids, dtype=np.int64).reshape(-1)[:n_groups * k]
    return nu.gather_clamped(table[:, :K], ids)


def _t(x, device=None):
    if isinstance(x, torch.Tensor):
        return x if device is None else x.to(device)
    return torch.from_numpy(np.ascontiguousarray(x)).to(device or "cpu")


def _operands(X, W, bias):
    """(X fp64, Wm as bf16 RNE in fp64, b fp64 [hidden]) on X's device."""
    X = _t(X)
    dev = X.device
    W = W.detach().cpu().numpy() if isinstance(W, torch.Tensor) else np.asarray(W)
    Wb = _t(nu.bf16_rne(W), dev).double()
    if bias is None:
        b = torch.zeros(Wb.shape[1], dtype=torch.float64, device=dev)
    else:
        b = _t(np.asarray(bias.detach().cpu() if isinstance(bias, torch.Tensor) else bias, np.float32), dev).double()
    return X.double(), Wb, b


def products(X, W, bias=None):
    """(pre, S1, S2, b): pre = X Wm exactly (fp64 holds a product of a bf16 row and a bf16 column of K <= 640 terms within
    2^-40 relative of S1, far below what the checks resolve), S1 = |X| |Wm|, S2 = sqrt((X * X) (Wm * Wm)), all
    [n_groups * k, hidden] fp64; b the bias as fp64."""
    X, Wb, b = _operands(X, W, bias)
    return X @ Wb, X.abs() @ Wb.abs(), torch.sqrt((X * X) @ (Wb * Wb)), b


def _quantum_exp(x):
    """p such that 2^p is the largest power of two dividing every element of x (fp64 tensor), or None if x is all 0."""
    x = x.reshape(-1)
    x = x[x != 0]
    if x.numel() == 0:
        return None
    m, e = torch.frexp(x)                               # x = m 2^e, 0.5 <= |m| < 1: m 2^53 is an integer
    M = (m.abs() * 2.0 ** 53).to(torch.int64)
    low = M & (-M)
    return int((torch.log2(low.double()).round().to(torch.int64) + e.to(torch.int64)).min()) - 53


def _min_exp(*ps):
    ps = [p for p in ps if p is not None]
    return min(ps) if ps else None


def grid_reference(X, W, bias, k, pool):
    """The contract's one answer on grid operands (module docstring), float32 [n_groups, hidden] on X's device.  Raises
    AssertionError when the operands do not make every fp32 operation of the contract exact."""
    if pool not in POOLS:
        raise ValueError("pool must be 'max' or 'mean'")
    X, Wb, b = _operands(X, W, bias)
    pre, S1 = X @ Wb, X.abs() @ Wb.abs()
    n = pre.shape[0] // k
    px, pw = _quantum_exp(X), _quantum_exp(Wb)
    p_pre = None if px is None or pw is None else px + pw
    p = _min_exp(p_pre, _quantum_exp(b))
    lim = 2.0 ** (24 + p) if p is not None else math.inf
    if p_pre is not None:
        assert float(S1.max()) < 2.0 ** (24 + p_pre), "pre is not exact in fp32 in every order"
    z = pre + b                                          # exact in fp64: < 2^53 quanta
    assert float((S1 + b.abs()).max()) < lim, "pre + b is not exact in fp32"
    assert torch.equal(pre.float().double(), pre) and torch.equal((pre.float() + b.float()).double(), z)
    z = z.reshape(n, k, -1)
    if pool == "max":
        out = torch.relu(z.max(dim=1).values)
        out32 = torch.clamp_min(pre.float().reshape(n, k, -1).max(dim=1).values + b.float(), 0.0)
        assert torch.equal(out32.double(), out)
        return out32
    t = torch.relu(z)
    s64 = t.sum(dim=1)
    assert s64.numel() == 0 or float(s64.max()) < lim, "the mean's sum is not exact in fp32"
    t32 = t.float()
    s32 = torch.zeros_like(t32[:, 0])
    for j in range(k):
        s32 = s32 + t32[:, j]
    assert torch.equal(s32.double(), s64), "fp32 in j order and fp64 disagree"
    return s32 / torch.tensor(float(k), dtype=torch.float32, device=s32.device)


def _ulp32(x):
    """ulp of |x| rounded to fp32 (fp64 tensor in, fp64 out): the spacing above it; 2^-149 at 0."""
    a = x.abs().float()
    return (torch.nextafter(a, torch.full_like(a, math.inf)).double() - a.double())


def bounded_reference(X, W, bias, k, pool):
    """(ref, bound, s2, r): the fp64 contract output [n_groups, hidden], the derived bound on |out - ref|, and the S2*
    and R of the RMS statistic (module docstring), all fp64 on X's device."""
    if pool not in POOLS:
        raise ValueError("pool must be 'max' or 'mean'")
    pre, S1, S2, b = products(X, W, bias)
    K = _t(X).shape[1]
    n = pre.shape[0] // k
    hid = pre.shape[1]
    e = (K * 2.0 ** -23) * S1.reshape(n, k, hid)
    z = (pre + b).reshape(n, k, hid)
    S2 = S2.reshape(n, k, hid)
    if pool == "max":
        r, arg = z.max(dim=1)
        ref = torch.relu(r)
        E = e.max(dim=1).values
        return ref, E + _ulp32(ref + E), torch.gather(S2, 1, arg[:, None, :])[:, 0], _ulp32(ref)
    ref = torch.relu(z).mean(dim=1)
    gamma = (k - 1) * U / (1 - (k - 1) * U)

    def bound(e):
        D = (e + U * (z.abs() + e) + TINY).mean(dim=1)
        B = D + gamma * (ref + D) + (k - 1) * TINY / k
        return B + U * (ref + B) + TINY

    return ref, bound(e), S2.mean(dim=1), bound(torch.zeros_like(e))


def errors(out, ref, bound, s2, r):
    """(worst, rms): worst = max |out - ref| / bound (<= 1 required; a NaN or inf output is inf), rms = the RMS of
    max(|out - ref| - R, 0) / S2* (a nonzero one where S2* = 0 is inf)."""
    out = _t(out, ref.device).double()
    err = torch.where(torch.isfinite(out), (out - ref).abs(), torch.full_like(out, math.inf))
    if err.numel() == 0:
        return 0.0, 0.0
    worst = float((err / bound).max())
    acc = torch.clamp_min(err - r, 0.0)
    rel = torch.where(s2 > 0, acc / torch.where(s2 > 0, s2, torch.ones_like(s2)),
                      torch.where(acc > 0, torch.full_like(acc, math.inf), torch.zeros_like(acc)))
    return worst, float(torch.sqrt(torch.mean(rel * rel)))


def check_bounded(out, ref, bound, s2, r, rms_bound=nu.RMS_BOUND):
    """(ok, worst, rms): |out - ref| <= bound everywhere and the RMS statistic <= rms_bound."""
    worst, rms = errors(out, ref, bound, s2, r)
    return worst <= 1.0 and rms <= rms_bound, worst, rms


def same_values(a, b):
    """float32 tensors equal bit for bit except that -0 equals +0 (NaN never equals a number)."""
    a, b = _t(a), _t(b, _t(a).device)
    if a.shape != b.shape or a.dtype != torch.float32 or b.dtype != torch.float32:
        return False
    return torch.equal((a + 0.0).view(torch.int32), (b + 0.0).view(torch.int32))
