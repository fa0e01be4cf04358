"""Operand-exact contract of the pooling backward through the fused bf16 kernels: B1 gs_pool_mlp_backward_dp
(maxpool_mlp_kernel<true, 128, 1, 0, kGrad> in csrc/maxpool_tc.cu), B2 gs_pool_mlp_backward_dw and B3
gs_pool_mlp_backward_dx (csrc/maxpool_bwd_tc.cu).  Notation as in oracle/pool_grad.py: one hop of n groups of k rows,
X [n k, K] the gathered rows (pool_forward.gather: the table's bf16 rows, columns < K, ids outside [0, n_rows) read row
n_rows - 1), Wm [K, hidden] rounded to bf16 to nearest even, b the bias (0 when NULL), dhp [n, hidden] (row stride
lddhp >= hidden).

B1, teacher-forced on K4's own pre-activations.  Let pre_K4[g, j, u] be the fp32 value the default K4 forward (rows as
A, 128-row tiles of G = 128 // k groups, one wgmma group in flight, cp.async rows, no cluster: B1's template
arguments) accumulates for row (g, j) at its own tile slot.  Then, bit for bit:
  dP        == bf16_rne(pool_grad.dpre(pre_K4, b, dhp, k, pool)) at every gathered row, +0 at every padding slot
  partials  == pool_grad.dbm_partials(pool_grad.dpre(pre_K4, ...))
So one contract covers B1's semantics (the ReLU mask and tie rule after the bias, the division by the count or by k,
the one rounding to bf16, the parity streams of the dbm partials) and its agreement with the forward: dhp goes to the
rows whose values the forward returned, including at near-ties that depend on how the sum was rounded.

The probe (probe_rows).  pre_K4 is not an output of any kernel, but it can be read off K4 exactly.  Run the default
K4 max forward with a NULL bias on ids that put the real row of (g, j) at position j of group g and an all-zero row
at every other position, once with Wm and once with -Wm.  Each output element is then fmaxf(max(p, z), 0) where p is
the real row's accumulator at slot (g, j) and z the zero rows' (+-0): out(Wm) = fmaxf(p, 0), and with -Wm the
accumulator is exactly -p (negating a bf16 weight is exact, every product changes sign, and the accumulator's
rounding, truncating or to nearest, is symmetric in sign), so out(-Wm) = fmaxf(-p, 0) and
  out(Wm) - out(-Wm) = p    exactly (one of the two terms is 0, the other is |p|).
The row sits at the slot it occupies in B1, so no assumption about slots being independent is needed; k positions x
2 signs = 2 k forward calls give pre_K4 of every row.

Probe-free window.  Every pre_K4 lies within K4's accumulation bound of the exact product:
  |pre_K4 - X Wm| <= K 2^-23 S1,  S1 = |X| |Wm|          (pool_forward.bounded_reference's e_j)
so a B1 that shared a wrong main loop with K4 (a pad column read, a k16 step dropped) is caught without the probe.

B2.  dWm_out == fl32(dWm_in + D) bit for bit, D the kernel's sum into a zero dWm, and D against the float64 product
X^T dP_kernel (dP_kernel: B1's own bf16 dP) by criteria (a) and (b) of numerics.check_gemm, with n k products per
element.  dbm_out == fl32(dbm_in + pool_grad.dbm_combine(pool_grad.dbm_partials(teacher-forced dpre))) bit for bit:
the tile partials are summed in B2's fixed order and added once.
  The accumulation: chunks of L = 64 * pool_grad.dw_chunks(n, k)[1] row slots, each a chain of L / 16 truncating k16
  steps from 0, then the chunk partials added in order (round to nearest).  A truncating chain biases every step
  toward zero by up to one ulp of the running sum, so its criterion-(b) statistic grows about linearly with L; a
  numpy model of it gives about 2^-21.6 at 512-slot chunks and 2^-18.1 at the 4,096-slot chunks of the 5,120-group,
  k = 25 training hop, and an H100 measures 2^-17.9 there (0.54 of numerics.RMS_BOUND).  4,096 slots is the chunk of
  every launch up to 1,024 tiles; a larger launch has longer chunks and would need a bound that grows with L.

UNDERFLOW.  Criterion (b) is relative to S2, which does not scale an error the fp32 accumulator makes below its
subnormal quantum: an output near 2^-135 (subnormal dhp reach dP) keeps only a few significant bits whatever the
order.  Each rounding of such a partial sum is off by less than 2^-149, and a chain of K / 16 k16 steps (plus B2's at
most 32 chunk adds) rounds far fewer than K / 2 times, so before dividing by S2 the statistic subtracts K 2^-150: far
below the error of any output in the normal range.

B3.  dx[:, :Kd] against the float64 product dP_kernel bf16(Wm)^T[:, :Kd] by criteria (a) and (b), hidden products per
element; nothing outside dx's [n k, Kd] view is written.

The large references run in torch float64 on the device of their inputs (numpy inputs: the CPU).

Test infrastructure - not imported by the product.
"""
import math

import numpy as np
import torch

from . import numerics as nu
from . import pool_forward as pf
from . import pool_grad

U23 = 2.0 ** -23


def _t(x, device=None):
    return pf._t(x, device)


def probe_rows(rows, n, k, j, zero_row):
    """The probe's ids for position j: row (g, j) of `rows` (the clamped table row of every (g, j), pf.row_index) at
    position j of group g, `zero_row` (an all-zero table row) everywhere else.  int32 [n k]."""
    ids = np.full((n, k), zero_row, np.int64)
    ids[:, j] = np.asarray(rows, np.int64).reshape(n, k)[:, j]
    return ids.reshape(-1).astype(np.int32)


def teacher_forced(pre_k4, bias, dhp, n, k, pool):
    """(dP, dpre, partials): the contract's B1 outputs for K4's own pre [n k, hidden] fp32 - dP = bf16_rne(dpre) and
    the dbm partials [n_tiles, hidden] - numpy float32."""
    hid = np.asarray(pre_k4).shape[-1]
    b = np.zeros(hid, np.float32) if bias is None else np.asarray(bias, np.float32)
    d = pool_grad.dpre(np.asarray(pre_k4, np.float32).reshape(n * k, hid), b, np.asarray(dhp, np.float32), k, pool)
    return nu.bf16_rne(d), d, pool_grad.dbm_partials(d, n, k)


def check_b1(buf, pre_k4, bias, dhp, n, k, pool):
    """(bad, dP, dpre): bad = [] when B1's output buffer (uint8: images, then partials) is the contract's answer for
    pre_k4, else a list of what differs; dP the buffer's dP [n k, hidden] and dpre the teacher-forced one, fp32."""
    hid = np.asarray(pre_k4).shape[-1]
    dP, full, parts = pool_grad.dp_images_to_rows(np.asarray(buf), n, k, hid)
    want, dpre, want_parts = teacher_forced(pre_k4, bias, dhp, n, k, pool)
    bad = []
    if not nu.bits_equal(dP, want):
        d = np.argwhere(dP.view(np.uint32) != want.view(np.uint32))
        r, u = d[0]
        bad.append("dP: %d elements differ, first (row %d, unit %d): got %r want %r" % (len(d), r, u, dP[r, u], want[r, u]))
    pad = full[pool_grad.tile_rows(n, k) < 0]
    if pad.size and pad.view(np.uint32).any():
        bad.append("padding slots not +0")
    if not nu.bits_equal(parts, want_parts):
        d = np.argwhere(parts.view(np.uint32) != want_parts.view(np.uint32))
        t, u = d[0]
        bad.append("dbm partials: %d differ, first (tile %d, unit %d): got %r want %r"
                   % (len(d), t, u, parts[t, u], want_parts[t, u]))
    return bad, dP, dpre


def window(pre_k4, X, W):
    """(ok, worst): worst = max |pre_K4 - X Wm| / (K 2^-23 S1) (0 / 0 counts as 0, anything else over a zero bound as
    inf); ok when <= 1.  Computed in float64 on X's device."""
    pre, S1, _, _ = pf.products(X, W)
    K = _t(X).shape[1]
    p = _t(pre_k4, pre.device).double().reshape(pre.shape)
    err = torch.where(torch.isfinite(p), (p - pre).abs(), torch.full_like(p, math.inf))
    bound = K * U23 * S1
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    return worst <= 1.0, worst


def gemm_reference(A, B):
    """(ref, S1, S2, K) of A B in float64 on A's device: the products of numerics.gemm_reference for operands that are
    already the multiplied values (bf16 values held in fp32)."""
    A = _t(A).double()
    B = _t(B, A.device).double()
    return A @ B, A.abs() @ B.abs(), torch.sqrt((A * A) @ (B * B)), A.shape[1]


def gemm_errors(out, ref, S1, S2, K):
    """numerics.gemm_errors on torch tensors: (worst, rms) of criteria (a) and (b), where (b) first subtracts the
    underflow allowance K 2^-150 (UNDERFLOW in the module docstring)."""
    out = _t(out, ref.device).double()
    err = torch.where(torch.isfinite(out), (out - ref).abs(), torch.full_like(out, math.inf))
    if err.numel() == 0:
        return 0.0, 0.0
    worst = float((err / (K * U23 * S1 + pf._ulp32(ref))).max())
    acc = torch.clamp_min(err - K * pf.TINY, 0.0)
    rel = torch.where(S2 > 0, acc / torch.where(S2 > 0, S2, torch.ones_like(S2)),
                      torch.where(acc > 0, torch.full_like(acc, math.inf), torch.zeros_like(acc)))
    return worst, float(torch.sqrt(torch.mean(rel * rel)))


def check_gemm(out, ref, S1, S2, K, rms_bound=nu.RMS_BOUND):
    """(ok, worst, rms): both criteria of numerics.check_gemm."""
    worst, rms = gemm_errors(out, ref, S1, S2, K)
    return worst <= 1.0 and rms <= rms_bound, worst, rms


def dw_reference(X, dP):
    """B2's (ref, S1, S2, K): X^T dP_kernel, X [n k, K] the gathered rows, dP [n k, hidden] B1's bf16 dP."""
    X = _t(X)
    return gemm_reference(X.t(), _t(dP, X.device))


def dx_reference(dP, W, Kd):
    """B3's (ref, S1, S2, K): dP_kernel bf16_rne(Wm)^T[:, :Kd]."""
    W = W.detach().cpu().numpy() if isinstance(W, torch.Tensor) else np.asarray(W)
    dP = _t(dP)
    return gemm_reference(dP, _t(np.ascontiguousarray(nu.bf16_rne(W)[:Kd].T), dP.device))


def dbm_reference(dpre, n, k, dbm0=None):
    """B2's dbm: fl32(dbm0 + dbm_combine(dbm_partials(dpre))), dbm0 = 0 when None."""
    s = pool_grad.dbm_combine(pool_grad.dbm_partials(dpre, n, k))
    return s if dbm0 is None else (np.asarray(dbm0, np.float32) + s).astype(np.float32)
