"""CPU: the checks of oracle/pool2_forward.py (K5's forward contract) reject subtly wrong kernels.

A numpy emulation of K5 - fp32 accumulation in 64-column chunks of h1, as the kernel walks it - passes both checks: bit
for bit on grid operands and within the derived bound on random ones.  Each mutant below changes one detail a kernel
could get wrong, and at least one of the two checks must reject it (tests/test_zz_gpu_twomax.py runs the same checks on
the real kernel)."""
import numpy as np
import pytest
import torch

from oracle import numerics as nu
from oracle import pool2_forward as p2

N_ROWS, N, k, K, H1, H2 = 300, 12, 5, 70, 128, 256
MUTANTS = ("h1_fp32", "h1_truncated", "b1_dropped", "b1_after_rounding", "last_h1_chunk_missing", "W2_truncated",
           "neighbour_row_in_max", "wrong_clamp_row")


def _trunc_bf16(x):
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def emulate(table, ids, W1, b1, W2, b2, mutant=None):
    """K5 in numpy: gather (clamped), fp32 layer 1, bf16 h1, fp32 layer 2 over 64-wide h1 chunks, max, + b2, ReLU."""
    ids = np.asarray(ids, np.int64)
    bad = (ids < 0) | (ids >= table.shape[0])
    rows = np.where(bad, 0 if mutant == "wrong_clamp_row" else table.shape[0] - 1, ids)
    X = table[rows, :K].astype(np.float32)
    if mutant == "neighbour_row_in_max":
        X = X.copy()
        X[k - 1] = X[k]                                   # group 0's last row is group 1's first
    W1b = nu.bf16_rne(W1)
    W2b = _trunc_bf16(W2) if mutant == "W2_truncated" else nu.bf16_rne(W2)
    pre1 = X @ W1b
    z = pre1 if mutant == "b1_dropped" else (pre1 + b1).astype(np.float32)
    if mutant == "h1_fp32":
        h1 = np.maximum(z, 0)
    elif mutant == "h1_truncated":
        h1 = _trunc_bf16(np.maximum(z, 0))
    elif mutant == "b1_after_rounding":
        h1 = np.maximum(nu.bf16_rne(pre1) + b1, 0).astype(np.float32)
    else:
        h1 = nu.bf16_rne(np.maximum(z, 0))
    pre2 = np.zeros((X.shape[0], H2), np.float32)
    chunks = H1 // 64 - (1 if mutant == "last_h1_chunk_missing" else 0)
    for c in range(chunks):
        pre2 = (pre2 + h1[:, 64 * c:64 * c + 64] @ W2b[64 * c:64 * c + 64]).astype(np.float32)
    m = pre2.reshape(N, k, H2).max(axis=1)
    return np.maximum((m + b2).astype(np.float32), 0)


def inputs(grid, seed=0):
    rs = np.random.RandomState(seed)
    table = np.full((N_ROWS, K + 10), np.nan, np.float32)
    ids = rs.randint(0, N_ROWS, size=N * k)
    ids[3], ids[11], ids[17] = -1, N_ROWS, 2 ** 31 - 1    # out of range: the last row
    live = np.unique(np.concatenate([ids[(ids >= 0) & (ids < N_ROWS)], [N_ROWS - 1, 0]]))
    if grid:
        table[live, :K] = rs.randint(-4, 5, size=(live.size, K)) / 4.0
        table[0, :K] = 1.0                                # the wrong clamp row differs from the right one
        W1, W2 = rs.randint(-4, 5, size=(K, H1)) / 16.0, rs.randint(-4, 5, size=(H1, H2)) / 16.0
        b1, b2 = rs.randint(-16, 17, size=H1) / 64.0, rs.randint(-16, 17, size=H2) / 64.0
    else:
        table[live, :K] = nu.bf16_rne(rs.randn(live.size, K))
        W1, W2 = rs.randn(K, H1) / np.sqrt(K), rs.randn(H1, H2) / np.sqrt(H1 / 2)
        b1, b2 = rs.randn(H1) * 0.5, rs.randn(H2) * 0.1
    f = lambda a: np.asarray(a, np.float32)               # noqa: E731
    return table, ids.astype(np.int32), f(W1), f(b1), f(W2), f(b2)


def _checks(mutant):
    """(grid bit for bit, random within the bound) for the emulation with `mutant`."""
    table, ids, W1, b1, W2, b2 = inputs(True)
    X = torch.from_numpy(p2.gather(table, K, N, k, ids))
    grid_ok = p2.same_values(torch.from_numpy(emulate(table, ids, W1, b1, W2, b2, mutant)),
                             p2.grid_reference(X, W1, b1, W2, b2, k))
    table, ids, W1, b1, W2, b2 = inputs(False, seed=1)
    X = torch.from_numpy(p2.gather(table, K, N, k, ids))
    refs = p2.bounded_reference(X, W1, b1, W2, b2, k)
    bounded_ok = p2.check_bounded(torch.from_numpy(emulate(table, ids, W1, b1, W2, b2, mutant)), *refs)[0]
    return grid_ok, bounded_ok


def test_the_emulated_kernel_passes_both_checks():
    assert _checks(None) == (True, True)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_each_mutant_is_rejected(mutant):
    assert _checks(mutant) != (True, True), mutant


def test_the_grid_reference_refuses_operands_that_round():
    table, ids, W1, b1, W2, b2 = inputs(True)
    X = torch.from_numpy(p2.gather(table, K, N, k, ids))
    with pytest.raises(AssertionError):
        p2.grid_reference(X, W1 + np.float32(2.0 ** -20), b1, W2, b2, k)
