"""numpy restatement of gs_sgd_orders / gs_sgd_fit (csrc/sgd.cu): scikit-learn's plain SGD for
SGDClassifier(loss="log_loss", max_iter=5, tol=None) on float64 X, with the kernel's dot-product order.

Line numbers cite the installed scikit-learn sources:
  P = sklearn/linear_model/_sgd_fast.pyx.tp       (_plain_sgd64)
  W = sklearn/utils/_weight_vector.pyx.tp          (WeightVector64)
  D = sklearn/utils/_seq_dataset.pyx.tp            (SequentialDataset64 / ArrayDataset64)
  R = sklearn/utils/_random.pxd                    (our_rand_r)
  L = sklearn/_loss/_loss.pyx.tp                   (cgradient_half_binomial)
The problems step in lockstep: one numpy operation per step covers all of them.
"""
import math

import numpy as np

RAND_R_MOD = 2 ** 31          # R:34  seed % (RAND_R_MAX + 1)
MAX_DLOSS = 1e12              # P:439
RESET_WSCALE = 1e-9           # W:16  reset_wscale_threshold of WeightVector64
LANES = 32
_libm_exp = np.frompyfunc(math.exp, 1, 1)     # L:29 cimports exp from libc.math: the C library's, not numpy's


def our_rand_r(state):
    """R:20-34 -> (new state, draw)."""
    if state == 0:                                       # R:23-24
        state = 1
    state ^= (state << 13) & 0xFFFFFFFF                  # R:26
    state ^= state >> 17                                 # R:27
    state ^= (state << 5) & 0xFFFFFFFF                   # R:28
    return state, state % RAND_R_MOD                     # R:34


def sigma(seed, n):
    """D:137-145 shuffle(seed) applied to arange(n): the Fisher-Yates chain from seed (taken by value)."""
    ind = np.arange(n, dtype=np.int32)
    state = int(seed) & 0xFFFFFFFF
    for i in range(n - 1):                               # D:143
        state, r = our_rand_r(state)
        j = i + r % (n - i)                              # D:144
        ind[i], ind[j] = ind[j], ind[i]                  # D:145
    return ind


def epoch_orders(sig, epochs):
    """P:473-474 shuffles before every epoch with the same seed, so the swaps of sigma are re-applied to the previous
    order: order_0 = sigma, order_e = sigma[order_{e-1}]  -> int32 [epochs, n]."""
    out = [np.asarray(sig, dtype=np.int32)]
    for _ in range(1, epochs):
        out.append(out[0][out[-1]])
    return np.stack(out)


def kernel_dot(w, x):
    """sum_j w[:, j] * x[:, j] per row in the kernel's order: lane l adds its columns l, l + 32, ... left to right from
    0.0, then the 32 lane sums meet in the xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same value)."""
    P, d = w.shape
    prod = w * x
    acc = np.zeros((P, LANES))
    for k in range(0, d, LANES):
        chunk = prod[:, k:k + LANES]
        acc[:, :chunk.shape[1]] = acc[:, :chunk.shape[1]] + chunk
    lanes = np.arange(LANES)
    for m in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ m]
    return acc[:, 0]


def sequential_dot(w, x):
    """W:179-181 as written: one running sum over j."""
    acc = np.zeros(w.shape[0])
    for j in range(w.shape[1]):
        acc = acc + w[:, j] * x[:, j]
    return acc


def fit(X, labels, orders, alpha, optimal_init, dot=kernel_dot):
    """_plain_sgd64 for every problem p: X [n, d] (widened to float64), labels [P, n] (> 0 positive), orders
    [P, epochs, n].  Returns (coef [P, d], intercept [P]) as w.reset_wscale() (P:635) leaves them."""
    X = np.asarray(X, dtype=np.float64)
    labels = np.asarray(labels)
    P, epochs, n = orders.shape
    d = X.shape[1]
    rows = np.arange(P)
    w = np.zeros((P, d))                                  # W:69 wscale = 1.0
    wscale = np.ones(P)
    intercept = np.zeros(P)
    t = 1.0                                               # est.t_ = 1.0
    for e in range(epochs):                               # P:467
        for i in range(n):                                # P:475
            idx = orders[:, e, i]                         # D:148-154 next(), D:269 index_data_ptr[current_index]
            x = X[idx]
            y = (labels[rows, idx] > 0).astype(np.float64)   # _prepare_fit_binary: y in {0, 1} for the log loss
            p = dot(w, x) * wscale + intercept            # P:484, W:182
            eta = 1.0 / (alpha * (optimal_init + t - 1))  # P:486
            big = p > -37                                 # L:720
            ex = _libm_exp(np.where(big, -p, p)).astype(np.float64)      # arguments < 37: no overflow
            dloss = np.where(big, ((1 - y) - y * ex) / (1 + ex), ex - y)   # L:721-725
            dloss = np.clip(dloss, -MAX_DLOSS, MAX_DLOSS)  # P:526-529
            update = -eta * dloss                         # P:530
            # P:540 update *= class_weight * sample_weight: both 1.0
            c = max(0.0, 1.0 - (1.0 - 0.0) * eta * alpha)   # P:545 (l1_ratio = 0 for L2)
            wscale = wscale * c                           # W:190
            low = wscale < RESET_WSCALE                   # W:194-195
            if low.any():
                w[low] = wscale[low, None] * w[low]       # W:206
                wscale[low] = 1.0                         # W:207
            nz = update != 0.0                            # P:547
            if nz.any():
                step = update[nz] / wscale[nz]            # W:110 c / wscale
                w[nz] = w[nz] + x[nz] * step[:, None]     # W:110
                intercept[nz] = intercept[nz] + update[nz]   # P:549-554 (intercept_decay = 1.0 for dense X)
            t += 1                                        # P:570
    return wscale[:, None] * w, intercept                 # P:635, W:206


def fit_problems(X, labels, seeds, alpha, optimal_init, epochs=5, dot=kernel_dot):
    """sigma, the epoch orders and the fit of every problem from its shuffle seed: what one gs_sgd_orders +
    gs_sgd_fit computes."""
    orders = np.stack([epoch_orders(sigma(s, X.shape[0]), epochs) for s in seeds])
    return fit(X, labels, orders, alpha, optimal_init, dot=dot)
