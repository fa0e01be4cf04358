"""CPU: oracle/pool_backward.py - the contract tests/test_zz_gpu_pool_backward.py holds B1, B2 and B3 to - and the
evidence that its checks have teeth.  A numpy emulation of the kernels passes every check the GPU file applies, at its
shapes: K4 and B1 share one main loop (truncating k16 steps in a perturbed order, so nothing relies on the natural
order), the probe over the emulated K4 returns exactly that loop's pre, B2 accumulates chunks of truncating k16 steps
and adds the chunk partials in order, B3 accumulates over hidden in truncating k16 steps.  Each mutant below (a subtly
wrong kernel) fails at least one of those checks."""
import numpy as np
import pytest
import torch

from oracle import numerics as nu
from oracle import pool_backward as pb
from oracle import pool_forward as pf
from oracle import pool_grad
from test_numerics_cpu import _accumulate, _trunc_bf16
from test_zz_gpu_pool_backward import CASES, _finish_bias, _forward_epilogue, case_inputs

STEP = 16                                    # bf16 wgmma: K = 16 per MMA step
KBLOCK = 64

MUTANTS = [
    "ties_before_bias",   # max: ties compared before the bias (pre_j == max pre)
    "no_relu_mask",       # the ReLU mask dropped (max: hp = m + b, no hp > 0 test; mean: every row gets dhp / k)
    "first_argmax",       # max: the whole dhp to the first argmax
    "no_tie_division",    # max: every tied row gets the whole dhp
    "reciprocal",         # dhp * fl(1 / count) (max) or dhp * fl(1 / k) (mean) for the division
    "mean_ge",            # mean: z >= 0 in the mask
    "dp_trunc",           # dP truncated to bf16
    "dbm_from_bf16",      # the dbm partials summed from the bf16 dP
    "dbm_one_stream",     # the dbm parity streams merged into one stream in g order
    "dhp_stride",         # dhp read at row stride hidden instead of lddhp
    "next_row_in_max",    # the max and the ties over k + 1 rows: the next group's first row (or a padding slot)
    "b1_order",           # B1's pre accumulated in a different k16 order than K4's
    "b2_last_chunk",      # B2's last chunk dropped
    "pad_read",           # a pad column read as data, in the main loop K4 and B1 share
    "b3_last_slice",      # B3's last 128-unit hidden slice dropped
]
POOL_ONLY = {"ties_before_bias": "max", "first_argmax": "max", "no_tie_division": "max", "mean_ge": "mean",
            "next_row_in_max": "max"}
# n = 400 groups of 3: G = 42, 10 tiles (20 row blocks: B2 chunks of 8, 8 and 4), K = 65 (a partial K-block, NaN pad
# columns), two hidden slices; the GPU file's edges (ties of 2, 3 and k, a zero-row group, z = 0, 2^22 biases, -4096)
MUTANT_CASE = ("mutants", 400, 3, 65, 256, "ids", "special")


def _case(name):
    return next(c for c in CASES if c[0] == name)


# ---------------------------------------------------------------- the emulation
def slot_rows(n, k, rows):
    """table row of every B1 tile slot [n_tiles * 128] (-1: a padding slot, zero-filled)"""
    tr = pool_grad.tile_rows(n, k).reshape(-1)
    rows = np.asarray(rows, np.int64)
    return np.where(tr >= 0, rows[np.maximum(tr, 0)], -1)


def slot_X(table, slots, cols):
    """the tile images' rows [slots, ceil(cols / 64) * 64]: columns < cols of each slot's row, zeros elsewhere"""
    X = np.zeros((slots.size, -(-cols // KBLOCK) * KBLOCK), np.float32)
    v = slots >= 0
    X[v, :cols] = table[slots[v], :cols]
    return X


def k16_order(nsteps, natural=False):
    """the main loop's k16 steps: a fixed perturbation of the natural order (steps 1, 0, 3, 2 of each K-block)"""
    order = np.arange(nsteps)
    return order if natural else order.reshape(-1, 4)[:, [1, 0, 3, 2]].reshape(-1)


def emulate_pre(inp, slots, W, mutant=None, natural=False):
    """the main loop K4 and B1 share: truncating k16 steps over the packed Wm image (zero rows >= K) -> the staging
    tile [n_tiles, 129, hidden] (slot 128: the row after the tile, zero)"""
    cols = inp["pitch"] if mutant == "pad_read" else inp["K"]
    X = slot_X(inp["table"], slots, cols)
    Wimg = np.zeros((X.shape[1], W.shape[1]), np.float32)
    Wimg[:inp["K"]] = nu.bf16_rne(W)
    acc = np.zeros((X.shape[0], W.shape[1]), np.float32)
    with np.errstate(invalid="ignore"):
        for s in k16_order(X.shape[1] // STEP, natural):
            acc = _accumulate(acc, X[:, s * STEP:(s + 1) * STEP], Wimg[s * STEP:(s + 1) * STEP], "rz")
    st = acc.reshape(-1, 128, W.shape[1])
    return np.concatenate([st, np.zeros_like(st[:, :1])], axis=1)


def group_view(st, n, k, kk):
    """[n, kk, hidden]: group g's rows j < kk of the staging tile (kk = k + 1 runs into the next slot)"""
    G = 128 // k
    idx = np.arange(G)[:, None] * k + np.arange(kk)[None, :]
    return st[:, idx].reshape(-1, kk, st.shape[-1])[:n]


def emulate_k4(inp, n, slots, W, bias, pool, mutant=None):
    """K4's forward over the staging tile: fmaxf(max_j p_j + b, 0) or the mean epilogue, fp32"""
    k = inp["k"]
    p = group_view(emulate_pre(inp, slots, W, mutant), n, k, k)
    b = np.zeros(p.shape[-1], np.float32) if bias is None else bias
    if pool == "max":
        return np.maximum(p.max(axis=1) + b, np.float32(0))
    s = np.zeros((n, p.shape[-1]), np.float32)
    with np.errstate(invalid="ignore"):
        for j in range(k):
            s = s + np.maximum(p[:, j] + b, np.float32(0))
    return s / np.float32(k)


def emulate_probe(inp, W, mutant=None):
    """the GPU file's probe over the emulated K4: [n k, hidden]"""
    n, k = inp["n"], inp["k"]
    rows = pf.row_index(inp["n_rows"], n, k, inp["ids"], inp["row0"])
    pre = np.zeros((n, k, W.shape[1]), np.float32)
    for j in range(k):
        slots = slot_rows(n, k, pb.probe_rows(rows, n, k, j, inp["zero_row"]))
        pos = emulate_k4(inp, n, slots, W, None, "max", mutant)
        neg = emulate_k4(inp, n, slots, -W, None, "max", mutant)
        pre[:, j] = pos - neg
    return pre.reshape(n * k, -1)


def emulate_b1(inp, slots, bias, dhp_buf, lddhp, pool, mutant=None):
    """B1: the shared main loop, then the kGrad epilogue -> the output buffer (images, then partials)"""
    n, k, hid = inp["n"], inp["k"], inp["hidden"]
    st = emulate_pre(inp, slots, inp["W"], mutant, natural=mutant == "b1_order")
    kk = k + 1 if mutant == "next_row_in_max" else k
    p = group_view(st, n, k, kk)
    b = np.zeros(hid, np.float32) if bias is None else bias
    ld = hid if mutant == "dhp_stride" else lddhp
    d = dhp_buf.reshape(-1)[np.arange(n)[:, None] * ld + np.arange(hid)[None, :]][:, None, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        z = (p + b).astype(np.float32)
        if pool == "mean":
            q = d * (np.float32(1) / np.float32(k)) if mutant == "reciprocal" else d / np.float32(k)
            mask = np.ones_like(z, bool) if mutant == "no_relu_mask" else z >= 0 if mutant == "mean_ge" else z > 0
            dp = np.where(mask, q, np.float32(0))
        else:
            m = p.max(axis=1, keepdims=True)
            hp = m + b if mutant == "no_relu_mask" else np.maximum(m + b, np.float32(0))
            sel = (p == m) if mutant == "ties_before_bias" else (z == hp)
            if mutant != "no_relu_mask":
                sel &= hp > 0
            if mutant == "first_argmax":
                sel &= np.cumsum(sel, axis=1) == 1
            cnt = np.maximum(sel.sum(axis=1, keepdims=True), 1).astype(np.float32)
            q = d if mutant in ("first_argmax", "no_tie_division") else \
                d * (np.float32(1) / cnt) if mutant == "reciprocal" else d / cnt
            dp = np.where(sel, q, np.float32(0))
    dp = dp[:, :k].astype(np.float32)
    dP = _trunc_bf16(dp) if mutant == "dp_trunc" else nu.bf16_rne(dp)
    src = dP if mutant == "dbm_from_bf16" else dp
    s = np.zeros((n, hid), np.float32)
    for j in range(k):
        s = s + src[:, j]
    G = 128 // k
    T = -(-n // G)
    sg = np.zeros((T * G, hid), np.float32)
    sg[:n] = s
    sg = sg.reshape(T, G, hid)
    acc = np.zeros((2, T, hid), np.float32)
    for g in range(G):
        par = 0 if mutant == "dbm_one_stream" else g & 1
        acc[par] = acc[par] + sg[:, g]
    parts = (acc[0] + acc[1]).astype(np.float32)
    buf = pool_grad.rows_to_dp_images(dP.reshape(n * k, hid), n, k)
    buf[T * hid * 256:] = parts.reshape(-1).view(np.uint8)
    return buf


def emulate_b2(inp, slots, buf, dWm0, dbm0, mutant=None):
    """B2: chunks of truncating k16 steps over the row slots, chunk partials added in order, then into dWm0; dbm:
    the partials' fixed-order combine into dbm0"""
    n, k, K, hid = inp["n"], inp["k"], inp["K"], inp["hidden"]
    _, full, parts = pool_grad.dp_images_to_rows(buf, n, k, hid)
    F = full.reshape(-1, hid)
    X = slot_X(inp["table"], slots, K)[:, :K]
    _, per, chunks = pool_grad.dw_chunks(n, k)
    tot = np.zeros((K, hid), np.float32)
    for c in range(chunks - (mutant == "b2_last_chunk")):
        acc = np.zeros((K, hid), np.float32)
        for s in range(c * per * 64, min((c + 1) * per * 64, F.shape[0]), STEP):
            acc = _accumulate(acc, X[s:s + STEP].T, F[s:s + STEP], "rz")
        tot = tot + acc
    return dWm0 + tot, dbm0 + pool_grad.dbm_combine(parts)


def emulate_b3(inp, buf, Kd, mutant=None):
    """B3: dx = dP Wm^T[:, :Kd] in truncating k16 steps over hidden"""
    n, k, hid = inp["n"], inp["k"], inp["hidden"]
    dP, _, _ = pool_grad.dp_images_to_rows(buf, n, k, hid)
    Wt = np.ascontiguousarray(nu.bf16_rne(inp["W"])[:Kd].T)
    acc = np.zeros((n * k, Kd), np.float32)
    for h in range(0, hid - 128 * (mutant == "b3_last_slice"), STEP):
        acc = _accumulate(acc, dP[:, h:h + STEP], Wt[h:h + STEP], "rz")
    return acc


# ---------------------------------------------------------------- the GPU file's checks on the emulation
def failed_checks(case, pool, mutant=None):
    """run the emulated kernels through every check of tests/test_zz_gpu_pool_backward.py; the names that fail"""
    inp = case_inputs(case, pool)
    n, k, K, hid = inp["n"], inp["k"], inp["K"], inp["hidden"]
    rows = pf.row_index(inp["n_rows"], n, k, inp["ids"], inp["row0"])
    slots = slot_rows(n, k, rows)
    X = pf.gather(inp["table"], K, n, k, inp["ids"], inp["row0"])
    shared = mutant if mutant == "pad_read" else None             # the main loop K4 and B1 share
    pre = emulate_probe(inp, inp["W"], shared)
    failed = []
    if not pb.window(pre, X, inp["W"])[0]:
        failed.append("window")
    pre_t = torch.from_numpy(pre)
    bias = _finish_bias(inp, pre_t)
    fwd = emulate_k4(inp, n, slots, inp["W"], bias, pool, shared)
    if not pf.same_values(torch.from_numpy(fwd), _forward_epilogue(pre_t, None if bias is None else
                                                                   torch.from_numpy(bias), n, k, pool)):
        failed.append("forward")
    dhp_buf = np.full((n, hid + 24), np.nan, np.float32)
    dhp_buf[:, :hid] = inp["dhp"]
    buf = emulate_b1(inp, slots, bias, dhp_buf, hid + 24, pool, mutant)
    bad, dP, dpre = pb.check_b1(buf, pre, bias, inp["dhp"], n, k, pool)
    if bad:
        failed.append("b1")
    rs = np.random.RandomState(5)
    dW0, db0 = emulate_b2(inp, slots, buf, np.zeros((K, hid), np.float32), np.zeros(hid, np.float32), mutant)
    dWm_in, dbm_in = rs.randn(K, hid).astype(np.float32), rs.randn(hid).astype(np.float32)
    dWm, dbm = emulate_b2(inp, slots, buf, dWm_in, dbm_in, mutant)
    if not nu.bits_equal(dWm, dWm_in + dW0) or not nu.bits_equal(dbm, pb.dbm_reference(dpre, n, k, dbm_in)):
        failed.append("b2_add")
    if not pb.check_gemm(dW0, *pb.dw_reference(X, dP))[0]:
        failed.append("b2")
    for Kd in sorted({K, max(1, K // 3)}):
        if not pb.check_gemm(emulate_b3(inp, buf, Kd, mutant), *pb.dx_reference(dP, inp["W"], Kd))[0]:
            failed.append("b3")
    return failed


EMULATED = ["k1_K1", "k2_K7", "k3_K8", "k25_K63", "k43_K64", "k64_K65"]


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("name", EMULATED + ["mutants"])
def test_emulation_passes_every_check(name, pool):
    case = MUTANT_CASE if name == "mutants" else _case(name)
    assert failed_checks(case, pool) == []


@pytest.mark.parametrize("name", ["k64_K65", "mutants"])
def test_the_probe_returns_the_shared_main_loops_pre(name):
    """out(Wm) - out(-Wm) over the emulated K4 is exactly the main loop's pre at every row's own slot, and that pre
    differs from the float64 product (the accumulation rounds) and from the natural k16 order in places"""
    inp = case_inputs(MUTANT_CASE if name == "mutants" else _case(name), "max")
    n, k = inp["n"], inp["k"]
    slots = slot_rows(n, k, pf.row_index(inp["n_rows"], n, k, inp["ids"], inp["row0"]))
    live = pool_grad.tile_rows(n, k).reshape(-1) >= 0
    want = emulate_pre(inp, slots, inp["W"])[:, :128].reshape(-1, inp["hidden"])[live]
    pre = emulate_probe(inp, inp["W"])
    assert nu.bits_equal(pre, want)
    natural = emulate_pre(inp, slots, inp["W"], natural=True)[:, :128].reshape(-1, inp["hidden"])[live]
    assert not nu.bits_equal(natural, want)
    X = pf.gather(inp["table"], inp["K"], n, k, inp["ids"], inp["row0"])
    exact = X.astype(np.float64) @ nu.bf16_rne(inp["W"]).astype(np.float64)
    assert (pre != exact).any() and pb.window(pre, X, inp["W"])[0]


def test_mutant_case_has_the_edges():
    """the mutant case reaches what the mutants need: several B2 chunks with a short last one, two hidden slices,
    ties of 2, 3 and k, a zero-row group, bias columns with z = 0 and with 2^22 max|pre|, hp = 0 columns"""
    inp = case_inputs(MUTANT_CASE, "max")
    n, k, K = inp["n"], inp["k"], inp["K"]
    blocks, per, chunks = pool_grad.dw_chunks(n, k)
    assert chunks == 3 and blocks % per and inp["hidden"] == 256 and K % KBLOCK and inp["pitch"] > K
    ids = inp["ids"].reshape(n, k)
    assert (ids[0] == ids[0, 0]).all() and ids[1, 0] == ids[1, k - 1] and (ids[3] == inp["zero_row"]).all()
    assert ((ids < 0) | (ids >= inp["n_rows"])).any()
    pre = emulate_probe(inp, inp["W"])
    b = _finish_bias(inp, torch.from_numpy(pre))
    z = pre.reshape(n, k, -1) + b
    assert (z.max(axis=1)[:, 8:24] == 0).sum() >= 16 and (b[-2:] == -4096).all()
    assert (pre.reshape(n, k, -1)[:, :, 2].std(axis=1) > 0).any()
    tied = (z[:, :, 2] == z[:, :, 2].max(axis=1, keepdims=True)).sum(axis=1)
    assert (tied > 1).sum() > n // 4                               # post-bias ties that are not pre ties


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("mutant", MUTANTS)
def test_each_mutant_fails_a_check(mutant, pool):
    if POOL_ONLY.get(mutant, pool) != pool:
        pytest.skip("a %s-pool mutant" % POOL_ONLY[mutant])
    assert failed_checks(MUTANT_CASE, pool, mutant) != [], mutant


# ---------------------------------------------------------------- the oracle itself
def test_torch_gemm_errors_equal_numerics():
    rs = np.random.RandomState(1)
    A, B = nu.bf16_rne(rs.randn(300, 70)), nu.bf16_rne(rs.randn(70, 130))
    ref, S1, S2, K = nu.gemm_reference([(A, B)], "bf16")
    out = (A.astype(np.float64) @ B.astype(np.float64)).astype(np.float32)
    out[3, 4] = np.nextafter(out[3, 4], np.float32(np.inf))
    want = nu.gemm_errors(out, ref, S1, S2, K)
    got = pb.gemm_errors(out, *pb.gemm_reference(A, B))
    assert np.allclose(got, want, rtol=1e-12, atol=0)


def test_probe_rows_and_teacher_forced():
    rows = np.arange(12) * 10
    ids = pb.probe_rows(rows, 4, 3, 1, 99).reshape(4, 3)
    assert (ids[:, 1] == rows.reshape(4, 3)[:, 1]).all() and (ids[:, [0, 2]] == 99).all() and ids.dtype == np.int32
    pre = np.array([[1.0], [3.0], [3.0], [-1.0], [0.5], [2.0]], np.float32)      # two groups of 3, one column
    dP, dpre, parts = pb.teacher_forced(pre, np.zeros(1, np.float32), np.array([[3.0], [6.0]], np.float32), 2, 3,
                                        "max")
    assert dpre.reshape(-1).tolist() == [0.0, 1.5, 1.5, 0.0, 0.0, 6.0] and parts.tolist() == [[9.0]]
