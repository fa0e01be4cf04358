"""CPU: oracle/pool_forward.py - the contract tests/test_zz_gpu_pool_forward.py holds K4's forward to - and the evidence
that its checks have teeth: a numpy emulation of the kernel passes them at the GPU file's shapes, on grid inputs the
contract is the reference's max-pool / mean-pool semantics, and each mutant below (a subtly wrong kernel) fails a check
the GPU file applies, at one of its shapes."""
import numpy as np
import pytest
import torch

import oracle
from oracle import numerics as nu
from oracle import pool_forward as pf
from test_numerics_cpu import _accumulate, _trunc_bf16
from test_zz_gpu_pool_forward import CASES, case_inputs

STEP = 16                                  # bf16 wgmma: K = 16 per MMA step
KBLOCK = 64                                # bf16 columns per K-block

MUTANTS = [
    "w_trunc",            # Wm truncated to bf16 instead of rounded to nearest even
    "drop_last_k16",      # the last k16 step of a partial last K-block skipped
    "pad_read",           # the table's pad columns read (against the zero weight image: NaN pads give NaN)
    "k_minus_1",          # the pool over k - 1 rows
    "k_plus_1",           # the pool over k + 1 rows: the next group's first row (or a padding row)
    "tile_stride",        # tile t's rows at t * NT + r instead of t * G * k + r
    "oob_row0",           # ids outside [0, n_rows) read row 0
    "mean_relu_after",    # mean: ReLU applied after the mean
    "mean_div_k_plus_1",  # mean: divided by k + 1
    "max_relu_then_bias", # max: relu(m) + b
    "slice0",             # hidden slices >= 1 write slice 0's columns
    "bf16_accumulate",    # the accumulator rounded to bf16 after each step
]
POOL_ONLY = {"mean_relu_after": "mean", "mean_div_k_plus_1": "mean", "max_relu_then_bias": "max"}


def _case(name):
    return next(c for c in CASES if c[0] == name)


def emulate_k4(inp, n, pool, NT=128, mutant=None):
    """maxpool_mlp_kernel in numpy: tiles of NT rows (G = NT // k whole groups, zero rows after them), one fp32
    accumulator per (row, hidden unit) that takes one k16 step at a time and truncates (how the H100's tensor cores
    accumulate), then the epilogue of the staging tile.  Returns float32 [n, hidden]."""
    table, k, K, hidden, n_rows = inp["table"], inp["k"], inp["K"], inp["hidden"], inp["n_rows"]
    G = NT // k
    n_tiles = -(-n // G)
    W = _trunc_bf16(inp["W"]) if mutant == "w_trunc" else nu.bf16_rne(inp["W"])
    Kr = inp["pitch"] if mutant == "pad_read" else K
    Wimg = np.zeros((-(-Kr // KBLOCK) * KBLOCK, hidden), np.float32)    # the packed image: zero for k >= K
    Wimg[:K] = W
    # the tile's row slots -> table rows
    t = np.arange(n_tiles)[:, None]
    r = np.arange(NT)[None, :]
    flat = (t * NT if mutant == "tile_stride" else t * G * k) + r
    valid = (r < G * k) & (flat < n * k)
    if inp["ids"] is None:
        ids = inp["row0"] + flat.astype(np.int64)
    else:
        ids = np.asarray(inp["ids"], np.int64)[np.minimum(flat, n * k - 1)]
    oob = (ids < 0) | (ids >= n_rows)
    ids = np.where(oob, 0 if mutant == "oob_row0" else n_rows - 1, ids)
    X = np.zeros((n_tiles * NT, Wimg.shape[0]), np.float32)
    X[valid.reshape(-1), :Kr] = table[ids[valid], :Kr]
    # main loop
    acc = np.zeros((X.shape[0], hidden), np.float32)
    last = (K - 1) // STEP * STEP
    with np.errstate(invalid="ignore"):
        for k0 in range(0, Wimg.shape[0], STEP):
            if mutant == "drop_last_k16" and K % KBLOCK and k0 == last:
                continue
            acc = _accumulate(acc, X[:, k0:k0 + STEP], Wimg[k0:k0 + STEP], "rz")
            if mutant == "bf16_accumulate":
                acc = nu.bf16_rne(acc)
    stage = np.concatenate([acc.reshape(n_tiles, NT, hidden), np.zeros((n_tiles, 1, hidden), np.float32)], axis=1)
    # epilogue
    kk = k - 1 if mutant == "k_minus_1" else k + 1 if mutant == "k_plus_1" else k
    idx = np.arange(G)[:, None] * k + np.arange(kk)[None, :]
    p = stage[:, idx].reshape(n_tiles * G, kk, hidden)[:n]                # [group, j, hidden]
    b = np.zeros(hidden, np.float32) if inp["bias"] is None else inp["bias"]
    if pool == "max":
        m = p.max(axis=1)
        res = np.maximum(m, np.float32(0)) + b if mutant == "max_relu_then_bias" else np.maximum(m + b, np.float32(0))
    else:
        s = np.zeros((n, hidden), np.float32)
        for j in range(kk):
            s = s + (p[:, j] + b if mutant == "mean_relu_after" else np.maximum(p[:, j] + b, np.float32(0)))
        res = s / np.float32(k + 1 if mutant == "mean_div_k_plus_1" else k)
        if mutant == "mean_relu_after":
            res = np.maximum(res, np.float32(0))
    out = np.full((n, hidden), np.nan, np.float32)
    for sl in range(hidden // 128):
        dst = 0 if mutant == "slice0" else sl
        out[:, dst * 128:(dst + 1) * 128] = res[:, sl * 128:(sl + 1) * 128]
    return out


def _grid_ok(inp, n, pool, out):
    ref = pf.grid_reference(pf.gather(inp["table"], inp["K"], n, inp["k"], inp["ids"], inp["row0"]), inp["W"],
                            inp["bias"], inp["k"], pool)
    return pf.same_values(torch.from_numpy(out), ref)


def _bounded(inp, n, pool, out):
    X = pf.gather(inp["table"], inp["K"], n, inp["k"], inp["ids"], inp["row0"])
    return pf.check_bounded(out, *pf.bounded_reference(X, inp["W"], inp["bias"], inp["k"], pool))


# ---------------------------------------------------------------- the oracle itself
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_row_index_reads_what_gather_clamped_reads(case):
    inp = case_inputs(case, grid=True)
    n = inp["nmax"]
    idx = pf.row_index(inp["n_rows"], n, inp["k"], inp["ids"], inp["row0"])
    X = pf.gather(inp["table"], inp["K"], n, inp["k"], inp["ids"], inp["row0"])
    assert nu.bits_equal(inp["table"][idx, :inp["K"]], X)
    assert not np.isnan(X).any()                                 # every row a group reads is live
    ids = inp["ids"].astype(np.int64) if inp["ids"] is not None else inp["row0"] + np.arange(n * inp["k"])
    if n > 1:                                                   # past group 0 (one repeated id), some are clamped
        assert ((ids < 0) | (ids >= inp["n_rows"])).any()


@pytest.mark.parametrize("case", [c for c in CASES if c[0] != "bench"], ids=[c[0] for c in CASES if c[0] != "bench"])
def test_grid_cases_are_exact(case):
    """grid_reference accepts every grid case (its exactness assertions hold) at the largest launch; on the GPU the
    bench case is checked the same way."""
    inp = case_inputs(case, grid=True)
    X = pf.gather(inp["table"], inp["K"], inp["nmax"], inp["k"], inp["ids"], inp["row0"])
    for pool in pf.POOLS:
        out = pf.grid_reference(X, inp["W"], inp["bias"], inp["k"], pool)
        assert out.dtype == torch.float32 and tuple(out.shape) == (inp["nmax"], inp["hidden"])


def test_grid_reference_refuses_operands_that_round():
    rs = np.random.RandomState(0)
    X = (rs.randint(-32, 33, size=(256 * 4, 640)) / 16.0).astype(np.float32)
    W = (rs.randint(-16, 17, size=(640, 128)) / 16.0).astype(np.float32)
    pf.grid_reference(X, W, None, 256, "max")
    fine = X.copy()
    fine[:, 0] = 2.0 ** -12                                     # products on 2^-16, |X| |W| about 2^8: 2^24 quanta
    with pytest.raises(AssertionError):
        pf.grid_reference(fine, W, None, 4, "max")
    with pytest.raises(AssertionError):                         # fp32(1 / 3) is on a 2^-25 grid
        pf.grid_reference(X, W, np.full(128, 1 / 3, np.float32), 4, "max")
    # each pre + b is exact (on 2^-6, below 2^15), but 256 of them near 6000 sum past 2^24 quanta: only the mean refuses
    big = np.full(128, 6000.0, np.float32)
    pf.grid_reference(X * 4, W, big, 256, "max")
    with pytest.raises(AssertionError):
        pf.grid_reference(X * 4, W, big, 256, "mean")


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("name", ["k25_K63", "k65_K256", "k7_K9"])
def test_grid_contract_is_the_reference_semantics(name, pool):
    """On grid inputs the contract is oracle.maxpool_aggregator's neighbour branch (identity self / neighbour weights)
    and the fp64 mean of the ReLU'd rows, exactly."""
    inp = case_inputs(_case(name), grid=True)
    n, k, K, hidden = inp["counts"][128], inp["k"], inp["K"], inp["hidden"]
    X = pf.gather(inp["table"], K, n, k, inp["ids"], inp["row0"])
    got = pf.grid_reference(X, inp["W"], inp["bias"], k, pool).numpy()
    Wr = nu.bf16_rne(inp["W"]).astype(np.float64)
    b = (np.zeros(hidden) if inp["bias"] is None else inp["bias"]).astype(np.float64)
    neigh = X.astype(np.float64).reshape(n, k, K)
    if pool == "max":
        want = oracle.maxpool_aggregator(np.zeros((n, 1)), neigh, Wr, b, np.eye(hidden), np.zeros((1, hidden)),
                                         concat=False, act=lambda x: x)
    else:
        want = np.maximum(neigh.reshape(n * k, K) @ Wr + b, 0).reshape(n, k, hidden).mean(axis=1)
    assert np.array_equal(got, want.astype(np.float32))
    if pool == "max":
        assert np.array_equal(got.astype(np.float64), want)
    assert (got > 0).any() and (got == 0).any()


def test_bounded_reference_is_exact_on_the_grid_and_the_bound_scales():
    inp = case_inputs(_case("k25_K63"), grid=True)
    n = inp["counts"][128]
    X = pf.gather(inp["table"], inp["K"], n, inp["k"], inp["ids"], inp["row0"])
    for pool in pf.POOLS:
        ref, bound, s2, r = pf.bounded_reference(X, inp["W"], inp["bias"], inp["k"], pool)
        grid = pf.grid_reference(X, inp["W"], inp["bias"], inp["k"], pool).double()
        assert bool((torch.abs(grid - ref) <= pf.U * ref.abs() * (pool == "mean")).all())   # the mean: one division
        assert bool((bound > r).all()) and bool((r > 0).all()) and bool((s2 >= 0).all())
        # the grid answer is what an exact accumulator gives: inside R, so it adds nothing to the RMS statistic
        assert pf.errors(grid, ref, bound, s2, r)[1] == 0.0


# ---------------------------------------------------------------- the emulation passes
EMULATED = ["k1_K1", "k3_K8", "k7_K9", "k25_K63", "k64_K65", "k65_K256", "k25_K640", "k129_K602", "k200_K65",
            "k256_K640"]


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("name", EMULATED)
def test_emulation_passes_both_checks(name, pool):
    case = _case(name)
    for grid in (True, False):
        inp = case_inputs(case, grid=grid)
        for NT, n in inp["counts"].items():
            out = emulate_k4(inp, n, pool, NT)
            if grid:
                assert _grid_ok(inp, n, pool, out), (name, NT)
            else:
                ok, worst, rms = _bounded(inp, n, pool, out)
                assert ok, (name, NT, worst, rms)


# ---------------------------------------------------------------- each mutant fails
MUTANT_CASE = "k25_K63"      # 8 hidden slices, NT % k != 0, two tiles, a partial K-block, out-of-range ids, pad columns


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("mutant", MUTANTS)
def test_each_mutant_fails_a_check(mutant, pool):
    if POOL_ONLY.get(mutant, pool) != pool:
        pytest.skip("a %s-pool mutant" % POOL_ONLY[mutant])
    case = _case(MUTANT_CASE)
    grid_inp, rand_inp = case_inputs(case, grid=True), case_inputs(case, grid=False)
    n = grid_inp["counts"][128]
    assert 128 % grid_inp["k"] and n > 128 // grid_inp["k"] and grid_inp["K"] % KBLOCK
    with np.errstate(invalid="ignore"):
        grid_ok = _grid_ok(grid_inp, n, pool, emulate_k4(grid_inp, n, pool, 128, mutant))
        rand_ok = _bounded(rand_inp, n, pool, emulate_k4(rand_inp, n, pool, 128, mutant))[0]
    assert not (grid_ok and rand_ok), mutant
