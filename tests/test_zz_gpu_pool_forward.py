"""GPU: K4's forward (gs_maxpool_mlp_fused / gs_meanpool_mlp_fused) against the operand-exact contract of
oracle/pool_forward.py, in all nine named kernel variants (test_gpu_parity.K4_VARIANTS) and both pools.

* Grid inputs, bit for bit (zeros by value).  Every pad column of the table and every row no group should read is NaN,
  so a read of either shows.  Ids repeat (exact ties), one group reads one id k times, ids fall outside [0, n_rows) and
  row0 ranges run past the table.  One bias column is -4096 (output 0), one makes pre + b exactly 0 on some rows, and
  some cases pass no bias.  The output is a column slice of a NaN-filled wider buffer that must stay NaN around it.  Two
  calls are bit-identical and the variants agree.
* Random operands at the same shapes within the derived bounds; the worst bound ratio and the RMS statistic per
  (variant, pool) are printed at the end.
* The refusals: a fanout above the tile, K > 640, hidden % 128 != 0; n_groups = 0 launches nothing.

tests/test_pool_forward_numerics_cpu.py shows on a numpy emulation of the kernel that these checks reject subtly wrong
kernels at these shapes."""
import numpy as np
import pytest
import torch

from oracle import numerics as nu
from oracle import pool_forward as pf

pytestmark = pytest.mark.gpu

# (name, n_groups, k, K, hidden, rows addressed by "ids" | "row0", bias "special" | None).  n_groups is a count or, in
# terms of the tile's G = tile // k groups, "1", "G-1", "G", "G+1" or "waves" (300 tiles: several waves of CTAs).
# Fanouts 1 .. 128 run in every variant; 129 .. 256 only with 256-row tiles (the others must refuse them).  Hidden 128,
# 384, 640, 1024, 1280 are 1, 3, 5, 8, 10 slices, so k4_cluster 2 and -1 clamp to 1, 2, 3, 5 and 8 CTAs.
CASES = [
    ("k1_K1", "1", 1, 1, 128, "ids", "special"),
    ("k3_K8", "G-1", 3, 8, 384, "ids", None),
    ("k7_K9", "G", 7, 9, 640, "row0", "special"),
    ("k25_K63", "G+1", 25, 63, 1024, "ids", "special"),
    ("k43_K64", "waves", 43, 64, 1280, "ids", "special"),
    ("k64_K65", "G+1", 64, 65, 128, "row0", "special"),
    ("k65_K256", "G+1", 65, 256, 384, "ids", "special"),
    ("k128_K602", "waves", 128, 602, 640, "ids", "special"),
    ("k25_K640", "G-1", 25, 640, 1280, "ids", None),
    ("k3_K1", "waves", 3, 1, 1024, "row0", "special"),
    ("bench", 5120, 25, 602, 512, "ids", "special"),          # configs[2]'s hop-2 launch of layer 0
    ("k129_K602", "G+1", 129, 602, 384, "ids", "special"),
    ("k200_K65", "1", 200, 65, 128, "row0", None),
    ("k256_K640", "G", 256, 640, 640, "ids", "special"),
]
TILES = (128, 256)
WAVES = 300
BAD_IDS = (-1, -7, -2 ** 31, 2 ** 31 - 1)             # plus n_rows and n_rows + 5: all read the last row

# the largest ratios seen: {(variant, pool): [worst |err| / bound, rms |err| / S2*]}, printed at the end
MEASURED = {}


def group_count(spec, k, tile):
    G = tile // k
    if not isinstance(spec, str):
        return spec
    return {"1": 1, "G-1": G - 1, "G": G, "G+1": G + 1, "waves": WAVES * G}[spec]


def case_inputs(case, grid, seed=0):
    """numpy inputs of a case: a float32 table of bf16 values with NaN pad columns (pitch = pad_cols(K) + 8) and NaN in
    every row no group reads, row ids or row0, W [K, hidden] fp32, bias fp32 or None, and the group count per tile.
    grid: operands on multiples of 2^-4 (the contract's exact answer); else Gaussian X (bf16) and W / sqrt(K)."""
    name, spec, k, K, hidden, form, bias_kind = case
    counts = {t: group_count(spec, k, t) for t in TILES if k <= t}
    nmax, nmin = max(counts.values()), min(counts.values())
    rs = np.random.RandomState(seed + 1000 * k + 7 * K + hidden)
    pitch = (K + 7) // 8 * 8 + 8
    if form == "ids":
        n_rows = 4096
        pool = rs.choice(np.arange(1, n_rows - 1), size=256, replace=False)   # row 0 stays NaN
        ids = pool[rs.randint(0, pool.size, size=nmax * k)].astype(np.int64)
        ids[:k] = pool[0]                                                     # one group of one repeated id
        bad = np.array(BAD_IDS + (n_rows, n_rows + 5), dtype=np.int64)
        pos = np.concatenate([np.arange(k, min(nmax * k, k + bad.size)), rs.randint(0, nmax * k, size=nmax * k // 50)])
        ids[pos] = bad[np.arange(pos.size) % bad.size]
        ids = ids.astype(np.int32)
        row0 = 0
        live = np.concatenate([pool, [n_rows - 1]])
    else:
        n_rows = max(3000, nmin * k)
        row0 = n_rows - max(1, nmin * k // 2)                  # the smallest launch already runs past the table
        ids = None
        live = np.arange(row0, n_rows)
    table = np.full((n_rows, pitch), np.nan, np.float32)
    if grid:
        vals = rs.randint(-32, 33, size=(live.size, K)) / 16.0
        vals[:, 0] = rs.choice([-0.5, 0.0, 0.5, 1.0], size=live.size)
        W = rs.randint(-16, 17, size=(K, hidden)) / 16.0
        b = rs.randint(-32, 33, size=hidden) / 16.0
    else:
        vals = nu.bf16_rne(rs.randn(live.size, K))
        W = rs.randn(K, hidden) / np.sqrt(K)
        b = rs.randn(hidden)
    table[live, :K] = vals
    W = W.astype(np.float32)
    bias = None
    if bias_kind == "special":
        bias = b.astype(np.float32)
        bias[hidden - 1] = -4096.0                              # every pre + b < 0: the output is 0
        if grid and hidden > 2:
            W[:, 1] = 0.0                                       # pre = X[:, 0] in {-0.5, 0, 0.5, 1}: pre + b hits 0
            W[0, 1] = 1.0
            bias[1] = -0.5
    return dict(case=case, table=table, n_rows=n_rows, pitch=pitch, K=K, k=k, hidden=hidden, ids=ids, row0=row0,
                W=W, bias=bias, counts=counts, nmax=nmax)


def reference_X(inp, n, device=None):
    """X [n * k, K] fp32 of the first n groups: numpy (device None) or gathered on the device from the same table."""
    k, K = inp["k"], inp["K"]
    if device is None:
        return pf.gather(inp["table"], K, n, k, inp["ids"], inp["row0"])
    idx = torch.from_numpy(pf.row_index(inp["n_rows"], n, k, inp["ids"], inp["row0"])).to(device)
    return torch.from_numpy(inp["table"][:, :K]).to(device)[idx]


# ---------------------------------------------------------------- GPU side
@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    yield graphsage_b200
    if MEASURED:
        print("\nK4 forward, measured on %s:" % torch.cuda.get_device_name())
        for (variant, pool), (worst, rms) in sorted(MEASURED.items()):
            print("  %-16s %-4s worst |err| / bound = %.3e   rms |err| / S2 = %.3e (2^%.1f)"
                  % (variant, pool, worst, rms, np.log2(rms) if rms > 0 else -np.inf))


@pytest.fixture(autouse=True)
def _default_tuning(gs):
    """Every case switches the K4 variant; the default comes back even when it fails (later files run with it)."""
    from test_gpu_parity import K4_DEFAULT, _k4_select
    try:
        yield
    finally:
        _k4_select(gs, K4_DEFAULT)


def _variants():
    from test_gpu_parity import K4_VARIANTS
    return K4_VARIANTS


def _device_inputs(gs, inp):
    tab = torch.from_numpy(inp["table"]).cuda().to(torch.bfloat16)
    return dict(table=tab, W=torch.from_numpy(inp["W"]).cuda(),
                bias=None if inp["bias"] is None else torch.from_numpy(inp["bias"]).cuda(),
                ids=None if inp["ids"] is None else torch.from_numpy(inp["ids"]).cuda(),
                packed=gs.ops.PackedMlpWeights())


def _call(gs, inp, d, n, pool, out=None):
    k, K = inp["k"], inp["K"]
    ids = None if d["ids"] is None else d["ids"][:n * k]
    return gs.ops.maxpool_mlp_fused(d["table"][:, :K], n, k, d["W"], d["bias"], d["packed"], row_ids=ids,
                                    row0=inp["row0"], out=out, pool=pool)


def _run_variants(gs, inp, d, pool, check):
    """Run every variant on inp: a refusal when the fanout exceeds its tile, else the output into a column slice of a
    NaN-filled wider buffer (left NaN around it) and again into a fresh buffer (the same bits); check(variant, n, out).
    Then the variants of each tile width agree with each other (zeros by value)."""
    from test_gpu_parity import _k4_select
    hidden, k = inp["hidden"], inp["k"]
    outs = {}
    for name, (_, tile, _, _, _) in _variants().items():
        _k4_select(gs, name)
        if k > tile:
            with pytest.raises(RuntimeError, match="k <= %d" % tile):
                _call(gs, inp, d, 1, pool)
            continue
        n = inp["counts"][tile]
        full = torch.full((n + 2, hidden + 9), float("nan"), device="cuda")
        out = _call(gs, inp, d, n, pool, out=full[:n, 5:5 + hidden])
        assert out.stride(0) == hidden + 9
        again = _call(gs, inp, d, n, pool)
        torch.cuda.synchronize()
        rest = torch.cat([full[n:].reshape(-1), full[:n, :5].reshape(-1), full[:n, 5 + hidden:].reshape(-1)])
        assert bool((rest.view(torch.int32) == 0x7FC00000).all()), (name, pool, "wrote outside the output slice")
        assert torch.equal(out.view(torch.int32), again.view(torch.int32)), (name, pool, "two calls differ")
        check(name, n, out)
        outs.setdefault(tile, []).append((name, out.clone()))
    for lst in outs.values():
        for name, o in lst[1:]:
            assert pf.same_values(o, lst[0][1]), (name, lst[0][0], pool)


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_grid_inputs_bit_for_bit(gs, case, pool):
    inp = case_inputs(case, grid=True)
    ref = pf.grid_reference(reference_X(inp, inp["nmax"], "cuda"), inp["W"], inp["bias"], inp["k"], pool)
    if inp["bias"] is not None:
        assert bool((ref[:, -1] == 0).all())

    def check(name, n, out):
        if not pf.same_values(out, ref[:n]):
            bad = torch.nonzero((out + 0.0).view(torch.int32) != (ref[:n] + 0.0).view(torch.int32))
            pytest.fail("%s %s %s: %d elements differ, first (group, unit) %s: got %r want %r"
                        % (case[0], name, pool, bad.shape[0], bad[0].tolist(), float(out[tuple(bad[0])]),
                           float(ref[tuple(bad[0])])))

    _run_variants(gs, inp, _device_inputs(gs, inp), pool, check)


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_random_operands_within_the_derived_bound(gs, case, pool):
    inp = case_inputs(case, grid=False)
    refs = pf.bounded_reference(reference_X(inp, inp["nmax"], "cuda"), inp["W"], inp["bias"], inp["k"], pool)

    def check(name, n, out):
        ok, worst, rms = pf.check_bounded(out, *(x[:n] for x in refs))
        w, r = MEASURED.get((name, pool), (0.0, 0.0))
        MEASURED[(name, pool)] = [max(w, worst), max(r, rms)]
        assert ok, (case[0], name, pool, worst, rms)

    _run_variants(gs, inp, _device_inputs(gs, inp), pool, check)


def test_refusals_and_an_empty_launch(gs):
    from test_gpu_parity import K4_VARIANTS, _k4_select
    table = torch.zeros((64, 648), dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(600, dtype=torch.int32, device="cuda")
    W = torch.zeros((64, 128), device="cuda")
    packed = gs.ops.PackedMlpWeights()
    for pool in pf.POOLS:
        for name, (_, tile, _, _, _) in K4_VARIANTS.items():
            _k4_select(gs, name)
            gs.ops.maxpool_mlp_fused(table[:, :64], 2, tile, W, None, packed, row_ids=ids, pool=pool)
            with pytest.raises(RuntimeError, match="k <= %d" % tile):
                gs.ops.maxpool_mlp_fused(table[:, :64], 1, tile + 1, W, None, packed, row_ids=ids, pool=pool)
        _k4_select(gs, "round1")
        with pytest.raises(RuntimeError, match="K <= 640"):
            gs.ops.maxpool_mlp_fused(table[:, :641], 2, 3, torch.zeros((641, 128), device="cuda"), None,
                                     gs.ops.PackedMlpWeights(), row_ids=ids, pool=pool)
        with pytest.raises(RuntimeError, match="hidden % 128 == 0"):
            gs.ops.maxpool_mlp_fused(table[:, :64], 2, 3, torch.zeros((64, 200), device="cuda"), None,
                                     gs.ops.PackedMlpWeights(), row_ids=ids, pool=pool)
    # n_groups = 0: success without touching a pointer (all NULL) and nothing launched through the wrappers
    lib = gs._lib.lib()
    for fn in (lib.gs_maxpool_mlp_fused, lib.gs_meanpool_mlp_fused):
        assert fn(None, 64, 64, 64, None, 0, 0, 3, None, None, 128, None, 128, None) == 0
    packed.get(W)
    before = gs.ops.LAUNCHES
    full = torch.full((1, 128), float("nan"), device="cuda")
    out = gs.ops.maxpool_mlp_fused(table[:, :64], 0, 3, W, None, packed, row_ids=ids[:0], out=full[:0])
    torch.cuda.synchronize()
    assert tuple(out.shape) == (0, 128) and gs.ops.LAUNCHES == before
    assert bool(torch.isnan(full).all())
