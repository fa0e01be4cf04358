"""GPU: the pooling backward through the fused bf16 kernels - B1 gs_pool_mlp_backward_dp, B2 gs_pool_mlp_backward_dw, B3
gs_pool_mlp_backward_dx - against the contract of oracle/pool_backward.py, on random bf16 operands.

* B1 bit for bit, teacher-forced on K4's own pre-activations: pre_K4 is read off the default K4 forward by the probe
  (probe() below: the real row at position j of every group, zero rows elsewhere, out(Wm) - out(-Wm)), and B1's dP
  and dbm partials must equal pool_grad's dpre of it.  Every pre_K4 also lies within K4's accumulation bound of the
  float64 product, and the default K4 forward equals the max / mean epilogue of pre_K4 bit for bit (zeros by value).
* Edges in the B1 cases: exact ties from duplicate ids inside a group (count 2, 3 and k), an all-zero-row group, a
  bias column of 2^22 max|pre| (post-bias ties that are not pre-activation ties), bias columns that make pre + b exactly
  0 at a group's largest row, b = -4096 columns, a NULL bias, and dhp with -0.0, subnormals and c x values whose
  division by the tie count or by k is a bf16 rounding tie.
* Addressing: NaN in pad columns and in rows no id reads; ids -1, n_rows and 2^31 - 1; a row0 range running past the
  table; dhp a view of a NaN-padded wider buffer (lddhp > hidden).  B1's buffer and B2's workspace start as NaN
  bytes and B1 must write every byte it owns (padding slots +0) and nothing after it; B3 writes into a NaN frame with
  ldx > Kd and extra rows that must stay NaN.
* B2: criteria (a) and (b) of numerics.check_gemm for X^T dP_kernel, the add into a nonzero dWm is fl32(dWm0 + sum),
  dbm is the fixed-order combine of the teacher-forced partials added once.  B3: (a) and (b) for dP_kernel Wm^T[:, :Kd].
  The training shapes of tools/pool_train_bench.py (layer 0 hop 2: 5,120 groups of 25 rows, K = 602, hidden 512 and
  1024; layer 1: 512 groups of 10, K = 256) are among the cases.  The largest ratios are printed at the end.
* The probe under every K4 variant (informational: whether a non-default tuning accumulates the same bits), two calls
  bit-identical, empty calls and the refusals.

tests/test_pool_backward_numerics_cpu.py shows on a numpy emulation of the kernels that these checks reject subtly
wrong kernels."""
import numpy as np
import pytest
import torch

from oracle import numerics as nu
from oracle import pool_backward as pb
from oracle import pool_forward as pf

pytestmark = pytest.mark.gpu

# (name, n_groups, k, K, hidden, rows addressed by "ids" | "row0", bias "special" | None).  G = 128 // k groups per tile.
CASES = [
    ("k1_K1", 300, 1, 1, 128, "ids", "special"),            # G = 128: three tiles, the last one partial
    ("k2_K7", 1, 2, 7, 384, "row0", None),                   # one group
    ("k3_K8", 85, 3, 8, 640, "ids", "special"),              # G = 42: two padding slots per tile, last tile partial
    ("k25_K63", 11, 25, 63, 512, "ids", None),
    ("k43_K64", 40, 43, 64, 384, "ids", "special"),          # G = 2: 42 padding slots per tile
    ("k64_K65", 9, 64, 65, 128, "row0", "special"),
    ("k65_K602", 7, 65, 602, 640, "ids", "special"),         # G = 1: 63 padding slots per tile
    ("k127_K640", 3, 127, 640, 1024, "ids", "special"),
    ("k128_K602", 4, 128, 602, 128, "ids", None),
    ("waves", 20000, 3, 65, 384, "row0", "special"),         # 477 tiles x 3 slices: several waves of CTAs
    ("layer1", 512, 10, 256, 512, "ids", "special"),         # layer 1 of the training shape
    ("hop2_512", 5120, 25, 602, 512, "ids", "special"),      # layer 0 hop 2 of the training shape, "small"
    ("hop2_1024", 5120, 25, 602, 1024, "ids", "special"),    # ... "big"
]
BAD_IDS = (-1, 2 ** 31 - 1)                                  # plus n_rows: all read the last row
NAN_BYTE = 0xFF                                              # 0xFFFF (bf16) and 0xFFFFFFFF (fp32) are NaN
GUARD = 256

# the largest ratios seen, printed at the end: {(kernel, case): [worst |err| / bound, rms]}
MEASURED = {}
VARIANT_PROBE = {}


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    yield graphsage_b200
    if MEASURED:
        print("\npooling backward, measured on %s:" % torch.cuda.get_device_name())
        for key, (worst, rms) in sorted(MEASURED.items()):
            print("  %-3s %-16s worst |err| / bound = %.3e   rms = %.3e (2^%.1f)"
                  % (key[0], key[1], worst, rms, np.log2(rms) if rms > 0 else -np.inf))
    for key, same in sorted(VARIANT_PROBE.items()):
        print("  probe %-16s %-10s pre bits %s round1's" % (key[0], key[1], "equal" if same else "DIFFER from"))


@pytest.fixture(autouse=True)
def _default_tuning(gs):
    """The probe reads the default K4 (round1); the default stays selected whatever a test does."""
    from test_gpu_parity import K4_DEFAULT, _k4_select
    _k4_select(gs, K4_DEFAULT)
    try:
        yield
    finally:
        _k4_select(gs, K4_DEFAULT)


def _tie_values(rs, shape):
    """x = +-(1 + m 2^-7 + 2^-8) 2^e: exactly halfway between two bf16 values, 9 significant bits"""
    m = rs.randint(0, 128, size=shape)
    e = rs.randint(-12, 3, size=shape)
    s = rs.choice([-1.0, 1.0], size=shape)
    return (s * (1.0 + m * 2.0 ** -7 + 2.0 ** -8) * 2.0 ** e).astype(np.float32)


def case_inputs(case, pool, seed=0):
    """numpy inputs: a float32 table of bf16 values with NaN pad columns and NaN in every row nothing reads, an all-zero
    row for the probe, ids (or row0), W, the bias before its probe-dependent columns, and dhp."""
    name, n, k, K, hidden, form, bias_kind = case
    rs = np.random.RandomState(seed + 1000 * k + 7 * K + hidden + (pool == "mean"))
    pitch = (K + 7) // 8 * 8 + 8
    if form == "ids":
        n_rows = max(4096, n * k // 4)
        live = rs.choice(np.arange(2, n_rows - 1), size=min(n_rows // 2, max(256, n * k // 8)), replace=False)
        zero_row = 1
        ids = live[rs.randint(0, live.size, size=n * k)].astype(np.int64).reshape(n, k)
        keep = np.zeros((n, k), bool)                           # the tie and zero-row positions below
        if k >= 2:
            ids[0] = live[0]                                    # count k: one id k times
            keep[0] = True
        if k >= 2 and n > 1:
            ids[1, k - 1] = ids[1, 0]                           # count 2 (at least)
            keep[1, [0, k - 1]] = True
        if k >= 3 and n > 2:
            ids[2, [k // 2, k - 1]] = ids[2, 0]                 # count 3 (at least)
            keep[2, [0, k // 2, k - 1]] = True
        if n > 3:
            ids[3] = zero_row                                   # an all-zero-row group
            keep[3] = True
        ids, keep = ids.reshape(-1), keep.reshape(-1)
        free = np.flatnonzero(~keep)
        pos = rs.choice(free, size=min(free.size, max(3, n * k // 40)), replace=False)
        bad = np.array(BAD_IDS + (n_rows,), dtype=np.int64)
        ids[pos] = bad[np.arange(pos.size) % bad.size]
        ids = ids.astype(np.int32)
        row0 = 0
        live = np.concatenate([live, [n_rows - 1]])
    else:
        n_rows = max(3000, n * k // 2 + 8)
        row0 = n_rows - max(1, n * k // 2)                     # the range runs past the table
        zero_row = row0 - 2                                     # read by the probe only
        ids = None
        live = np.arange(row0, n_rows)
    table = np.full((n_rows, pitch), np.nan, np.float32)
    table[live, :K] = nu.bf16_rne(rs.randn(live.size, K))
    table[zero_row, :K] = 0.0
    W = (rs.randn(K, hidden) / np.sqrt(K)).astype(np.float32)
    bias = None
    if bias_kind == "special":
        bias = rs.randn(hidden).astype(np.float32) * np.float32(0.5)
        bias[hidden - 2:] = -4096.0                            # hp = 0: no gradient
    x = _tie_values(rs, (n, hidden))
    c = np.ones((n, 1), np.float32)
    if pool == "mean":
        c[:] = k
    else:
        c[:min(n, 4)] = np.array([k, 2, 3, k], np.float32)[:min(n, 4), None]
    dhp = np.where(rs.rand(n, hidden) < 0.5, c * x, rs.randn(n, hidden)).astype(np.float32)
    flat = dhp.reshape(-1)
    pick = rs.choice(flat.size, size=max(2, flat.size // 50), replace=False)
    half = pick.size // 2
    flat[pick[:half]] = -0.0
    flat[pick[half:]] = (rs.randint(1, 2 ** 20, size=pick.size - half) * rs.choice([-1.0, 1.0], size=pick.size - half)
                         * 2.0 ** -149).astype(np.float32)     # subnormals
    return dict(case=case, n=n, k=k, K=K, hidden=hidden, table=table, n_rows=n_rows, pitch=pitch, ids=ids, row0=row0,
                zero_row=zero_row, W=W, bias=bias, dhp=dhp)


def _device(gs, inp):
    n, hidden = inp["n"], inp["hidden"]
    dhp_buf = torch.full((n, hidden + 24), float("nan"), device="cuda")
    dhp_buf[:, :hidden] = torch.from_numpy(inp["dhp"]).cuda()
    W = torch.from_numpy(inp["W"]).cuda()
    return dict(table=torch.from_numpy(inp["table"]).cuda().to(torch.bfloat16), W=W, Wneg=-W,
                ids=None if inp["ids"] is None else torch.from_numpy(inp["ids"]).cuda(),
                dhp=dhp_buf[:, :hidden], packed=gs.ops.PackedMlpWeights(), packed_neg=gs.ops.PackedMlpWeights())


def probe(gs, inp, d):
    """pre_K4 [n k, hidden] fp32 on the device, read off the current K4 forward (oracle/pool_backward.py: the probe)."""
    n, k, K, hidden = inp["n"], inp["k"], inp["K"], inp["hidden"]
    rows = pf.row_index(inp["n_rows"], n, k, inp["ids"], inp["row0"])
    pre = torch.empty((n, k, hidden), dtype=torch.float32, device="cuda")
    for j in range(k):
        ids = torch.from_numpy(pb.probe_rows(rows, n, k, j, inp["zero_row"])).cuda()
        pos = gs.ops.maxpool_mlp_fused(d["table"][:, :K], n, k, d["W"], None, d["packed"], row_ids=ids)
        neg = gs.ops.maxpool_mlp_fused(d["table"][:, :K], n, k, d["Wneg"], None, d["packed_neg"], row_ids=ids)
        assert bool(((pos == 0) | (neg == 0)).all())
        pre[:, j] = pos - neg
    return pre.reshape(n * k, hidden)


def _finish_bias(inp, pre):
    """the probe-dependent bias columns: a 2^22 max|pre| column (post-bias ties) and columns with b = -pre at the
    largest row of one group (z = 0 exactly at the max)."""
    if inp["bias"] is None:
        return None
    n, k, hidden = inp["n"], inp["k"], inp["hidden"]
    b = inp["bias"].copy()
    p = pre.reshape(n, k, hidden)
    for u in (2, 5):
        m = float(p[:, :, u].abs().max())
        b[u] = 2.0 ** (np.ceil(np.log2(m)) + 22) if m > 0 else 1.0
    for i, u in enumerate(range(8, min(hidden - 2, 8 + 16))):
        g0 = (i * 7919) % n
        b[u] = -float(p[g0, :, u].max())
    return b


def _forward_epilogue(pre, bias, n, k, pool):
    """fmaxf(max_j pre_j + b, 0) (max) or the fp32 sum in j order of fmaxf(pre_j + b, 0) over fp32(k) (mean)"""
    hid = pre.shape[-1]
    p = pre.reshape(n, k, hid)
    b = torch.zeros(hid, device=pre.device) if bias is None else bias
    if pool == "max":
        return torch.clamp_min(p.max(dim=1).values + b, 0.0)
    s = torch.zeros((n, hid), dtype=torch.float32, device=pre.device)
    for j in range(k):
        s = s + torch.clamp_min(p[:, j] + b, 0.0)
    return s / torch.tensor(float(k), dtype=torch.float32, device=pre.device)


def _nan_bytes(nbytes):
    return torch.full((nbytes + GUARD,), NAN_BYTE, dtype=torch.uint8, device="cuda")


def _b1(gs, inp, d, bias_t, pool):
    """B1 through the C ABI into a NaN buffer with a guard region after it -> (buffer, guard untouched)"""
    from graphsage_b200 import ops
    n, k, K, hidden = inp["n"], inp["k"], inp["K"], inp["hidden"]
    nbytes = gs._lib.lib().gs_pool_mlp_dp_bytes(n, k, hidden)
    buf = _nan_bytes(nbytes)
    rc = gs._lib.lib().gs_pool_mlp_backward_dp(
        ops.ptr(d["table"]), inp["n_rows"], K, d["table"].stride(0), ops.ptr(d["ids"]), inp["row0"], n, k,
        ops.ptr(d["packed"].get(d["W"])), ops.ptr(bias_t), hidden, ops.ptr(d["dhp"]), d["dhp"].stride(0),
        int(pool == "mean"), ops.ptr(buf), ops.stream_ptr())
    assert rc == 0, gs._lib.last_error() if hasattr(gs._lib, "last_error") else rc
    torch.cuda.synchronize()
    return buf[:nbytes], bool((buf[nbytes:] == NAN_BYTE).all())


def _b2(gs, inp, d, buf, dWm, dbm):
    from graphsage_b200 import ops
    n, k, K, hidden = inp["n"], inp["k"], inp["K"], inp["hidden"]
    nbytes = gs._lib.lib().gs_pool_mlp_dw_workspace_bytes(n, k, K, hidden)
    ws = _nan_bytes(nbytes)
    rc = gs._lib.lib().gs_pool_mlp_backward_dw(
        ops.ptr(d["table"]), inp["n_rows"], K, d["table"].stride(0), ops.ptr(d["ids"]), inp["row0"], n, k, hidden,
        ops.ptr(buf), ops.ptr(ws), nbytes, ops.ptr(dWm), hidden, ops.ptr(dbm), ops.stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()


def _record(kernel, name, worst, rms):
    w, r = MEASURED.get((kernel, name), (0.0, 0.0))
    MEASURED[(kernel, name)] = [max(w, worst), max(r, rms)]


@pytest.mark.parametrize("pool", pf.POOLS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_backward_against_the_contract(gs, case, pool):
    name = case[0]
    inp = case_inputs(case, pool)
    n, k, K, hidden = inp["n"], inp["k"], inp["K"], inp["hidden"]
    d = _device(gs, inp)
    idx = torch.from_numpy(pf.row_index(inp["n_rows"], n, k, inp["ids"], inp["row0"])).cuda()
    X = torch.from_numpy(inp["table"][:, :K]).cuda()[idx]                # the gathered rows, fp32
    assert not bool(torch.isnan(X).any())

    # pre_K4 by the probe, and the probe-free window
    pre = probe(gs, inp, d)
    ok, worst = pb.window(pre, X, inp["W"])
    _record("pre", name, worst, 0.0)
    assert ok, (name, "pre_K4 outside K4's accumulation bound", worst)
    bias = _finish_bias(inp, pre)
    bias_t = None if bias is None else torch.from_numpy(bias).cuda()

    # the default K4 forward is the epilogue of pre_K4
    out = gs.ops.maxpool_mlp_fused(d["table"][:, :K], n, k, d["W"], bias_t, d["packed"], row_ids=d["ids"],
                                   row0=inp["row0"], pool=pool)
    assert pf.same_values(out, _forward_epilogue(pre, bias_t, n, k, pool)), (name, "K4 is not the epilogue of pre_K4")

    # B1, twice
    buf, guard = _b1(gs, inp, d, bias_t, pool)
    again, _ = _b1(gs, inp, d, bias_t, pool)
    assert guard, (name, "B1 wrote past its buffer")
    assert torch.equal(buf, again), (name, "two B1 calls differ")
    pre_np = pre.cpu().numpy()
    buf_np = buf.cpu().numpy()
    bad, dP, dpre = pb.check_b1(buf_np, pre_np, bias, inp["dhp"], n, k, pool)
    assert not bad, (name, pool, bad)
    if bias is not None and pool == "max":
        assert not dP[:, hidden - 1].any() and dP[:, 2].any()
    assert dP.any()

    # B2: into zeros, then into a nonzero dWm / dbm (added once)
    rs = np.random.RandomState(5)
    dW0 = torch.zeros((K, hidden), dtype=torch.float32, device="cuda")
    db0 = torch.zeros((hidden,), dtype=torch.float32, device="cuda")
    _b2(gs, inp, d, buf, dW0, db0)
    dWm_in = rs.randn(K, hidden).astype(np.float32)
    dbm_in = rs.randn(hidden).astype(np.float32)
    dWm, dbm = torch.from_numpy(dWm_in).cuda(), torch.from_numpy(dbm_in).cuda()
    _b2(gs, inp, d, buf, dWm, dbm)
    assert torch.equal(dWm, torch.from_numpy(dWm_in).cuda() + dW0), (name, "dWm is not fl32(dWm0 + sum)")
    assert nu.bits_equal(dbm.cpu().numpy(), pb.dbm_reference(dpre, n, k, dbm_in)), (name, "dbm")
    dP_dev = torch.from_numpy(dP).cuda()
    ok, worst, rms = pb.check_gemm(dW0, *pb.dw_reference(X, dP_dev))
    _record("B2", name, worst, rms)
    assert ok, (name, pool, "B2", worst, rms)

    # B3 into a NaN frame: ldx > Kd, extra rows
    for Kd in sorted({K, max(1, K // 3)}):
        frame = torch.full((n * k + 3, Kd + 13), float("nan"), device="cuda")
        dx = gs.ops.pool_mlp_backward_dx(buf, n, k, d["W"], gs.ops.PackedMlpDxWeights(Kd), out=frame[:n * k, :Kd])
        torch.cuda.synchronize()
        assert dx.stride(0) == Kd + 13
        rest = torch.cat([frame[n * k:].reshape(-1), frame[:n * k, Kd:].reshape(-1)])
        assert bool((rest.view(torch.int32) == 0x7FC00000).all()), (name, "B3 wrote outside its view")
        ok, worst, rms = pb.check_gemm(dx, *pb.dx_reference(dP_dev, inp["W"], Kd))
        _record("B3", name, worst, rms)
        assert ok, (name, pool, "B3", Kd, worst, rms)


PROBE_CASES = ("k3_K8", "k25_K63", "layer1")


@pytest.mark.parametrize("name", PROBE_CASES)
def test_probe_under_every_k4_variant(gs, name):
    """Informational: whether each K4 variant accumulates the pre bits of the default (printed at the end; only the
    default is B1's forward).  Every variant's pre must lie in the window, as K4's contract requires."""
    from test_gpu_parity import K4_VARIANTS, _k4_select
    case = next(c for c in CASES if c[0] == name)
    inp = case_inputs(case, "max")
    d = _device(gs, inp)
    idx = torch.from_numpy(pf.row_index(inp["n_rows"], inp["n"], inp["k"], inp["ids"], inp["row0"])).cuda()
    X = torch.from_numpy(inp["table"][:, :inp["K"]]).cuda()[idx]
    base = probe(gs, inp, d)
    for variant, (_, tile, _, _, _) in K4_VARIANTS.items():
        if inp["k"] > tile:
            continue
        _k4_select(gs, variant)
        pre = probe(gs, inp, d)
        assert pb.window(pre, X, inp["W"])[0], variant
        VARIANT_PROBE[(name, variant)] = bool(torch.equal(pre.view(torch.int32), base.view(torch.int32))) or \
            pf.same_values(pre, base)
    assert VARIANT_PROBE[(name, "round1")]


def test_refusals_and_empty_calls(gs):
    from graphsage_b200 import ops
    lib = gs._lib.lib()
    # n_groups = 0: success with every pointer NULL, and nothing written
    assert lib.gs_pool_mlp_backward_dp(None, 64, 64, 64, None, 0, 0, 3, None, None, 128, None, 128, 0, None, None) == 0
    assert lib.gs_pool_mlp_backward_dw(None, 64, 64, 64, None, 0, 0, 3, 128, None, None, 0, None, 128, None, None) == 0
    assert lib.gs_pool_mlp_backward_dx(0, 3, 128, None, None, 64, None, 64, None) == 0
    table = torch.zeros((64, 648), dtype=torch.bfloat16, device="cuda")
    W = torch.zeros((64, 128), device="cuda")
    dWm = torch.full((64, 128), float("nan"), device="cuda")
    dbm = torch.full((128,), float("nan"), device="cuda")
    buf = _nan_bytes(0)
    gs.ops.pool_mlp_backward_dw(table[:, :64], 0, 3, buf, dWm, dbm, row0=0)
    dx = gs.ops.pool_mlp_backward_dx(buf, 0, 3, W, gs.ops.PackedMlpDxWeights(64))
    torch.cuda.synchronize()
    assert tuple(dx.shape) == (0, 64) and bool(torch.isnan(dWm).all()) and bool(torch.isnan(dbm).all())
    assert bool((buf == NAN_BYTE).all())
    # fanout, K and hidden limits
    dhp = torch.zeros((2, 128), device="cuda")
    ids = torch.zeros(2 * 129, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="k <= 128"):
        gs.ops.pool_mlp_backward_dp(table[:, :64], 2, 129, W, None, gs.ops.PackedMlpWeights(), dhp, row_ids=ids)
    with pytest.raises(RuntimeError, match="K <= 640"):
        gs.ops.pool_mlp_backward_dp(table[:, :641], 2, 3, torch.zeros((641, 128), device="cuda"), None,
                                    gs.ops.PackedMlpWeights(), dhp, row_ids=ids)
    assert lib.gs_pool_mlp_dp_bytes(2, 3, 200) == -1 and lib.gs_pool_mlp_dp_bytes(2, 129, 128) == -1
    assert lib.gs_pool_mlp_dw_workspace_bytes(2, 3, 64, 200) == -1
    assert lib.gs_pool_mlp_dx_pack_bytes(64, 200) == -1
    with pytest.raises(ValueError, match="lddhp|unit column stride|matrix"):
        gs.ops.pool_mlp_backward_dp(table[:, :64], 2, 3, W, None, gs.ops.PackedMlpWeights(), dhp[:, :100],
                                    row_ids=ids)
    # B2: ldw != hidden and a short workspace; B3: ldx < Kd
    n, k, K = 2, 3, 64
    grad = gs.ops.pool_mlp_backward_dp(table[:, :K], n, k, W, None, gs.ops.PackedMlpWeights(), dhp, row_ids=ids[:6])
    nb = lib.gs_pool_mlp_dw_workspace_bytes(n, k, K, 128)
    ws = _nan_bytes(nb)
    dW = torch.zeros((K, 128), device="cuda")
    db = torch.zeros((128,), device="cuda")
    args = (ops.ptr(table), 64, K, table.stride(0), ops.ptr(ids), 0, n, k, 128, ops.ptr(grad), ops.ptr(ws))
    assert lib.gs_pool_mlp_backward_dw(*args, nb, ops.ptr(dW), 129, ops.ptr(db), ops.stream_ptr()) != 0
    assert lib.gs_pool_mlp_backward_dw(*args, nb - 4, ops.ptr(dW), 128, ops.ptr(db), ops.stream_ptr()) != 0
    packed = gs.ops.PackedMlpDxWeights(K).get(W)
    out = torch.full((n * k, K), float("nan"), device="cuda")
    assert lib.gs_pool_mlp_backward_dx(n, k, 128, ops.ptr(grad), ops.ptr(packed), K, ops.ptr(out), K - 1,
                                       ops.stream_ptr()) != 0
    with pytest.raises(ValueError, match="out must be"):
        gs.ops.pool_mlp_backward_dx(grad, n, k, W, gs.ops.PackedMlpDxWeights(K), out=out[:, :K - 1])
    torch.cuda.synchronize()
    assert bool(torch.isnan(out).all()) and not dW.any() and not db.any()
