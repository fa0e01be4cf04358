"""GPU: the aggregation kernels against operand-exact references (oracle/numerics.py).

* Fanout means (every gs_gather_mean form, gs_gather_mean_dropout) bit for bit against numerics.mean_f32.
* The K3 GEMM (gs_sage_gemm, one-shot and prepacked) in all four math modes against the float64 product of the operands
  the mode multiplies, within numerics.check_gemm's worst-case and RMS bounds.
* gs_sage_layer_small (mean -> GEMM -> bias -> ReLU -> l2-normalise in one launch), gs_segment_max and
  gs_l2_normalize_rows.

tests/test_numerics_cpu.py shows on an emulation that each check rejects a subtly wrong kernel."""
import numpy as np
import pytest
import torch

from oracle import dropout
from oracle import numerics as nu

pytestmark = pytest.mark.gpu

# the largest ratios seen per math mode: {mode: [worst-case fraction of bound (a), RMS statistic (b)]}, printed at the end
MEASURED = {}


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    yield graphsage_b200
    if MEASURED:
        print("\nmeasured on %s:" % torch.cuda.get_device_name())
        for mode, (worst, rms) in sorted(MEASURED.items()):
            print("  %-12s worst |err| / bound (a) = %.3e   rms |err| / S2 = %.3e (2^%.1f)"
                  % (mode, worst, rms, np.log2(rms) if rms > 0 else -np.inf))


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def _note(mode, worst, rms):
    w, r = MEASURED.get(mode, (0.0, 0.0))
    MEASURED[mode] = [max(w, worst), max(r, rms)]


# ---------------------------------------------------------------- fanout means, bit for bit
FORMS = ["tma2", "tma", "ldg", "scalar", "bf16"]
VARIANT = {"tma2": 2, "tma": 1, "ldg": 0, "scalar": 2, "bf16": 2}
# one gather call per list: (n, k) per segment - mixed size order, empty segments, every fanout
CALLS = [[(40, 25), (0, 13), (9, 128), (17, 1)],
         [(5, 2), (33, 7), (0, 3), (21, 5)],
         [(12, 64), (30, 2)]]
N_SRC = 700


def _special_table(rs, F):
    """Normal rows plus rows of -0.0, of subnormals, of 3e38 (two of them overflow to +inf) and of mixed tiny values."""
    x = rs.randn(N_SRC, F).astype(np.float32)
    x[0] = -0.0
    x[1] = rs.choice([1e-45, -1e-45, 1e-40, -2e-39, 5e-39], size=F)
    x[2] = 3.0e38
    x[3] = rs.choice([-0.0, 0.0, 1e-44, -1e-38], size=F)
    return x


def _segment_ids(rs, n, k, s):
    """Self / neighbour ids: out-of-range ids (read the last row), and in segment s % 2 == 1 ids from a pool of six rows
    (the special ones among them), repeated many times."""
    if s % 2:
        nb = rs.randint(0, 6, size=n * k)
    else:
        nb = rs.randint(-3, N_SRC + 3, size=n * k)
    sf = rs.randint(-2, N_SRC + 2, size=n)
    sf[:min(n, 4)] = np.arange(min(n, 4))
    return sf.astype(np.int32), nb.astype(np.int32)


def _gather_src(gs, x, form):
    F = x.shape[1]
    if form == "scalar":                        # a row pitch that is not a multiple of 4 floats: the scalar kernel
        pitch = F if F % 4 else F + 1
        t = torch.full((N_SRC, pitch), 7.0, dtype=torch.float32, device="cuda")
        t[:, :F] = dev(x)
        return t[:, :F], x
    t = torch.full((N_SRC, gs.ops.pad_cols(F)), 7.0, dtype=torch.float32, device="cuda")   # poisoned pad columns
    t[:, :F] = dev(x)
    if form == "bf16":
        return t.to(torch.bfloat16)[:, :F], nu.bf16_rne(x)
    return t[:, :F], x


def _expected(ref_table, calls, include_self, pitch):
    rows = max(r0 + n for (n, k, sf, nb, r0) in calls)
    F = ref_table.shape[1]
    xm = np.zeros((rows, pitch), np.float32)
    xs = np.zeros((rows, pitch), np.float32)
    for n, k, sf, nb, r0 in calls:
        if n == 0:
            continue
        s = nu.gather_clamped(ref_table, sf)
        xm[r0:r0 + n, :F] = nu.mean_f32(nu.gather_clamped(ref_table, nb), k, s, include_self)
        xs[r0:r0 + n, :F] = s
    return xs, xm


@pytest.mark.parametrize("F", [4, 7, 8, 50, 602, 1300])
@pytest.mark.parametrize("form", FORMS)
def test_gather_mean_bit_exact(gs, form, F):
    rs = np.random.RandomState(F)
    src, ref_table = _gather_src(gs, _special_table(rs, F), form)
    pitch = gs.ops.pad_cols(F)
    gs._lib.set_tuning("gather_variant", VARIANT[form])
    try:
        for spec in CALLS:
            total = sum(n for n, _ in spec)
            segs, calls, r0 = [], [], total
            for s, (n, k) in enumerate(spec):
                r0 -= n                                     # segment 0 writes the last rows
                sf, nb = _segment_ids(rs, n, k, s)
                segs.append(gs.ops.Seg(n, k, self_ids=dev(sf), neigh_ids=dev(nb), out_row0=r0))
                calls.append((n, k, sf, nb, r0))
            for include_self in (False, True):
                xs_ref, xm_ref = _expected(ref_table, calls, include_self, pitch)
                for want_self in (False, True):
                    xs, xm = gs.ops.gather_mean(src, segs, include_self=include_self, want_self=want_self)
                    assert nu.bits_equal(xm.cpu().numpy(), xm_ref), (form, F, spec, include_self, want_self)
                    if want_self:
                        assert nu.bits_equal(xs.cpu().numpy(), xs_ref), (form, F, spec, include_self)
                    else:
                        assert xs is None
        # rows addressed by ranges (no id lists); row ranges running past the table read its last row
        n, k = 37, 5
        segs = [gs.ops.Seg(n, k, self_row0=N_SRC - 20, neigh_row0=N_SRC - 150)]
        _, xm = gs.ops.gather_mean(src, segs, include_self=True, want_self=False)
        sf = np.arange(N_SRC - 20, N_SRC - 20 + n)
        nb = np.arange(N_SRC - 150, N_SRC - 150 + n * k)
        assert nu.bits_equal(xm.cpu().numpy(), _expected(ref_table, [(n, k, sf, nb, 0)], True, pitch)[1])
    finally:
        gs._lib.set_tuning("gather_variant", 2)


@pytest.mark.parametrize("F", [7, 50, 602])
def test_gather_mean_dropout_bit_exact(gs, F):
    """gs_gather_mean_dropout at p = 0.5: the masks of oracle.dropout, x / fp32(1 - p) on the kept elements, then the
    fp32 mean (F = 7 runs the scalar kernel, the others the bulk-copy one)."""
    rs = np.random.RandomState(100 + F)
    x = _special_table(rs, F)
    src = dev(x) if F == 7 else torch.zeros((N_SRC, gs.ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    if F != 7:
        src[:, :F] = dev(x)
        src = src[:, :F]
    pitch = gs.ops.pad_cols(F)
    spec = [(40, 25), (0, 13), (9, 10), (17, 1)]
    segs, calls, r0 = [], [], 0
    nsites, ssites = [], []
    for s, (n, k) in enumerate(spec):
        sf, nb = _segment_ids(rs, n, k, s)
        segs.append(gs.ops.Seg(n, k, self_ids=dev(sf), neigh_ids=dev(nb), out_row0=r0))
        calls.append((n, k, sf, nb, r0))
        nsites.append((77, 10 + 2 * s, 0.5))
        ssites.append((77, 11 + 2 * s, 0.5))
        r0 += n
    for include_self in (False, True):
        xs, xm = gs.ops.gather_mean_dropout(src, segs, nsites, ssites, include_self=include_self)
        xm_ref = np.zeros((r0, pitch), np.float32)
        xs_ref = np.zeros((r0, pitch), np.float32)
        for (n, k, sf, nb, o), ns, ss in zip(calls, nsites, ssites):
            if n == 0:
                continue
            srow = nu.gather_clamped(x, sf)
            xm_ref[o:o + n, :F] = nu.mean_f32(nu.gather_clamped(x, nb), k, srow, include_self, neigh_site=ns, self_site=ss)
            with np.errstate(over="ignore"):
                xs_ref[o:o + n, :F] = dropout.apply(srow, *ss)
        assert nu.bits_equal(xm.cpu().numpy(), xm_ref), (F, include_self)
        assert nu.bits_equal(xs.cpu().numpy(), xs_ref), (F, include_self)


# ---------------------------------------------------------------- K3: gs_sage_gemm in every math mode
GEMM_CASES = [
    # (M, [(K, N), ...], combine, bias, relu, A layout, out with extra columns)
    (1, [(1, 1)], "add", False, False, "dense", False),
    (63, [(4, 2)], "add", True, False, "padded", True),
    (64, [(7, 3)], "add", False, True, "odd", False),
    (65, [(31, 127)], "add", True, True, "offset", True),
    (127, [(32, 128)], "add", False, False, "padded", False),
    (128, [(33, 129)], "add", True, False, "odd", True),
    (129, [(63, 200)], "add", False, True, "offset", False),
    (257, [(64, 256)], "add", True, True, "dense", True),
    (129, [(65, 129), (65, 129)], "add", True, True, "padded", False),
    (257, [(602, 200), (640, 56)], "concat", True, False, "odd", True),      # part-0 N not a multiple of 128
    (65, [(33, 3), (7, 127)], "concat", True, True, "offset", False),
    (63, [(640, 1)], "add", True, False, "padded", True),
    (0, [(32, 128)], "add", True, False, "dense", False),
    (5632, [(602, 128), (602, 128)], "concat", False, True, "padded", False),  # configs[1] layer 0
    (512, [(256, 128), (256, 128)], "concat", False, False, "dense", False),   # configs[1] layer 1
]
# configs[2] (max-pool, --math bf16): the self and neighbour GEMMs of both layers
BF16_CASES = [
    (5632, [(602, 128), (512, 128)], "concat", False, True, "padded", False),
    (512, [(256, 128), (512, 128)], "concat", False, False, "dense", False),
]
MODES = {"fp32": "MATH_FP32_SIMT", "tf32x3": "MATH_TF32X3", "tf32": "MATH_TF32", "bf16": "MATH_BF16"}


def _a_operand(rs, M, K, layout):
    """A [M, K] fp32 as the layout asks; every other element of its storage is NaN, so a read past K shows."""
    a = rs.randn(M, K).astype(np.float32)
    if layout == "dense":
        return torch.empty((M, K), device="cuda").copy_(torch.from_numpy(a)), a
    if layout == "padded":                                # 16-byte-aligned rows, lda = pad_cols(K)
        store = torch.full((M, (K + 7) // 8 * 8), float("nan"), device="cuda")
        view = store[:, :K]
    elif layout == "odd":                                 # odd lda
        store = torch.full((M, K + 1 if K % 2 == 0 else K + 2), float("nan"), device="cuda")
        view = store[:, :K]
    else:                                                 # "offset": starts one column in -> not 16-byte aligned
        store = torch.full((M, (K + 8) // 8 * 8), float("nan"), device="cuda")
        view = store[:, 1:1 + K]
    view.copy_(dev(a))
    return view, a


def _run_gemm(gs, case, math):
    M, kn, combine, use_bias, relu, layout, wide_out = case
    rs = np.random.RandomState(M * 7 + sum(k for k, _ in kn))
    parts, np_parts = [], []
    for K, N in kn:
        A, a = _a_operand(rs, M, K, layout)
        B = (rs.randn(K, N) / np.sqrt(K)).astype(np.float32)
        parts.append((A, K, dev(B)))
        np_parts.append((a, B))
    ntot = sum(n for _, n in kn) if combine == "concat" else kn[0][1]
    bias = rs.randn(ntot).astype(np.float32) if use_bias else None
    kw = dict(combine=gs.ops.COMBINE_CONCAT if combine == "concat" else gs.ops.COMBINE_ADD,
              bias=None if bias is None else dev(bias), act=gs.ops.ACT_RELU if relu else gs.ops.ACT_NONE,
              math=getattr(gs.ops, MODES[math]))
    outs = []
    for packed in (None, gs.ops.PackedWeights()):
        if wide_out:                                      # ldo > ntot: the extra columns hold NaN and must stay so
            full = torch.full((M, ntot + 5), float("nan"), device="cuda")
            out = gs.ops.sage_gemm(parts, out=full[:, :ntot], packed=packed, **kw)
            assert out.stride(0) == ntot + 5
            extra = full[:, ntot:].cpu().numpy()
            assert np.array_equal(nu.f32_bits(extra), np.full(extra.shape, 0x7FC00000, np.uint32))
        else:
            out = gs.ops.sage_gemm(parts, packed=packed, **kw)
        assert tuple(out.shape) == (M, ntot)
        outs.append(out.cpu().numpy())
    torch.cuda.synchronize()
    assert nu.bits_equal(outs[0], outs[1]), "one-shot and prepacked results differ (%s, %r)" % (math, case)
    ref, S1, S2, Kc = nu.gemm_reference(np_parts, math, combine, bias, "relu" if relu else None)
    ok, worst, rms = nu.check_gemm(outs[1], ref, S1, S2, Kc)
    _note(math, worst, rms)
    assert ok, (math, case, worst, rms)


@pytest.mark.parametrize("math", list(MODES))
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: "M%d_%s_%s" % (c[0], "_".join("%dx%d" % kn for kn in c[1]), c[5]))
def test_sage_gemm_operand_exact(gs, case, math):
    _run_gemm(gs, case, math)


@pytest.mark.parametrize("case", BF16_CASES, ids=["layer0", "layer1"])
def test_sage_gemm_bf16_maxpool_shapes(gs, case):
    _run_gemm(gs, case, "bf16")


# ---------------------------------------------------------------- gs_sage_layer_small
# (path, output width) -> (n, k, F, kind, bias, out_row0); every nslices regime of both paths.  kind: gcn (one part, mean
# with the self row), mean1 (one part, neighbour mean), add / concat (self part + neighbour part).
LS_CASES = {
    ("vec", 4): (1, 1, 4, "gcn", True, 0),
    ("vec", 16): (3, 3, 256, "concat", False, 2),
    ("vec", 40): (4, 5, 2048, "concat", True, 0),
    ("vec", 128): (5, 6, 256, "add", True, 1),
    ("vec", 256): (301, 10, 256, "gcn", True, 0),
    ("vec", 500): (301, 5, 256, "concat", True, 7),
    ("vec", 512): (2048, 3, 4, "add", False, 0),
    ("vec", 1024): (5, 128, 2048, "concat", True, 0),
    ("scalar", 4): (2048, 6, 7, "mean1", True, 0),
    ("scalar", 16): (301, 10, 2048, "gcn", False, 3),
    ("scalar", 40): (5, 1, 50, "add", True, 0),
    ("scalar", 128): (4, 128, 602, "concat", True, 0),
    ("scalar", 256): (3, 3, 4, "concat", True, 1),
    ("scalar", 500): (301, 5, 602, "concat", True, 0),
    ("scalar", 512): (1, 10, 256, "add", False, 0),
    ("scalar", 1024): (5, 6, 50, "gcn", True, 2),
}


@pytest.mark.parametrize("key", list(LS_CASES), ids=lambda k: "%s_w%d" % k)
def test_sage_layer_small_operand_exact(gs, key):
    path, width = key
    n, k, F, kind, use_bias, out_row0 = LS_CASES[key]
    rs = np.random.RandomState(width + F + n)
    n_src = 300
    x = rs.randn(n_src, F).astype(np.float32)
    x[0] = 0.0                                                # the zero row: rows built from it come out all zero
    if path == "vec":
        assert F % 4 == 0
        store = torch.zeros((n_src, F), dtype=torch.float32, device="cuda")
        src = store
    else:                                                     # one column in: not 16-byte aligned -> the scalar path
        store = torch.full((n_src, F + 5), float("nan"), device="cuda")
        src = store[:, 1:1 + F]
    src.copy_(dev(x))
    sf = rs.randint(-2, n_src + 2, size=n).astype(np.int32)   # out-of-range ids read the last row
    nb = rs.randint(-2, n_src + 2, size=n * k).astype(np.int32)
    zero = [i for i in (0, n // 2) if i < n]
    sf[zero] = 0
    nb.reshape(n, k)[zero] = 0
    seg = gs.ops.Seg(n, k, self_ids=dev(sf), neigh_ids=dev(nb), out_row0=out_row0)
    if kind in ("add", "concat"):
        n0 = width // 2 // 4 * 4 if kind == "concat" else width
        widths = [n0, width - n0] if kind == "concat" else [width, width]
    else:
        widths = [width]
    Bs = [(rs.randn(F, w) / np.sqrt(F)).astype(np.float32) for w in widths]
    relu = kind != "add"
    # a negative bias: rows built from the zero row come out all zero after the ReLU
    bias = (-0.5 * np.abs(rs.randn(width)) - 0.05).astype(np.float32) if use_bias else None
    selfv = nu.gather_clamped(x, sf)
    mean = nu.mean_f32(nu.gather_clamped(x, nb), k, selfv, kind == "gcn")
    np_parts = [(selfv, Bs[0]), (mean, Bs[1])] if len(Bs) == 2 else [(mean, Bs[0])]
    combine = "concat" if kind == "concat" else "add"
    ref, S1, S2, Kc = nu.gemm_reference(np_parts, "fp32", combine, bias, "relu" if relu else None)
    for l2 in (False, True):
        out = gs.ops.sage_layer_small(src, seg, [(None, F, dev(B)) for B in Bs],
                                      combine=gs.ops.COMBINE_CONCAT if combine == "concat" else gs.ops.COMBINE_ADD,
                                      include_self=(kind == "gcn"), bias=None if bias is None else dev(bias),
                                      act=gs.ops.ACT_RELU if relu else gs.ops.ACT_NONE, l2_normalize=l2)
        got = out.cpu().numpy()[out_row0:out_row0 + n]
        if l2:
            ok, worst = nu.check_l2_normalized(got, ref, nu.gemm_bound(ref, S1, Kc))
            assert ok, (key, worst)
        else:
            ok, worst, rms = nu.check_gemm(got, ref, S1, S2, Kc)
            _note("layer_small", worst, rms)
            assert ok, (key, worst, rms)
        if relu:                                              # zero, not NaN, also after the l2-normalisation
            assert (got[zero] == 0).all()


# ---------------------------------------------------------------- gs_segment_max, gs_l2_normalize_rows
@pytest.mark.parametrize("n,k,C", [(2000, 1, 1), (1100, 2, 255), (300, 25, 256), (2000, 2, 257), (40, 128, 1024),
                                   (1500, 25, 1), (2000, 1, 1024), (90, 128, 257)])
def test_segment_max_exact(gs, n, k, C):
    rs = np.random.RandomState(n + k + C)
    x = rs.randn(n * k, C).astype(np.float32)
    x[rs.rand(n * k, C) < 0.2] = 0.0
    x[rs.rand(n * k, C) < 0.2] = -0.0
    x[rs.rand(n * k, C) < 0.01] = -np.inf
    x[: 3 * k] = -rs.rand(3 * k, C).astype(np.float32)            # rows whose max is negative
    store = torch.full((n * k, C + 3), float("nan"), device="cuda")  # ldx > C: the extra columns are never read
    store[:, :C] = dev(x)
    got = gs.ops.segment_max(store[:, :C], n, k).cpu().numpy()
    want = x.reshape(n, k, C).max(axis=1)
    assert np.array_equal(got, want)                              # by value: fmaxf(-0, +0) may return either zero
    nz = want != 0
    assert np.array_equal(nu.f32_bits(got)[nz], nu.f32_bits(want)[nz])


@pytest.mark.parametrize("n,C", [(9000, 1), (300, 31), (9000, 32), (257, 33), (2000, 256), (100, 1024)])
def test_l2_normalize_rows(gs, n, C):
    rs = np.random.RandomState(n + C)
    x = (rs.randn(n, C) * np.exp(rs.uniform(-8, 8, size=(n, 1)))).astype(np.float32)
    x[0] = 0.0
    x[1] = rs.randn(C).astype(np.float32) * 1e-9                 # sum of squares < 1e-12: scaled by 1 / sqrt(1e-12)
    x[2] = -0.0
    store = torch.full((n, C + 5), float("nan"), device="cuda")   # strided rows
    store[:, :C] = dev(x)
    v = store[:, :C]
    gs.ops.l2_normalize_rows_(v)
    got = v.cpu().numpy()
    assert nu.bits_equal(store[:, C:].cpu().numpy(), np.full((n, 5), np.nan, np.float32))
    x64 = x.astype(np.float64)
    ss = np.sum(x64 * x64, axis=1)
    big = ss >= 2e-12                                             # clear of the epsilon
    ref = x64[big] / np.sqrt(ss[big])[:, None]
    assert np.all(np.abs(got[big] - ref) <= (C + 2) * 2.0 ** -24 * np.abs(ref))
    tiny = ss < 0.5e-12
    inv = np.float32(1) / np.sqrt(np.float32(1e-12))
    assert nu.bits_equal(got[tiny], x[tiny] * inv)
    assert (got[0] == 0).all() and (got[2] == 0).all() and tiny[1]
