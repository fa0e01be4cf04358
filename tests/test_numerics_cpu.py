"""CPU: oracle/numerics.py - the operand-exact references the GPU file tests/test_zz_gpu_numerics.py compares the
aggregation kernels with - and the evidence that its checks have teeth: a numpy emulation of each kernel passes them,
and each mutant below (a subtly wrong kernel) fails them at the shapes the GPU file uses."""
import numpy as np
import pytest
import torch

from oracle import numerics as nu


# ---------------------------------------------------------------- operand rounding
def _special_f32():
    """+-0, subnormals, the smallest / largest normals, +-inf, and values at and next to the bf16 halfway points."""
    vals = [0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.17549435e-38, 3.4028235e38, -3.4028235e38, np.inf, -np.inf, 1.0, -1.5]
    bits = [np.float32(v).view(np.uint32) for v in vals]
    for base in (0x3F800000, 0x3F810000, 0xBF830000, 0x00010000, 0x7F7F0000, 0x00000000):
        for low in (0x7FFF, 0x8000, 0x8001, 0xFFFF, 0x0001):      # below, at, above the halfway point; odd / even kept bit
            bits.append(np.uint32(base | low))
    rs = np.random.RandomState(0)
    bits.extend(rs.randint(0, 2 ** 32, size=20000, dtype=np.uint64).astype(np.uint32))
    b = np.array(bits, dtype=np.uint32)
    b = b[(b & 0x7FFFFFFF) <= 0x7F800000]                          # no NaN: out of scope
    return b.view(np.float32)


def test_bf16_rne_equals_torch_bit_for_bit():
    x = _special_f32()
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).to(torch.float32).numpy()
    assert nu.bits_equal(nu.bf16_rne(x), want)
    assert nu.bits_equal(nu.bf16_widen(torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)),
                         want)


def test_tf32_truncation_and_split():
    x = _special_f32()
    x = x[np.isfinite(x)]
    t = nu.tf32_trunc(x)
    assert np.array_equal(t.view(np.uint32), x.view(np.uint32) & 0xFFFFE000)
    hi, lo = nu.tf32x3_split(x)
    assert np.array_equal(hi.view(np.uint32) & 0x1FFF, np.zeros_like(hi.view(np.uint32)))
    assert np.array_equal(lo.view(np.uint32) & 0x1FFF, np.zeros_like(lo.view(np.uint32)))
    # x - hi is the 13 low mantissa bits; lo keeps the leading 11 of them, so hi + lo is within 2^-21 |x| while lo stays
    # normal (near the subnormal range lo loses more)
    x = x[np.abs(x) >= 2.0 ** -100]
    hi, lo = nu.tf32x3_split(x)
    r = np.abs(hi.astype(np.float64) + lo.astype(np.float64) - x.astype(np.float64)) / np.abs(x.astype(np.float64))
    assert np.all(r < 2.0 ** -21) and r.max() > 2.0 ** -22


def test_mean_f32_against_float64():
    rs = np.random.RandomState(1)
    for k, inc in ((1, False), (5, True), (25, False), (128, True)):
        rows = rs.randn(300 * k, 50).astype(np.float32)
        selfv = rs.randn(300, 50).astype(np.float32)
        m = nu.mean_f32(rows, k, selfv, inc)
        r64 = rows.astype(np.float64).reshape(300, k, 50)
        s = r64.sum(1) + (selfv if inc else 0)
        absum = np.abs(r64).sum(1) + (np.abs(selfv) if inc else 0)
        d = k + inc
        ref = s / d
        # k + inc - 1 additions and one division, each within 2^-24 relative
        assert np.all(np.abs(m - ref) <= (d * 2.0 ** -24 * absum) / d + 2.0 ** -24 * np.abs(ref))
        assert m.dtype == np.float32


def test_gather_clamped_reads_the_last_row():
    t = np.arange(12, dtype=np.float32).reshape(4, 3)
    np.testing.assert_array_equal(nu.gather_clamped(t, [-1, 0, 3, 4, 99]), t[[3, 0, 3, 3, 3]])


# ---------------------------------------------------------------- emulation of the kernels and their mutants
def _accumulate(acc, a, b, rounding="rne"):
    """acc (fp32) += a @ b, the products of the step summed exactly and rounded once to fp32 (one MMA step)."""
    return _to_f32(acc.astype(np.float64) + a.astype(np.float64) @ b.astype(np.float64), rounding)


def _trunc_bf16(x):
    return (nu._f32(x).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def _to_f32(x64, rounding):
    """float64 -> fp32, to nearest ("rne") or toward zero ("rz", how the H100's tensor cores accumulate)."""
    f = x64.astype(np.float32)
    if rounding == "rz":
        over = np.abs(f.astype(np.float64)) > np.abs(x64)
        f[over] = np.nextafter(f[over], np.float32(0))
    return f


def emulate_k3(parts, math, combine="add", bias=None, act=None, mutant=None, rounding="rz"):
    """fp32: one FMA per k, rounded to nearest.  Tensor-core modes: one k8 (tf32) / k16 (bf16) step at a time into an
    fp32 accumulator (`rounding`); tf32x3 runs hi*hi, hi*lo, lo*hi per step.  K-blocks are 32 (tf32 modes) / 64 (bf16)
    wide."""
    step = 1 if math == "fp32" else 16 if math == "bf16" else 8
    bk = 64 if math == "bf16" else 32
    outs = []
    for pi, (A, B) in enumerate(parts):
        K = A.shape[1]
        if math == "bf16":
            a = _trunc_bf16(A) if mutant == "bf16_a_trunc" else nu.bf16_rne(A)
            b = _trunc_bf16(B) if mutant == "bf16_b_trunc" else nu.bf16_rne(B)
            terms = [(a, b)]
        elif math == "tf32x3":
            (ah, al), (bh, bl) = nu.tf32x3_split(A), nu.tf32x3_split(B)
            terms = [(ah, bh)] if mutant == "tf32x3_no_lo" else [(ah, bh), (ah, bl), (al, bh)]
        else:
            terms = [(nu.operands(A, math)[0], nu.operands(B, math)[0])]
        kend = K
        if mutant == "drop_partial_kblock" and pi == 0 and K % bk:
            kend = K - K % bk
        last_block = (K - 1) // bk * bk
        acc = np.zeros((A.shape[0], B.shape[1]), dtype=np.float32)
        for k0 in range(0, kend, step):
            k1 = min(k0 + step, kend)
            for t, (a, b) in enumerate(terms):
                if mutant == "tf32x3_no_lo_hi_last_block" and t == 2 and k0 >= last_block:
                    continue
                acc = _accumulate(acc, a[:, k0:k1], b[k0:k1], "rne" if math == "fp32" else rounding)
        outs.append(acc)
    if combine == "concat":
        out = np.concatenate(outs, axis=1)
    else:
        out = outs[0]
        for o in outs[1:]:
            out = out + o
    if bias is not None:
        b = nu._f32(bias)
        if mutant == "bias_wrong_half":
            n0 = parts[0][1].shape[1]
            b = np.concatenate([b[:n0], b[:out.shape[1] - n0]])
        out = out + b
    if act == "relu":
        out = np.maximum(out, np.float32(0))
    return out


def emulate_mean(rows, k, self_rows, include_self, mutant=None):
    """The gather kernels' mean: neighbour rows in groups (gather_mean_tma2_kernel's 13-row groups), fp32, j order."""
    rows = nu._f32(rows).reshape(-1, k, rows.shape[-1])
    acc = np.zeros((rows.shape[0], rows.shape[2]), dtype=np.float32)
    if mutant == "pairwise":
        level = [rows[:, j] for j in range(k)]
        while len(level) > 1:
            level = [level[i] + level[i + 1] if i + 1 < len(level) else level[i] for i in range(0, len(level), 2)]
        acc = acc + level[0]
    else:
        for g in range(0, k, 13):
            for j in range(g, min(g + 13, k)):
                acc = acc + rows[:, j]
    if include_self or mutant == "self_when_excluded":
        acc = acc + self_rows
    div = np.float32(k + (1 if include_self else 0))
    if mutant == "reciprocal":
        return acc * (np.float32(1) / div)
    return acc / div


# the GEMM shapes of the GPU file this table runs at: (M, [(K, N), ...], combine, bias, act)
GEMM_SHAPES = [
    (257, [(602, 200), (640, 56)], "concat", True, None),
    (129, [(65, 129), (65, 129)], "add", True, "relu"),
    (512, [(256, 128), (512, 128)], "concat", False, None),
]

GEMM_MUTANTS = [
    ("bf16_a_trunc", "bf16"),
    ("bf16_b_trunc", "bf16"),
    ("tf32x3_no_lo_hi_last_block", "tf32x3"),
    ("tf32x3_no_lo", "tf32x3"),
    ("drop_partial_kblock", "tf32x3"),
    ("drop_partial_kblock", "tf32"),
    ("drop_partial_kblock", "bf16"),
    ("bias_wrong_half", "fp32"),
    ("bias_wrong_half", "tf32x3"),
]


def _gemm_case(shape, seed=0):
    M, kn, combine, use_bias, act = shape
    rs = np.random.RandomState(seed + M)
    parts = [(rs.randn(M, K).astype(np.float32), (rs.randn(K, N) / np.sqrt(K)).astype(np.float32)) for K, N in kn]
    ntot = sum(n for _, n in kn) if combine == "concat" else kn[0][1]
    bias = rs.randn(ntot).astype(np.float32) if use_bias else None
    return parts, combine, bias, act


@pytest.mark.parametrize("rounding", ["rne", "rz"])
@pytest.mark.parametrize("math", nu.MATHS)
@pytest.mark.parametrize("shape", GEMM_SHAPES)
def test_check_gemm_accepts_the_emulated_kernel(math, shape, rounding):
    parts, combine, bias, act = _gemm_case(shape)
    out = emulate_k3(parts, math, combine, bias, act, rounding=rounding)
    ok, worst, rms = nu.check_gemm(out, *nu.gemm_reference(parts, math, combine, bias, act))
    assert ok and worst < 0.1, (worst, rms)
    if rounding == "rne":
        assert rms < nu.RMS_BOUND / 16


@pytest.mark.parametrize("mutant,math", GEMM_MUTANTS)
@pytest.mark.parametrize("shape", GEMM_SHAPES)
def test_check_gemm_rejects_each_mutant(mutant, math, shape):
    parts, combine, bias, act = _gemm_case(shape)
    if mutant == "bias_wrong_half" and (combine != "concat" or bias is None):
        pytest.skip("needs a biased concat")
    if mutant == "drop_partial_kblock" and parts[0][0].shape[1] % (64 if math == "bf16" else 32) == 0:
        pytest.skip("part 0 has no partial K-block")
    out = emulate_k3(parts, math, combine, bias, act, mutant=mutant)
    ok, worst, rms = nu.check_gemm(out, *nu.gemm_reference(parts, math, combine, bias, act))
    assert not ok, (mutant, math, worst, rms)


def test_the_rms_criterion_is_what_catches_the_dropped_product():
    """A tf32x3 kernel that skips A_lo * B_hi in its last K-block stays inside the worst-case bound: (b) is needed."""
    parts, combine, bias, act = _gemm_case(GEMM_SHAPES[0])
    out = emulate_k3(parts, "tf32x3", combine, bias, act, mutant="tf32x3_no_lo_hi_last_block")
    worst, rms = nu.gemm_errors(out, *nu.gemm_reference(parts, "tf32x3", combine, bias, act))
    assert worst <= 1.0 and rms > 4 * nu.RMS_BOUND


MEAN_MUTANTS = ["reciprocal", "pairwise", "self_when_excluded"]


@pytest.mark.parametrize("k", [1, 2, 5, 7, 25, 64, 128])
@pytest.mark.parametrize("include_self", [False, True])
def test_mean_emulation_is_bit_exact(k, include_self):
    rs = np.random.RandomState(k)
    rows, selfv = rs.randn(200 * k, 602).astype(np.float32), rs.randn(200, 602).astype(np.float32)
    assert nu.bits_equal(emulate_mean(rows, k, selfv, include_self), nu.mean_f32(rows, k, selfv, include_self))


@pytest.mark.parametrize("mutant", MEAN_MUTANTS)
@pytest.mark.parametrize("k", [5, 7, 25])           # the reciprocal of a power of two is exact: k = 64, 128 cannot tell
def test_bit_exact_mean_check_rejects_each_mutant(mutant, k):
    rs = np.random.RandomState(k)
    rows, selfv = rs.randn(200 * k, 602).astype(np.float32), rs.randn(200, 602).astype(np.float32)
    got = emulate_mean(rows, k, selfv, False, mutant=mutant)
    assert not nu.bits_equal(got, nu.mean_f32(rows, k, selfv, False))
    # ... which a 1e-5 relative comparison with float64 lets through, except for the self row
    if mutant != "self_when_excluded":
        ref = rows.astype(np.float64).reshape(200, k, 602).mean(1)
        assert np.max(np.abs(got - ref)) / np.max(np.abs(ref)) < 1e-5


def test_mean_f32_dropout_matches_the_dropout_oracle():
    from oracle import dropout
    rs = np.random.RandomState(4)
    n, k, F = 50, 7, 13
    rows, selfv = rs.randn(n * k, F).astype(np.float32), rs.randn(n, F).astype(np.float32)
    ns, ss = (5, 2, 0.5), (5, 3, 0.5)
    got = nu.mean_f32(rows, k, selfv, True, neigh_site=ns, self_site=ss)
    nb = dropout.apply(rows, *ns).reshape(n, k, F)
    acc = np.zeros((n, F), np.float32)
    for j in range(k):
        acc = acc + nb[:, j]
    acc = acc + dropout.apply(selfv, *ss)
    assert nu.bits_equal(got, acc / np.float32(k + 1))
    assert 0.3 < float(np.mean(nb == 0)) < 0.7


def test_l2_check_accepts_fp32_normalisation_and_rejects_a_missing_epsilon_or_relu():
    parts, combine, bias, act = _gemm_case((129, [(65, 129), (65, 129)], "add", True, "relu"))
    v = emulate_k3(parts, "fp32", combine, bias, act)
    v[:3] = 0                                                 # rows that come out all zero
    ref, S1, S2, K = nu.gemm_reference(parts, "fp32", combine, bias, act)
    ref[:3] = 0
    bound = nu.gemm_bound(ref, S1, K)
    ss = np.zeros(v.shape[0], np.float32)
    for c in range(v.shape[1]):
        ss = ss + v[:, c] * v[:, c]
    out = v * (np.float32(1) / np.sqrt(np.maximum(ss, np.float32(1e-12))))[:, None]
    assert nu.check_l2_normalized(out, ref, bound)[0]
    with np.errstate(invalid="ignore", divide="ignore"):
        no_eps = v * (np.float32(1) / np.sqrt(ss))[:, None]
    assert not nu.check_l2_normalized(no_eps, ref, bound)[0]
    pre = emulate_k3(parts, "fp32", combine, bias, None)
    pss = np.sum(pre.astype(np.float64) ** 2, axis=1)
    assert not nu.check_l2_normalized((pre / np.sqrt(pss)[:, None]).astype(np.float32), ref, bound)[0]
