"""CPU: the teacher-forced references of the LSTM recurrence kernels (oracle/seq.py: lstm_step_reference,
lstm_bptt_step_reference and the checks built on them, which tests/test_zz_gpu_seq_kernels.py applies to
gs_lstm_forward / gs_lstm_backward) and the evidence that the checks have teeth: a numpy fp32 emulation of both kernels,
in their order of evaluation, passes them, and each mutant below (a subtly wrong kernel) fails them."""
import numpy as np
import pytest

from oracle import seq as oseq

f32 = np.float32
S128 = 32                          # sequences per CTA tile at H = 128 (csrc/lstm.cu SeqTile)


def _sigmoid32(x):
    with np.errstate(over="ignore"):
        return f32(1) / (f32(1) + np.exp(-x))


def _fma_chain(acc, a, b):
    """acc (fp32) + sum_m a[:, m] b[m] as the kernels' fmaf chain, m ascending: each product is exact in float64 and
    each step is rounded once to fp32 (a double rounding via float64 that is within the bound's 1 u per step)."""
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    for m in range(a.shape[1]):
        acc = (acc.astype(np.float64) + a64[:, m, None] * b64[m]).astype(f32)
    return acc


def _tile_lengths(lengths, k, S, mutant):
    L = np.clip(np.asarray(lengths, np.int64), 0, k)
    if mutant == "neighbour_tile_length":          # sequence S + 3 runs with the length of sequence 3 (tile 0)
        L = L.copy()
        L[S + 3] = L[3]
    return L


def emulate_forward(P, Wh, lengths, mutant=None):
    """lstm_forward_kernel in fp32: (h_last, gates, c, h_prev), P [n, k, 4H]."""
    P, Wh = P.astype(f32), Wh.astype(f32)
    n, k, G = P.shape
    H = G // 4
    L = _tile_lengths(lengths, k, S128, mutant)
    h, c = np.zeros((n, H), f32), np.zeros((n, H), f32)
    gates, cs, hp = np.zeros((n, k, G), f32), np.zeros((n, k, H), f32), np.zeros((n, k, H), f32)
    W = Wh[:-1] if mutant == "drop_wh_term" else Wh  # the last m of the last unrolled block is skipped
    for t in range(k):
        on = (t < L)[:, None]
        acc = np.where(on, P[:, t], f32(0))
        acc = _fma_chain(acc, h[:, :W.shape[0]], W)
        zf = acc[:, 2 * H:3 * H] if (mutant == "forget_bias_skipped" and t == 1) else acc[:, 2 * H:3 * H] + f32(1)
        ig, jg, fg, og = _sigmoid32(acc[:, :H]), np.tanh(acc[:, H:2 * H]), _sigmoid32(zf), _sigmoid32(acc[:, 3 * H:])
        cn = c * fg + ig * jg
        hn = np.tanh(cn) * og
        gates[:, t] = np.where(on, np.concatenate([ig, jg, fg, og], axis=1), f32(0))
        cs[:, t] = np.where(on, cn, f32(0))
        hp[:, t] = np.where(on, h, f32(0))
        c, h = np.where(on, cn, c), np.where(on, hn, h)
    return h, gates, cs, hp


def emulate_backward(dh_last, gates, cs, lengths, Wh, mutant=None):
    """lstm_backward_kernel in fp32: dZ [n, k, 4H]."""
    gates, cs, Wh, dh_last = gates.astype(f32), cs.astype(f32), Wh.astype(f32), dh_last.astype(f32)
    n, k, G = gates.shape
    H = G // 4
    L = _tile_lengths(lengths, k, S128, mutant)
    last_at = L - 2 if mutant == "dh_last_off_by_one" else L - 1
    back = 2 if mutant == "cp_two_back" else 1
    dZ = np.zeros((n, k, G), f32)
    dh, dc = np.zeros((n, H), f32), np.zeros((n, H), f32)
    one = f32(1)
    for t in range(k - 1, -1, -1):
        on = (t < L)[:, None]
        ig, jg, fg, og = (gates[:, t, g * H:(g + 1) * H] for g in range(4))
        ct = cs[:, t]
        cp = cs[:, t - back] if t >= back else np.zeros((n, H), f32)
        d = dh + np.where((t == last_at)[:, None], dh_last, f32(0))
        tc = np.tanh(ct)
        zo = d * tc * og * (one - og)
        dct = dc + d * og * (one - tc * tc)
        z = np.concatenate([dct * jg * ig * (one - ig), dct * ig * (one - jg * jg), dct * cp * fg * (one - fg), zo], axis=1)
        z = np.where(on, z, f32(0))
        dZ[:, t] = z
        dc = np.where(on, dct * fg, dc)
        dh = _fma_chain(np.zeros((n, H), f32), z, Wh.T)
    return dZ


def _case(n=70, k=25, H=128, seed=0, saturate=False):
    """Inputs at the kernels' scale: W_h glorot for K = 50, P ~ 0.8 N(0, 1) (with saturate, every third unit's four
    gate columns scaled by 60, so |z| reaches 30 - 100+), lengths with a ragged last tile, one tile shorter than k, a
    length above k and one of 0."""
    rs = np.random.RandomState(seed)
    r = np.sqrt(6.0 / (50 + 5 * H))
    Wh = rs.uniform(-r, r, size=(H, 4 * H)).astype(f32)
    P = (rs.randn(n, k, 4 * H) * 0.8).astype(f32)
    if saturate:
        P.reshape(n, k, 4, H)[..., ::3] *= 60
    lengths = rs.randint(1, k + 1, size=n).astype(np.int32)
    lengths[S128:2 * S128] = np.minimum(lengths[S128:2 * S128], max(k - 3, 1))   # tile 1 ends before k (when k > 3)
    lengths[:6] = [k, 1, k + 5, 1, 0, max(k // 2, 1)]
    lengths[S128 + 3] = max(k - 3, 1)                                           # differs from sequence 3's length 1
    dh = rs.randn(n, H).astype(f32)
    return P, Wh, lengths, dh


def test_references_reproduce_the_fp64_oracle_on_its_own_trajectory():
    """Fed the float64 trajectory of lstm_run / lstm_bptt, the teacher-forced references give that trajectory back."""
    rs = np.random.RandomState(5)
    n, k, H = 7, 5, 8
    P, Wh = rs.randn(n, k, 4 * H), rs.randn(H, 4 * H) * 0.3
    lengths = np.array([5, 1, 3, 2, 9, 0, 4], np.int32)
    h, gates, cs, hp = oseq.lstm_run(P, Wh, lengths, train=True, dtype=np.float64)
    c_prev = np.concatenate([np.zeros((n, 1, H)), cs[:, :-1]], axis=1)
    r = oseq.lstm_step_reference(P, Wh, hp, c_prev, lengths)
    np.testing.assert_allclose(r["gates"][0], gates, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(r["c"][0], cs, rtol=1e-13, atol=1e-15)
    saved = lengths[:, None] > np.arange(1, k)                      # h_t is saved as h_prev[t + 1] while t + 1 < len
    np.testing.assert_allclose(r["h"][0][:, :-1][saved], hp[:, 1:][saved], rtol=1e-13, atol=1e-15)
    dh = rs.randn(n, H)
    dZ = oseq.lstm_bptt(dh, gates, cs, np.clip(lengths, 0, k), Wh)
    ref, bound = oseq.lstm_bptt_step_reference(dh, gates, cs, lengths, Wh, dZ)
    np.testing.assert_allclose(ref, dZ, rtol=1e-12, atol=1e-14)
    assert not ref[5].any() and not bound[5].any()                  # len 0: nothing runs
    assert np.all(bound[lengths[:, None] > np.arange(k)] > 0)


@pytest.mark.parametrize("k,saturate", [(1, False), (2, False), (25, False), (128, False), (25, True)])
def test_checks_accept_the_emulated_kernels(k, saturate):
    P, Wh, lengths, dh = _case(n=70 if k < 128 else 40, k=k, saturate=saturate)
    h, g, c, hp = emulate_forward(P, Wh, lengths)
    ok, worst = oseq.check_lstm_forward(P, Wh, lengths, h, g, c, hp)
    assert ok, worst
    dZ = emulate_backward(dh, g, c, lengths, Wh)
    ok, wb = oseq.check_lstm_backward(dh, g, c, lengths, Wh, dZ)
    assert ok, wb
    if saturate:                                                    # gates at exactly 0 / 1 / +-1 zero their dZ
        sat = oseq.saturated(g) & (np.arange(k)[None, :, None] < np.clip(lengths, 0, k)[:, None, None])
        assert sat.mean() > 0.05 and not dZ[sat].any()
    print("k=%d saturate=%s worst ratios: forward %s, backward %.3f" % (k, saturate, worst, wb))


FORWARD_MUTANTS = ["drop_wh_term", "forget_bias_skipped", "neighbour_tile_length"]
BACKWARD_MUTANTS = ["cp_two_back", "dh_last_off_by_one", "neighbour_tile_length"]


@pytest.mark.parametrize("mutant", FORWARD_MUTANTS)
def test_forward_check_rejects_each_mutant(mutant):
    P, Wh, lengths, _ = _case()
    ok, worst = oseq.check_lstm_forward(P, Wh, lengths, *emulate_forward(P, Wh, lengths, mutant=mutant))
    assert not ok, (mutant, worst)


@pytest.mark.parametrize("mutant", BACKWARD_MUTANTS)
def test_backward_check_rejects_each_mutant(mutant):
    P, Wh, lengths, dh = _case()
    _, g, c, _ = emulate_forward(P, Wh, lengths)
    ok, worst = oseq.check_lstm_backward(dh, g, c, lengths, Wh, emulate_backward(dh, g, c, lengths, Wh, mutant=mutant))
    assert not ok, (mutant, worst)


def test_bound_ratio_requires_exact_zeros_where_the_bound_is_zero():
    ref, bound = np.zeros(3), np.array([0.0, 1e-7, 0.0])
    assert oseq.bound_ratio(np.array([0.0, 5e-8, -0.0]), ref, bound) == 0.5
    assert oseq.bound_ratio(np.array([1e-45, 0.0, 0.0]), ref, bound) == np.inf
    assert oseq.bound_ratio(np.array([0.0, np.nan, 0.0]), ref, bound) == np.inf
