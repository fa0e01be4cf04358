"""CPU: the int8 row format (oracle/int8_rows.py) on hand-computed rows, its byte layout and error bound, Int8Features'
argument checks, and the refusals that need no device."""
import numpy as np
import pytest
import torch

from oracle import int8_rows


def _f32(*v):
    return np.array([v], dtype=np.float32)


def test_hand_computed_rows():
    # s = 127 / 127 = 1: q = rint(x), ties to even
    q, s = int8_rows.quantize(_f32(0.5, 1.5, 2.5, -0.5, -1.5, 127.0))
    assert s[0] == 1 and q.tolist() == [[0, 2, 2, 0, -2, 127]]
    # all-zero row: s = 0, every q = 0
    q, s = int8_rows.quantize(np.zeros((1, 5), np.float32))
    assert s[0] == 0 and not q.any()
    # a single non-zero value: it maps to +-127 and comes back as fl(127 * s)
    q, s = int8_rows.quantize(_f32(0, 0, -3.0, 0))
    assert q.tolist() == [[0, 0, -127, 0]] and s[0] == np.float32(3.0) / np.float32(127)
    assert int8_rows.dequantize(q, s)[0, 2] == np.float32(-127) * s[0]
    # negative absmax: the scale is positive
    q, s = int8_rows.quantize(_f32(-254.0, 127.0, 1.0))
    assert s[0] == 2 and q.tolist() == [[-127, 64, 0]]           # 63.5 -> 64 (even), 0.5 -> 0
    # values a hair past 127 * s (s rounded down) clamp at +-127
    a = np.float32(1.0000001)
    q, s = int8_rows.quantize(_f32(a, -a, 0.25))
    assert np.abs(q).max() == 127 and q[0, 0] == 127 and q[0, 1] == -127


@pytest.mark.parametrize("F", [1, 3, 4, 5, 602, 1536])
def test_layout_and_padding(F):
    rs = np.random.RandomState(F)
    x = rs.randn(7, F).astype(np.float32)
    x[3] = 0
    rows = int8_rows.quantize_rows(x)
    p4 = (F + 3) // 4 * 4
    assert rows.shape == (7, int8_rows.pitch(F)) and rows.shape[1] % 16 == 0 and rows.shape[1] >= p4 + 4
    assert not rows[:, F:p4].any() and not rows[:, p4 + 4:].any()
    q, s = int8_rows.quantize(x)
    assert np.array_equal(rows[:, :F].view(np.int8), q)
    assert np.array_equal(rows[:, p4:p4 + 4].copy().view("<f4").reshape(-1), s)
    assert not rows[3].any()                                        # the zero (dummy) row is all zero bytes
    q2, s2 = int8_rows.unpack(rows, F)
    assert np.array_equal(q2, q) and np.array_equal(s2, s)


def test_pitch_matches_the_package():
    from graphsage_b200 import ops
    for F in list(range(1, 70)) + [602, 1536]:
        assert ops.i8row_pitch(F) == int8_rows.pitch(F)


def test_error_bound_on_random_rows():
    rs = np.random.RandomState(0)
    x = (rs.randn(500, 64) * rs.lognormal(0, 3, size=(500, 1))).astype(np.float32)
    q, s = int8_rows.quantize(x)
    deq = int8_rows.dequantize(q, s)
    bound = s[:, None] / 2 + np.spacing(np.abs(deq)) + np.spacing(s[:, None] * 127)
    assert (np.abs(x.astype(np.float64) - deq) <= bound).all()
    assert (np.abs(q) <= 127).all() and (np.abs(q).max(axis=1) == 127).all()


def test_oracle_refuses_non_finite():
    for bad in (np.inf, -np.inf, np.nan):
        with pytest.raises(ValueError, match="non-finite"):
            int8_rows.quantize(_f32(1.0, bad))


@pytest.mark.parametrize("bad,err,match", [
    (np.array([1.0, 0.0], np.float32), ValueError, "2-D"),
    (np.zeros((3, 0), np.float32), ValueError, "F >= 1"),
    (np.zeros((3, 2), np.int32), TypeError, "floating-point"),
    (np.array([[1.0, np.nan], [0.0, 0.0]], np.float32), ValueError, "non-finite"),
    (np.array([[1.0, np.inf], [0.0, 0.0]], np.float32), ValueError, "non-finite"),
    (np.array([[1.0, 2.0], [0.0, 1.0]], np.float32), ValueError, "dummy row"),
])
def test_argument_checks(bad, err, match):
    from graphsage_b200 import Int8Features
    with pytest.raises(err, match=match):
        Int8Features(bad)


def test_an_integer_tensor_is_still_not_a_table():
    from graphsage_b200 import ops
    with pytest.raises(TypeError, match="float32 or bfloat16"):
        ops._dtype_code(torch.zeros((2, 2), dtype=torch.int8))


# ------------------------------------------------------------------ refusals that need no device
def _fake_int8(F=4, n=10):
    """An Int8Features over oracle-made host rows (no device needed: the refusals look at the type and dtype)."""
    from graphsage_b200 import Int8Features, ops
    x = np.random.RandomState(0).randn(n + 1, F).astype(np.float32)
    x[n] = 0
    t = Int8Features.__new__(Int8Features)
    ops.I8Rows.__init__(t, torch.from_numpy(int8_rows.quantize_rows(x)), F)
    return t


def test_fake_table_looks_like_a_table():
    t = _fake_int8()
    assert t.shape == (11, 4) and t.dtype == torch.int8 and t.pitch == 16 and t.device.type == "cpu"
    assert np.array_equal(t.dequantize().numpy(), int8_rows.dequantize(*int8_rows.unpack(t.rows.numpy(), 4)))


def test_refusals_without_a_device():
    import graphsage_b200 as gs
    from graphsage_b200.aggregators import refuse_seq_table
    from graphsage_b200.full_neighbor_training import refuse_full_neighbor
    from graphsage_b200.supervised_models import refuse_dropout_table, refuse_fused_pool
    t = _fake_int8()
    with pytest.raises(NotImplementedError, match="identity_dim > 0 with an int8"):
        gs.SampleAndAggregate({}, t, np.zeros((11, 3), np.int32), None, [], identity_dim=4)
    for cls, args in ((gs.SupervisedGraphsage, (3, {})), (gs.UnsupervisedGraphsage, ({},))):
        with pytest.raises(NotImplementedError, match="distributed=True with an int8"):
            cls(*args, t, None, np.ones(10), [], distributed=True)
    with pytest.raises(NotImplementedError, match="seq aggregator with a torch.int8"):
        refuse_seq_table(t)
    with pytest.raises(NotImplementedError, match="training dropout with a torch.int8"):
        refuse_dropout_table(t)

    class M(object):
        features, aggregator_cls, fused_pool, aggregators = t, gs.MeanAggregator, True, [gs.MaxPoolingAggregator.__new__(
            gs.MaxPoolingAggregator)]
    M.aggregators[0].mlp_layers = []
    with pytest.raises(NotImplementedError, match="fused_pool=True with an int8"):
        refuse_fused_pool(M())
    for training in (False, True):
        with pytest.raises(NotImplementedError, match="full-neighbourhood .* with an int8"):
            refuse_full_neighbor(M(), training)
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        gs.parallel.ShardedFeatures(t, 10)
    with pytest.raises(ValueError, match="HostFeatures"):
        gs.SampleAndAggregate({}, t, np.zeros((11, 3), np.int32), None, [])
