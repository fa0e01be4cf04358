"""CPU: sampled blocks over host-memory and int8 feature tables - the layer-0 loader's numpy restatement
(tests/host_gather_ref.py) on hand-made rows, and the refusals of the sampled-block entry points, which take these
tables while the whole-graph ones keep refusing them."""
import numpy as np
import pytest
import torch

from host_gather_ref import gather_rows_f32, link_rows, widen
from oracle import int8_rows


def _host(n=6, F=3, seed=0):
    t = np.random.RandomState(seed).randn(n + 1, 8).astype(np.float32)
    t[:, F:] = 0
    t[n] = 0
    return t


# ------------------------------------------------------------------ the loader's restatement
def test_rows_come_from_the_cache_the_host_or_the_zero_row():
    host = _host()
    cache = np.full((2, 8), 7.0, np.float32)            # cached rows differ from the host's: the rule picks the source
    cache[:, 3:] = 0
    cache[1, :3] = [1, 2, 3]
    slot = np.array([-1, 0, -1, -1, 1, -1, -1])          # ids 1 and 4 cached
    ids = [4, 0, 6, -1, 100, 1, 4, 0]                    # cached, host, dummy N, out of range, duplicates
    out = gather_rows_f32(host, cache, slot, ids, 3, "f32")
    assert out.shape == (8, 8) and out.dtype == np.float32
    assert out[0, :3].tolist() == [1, 2, 3] and out[5, :3].tolist() == [7, 7, 7]
    assert np.array_equal(out[1, :3], host[0, :3]) and np.array_equal(out[7], out[1])
    assert np.array_equal(out[6], out[0])
    assert not out[2:5].any() and not out[:, 3:].any()                # zero rows, zeroed pad columns
    assert link_rows(ids, slot, 6).tolist() == [0, 0]


def test_out_pitch_and_empty_lists():
    host = _host(F=5)
    slot = np.full(7, -1)
    assert gather_rows_f32(host, host[:0], slot, [], 5, "f32").shape == (0, 8)
    out = gather_rows_f32(host, host[:0], slot, [2, 3], 5, "f32", out_pitch=12)
    assert out.shape == (2, 12) and np.array_equal(out[:, :5], host[2:4, :5]) and not out[:, 5:].any()


def test_bf16_rows_widen_exactly():
    x = torch.from_numpy(_host(F=8)).to(torch.bfloat16)
    bits = x.view(torch.int16).numpy().view(np.uint16)
    slot = np.array([-1, -1, 0, -1, -1, -1, -1])
    out = gather_rows_f32(bits, bits[2:3], slot, [2, 5, 6], 8, "bf16")
    assert np.array_equal(out[:2], x[[2, 5]].to(torch.float32).numpy()) and not out[2].any()
    assert np.array_equal(widen(bits, 8, "bf16"), x.to(torch.float32).numpy())


@pytest.mark.parametrize("F", [1, 3, 16, 50])
def test_int8_rows_dequantise_with_their_own_scale(F):
    rs = np.random.RandomState(F)
    x = (rs.randn(9, F) * rs.uniform(0.01, 10, size=(9, 1))).astype(np.float32)
    x[8] = 0
    rows = int8_rows.quantize_rows(x)
    deq = int8_rows.dequantize(*int8_rows.quantize(x))
    cache = int8_rows.quantize_rows(x[[3, 5]] * np.float32(2))      # other bytes and other scales than the host's
    slot = np.full(9, -1)
    slot[[3, 5]] = [0, 1]
    ids = [0, 3, 5, 7, 8, 3, -4]
    out = gather_rows_f32(rows, cache, slot, ids, F, "i8row")
    cdeq = int8_rows.dequantize(*int8_rows.unpack(cache, F))
    assert np.array_equal(out[0, :F], deq[0]) and np.array_equal(out[3, :F], deq[7])
    assert np.array_equal(out[1, :F], cdeq[0]) and np.array_equal(out[2, :F], cdeq[1])
    assert np.array_equal(out[5], out[1]) and not out[4].any() and not out[6].any() and not out[:, F:].any()


# ------------------------------------------------------------------ refusals
def _fake_host(dtype=torch.float32):
    from graphsage_b200 import HostFeatures
    h = HostFeatures.__new__(HostFeatures)
    h.shape, h.dtype, h._alias = (11, 4), dtype, None
    return h


def _fake_int8():
    from graphsage_b200 import Int8Features, ops
    x = np.random.RandomState(0).randn(11, 4).astype(np.float32)
    x[10] = 0
    t = Int8Features.__new__(Int8Features)
    ops.I8Rows.__init__(t, torch.from_numpy(int8_rows.quantize_rows(x)), 4)
    return t


def _model(features, agg=None, **kw):
    import graphsage_b200 as gs

    class M(object):
        pass
    m = M()
    m.features, m.aggregator_cls, m.dropout_rate, m.distributed = features, agg or gs.MeanAggregator, 0., False
    for k, v in kw.items():
        setattr(m, k, v)
    return m


TABLES = [("host fp32", lambda: _fake_host(), "host-memory"), ("host bf16", lambda: _fake_host(torch.bfloat16),
                                                                 "host-memory"),
          ("host int8", lambda: _fake_host(torch.int8), "host-memory"), ("int8", _fake_int8, "int8")]


@pytest.mark.parametrize("name,make,word", TABLES, ids=[t[0] for t in TABLES])
def test_sampled_entry_points_take_host_and_int8_tables(name, make, word):
    from graphsage_b200.full_neighbor_training import refuse_full_neighbor, refuse_sampled
    m = _model(make())
    for training in (False, True):
        refuse_sampled(m, training)
        refuse_sampled(m, training, dropout=0.)
        with pytest.raises(NotImplementedError, match="full-neighbourhood %s .*with an? %s" % (
                "training" if training else "inference", word)):
            refuse_full_neighbor(m, training)
        with pytest.raises(NotImplementedError, match="full-neighbourhood .*%s" % word):
            refuse_full_neighbor(m, training, dropout=0.5)


def test_the_whole_graph_messages_are_unchanged():
    from graphsage_b200.full_neighbor_training import refuse_full_neighbor
    with pytest.raises(NotImplementedError) as e:
        refuse_full_neighbor(_model(_fake_host()), True)
    assert str(e.value) == ("full-neighbourhood training (it reads the whole table) with a host-memory (HostFeatures) "
                            "feature table is not implemented")
    with pytest.raises(NotImplementedError) as e:
        refuse_full_neighbor(_model(_fake_int8()), False)
    assert str(e.value) == "full-neighbourhood inference with an int8 (Int8Features) feature table is not implemented"


def test_dropout_on_sampled_blocks_host_yes_int8_no():
    from graphsage_b200.full_neighbor_training import refuse_sampled
    refuse_sampled(_model(_fake_host()), True, dropout=0.5)
    refuse_sampled(_model(_fake_host(torch.bfloat16)), True, dropout=0.5)
    for t in (_fake_int8(), _fake_host(torch.int8)):
        with pytest.raises(NotImplementedError, match="training dropout with a torch.int8 feature table"):
            refuse_sampled(_model(t), True, dropout=0.5)
        refuse_sampled(_model(t), False, dropout=0.5)          # inference draws no masks
    with pytest.raises(NotImplementedError, match="needs the rate passed explicitly"):
        refuse_sampled(_model(_fake_host(), dropout_rate=0.3), True)


@pytest.mark.parametrize("name,make,word", TABLES, ids=[t[0] for t in TABLES])
def test_what_stays_refused(name, make, word, monkeypatch):
    import graphsage_b200 as gs
    from graphsage_b200.full_neighbor_training import refuse_sampled
    t = make()
    for training in (False, True):
        with pytest.raises(NotImplementedError, match="seq aggregator"):
            refuse_sampled(_model(t, gs.SeqAggregator), training)
    with pytest.raises(NotImplementedError, match="twomaxpool"):
        refuse_sampled(_model(t, gs.TwoMaxLayerPoolingAggregator), True)
    refuse_sampled(_model(t, gs.TwoMaxLayerPoolingAggregator), False)
    with pytest.raises(NotImplementedError, match="distributed=True"):
        refuse_sampled(_model(t, distributed=True), True)

    class Sharded(object):
        c_table, shape, dtype = None, (11, 4), torch.float32
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        refuse_sampled(_model(Sharded()), False)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="cannot be captured in a CUDA graph"):
        refuse_sampled(_model(t), False)


def test_identity_features_stay_refused_with_these_tables():
    import graphsage_b200 as gs
    for t, word in ((_fake_host(), "host-memory"), (_fake_int8(), "int8")):
        with pytest.raises(NotImplementedError, match="identity_dim > 0 .*%s" % word):
            gs.SampleAndAggregate({}, t, np.zeros((11, 3), np.int32), None, [], identity_dim=4)
