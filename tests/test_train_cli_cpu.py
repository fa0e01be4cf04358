"""CPU: the trainers' host side (graphsage_b200.supervised_train / unsupervised_train / train_cli) - flags, log
directories, F1 against sklearn, the stats-file formats, the epoch loop's schedule against a restatement of the
reference's loop, and the --model branches built on the CPU."""
import types

import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import supervised_train as sup, train_cli, unsupervised_train as unsup

# the reference's DEFINE_* lines (supervised_train.py:28-57, unsupervised_train.py:25-55): name -> (kind, default)
SUP_FLAGS = {
    "log_device_placement": ("boolean", False), "model": ("string", "graphsage_mean"), "learning_rate": ("float", 0.01),
    "model_size": ("string", "small"), "train_prefix": ("string", ""), "epochs": ("integer", 10),
    "dropout": ("float", 0.0), "weight_decay": ("float", 0.0), "max_degree": ("integer", 128),
    "samples_1": ("integer", 25), "samples_2": ("integer", 10), "samples_3": ("integer", 0), "dim_1": ("integer", 128),
    "dim_2": ("integer", 128), "random_context": ("boolean", True), "batch_size": ("integer", 512),
    "sigmoid": ("boolean", False), "identity_dim": ("integer", 0), "base_log_dir": ("string", "."),
    "validate_iter": ("integer", 5000), "validate_batch_size": ("integer", 256), "gpu": ("integer", 1),
    "print_every": ("integer", 5), "max_total_steps": ("integer", 10 ** 10),
}
UNSUP_FLAGS = {
    "log_device_placement": ("boolean", False), "model": ("string", "graphsage"), "learning_rate": ("float", 0.00001),
    "model_size": ("string", "small"), "train_prefix": ("string", ""), "epochs": ("integer", 1),
    "dropout": ("float", 0.0), "weight_decay": ("float", 0.0), "max_degree": ("integer", 100),
    "samples_1": ("integer", 25), "samples_2": ("integer", 10), "dim_1": ("integer", 128), "dim_2": ("integer", 128),
    "random_context": ("boolean", True), "neg_sample_size": ("integer", 20), "batch_size": ("integer", 512),
    "n2v_test_epochs": ("integer", 1), "identity_dim": ("integer", 0), "save_embeddings": ("boolean", True),
    "base_log_dir": ("string", "."), "validate_iter": ("integer", 5000), "validate_batch_size": ("integer", 256),
    "gpu": ("integer", 1), "print_every": ("integer", 50), "max_total_steps": ("integer", 10 ** 10),
}
PY_TYPE = {"boolean": bool, "string": str, "float": float, "integer": int}


@pytest.mark.parametrize("mod,table", [(sup, SUP_FLAGS), (unsup, UNSUP_FLAGS)])
def test_flags_names_types_defaults(mod, table):
    assert {n: (k, d) for n, k, d in mod.FLAGS_SPEC} == table
    flags = vars(mod.parse_flags([]))
    assert flags == {n: d for n, (_, d) in table.items()}
    for name, (kind, _) in table.items():
        assert type(flags[name]) is PY_TYPE[kind], name


def test_flag_spellings():
    f = sup.parse_flags(["--train_prefix", "./example_data/ppi", "--model=gcn", "--sigmoid", "--epochs", "3",
                         "--learning_rate=0.5", "--norandom_context", "--log_device_placement", "--gpu", "0"])
    assert (f.train_prefix, f.model, f.sigmoid, f.epochs, f.learning_rate) == ("./example_data/ppi", "gcn", True, 3, 0.5)
    assert f.random_context is False and f.log_device_placement is True and f.gpu == 0
    assert sup.parse_flags(["--sigmoid", "--nosigmoid"]).sigmoid is False
    assert sup.parse_flags(["--sigmoid=false"]).sigmoid is False and sup.parse_flags(["--sigmoid=True"]).sigmoid is True
    assert sup.parse_flags(["-epochs", "2"]).epochs == 2
    u = unsup.parse_flags(["--nosave_embeddings", "--n2v_test_epochs=4", "--max_total_steps", "1000"])
    assert (u.save_embeddings, u.n2v_test_epochs, u.max_total_steps) == (False, 4, 1000)


@pytest.mark.parametrize("argv", [["--nope", "1"], ["--sigmoid_x"], ["stray"], ["--epochs"], ["--epochs", "x"],
                                  ["--sigmoid=maybe"], ["--nomodel"], ["--samples_3", "2.5"]])
def test_bad_flags_are_refused(argv):
    with pytest.raises(SystemExit):
        sup.parse_flags(argv)
    with pytest.raises(train_cli.FlagError):
        train_cli.parse_flags(sup.FLAGS_SPEC, argv)


def test_unsupervised_only_flags_are_unknown_to_the_supervised_trainer():
    with pytest.raises(SystemExit):
        sup.parse_flags(["--neg_sample_size", "5"])
    with pytest.raises(SystemExit):
        unsup.parse_flags(["--sigmoid"])


def test_log_dirs(tmp_path):
    base = str(tmp_path)
    f = sup.parse_flags(["--train_prefix", "./example_data/ppi", "--base_log_dir", base])
    assert sup.log_dir(f) == base + "/sup-example_data/graphsage_mean_small_0.0100/"
    f = sup.parse_flags(["--train_prefix", "../data/reddit/reddit", "--base_log_dir", base, "--model", "gcn",
                         "--model_size", "big", "--learning_rate", "0.00123"])
    assert sup.log_dir(f) == base + "/sup-reddit/gcn_big_0.0012/"
    u = unsup.parse_flags(["--train_prefix", "./example_data/toy-ppi", "--base_log_dir", base, "--model", "n2v"])
    assert unsup.log_dir(u) == base + "/unsup-example_data/n2v_small_0.000010/"
    import os
    assert os.path.isdir(base + "/sup-reddit/gcn_big_0.0012/") and os.path.isdir(base + "/unsup-example_data/n2v_small_0.000010/")


def _sk(y_true, y_pred, sigmoid):
    metrics = pytest.importorskip("sklearn.metrics")
    y_pred = np.array(y_pred, copy=True)
    if not sigmoid:                                     # the reference's calc_f1, verbatim (supervised_train.py:63-70)
        y_true, y_pred = np.argmax(y_true, axis=1), np.argmax(y_pred, axis=1)
    else:
        y_pred[y_pred > 0.5] = 1
        y_pred[y_pred <= 0.5] = 0
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return metrics.f1_score(y_true, y_pred, average="micro"), metrics.f1_score(y_true, y_pred, average="macro")


@pytest.mark.parametrize("seed", range(6))
def test_calc_f1_equals_sklearn_multilabel(seed):
    rs = np.random.RandomState(seed)
    n, c = int(rs.randint(1, 60)), int(rs.randint(1, 15))
    y = (rs.rand(n, c) < 0.3).astype(np.float64)
    p = rs.rand(n, c)
    y[:, 0] = 0                                          # a column with no true labels
    p[:, -1] = 0.1                                       # a column never predicted
    if c > 2:
        y[:, 1], p[:, 1] = 0, 0.2                        # a column with neither: scores 0 in the macro mean
    p[0, :] = 0.5                                        # exactly 0.5 is a negative
    got, want = sup.calc_f1(y, p, True), _sk(y, p, True)
    assert np.allclose(got, want, rtol=0, atol=1e-12), (got, want)
    zeros = np.zeros_like(y)
    assert np.allclose(sup.calc_f1(y, zeros, True), _sk(y, zeros, True), rtol=0, atol=1e-12)


@pytest.mark.parametrize("seed", range(6))
def test_calc_f1_equals_sklearn_multiclass(seed):
    rs = np.random.RandomState(100 + seed)
    n, c = int(rs.randint(1, 60)), int(rs.randint(2, 12))
    y = np.eye(c)[rs.randint(0, max(1, c - 2), size=n)]          # the last classes never true
    p = rs.rand(n, c)
    p[:, 0] = -1                                                  # class 0 never predicted
    got, want = sup.calc_f1(y, p, False), _sk(y, p, False)
    assert np.allclose(got, want, rtol=0, atol=1e-12), (got, want)


def test_stats_file_formats():
    assert sup.val_stats_line(0.123456, 0.5, 0.25, 1.5) == "loss=0.12346 f1_micro=0.50000 f1_macro=0.25000 time=1.50000"
    assert sup.test_stats_line(np.float32(0.1), 1.0, 0.0) == "loss=0.10000 f1_micro=1.00000 f1_macro=0.00000"


# ------------------------------------------------------------------------------------------------ the loop's schedule
class _Iter(object):
    """A minibatch iterator over `n` items in batches of `bs` (the last one short); shuffles are logged to `events`."""

    def __init__(self, n, bs, supervised, events):
        self.n, self.bs, self.supervised, self.batch_num, self.events = n, bs, supervised, 0, events

    def shuffle(self):
        self.batch_num = 0
        self.events.append(("shuffle",))

    def end(self):
        return self.batch_num * self.bs >= self.n

    def next_minibatch_feed_dict(self):
        size = min(self.bs, self.n - self.batch_num * self.bs)
        self.batch_num += 1
        feed = {"batch_size": size}
        return (feed, None) if self.supervised else feed


def _reference_schedule(n, bs, flags):
    """supervised_train.py:262-312 restated: shuffles, steps (with whether the step must run eagerly: a print step or a
    short batch), validations and prints, with (iter, total_steps); and epoch_val_costs for validations costing 1.5."""
    events, epoch_val_costs = [], []
    total_steps = 0
    for epoch in range(flags.epochs):
        events.append(("shuffle",))
        it, batch_num = 0, 0
        epoch_val_costs.append(0)
        while not batch_num * bs >= n:
            size = min(bs, n - batch_num * bs)
            batch_num += 1
            events.append(("step", it, total_steps, total_steps % flags.print_every == 0 or size != bs))
            if it % flags.validate_iter == 0:
                events.append(("validate", it, total_steps))
                epoch_val_costs[-1] += 1.5
            if total_steps % flags.print_every == 0:
                events.append(("print", it, total_steps))
            it += 1
            total_steps += 1
            if total_steps > flags.max_total_steps:
                break
        if total_steps > flags.max_total_steps:
            break
    return events, total_steps, epoch_val_costs


@pytest.mark.parametrize("supervised", [True, False])
@pytest.mark.parametrize("n,bs,epochs,print_every,validate_iter,max_total", [
    (100, 10, 3, 5, 4, 10 ** 10),         # whole batches only
    (95, 10, 3, 3, 2, 10 ** 10),          # a short last batch each epoch
    (95, 10, 4, 7, 5, 23),                # max_total_steps stops mid-epoch (total_steps > 23, not >=)
    (95, 10, 4, 2, 100, 19),              # ... right at an epoch boundary
    (95, 10, 4, 2, 100, 20),
    (5, 10, 3, 1, 1, 10 ** 10),           # every batch short
])
def test_loop_schedule_matches_the_reference(supervised, n, bs, epochs, print_every, validate_iter, max_total):
    flags = types.SimpleNamespace(epochs=epochs, print_every=print_every, validate_iter=validate_iter,
                                  max_total_steps=max_total, batch_size=bs)
    events = []
    current = {}

    def step(item, i, total, eager):
        assert isinstance(item, tuple) == supervised
        events.append(("step", i, total, eager))
        current["at"] = (i, total)
        return total

    def validate():
        events.append(("validate",) + current["at"])
        return 1.5

    def after(out, i, total, printing):
        assert out == total and (i, total) == current["at"]
        if printing:
            events.append(("print", i, total))

    with_epochs = train_cli.train_loop(_Iter(n, bs, supervised, events), flags, step, validate, after)
    want, want_total, want_costs = _reference_schedule(n, bs, flags)
    assert events == want
    assert with_epochs == (want_total, want_costs)


# ------------------------------------------------------------------------------------------------ model construction
class _Sampler(object):
    def __init__(self, adj_info, **kw):
        self.adj_info, self.counter, self.counter_dev = adj_info, 0, None


def _minibatch(N=40):
    rs = np.random.RandomState(0)
    return types.SimpleNamespace(adj=rs.randint(0, N, size=(N + 1, 8)).astype(np.int32), deg=np.ones(N),
                                 id2idx={i: i for i in range(N)})


@pytest.mark.parametrize("model,samples_3,kind,concat,dims", [
    ("graphsage_mean", 0, "mean", True, [16, 12]),
    ("graphsage_mean", 5, "mean", True, [16, 12, 12]),
    ("gcn", 0, "gcn", False, [32, 24]),
    ("graphsage_seq", 0, "seq", True, [16, 12]),
    ("graphsage_maxpool", 0, "maxpool", True, [16, 12]),
    ("graphsage_meanpool", 0, "meanpool", True, [16, 12]),
])
def test_supervised_model_branches(monkeypatch, model, samples_3, kind, concat, dims):
    monkeypatch.setattr(sup, "UniformNeighborSampler", _Sampler)
    flags = sup.parse_flags(["--model", model, "--dim_1", "16", "--dim_2", "12", "--samples_3", str(samples_3),
                             "--sigmoid", "--identity_dim", "4", "--learning_rate", "0.02", "--weight_decay", "0.1"])
    feats = np.random.RandomState(1).randn(41, 6)
    m = sup.build_model(flags, feats, _minibatch(), 7, "cpu")
    assert isinstance(m, gs.SupervisedGraphsage) and m.aggregator_cls is gs.models._AGGREGATORS[kind]
    assert m.concat == concat and m.dims == [4 + 6] + dims and m.sigmoid_loss and m.num_classes == 7
    fanouts = [25, 10, 5][:len(dims)]
    assert [i.num_samples for i in m.layer_infos] == fanouts
    assert len({id(i.neigh_sampler) for i in m.layer_infos}) == 1
    assert (m.learning_rate, m.weight_decay, m.identity_dim) == (0.02, 0.1, 4)


def test_samples_3_only_for_mean_and_single_layer(monkeypatch):
    monkeypatch.setattr(sup, "UniformNeighborSampler", _Sampler)
    feats = np.zeros((41, 6))
    m = sup.build_model(sup.parse_flags(["--model", "graphsage_maxpool", "--samples_3", "5"]), feats, _minibatch(), 3, "cpu")
    assert len(m.layer_infos) == 2
    m = sup.build_model(sup.parse_flags(["--samples_2", "0"]), feats, _minibatch(), 3, "cpu")
    assert [i.num_samples for i in m.layer_infos] == [25]
    with pytest.raises(Exception, match="unrecognized"):
        sup.build_model(sup.parse_flags(["--model", "graphsage"]), feats, _minibatch(), 3, "cpu")


@pytest.mark.parametrize("model,kind,concat,dims", [
    ("graphsage_mean", "mean", True, [16, 12]), ("gcn", "gcn", False, [32, 24]), ("graphsage_seq", "seq", True, [16, 12]),
    ("graphsage_maxpool", "maxpool", True, [16, 12]), ("graphsage_meanpool", "meanpool", True, [16, 12]),
])
def test_unsupervised_model_branches(monkeypatch, model, kind, concat, dims):
    monkeypatch.setattr(unsup, "UniformNeighborSampler", _Sampler)
    flags = unsup.parse_flags(["--model", model, "--dim_1", "16", "--dim_2", "12", "--neg_sample_size", "7"])
    m = unsup.build_model(flags, np.zeros((41, 6)), _minibatch(), "cpu")
    assert isinstance(m, gs.UnsupervisedGraphsage) and m.aggregator_cls is gs.models._AGGREGATORS[kind]
    assert m.concat == concat and m.dims == [6] + dims and m.neg_sample_size == 7 and m.learning_rate == 0.00001


def test_unsupervised_n2v_and_unknown_models():
    flags = unsup.parse_flags(["--model", "n2v", "--dim_1", "8", "--learning_rate", "0.3"])
    m = unsup.build_model(flags, None, _minibatch(40), "cpu")
    assert isinstance(m, gs.Node2VecModel)
    assert tuple(m.target_embeds.shape) == (41, 16) and m.lr == 0.3 and m.neg_sample_size == 20
    with pytest.raises(Exception, match="unrecognized"):
        unsup.build_model(unsup.parse_flags([]), None, _minibatch(), "cpu")      # the default --model graphsage


def test_step_clock_reports_wall_time_per_step():
    calls = []
    clock = train_cli.StepClock(None, sync=lambda: calls.append(1))
    clock.t0 -= 10.0
    assert 4.9 < clock.avg(2) < 5.5 and calls == [1]


def test_gpu_flag_without_a_device_is_an_error(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        train_cli.select_device(0)
