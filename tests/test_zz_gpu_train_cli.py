"""GPU: the trainers end to end on the toy-ppi slice (tests/golden/toy_ppi.npz written back in the reference's file
layout): every supervised model, the stats files, reproducibility, replayed steps against an all-eager loop, no host
synchronisation outside print and validation steps, and the unsupervised embedding files (graphsage_mean, n2v)."""
import json
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

SMALL = ["--sigmoid", "--epochs", "2", "--dim_1", "16", "--dim_2", "16", "--batch_size", "128", "--print_every", "3",
         "--validate_iter", "4", "--validate_batch_size", "64", "--gpu", "0"]


@pytest.fixture(scope="module")
def toy(tmp_path_factory):
    """<dir>/toy-ppi/toy-ppi-{G.json, feats.npy, id_map.json, class_map.json, walks.txt}; val/test - train links added
    (every 5th val/test node to a train node, train_removed) so walks from val/test nodes reach the train graph, as on the
    whole dataset.  Returns the prefix."""
    d = np.load(os.path.join(GOLDEN, "toy_ppi.npz"))
    root = tmp_path_factory.mktemp("data") / "toy-ppi"
    root.mkdir()
    prefix = str(root / "toy-ppi")
    ids = [int(u) for u in d["ids"]]
    labels = np.unpackbits(d["labels"], axis=1)[:, :int(d["n_classes"])]
    links = [(int(a), int(b), bool(x), bool(y)) for a, b, x, y in zip(d["src"], d["dst"], d["test_removed"], d["train_removed"])]
    train = [i for i, (v, t) in enumerate(zip(d["val"], d["test"])) if not v and not t]
    other = [i for i, (v, t) in enumerate(zip(d["val"], d["test"])) if v or t]
    links += [(other[5 * k % len(other)], train[7 * k % len(train)], False, True) for k in range(60)]
    g = {"directed": False, "multigraph": False, "graph": {"name": "toy-ppi slice"},
         "nodes": [{"id": u, "val": bool(v), "test": bool(t)} for u, v, t in zip(ids, d["val"], d["test"])],
         "links": [{"source": a, "target": b, "test_removed": x, "train_removed": y} for a, b, x, y in links]}
    with open(prefix + "-G.json", "w") as fp:
        json.dump(g, fp)
    np.save(prefix + "-feats.npy", d["feats"])
    with open(prefix + "-id_map.json", "w") as fp:
        json.dump({str(u): i for i, u in enumerate(ids)}, fp)
    with open(prefix + "-class_map.json", "w") as fp:
        json.dump({str(u): [int(x) for x in row] for u, row in zip(ids, labels)}, fp)
    from graphsage_b200 import utils
    G = utils.load_data(prefix)[0]
    nodes = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    pairs = utils.run_random_walks(G.subgraph(nodes), nodes, num_walks=4, rng=random.Random(3))
    with open(prefix + "-walks.txt", "w") as fp:
        fp.write("\n".join("%d\t%d" % p for p in pairs))
    return prefix


def _stats(path):
    return dict(kv.split("=") for kv in open(path).read().split())


def _run(toy, tmp_path, model, *extra):
    from graphsage_b200 import supervised_train as sup
    argv = ["--train_prefix", toy, "--base_log_dir", str(tmp_path), "--model", model] + SMALL + list(extra)
    m = sup.main(argv)
    return m, sup.log_dir(sup.parse_flags(argv))


def _val_labels(toy):
    from graphsage_b200 import utils
    G, _, _, _, class_map = utils.load_data(toy)
    return np.array([class_map[n] for n in G.nodes() if G.node[n]["val"]], dtype=np.float64)


@pytest.mark.parametrize("model,extra", [
    ("graphsage_mean", ["--samples_3", "5"]),
    ("gcn", ["--identity_dim", "16"]),
    ("graphsage_seq", ["--samples_1", "10", "--samples_2", "5"]),
    ("graphsage_maxpool", ["--dropout", "0.5"]),
    ("graphsage_meanpool", []),
])
def test_supervised_models_write_stats_that_beat_all_negative(toy, tmp_path, capsys, model, extra):
    from graphsage_b200 import supervised_train as sup
    _, d = _run(toy, tmp_path, model, *extra)
    val, test = _stats(d + "val_stats.txt"), _stats(d + "test_stats.txt")
    assert set(val) == {"loss", "f1_micro", "f1_macro", "time"} and set(test) == {"loss", "f1_micro", "f1_macro"}
    assert all(np.isfinite(float(v)) for v in list(val.values()) + list(test.values()))
    y = _val_labels(toy)
    assert float(val["f1_micro"]) > sup.calc_f1(y, np.zeros_like(y), True)[0]
    out = capsys.readouterr().out
    assert "Epoch: 0002" in out and "Optimization Finished!" in out and "Full validation stats:" in out
    assert out.count("Iter:") >= 2 and "train_f1_mic=" in out


def test_two_runs_write_the_same_stats(toy, tmp_path):
    _, a = _run(toy, tmp_path / "a", "graphsage_mean", "--dropout", "0.5")
    _, b = _run(toy, tmp_path / "b", "graphsage_mean", "--dropout", "0.5")
    for name in ("val_stats.txt", "test_stats.txt"):
        sa, sb = _stats(a + name), _stats(b + name)
        sa.pop("time", None)
        sb.pop("time", None)
        assert sa == sb, name


def test_replayed_and_eager_steps_train_like_an_all_eager_loop(toy, tmp_path):
    import graphsage_b200 as gs
    from graphsage_b200 import supervised_train as sup, utils
    argv = ["--train_prefix", toy, "--base_log_dir", str(tmp_path), "--dropout", "0.5", "--identity_dim", "8"] + SMALL
    flags = sup.parse_flags(argv)
    data = utils.load_data(toy)
    dev = torch.device("cuda", 0)
    calls = {"replay": 0, "eager": 0}
    real = gs.GraphedTrainStep.__call__

    def counting(self, a, b):
        calls["replay"] += 1
        return real(self, a, b)

    gs.GraphedTrainStep.__call__ = counting
    try:
        got = sup.train(data, flags, device=dev)
    finally:
        gs.GraphedTrainStep.__call__ = real

    minibatch = sup.build_iterator(data, flags)
    feats = np.vstack([data[1], np.zeros((1, data[1].shape[1]))])
    m = sup.build_model(flags, feats, minibatch, minibatch.num_classes, dev)
    gs.make_adam_capturable(m.optimizer)
    sampler = m.layer_infos[0].neigh_sampler
    adj, test_adj = sampler.adj_info, torch.from_numpy(minibatch.test_adj).to(dev)
    for _ in range(flags.epochs):
        minibatch.shuffle()
        it = 0
        while not minibatch.end():
            feed, labels = minibatch.next_minibatch_feed_dict()
            m.train_step(torch.tensor(feed["batch"], dtype=torch.int32, device=dev),
                         torch.tensor(labels, dtype=torch.float32, device=dev))
            calls["eager"] += 1
            if it % flags.validate_iter == 0:
                sampler.set_adj(test_adj)
                sup.evaluate(m, minibatch, flags.validate_batch_size, flags, dev)
                sampler.set_adj(adj)
            it += 1
    assert calls["replay"] >= 2 and calls["eager"] > calls["replay"]
    assert all(torch.equal(p, q) for p, q in zip(got.parameters(), m.parameters()))


def test_no_host_synchronisation_outside_print_and_validation_steps(toy, tmp_path, monkeypatch):
    from graphsage_b200 import supervised_train as sup, train_cli
    guarded = []

    def loop(minibatch, flags, step, validate, after):
        def quiet_step(item, it, total, eager):
            if total % flags.print_every == 0:
                return step(item, it, total, eager)
            torch.cuda.set_sync_debug_mode("error")
            try:
                out = step(item, it, total, eager)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            guarded.append(eager)
            return out
        return train_cli.train_loop(minibatch, flags, quiet_step, validate, after)

    monkeypatch.setattr(sup, "train_loop", loop)
    _run(toy, tmp_path, "graphsage_mean", "--print_every", "4")
    assert False in guarded and True in guarded                  # replays and the eager short batches


def _first_occurrence(nodes):
    seen, out = set(), []
    for n in nodes:
        if n not in seen:
            seen.add(n)
            out.append(n)
    return out


@pytest.mark.parametrize("model", ["graphsage_mean", "n2v"])
def test_unsupervised_writes_the_embedding_files(toy, tmp_path, monkeypatch, capsys, model):
    from graphsage_b200 import unsupervised_train as unsup, utils
    made = []
    real = unsup.build_iterator

    def keep(train_data, flags):
        made.append(real(train_data, flags))
        return made[-1]

    monkeypatch.setattr(unsup, "build_iterator", keep)
    argv = ["--train_prefix", toy, "--base_log_dir", str(tmp_path), "--model", model, "--dim_1", "16", "--dim_2", "16",
            "--batch_size", "128", "--print_every", "5", "--validate_iter", "5", "--validate_batch_size", "64",
            "--max_total_steps", "25", "--learning_rate", "0.01", "--gpu", "0"]
    m = unsup.main(argv)
    d = unsup.log_dir(unsup.parse_flags(argv))
    ids = open(d + "val.txt").read().split("\n")
    emb = np.load(d + "val.npy")
    assert emb.shape == (len(ids), 32) and np.isfinite(emb).all()
    assert ids == [str(n) for n in _first_occurrence(made[0].nodes)]
    out = capsys.readouterr().out
    assert "train_mrr_ema=" in out and "val_mrr_ema=" in out and "Optimization Finished!" in out
    if model == "n2v":
        ids2 = open(d + "val-test.txt").read().split("\n")
        emb2 = np.load(d + "val-test.npy")
        assert ids2 == ids
        id_map = utils.load_data(toy)[2]
        rows = [id_map[int(n)] for n in ids2]
        assert np.array_equal(emb2, m.target_embeds.cpu().numpy()[rows])
        assert "Doing test training for n2v." in out and "Walk time: " in out and "Train time: " in out
    else:
        assert not os.path.exists(d + "val-test.npy")
