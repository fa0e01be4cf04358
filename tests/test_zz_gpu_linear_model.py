"""GPU: gs_sgd_orders / gs_sgd_fit against oracle/sgd.py (orders exact, coef and intercept within 1e-9 relative), the
SGDClassifier forms (binary, 41-class one-vs-rest, 121-column multi-output), reproducibility, and ppi_eval end to end on
embeddings from the unsupervised trainer.

The rows of X have norm <= 1, as l2-normalised embeddings do.  With the "optimal" schedule (eta = 10 at t = 1) a step
multiplies a perturbation by up to 1 + eta |x|^2 / 4, so on rows of large norm the ulp-level difference between CUDA's
exp and numpy's grows chaotically and no tolerance holds; on these rows it stays near 1e-15."""
import os
import shutil

import numpy as np
import pytest
import torch

import oracle.sgd as osgd
from test_linear_model_cpu import oracle_stand_in, unit_rows
from test_zz_gpu_train_cli import toy  # noqa: F401  (fixture: the toy-ppi dataset with walks)

pytestmark = pytest.mark.gpu

REL = 1e-9


def _close(got, ref):
    scale = max(np.abs(ref).max(), 1e-300)
    assert np.abs(got - ref).max() <= REL * scale, np.abs(got - ref).max() / scale


def _same_predictions(x, coef, intercept, coef_ref, intercept_ref):
    s, r = x @ coef.T + intercept, x @ coef_ref.T + intercept_ref
    near_tie = np.abs(r) < 1e-12
    assert ((s > 0) == (r > 0))[~near_tie].all()


def test_orders_equal_the_oracle():
    from graphsage_b200 import linear_model as lm
    for n, seeds in [(1, [5]), (2, [0, 1]), (1000, [0, 7, 2 ** 31 - 2]), (50000, [123456789, 42])]:
        got = lm.sgd_orders(seeds, n, "cuda").cpu().numpy()
        for p, s in enumerate(seeds):
            assert np.array_equal(got[p], osgd.epoch_orders(osgd.sigma(s, n), 5)), (n, s)


@pytest.mark.parametrize("n,d,dtype,P", [
    (2000, 1, np.float64, 3),
    (3000, 50, np.float32, 3),
    (50000, 256, np.float64, 2),
    (4000, 256, np.float32, 2),
    (2000, 858, np.float64, 2),
    (1500, 1024, np.float32, 2),
])
def test_fit_equals_the_oracle(n, d, dtype, P):
    from graphsage_b200 import linear_model as lm
    rs = np.random.RandomState(d + n)
    x = unit_rows(rs, n, d).astype(dtype)
    labels = np.where(rs.rand(P, n) < np.linspace(0.05, 0.5, P)[:, None], 1, -1).astype(np.int32)
    seeds = rs.randint(0, 2 ** 31 - 1, size=P)
    orders = lm.sgd_orders(seeds, n, "cuda")
    coef, intercept = lm.sgd_fit(torch.from_numpy(x).cuda(), torch.from_numpy(labels).cuda(), orders)
    coef, intercept = coef.cpu().numpy(), intercept.cpu().numpy()
    ref_c, ref_b = osgd.fit(x, labels, orders.cpu().numpy(), lm.ALPHA, lm.optimal_init())
    _close(coef, ref_c)
    _close(intercept, ref_b)
    _same_predictions(x.astype(np.float64), coef, intercept, ref_c, ref_b)


def _both(monkeypatch, X, y, **kw):
    from graphsage_b200 import linear_model as lm
    np.random.seed(1)
    got = lm.SGDClassifier(**kw).fit(X, y)
    with monkeypatch.context() as m:
        m.setattr(lm, "_fit_problems", oracle_stand_in(osgd.kernel_dot))
        np.random.seed(1)
        ref = lm.SGDClassifier(device="cpu", **kw).fit(X, y)
    return got, ref


def test_one_vs_rest_41_classes(monkeypatch):
    rs = np.random.RandomState(41)
    X = unit_rows(rs, 3000, 64)
    y = rs.randint(0, 41, size=3000)
    got, ref = _both(monkeypatch, X, y)
    assert got.coef_.shape == (41, 64)
    _close(got.coef_, ref.coef_)
    _close(got.intercept_, ref.intercept_)
    _same_predictions(X, got.coef_, got.intercept_, ref.coef_, ref.intercept_)


def test_multi_output_121_columns_with_an_unbalanced_one(monkeypatch):
    rs = np.random.RandomState(121)
    X = unit_rows(rs, 2000, 50).astype(np.float32)
    Y = (rs.rand(2000, 121) < rs.uniform(0.02, 0.6, size=121)).astype(np.int64)
    Y[:, 7] = 0
    Y[13, 7] = 1                                   # one positive row in 2000
    got, ref = _both(monkeypatch, X, Y)
    assert got.coef_.shape == (121, 50) and got.predict(X).shape == (2000, 121)
    _close(got.coef_, ref.coef_)
    _close(got.intercept_, ref.intercept_)
    _same_predictions(X.astype(np.float64), got.coef_, got.intercept_, ref.coef_, ref.intercept_)


def test_two_fits_are_bit_identical():
    from graphsage_b200 import linear_model as lm
    rs = np.random.RandomState(3)
    X = unit_rows(rs, 5000, 256)
    y = rs.randint(0, 5, size=5000)
    a = lm.SGDClassifier(random_state=9).fit(X, y)
    b = lm.SGDClassifier(random_state=9).fit(X, y)
    assert np.array_equal(a.coef_, b.coef_) and np.array_equal(a.intercept_, b.intercept_)


def test_ppi_eval_on_trained_embeddings(toy, tmp_path, capsys):   # noqa: F811
    from graphsage_b200 import unsupervised_train as unsup
    from graphsage_b200.eval_scripts import micro_f1, ppi_eval
    argv = ["--train_prefix", toy, "--base_log_dir", str(tmp_path), "--model", "graphsage_mean", "--dim_1", "16",
            "--dim_2", "16", "--batch_size", "64", "--print_every", "100", "--validate_iter", "50",
            "--validate_batch_size", "64", "--max_total_steps", "300", "--epochs", "3", "--learning_rate", "0.01",
            "--gpu", "0"]
    unsup.main(argv)
    embed_dir = unsup.log_dir(unsup.parse_flags(argv))
    data = tmp_path / "ppi"
    data.mkdir()
    for part in ("G.json", "class_map.json", "id_map.json", "feats.npy"):
        shutil.copy(toy + "-" + part, str(data / ("ppi-" + part)))
    capsys.readouterr()
    ppi_eval.main([str(data), embed_dir.rstrip("/"), "test", "--gpu", "0"])
    out = capsys.readouterr().out.splitlines()
    f1 = [float(l.split()[-1]) for l in out if l.startswith("F1 score")]
    assert out[:2] == ["Loading data...", "running " + embed_dir.rstrip("/")] and len(f1) == 121
    assert sum(l.startswith("Random baseline F1 score") for l in out) == 121
    sklearn = pytest.importorskip("sklearn")
    from sklearn.linear_model import SGDClassifier
    from sklearn.multioutput import MultiOutputClassifier
    from graphsage_b200.eval_scripts import read_embeddings, split_ids
    from graphsage_b200.graph import node_link_graph
    import json
    G = node_link_graph(json.load(open(str(data / "ppi-G.json"))))
    labels = {int(k): v for k, v in json.load(open(str(data / "ppi-class_map.json"))).items()}
    train_ids, test_ids = split_ids(G, "test")
    emb, id_map = read_embeddings(os.path.join(embed_dir, "val"), int)
    xtr, xte = emb[[id_map[i] for i in train_ids]], emb[[id_map[i] for i in test_ids]]
    ytr, yte = np.array([labels[i] for i in train_ids]), np.array([labels[i] for i in test_ids])
    np.random.seed(1)
    ref = MultiOutputClassifier(SGDClassifier(loss="log_loss", max_iter=5, tol=None), n_jobs=1)
    ref.fit(xtr.astype(np.float64), ytr)
    pred = ref.predict(xte.astype(np.float64))
    assert sklearn is not None
    assert f1 == [micro_f1(yte[:, i], pred[:, i]) for i in range(yte.shape[1])]
