"""CPU: oracle/sgd.py against the installed scikit-learn (SGDClassifier(loss="log_loss", max_iter=5, tol=None) on float64
X: binary, one-vs-rest, MultiOutputClassifier), the seed chains and the stratified dummy of graphsage_b200.linear_model,
the three eval scripts on the toy-ppi slice with the oracle standing in for the kernel, and the refusals."""
import json
import os

import numpy as np
import pytest

import oracle.sgd as osgd
from conftest import GOLDEN

REL = 1e-9


def unit_rows(rs, n, d):
    """Gaussian rows scaled to norms in [0.5, 1] (the l2-normalised embeddings the eval scripts score)."""
    x = rs.randn(n, d)
    return x / np.linalg.norm(x, axis=1, keepdims=True) * rs.uniform(0.5, 1.0, size=(n, 1))


def oracle_stand_in(dot):
    """A replacement for linear_model._fit_problems: the oracle with the given dot-product order."""
    from graphsage_b200 import linear_model as lm

    def fit(x, labels, seeds, device):
        return osgd.fit_problems(np.asarray(x, dtype=np.float64), labels, seeds, lm.ALPHA, lm.optimal_init(), dot=dot)
    return fit


@pytest.fixture
def on_oracle(monkeypatch):
    from graphsage_b200 import linear_model as lm

    def use(dot):
        monkeypatch.setattr(lm, "_fit_problems", oracle_stand_in(dot))
    return use


def _sklearn_fit(X, y, multi_output=False):
    pytest.importorskip("sklearn")
    from sklearn.linear_model import SGDClassifier
    from sklearn.multioutput import MultiOutputClassifier
    np.random.seed(1)
    est = SGDClassifier(loss="log_loss", max_iter=5, tol=None)
    if multi_output:
        m = MultiOutputClassifier(est, n_jobs=1).fit(np.asarray(X, dtype=np.float64), y)
        coef = np.vstack([e.coef_ for e in m.estimators_])
        intercept = np.hstack([e.intercept_ for e in m.estimators_])
        return m, coef, intercept
    est.fit(np.asarray(X, dtype=np.float64), y)
    return est, est.coef_, est.intercept_


def _ours(X, y):
    from graphsage_b200 import linear_model as lm
    np.random.seed(1)
    return lm.SGDClassifier(device="cpu").fit(X, y)


CASES = {
    "binary": lambda rs, n: rs.randint(0, 2, size=n) * 3 + 2,           # labels 2 and 5: classes_[1] = 5 is positive
    "ovr": lambda rs, n: rs.choice(np.array([-1, 4, 9, 11]), size=n),
    "multi_output": lambda rs, n: np.vstack([[1] * 6, [0] * 6,
                                             (rs.rand(n - 2, 6) < [0.1, 0.3, 0.5, 0.7, 0.9, 0.05]).astype(np.int64)]),
}


@pytest.mark.parametrize("form", sorted(CASES))
@pytest.mark.parametrize("n,d", [(7, 3), (60, 5), (400, 33)])
def test_oracle_in_sklearn_order_is_sklearn_bit_for_bit(on_oracle, form, n, d):
    rs = np.random.RandomState(n * d)
    X, y = rs.randn(n, d) * 3, CASES[form](rs, n)
    ref, coef, intercept = _sklearn_fit(X, y, form == "multi_output")
    on_oracle(osgd.sequential_dot)
    ours = _ours(X, y)
    assert np.array_equal(ours.coef_, coef) and np.array_equal(ours.intercept_, intercept)
    assert np.array_equal(ours.predict(X), ref.predict(X))


@pytest.mark.parametrize("form", sorted(CASES))
@pytest.mark.parametrize("n,d", [(60, 5), (400, 33), (300, 100)])
def test_oracle_in_kernel_order_is_within_1e9_of_sklearn(on_oracle, form, n, d):
    rs = np.random.RandomState(n + d)
    X, y = unit_rows(rs, n, d), CASES[form](rs, n)
    ref, coef, intercept = _sklearn_fit(X, y, form == "multi_output")
    on_oracle(osgd.kernel_dot)
    ours = _ours(X, y)
    assert np.abs(ours.coef_ - coef).max() <= REL * np.abs(coef).max()
    assert np.abs(ours.intercept_ - intercept).max() <= REL * max(np.abs(intercept).max(), np.abs(coef).max())
    assert np.array_equal(ours.predict(X), ref.predict(X))


def test_a_wrong_order_or_seed_is_far_outside_the_tolerance():
    from graphsage_b200 import linear_model as lm
    rs = np.random.RandomState(0)
    X, lab = unit_rows(rs, 50, 4), np.where(rs.rand(1, 50) < 0.4, 1, -1)
    good = osgd.fit_problems(X, lab, [77], lm.ALPHA, lm.optimal_init())[0]
    sig = osgd.sigma(77, 50)
    wrong = [osgd.fit_problems(X, lab, [78], lm.ALPHA, lm.optimal_init())[0],                  # neighbouring seed
             osgd.fit(X, lab, np.tile(sig, (1, 5, 1)), lm.ALPHA, lm.optimal_init())[0],        # sigma every epoch
             osgd.fit(X, lab, osgd.epoch_orders(sig, 6)[None, 1:], lm.ALPHA, lm.optimal_init())[0]]   # shifted
    for w in wrong:
        assert np.abs(w - good).max() > 1e3 * REL * np.abs(good).max()


def test_orders_follow_sklearn_shuffle():
    pytest.importorskip("sklearn")
    from sklearn.utils._seq_dataset import ArrayDataset64
    for n, seed in [(1, 3), (2, 0), (37, 12345), (500, 2 ** 31 - 2)]:
        ds = ArrayDataset64(np.zeros((n, 1)), np.zeros(n), np.ones(n), 1)
        want = []
        for _ in range(4):
            ds._shuffle_py(seed)
            want.append([ds._next_py()[3] for _ in range(n)])
        assert np.array_equal(osgd.epoch_orders(osgd.sigma(seed, n), 4), want)


def test_stratified_dummy_draws_like_sklearn():
    pytest.importorskip("sklearn")
    from sklearn.dummy import DummyClassifier as Reference
    from graphsage_b200.linear_model import DummyClassifier
    rs = np.random.RandomState(2)
    X = rs.randn(300, 3)
    for y in [rs.randint(0, 5, size=300), rs.choice(np.array(["a", "b"]), size=300),
              (rs.rand(300, 4) < 0.3).astype(int)]:
        np.random.seed(1)
        want = [Reference(strategy="stratified").fit(X, y).predict(X) for _ in range(2)]
        np.random.seed(1)
        got = [DummyClassifier().fit(X, y).predict(X) for _ in range(2)]
        for a, b in zip(got, want):
            assert a.shape == b.shape and np.array_equal(a, b)


def test_refusals():
    from graphsage_b200.linear_model import DummyClassifier, SGDClassifier
    for kw in [dict(loss="hinge"), dict(penalty="l1"), dict(learning_rate="constant"), dict(average=True)]:
        with pytest.raises(NotImplementedError):
            SGDClassifier(**kw)
    with pytest.raises(NotImplementedError):
        DummyClassifier(strategy="uniform")
    X = np.zeros((4, 2))
    with pytest.raises(ValueError, match="greater than one"):
        SGDClassifier(device="cpu").fit(X, [3, 3, 3, 3])
    with pytest.raises(ValueError, match="greater than one"):
        SGDClassifier(device="cpu").fit(X, np.array([[0, 1], [0, 1], [1, 1], [0, 1]]))
    with pytest.raises(ValueError, match="0/1"):
        SGDClassifier(device="cpu").fit(X, np.array([[0, 2], [1, 1], [1, 0], [0, 1]]))
    with pytest.raises(RuntimeError, match="CUDA"):
        SGDClassifier(device="cpu").fit(X, [0, 1, 0, 1])


# ------------------------------------------------------------------ the eval scripts on the toy-ppi slice

def write_dataset(root, name, str_ids=False, single_label=False):
    """tests/golden/toy_ppi.npz written as <root>/<name>-{G.json, feats.npy, id_map.json, class_map.json}.  Returns the
    node ids and the label of every node (a 121-column 0/1 row, or with single_label one of six classes)."""
    d = np.load(os.path.join(GOLDEN, "toy_ppi.npz"))
    ids = [int(u) for u in d["ids"]]
    labels = np.unpackbits(d["labels"], axis=1)[:, :int(d["n_classes"])]
    if single_label:
        labels = labels[:, :6].argmax(axis=1)
    key = str if str_ids else int
    g = {"directed": False, "multigraph": False, "graph": {},
         "nodes": [{"id": key(u), "val": bool(v), "test": bool(t)} for u, v, t in zip(ids, d["val"], d["test"])],
         "links": [{"source": int(a), "target": int(b), "test_removed": bool(x), "train_removed": bool(y)}
                   for a, b, x, y in zip(d["src"], d["dst"], d["test_removed"], d["train_removed"])]}
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, name + "-G.json"), "w") as fp:
        json.dump(g, fp)
    feats = np.abs(d["feats"]).astype(np.float64)        # counts-like columns 0 and 1 for the log transform
    np.save(os.path.join(root, name + "-feats.npy"), feats)
    with open(os.path.join(root, name + "-id_map.json"), "w") as fp:
        json.dump({str(u): i for i, u in enumerate(ids)}, fp)
    with open(os.path.join(root, name + "-class_map.json"), "w") as fp:
        json.dump({str(u): (int(l) if single_label else [int(x) for x in l]) for u, l in zip(ids, labels)}, fp)
    return ids, labels, d


def write_embeddings(path, ids, rs, dim=16):
    """val.npy (unit rows, a shuffled row order) and val.txt as the unsupervised trainer writes them."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    order = rs.permutation(len(ids))
    emb = unit_rows(rs, len(ids), dim).astype(np.float32)
    np.save(path + ".npy", emb)
    with open(path + ".txt", "w") as fp:
        fp.write("\n".join(str(ids[i]) for i in order))
    return emb, {ids[i]: r for r, i in enumerate(order)}


def _split(ids, d, setting="test"):
    train = [i for i, (v, t) in enumerate(zip(d["val"], d["test"])) if not v and not t]
    test = [i for i, (v, t) in enumerate(zip(d["val"], d["test"])) if (v if setting == "val" else t)]
    return train, test


def _reference_lines(xtr, ytr, xte, yte, kind):
    """The reference's run_regression print lines, computed with the installed scikit-learn."""
    pytest.importorskip("sklearn")
    from sklearn.dummy import DummyClassifier
    from sklearn.linear_model import SGDClassifier
    from sklearn.metrics import f1_score
    from sklearn.multioutput import MultiOutputClassifier
    xtr, xte = np.asarray(xtr, dtype=np.float64), np.asarray(xte, dtype=np.float64)
    np.random.seed(1)
    lines = []
    if kind == "ppi":
        dummy = MultiOutputClassifier(DummyClassifier(strategy="stratified")).fit(xtr, ytr)
        log = MultiOutputClassifier(SGDClassifier(loss="log_loss", max_iter=5, tol=None), n_jobs=1).fit(xtr, ytr)
        for i in range(yte.shape[1]):
            lines.append("F1 score %s" % f1_score(yte[:, i], log.predict(xte)[:, i], average="micro"))
        for i in range(yte.shape[1]):
            lines.append("Random baseline F1 score %s" % f1_score(yte[:, i], dummy.predict(xte)[:, i], average="micro"))
        return lines
    dummy = DummyClassifier(strategy="stratified").fit(xtr, ytr)
    log = SGDClassifier(loss="log_loss", max_iter=5, tol=None).fit(xtr, ytr)
    if kind == "reddit":
        return ["Test scores", str(f1_score(yte, log.predict(xte), average="micro")), "Train scores",
                str(f1_score(ytr, log.predict(xtr), average="micro")), "Random baseline",
                str(f1_score(yte, dummy.predict(xte), average="micro"))]
    return ["F1 score: %s" % f1_score(yte, log.predict(xte), average="micro"),
            "Random baseline f1 score: %s" % f1_score(yte, dummy.predict(xte), average="micro")]


def _scaled(train, test):
    from graphsage_b200.eval_scripts import scale_pair
    return scale_pair(train, test)


def _log(feats):
    from graphsage_b200.eval_scripts import log_counts
    return log_counts(feats)


@pytest.mark.parametrize("branch", ["embeddings", "feat"])
def test_ppi_eval_prints_the_reference_lines(tmp_path, capsys, on_oracle, branch):
    from graphsage_b200.eval_scripts import ppi_eval
    on_oracle(osgd.sequential_dot)            # sklearn's own order: the runs agree bit for bit, so the lines do
    ids, labels, d = write_dataset(str(tmp_path / "data"), "ppi")
    emb, rows = write_embeddings(str(tmp_path / "unsup" / "val"), ids, np.random.RandomState(4))
    train, test = _split(ids, d)
    if branch == "feat":
        feats = _log(np.load(str(tmp_path / "data" / "ppi-feats.npy")))
        xtr, xte = _scaled(feats[train], feats[test])
        embed_dir = "feat"
    else:
        xtr, xte = emb[[rows[ids[i]] for i in train]], emb[[rows[ids[i]] for i in test]]
        embed_dir = str(tmp_path / "unsup")
    ppi_eval.main([str(tmp_path / "data"), embed_dir, "test"], device="cpu")
    out = capsys.readouterr().out.splitlines()
    head = ["Loading data...", "running " + embed_dir] + (["Using only features.."] if branch == "feat" else [])
    assert out[:len(head) + 1] == head + ["Running regression.."]
    assert out[len(head) + 1:] == _reference_lines(xtr, labels[train], xte, labels[test], "ppi")


@pytest.mark.parametrize("branch", ["embeddings", "n2v", "feat"])
def test_reddit_eval_prints_the_reference_lines(tmp_path, capsys, on_oracle, branch):
    from graphsage_b200.eval_scripts import reddit_eval
    on_oracle(osgd.sequential_dot)
    ids, labels, d = write_dataset(str(tmp_path / "data"), "reddit", str_ids=True, single_label=True)
    rs = np.random.RandomState(5)
    embed_dir = str(tmp_path / ("unsup-n2v" if branch == "n2v" else "unsup"))
    emb, rows = write_embeddings(os.path.join(embed_dir, "val"), ids, rs)
    train, test = _split(ids, d, "val")
    xtr = emb[[rows[ids[i]] for i in train]]
    feats = np.load(str(tmp_path / "data" / "reddit-feats.npy"))
    if branch == "n2v":
        tuned, trows = write_embeddings(os.path.join(embed_dir, "val-test"), ids, rs)
        xte = tuned[[trows[ids[i]] for i in test]]
        want = (["Doing it N2V style.", "Running regression.."] + _reference_lines(xtr, labels[train], xte, labels[test],
                                                                                   "reddit"))
        ftr, fte = _scaled(np.hstack([feats[train], xtr]), np.hstack([feats[test], xte]))
        want += ["Running regression with feats.."] + _reference_lines(ftr, labels[train], fte, labels[test], "reddit")
    elif branch == "feat":
        embed_dir = "feat"
        f = _log(feats)
        ftr, fte = _scaled(f[train], f[test])
        want = ["Using only features..", "Running regression.."] + _reference_lines(ftr, labels[train], fte, labels[test],
                                                                                   "reddit")
    else:
        xte = emb[[rows[ids[i]] for i in test]]
        want = ["Running regression.."] + _reference_lines(xtr, labels[train], xte, labels[test], "reddit")
    reddit_eval.main([str(tmp_path / "data"), embed_dir, "val"], device="cpu")
    assert capsys.readouterr().out.splitlines() == ["Loading data..."] + want


@pytest.mark.parametrize("branch", ["embeddings", "n2v", "feat"])
def test_citation_eval_prints_the_reference_lines(tmp_path, capsys, on_oracle, branch):
    from graphsage_b200.eval_scripts import citation_eval
    on_oracle(osgd.sequential_dot)
    ids, labels, d = write_dataset(str(tmp_path / "data"), "isi", single_label=True)
    lab_dir = tmp_path / "labels"
    lab_dir.mkdir()
    for c, code in enumerate(citation_eval.SUBJECTS):
        with open(str(lab_dir / (code + ".tsv")), "w") as fp:
            fp.write("id\tsubject\n" + "".join("%d\t%s\n" % (u, code) for u, l in zip(ids, labels) if l == c))
    rs = np.random.RandomState(6)
    embed_dir = str(tmp_path / ("n2v-run" if branch == "n2v" else "unsup"))
    emb, rows = write_embeddings(os.path.join(embed_dir, "val"), ids, rs)
    train, test = _split(ids, d)
    xtr = emb[[rows[ids[i]] for i in train]]
    feats = np.load(str(tmp_path / "data" / "isi-feats.npy"))
    if branch == "n2v":
        tuned, trows = write_embeddings(os.path.join(embed_dir, "val-test"), ids, rs)
        xte = tuned[[trows[ids[i]] for i in test]]
        want = ["Using n2v vectors.", "Running regression.."] + _reference_lines(xtr, labels[train], xte, labels[test],
                                                                                  "citation")
        ftr, fte = _scaled(np.hstack([feats[train], xtr]), np.hstack([feats[test], xte]))
        want += ["Running regression with feats.."] + _reference_lines(ftr, labels[train], fte, labels[test], "citation")
    elif branch == "feat":
        embed_dir = "feat"
        want = ["Using only features..", "Running regression.."] + _reference_lines(feats[train], labels[train],
                                                                                   feats[test], labels[test], "citation")
    else:
        xte = emb[[rows[ids[i]] for i in test]]
        want = ["Running regression.."] + _reference_lines(xtr, labels[train], xte, labels[test], "citation")
    citation_eval.main([str(tmp_path / "data"), embed_dir, "test", "--labels_dir", str(lab_dir)], device="cpu")
    assert capsys.readouterr().out.splitlines() == ["Loading data..."] + want


def test_citation_labels_default_to_the_reference_location():
    from graphsage_b200.eval_scripts import citation_eval, parse_args
    assert citation_eval.LABELS_DIR == "/dfs/scratch0/scisurv/clean"
    args = parse_args("x", ["a", "b", "test"], "h", extra=[(("--labels_dir",), dict(default=citation_eval.LABELS_DIR))])
    assert args.labels_dir == citation_eval.LABELS_DIR and args.gpu == 0
