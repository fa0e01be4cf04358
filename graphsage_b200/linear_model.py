"""The classifiers of the reference's eval scripts (eval_scripts/{ppi,reddit,citation}_eval.py), on the GPU.

    SGDClassifier(loss="log")   scikit-learn's plain SGD for the log loss with its defaults of the reference's pin (0.19.1):
                                L2 penalty, alpha = 1e-4, an intercept, the "optimal" learning rate, 5 epochs, a shuffle
                                before every epoch, no averaging, no class weights, X in float64.  Every binary problem
                                (one for two classes, one per class one-vs-rest, one per column of a 2-D 0/1 label matrix)
                                runs in ONE launch of gs_sgd_fit, one warp per problem.
    DummyClassifier()           0.19.1's default strategy "stratified", on the host.

Both draw from numpy's global RandomState when random_state is None, as the reference's scripts rely on after
np.random.seed(1).  The seed chains (which draws feed which problem) are scikit-learn's:
  * binary: make_dataset draws randint(1, MAX_INT), then the shuffle seed is randint(MAX_INT);
  * one-vs-rest: randint(MAX_INT, size=n_classes) from random_state, then the binary chain on RandomState(seed_i);
  * multi-output (MultiOutputClassifier): the binary chain per column, in column order, on random_state.
The reference fitted with joblib workers, so its own stream is not reproducible; this is the sequential (n_jobs=1) chain.
"""
import copy

import numpy as np
import torch

from ._lib import GS_F32, GS_F64, check, lib, ptr, stream_ptr

ALPHA = 1e-4
EPOCHS = 5
MAX_INT = np.iinfo(np.int32).max


def check_random_state(seed):
    """sklearn.utils.check_random_state: None -> numpy's global RandomState, an int -> RandomState(int)."""
    if seed is None:
        return np.random.mtrand._rand
    if isinstance(seed, np.random.RandomState):
        return seed
    return np.random.RandomState(seed)


def optimal_init(alpha=ALPHA):
    """optimal_init of _plain_sgd for the log loss: eta at t = 1 is typw / max(1, -dloss(-typw, y=1))."""
    typw = np.sqrt(1.0 / np.sqrt(alpha))
    e = np.exp(typw)
    gradient = (0.0 - 1.0 * e) / (1.0 + e)
    initial_eta0 = typw / max(1.0, gradient)
    return 1.0 / (initial_eta0 * alpha)


def binary_seed(rs):
    """fit_binary's draws on its RandomState: make_dataset's seed (unused for dense X), then the shuffle seed."""
    rs.randint(1, MAX_INT)
    return int(rs.randint(MAX_INT))


def sgd_orders(seeds, n, device, epochs=EPOCHS):
    """int32 [P, epochs, n]: the sample order of every epoch of every problem (gs_sgd_orders)."""
    seeds = torch.from_numpy(np.asarray(seeds, dtype=np.uint32).view(np.int32).copy()).to(device)
    orders = torch.empty((len(seeds), epochs, n), dtype=torch.int32, device=device)
    check(lib().gs_sgd_orders(ptr(seeds), len(seeds), n, epochs, ptr(orders), stream_ptr()))
    return orders


def sgd_fit(x, labels, orders, alpha=ALPHA):
    """(coef fp64 [P, d], intercept fp64 [P]) of gs_sgd_fit.  x: CUDA fp32 or fp64 [n, d] with unit column stride;
    labels: CUDA int32 [P, n] (> 0 positive); orders: sgd_orders(...)."""
    if x.dtype not in (torch.float32, torch.float64) or x.dim() != 2 or x.stride(1) != 1:
        raise ValueError("sgd_fit: x must be a 2-D fp32 or fp64 tensor with unit column stride")
    P, epochs, n = orders.shape
    if labels.shape != (P, n) or labels.dtype != torch.int32 or not labels.is_contiguous() or x.shape[0] != n:
        raise ValueError("sgd_fit: labels must be contiguous int32 [%d, %d] and x must have %d rows" % (P, n, n))
    d = x.shape[1]
    coef = torch.empty((P, d), dtype=torch.float64, device=x.device)
    intercept = torch.empty(P, dtype=torch.float64, device=x.device)
    check(lib().gs_sgd_fit(ptr(x), GS_F64 if x.dtype == torch.float64 else GS_F32, n, d, x.stride(0), ptr(labels), n,
                           ptr(orders), P, epochs, alpha, optimal_init(alpha), ptr(coef), d, ptr(intercept),
                           stream_ptr()))
    return coef, intercept


def _fit_problems(x, labels, seeds, device):
    """Fit the binary problems labels[p] (+1 / -1 per row of x) with shuffle seeds seeds[p] on `device`.
    Returns host fp64 (coef [P, d], intercept [P])."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("SGDClassifier.fit needs a CUDA device (there is no CPU fallback)")
    xt = torch.from_numpy(np.ascontiguousarray(x)).to(device)
    lt = torch.from_numpy(np.ascontiguousarray(labels, dtype=np.int32)).to(device)
    coef, intercept = sgd_fit(xt, lt, sgd_orders(seeds, x.shape[0], device))
    return coef.cpu().numpy(), intercept.cpu().numpy()


def _as_x(X):
    X = np.asarray(X)
    if X.dtype != np.float32:
        X = X.astype(np.float64)
    if X.ndim != 2:
        raise ValueError("X must be 2-D (got shape %s)" % (X.shape,))
    return X


def _two_classes(y):
    classes = np.unique(y)
    if len(classes) < 2:
        raise ValueError("The number of classes has to be greater than one; got %d class" % len(classes))
    return classes


class SGDClassifier(object):
    """sklearn.linear_model.SGDClassifier(loss="log") of scikit-learn 0.19.1, fitted by gs_sgd_fit.

    fit(X, y) with a 1-D y: two classes make one problem (classes_[1] positive); more are one-vs-rest over the sorted
    classes.  fit(X, Y) with a 2-D 0/1 Y is the multi-output form (MultiOutputClassifier(SGDClassifier(loss="log"))):
    one problem per column, all in the same launch; predict returns a [n, columns] matrix and classes_ is a list of
    the columns' classes.  X may be fp32 (each element is widened exactly) or anything numpy converts to fp64."""

    def __init__(self, loss="log", penalty="l2", learning_rate="optimal", average=False, random_state=None,
                 device="cuda"):
        if loss not in ("log", "log_loss"):
            raise NotImplementedError("SGDClassifier: only loss='log' is implemented (got %r)" % (loss,))
        if penalty != "l2":
            raise NotImplementedError("SGDClassifier: only penalty='l2' is implemented (got %r)" % (penalty,))
        if learning_rate != "optimal":
            raise NotImplementedError("SGDClassifier: only learning_rate='optimal' is implemented (got %r)"
                                      % (learning_rate,))
        if average:
            raise NotImplementedError("SGDClassifier: averaging is not implemented")
        self.loss, self.penalty, self.learning_rate, self.average = loss, penalty, learning_rate, average
        self.random_state, self.device = random_state, device
        self.alpha = ALPHA

    def fit(self, X, y):
        X = _as_x(X)
        y = np.asarray(y)
        if y.shape[0] != X.shape[0]:
            raise ValueError("X has %d rows, y has %d" % (X.shape[0], y.shape[0]))
        if y.ndim == 2:
            if not np.isin(y, (0, 1)).all():
                raise ValueError("the multi-output form takes a 0/1 label matrix")
            self.classes_ = [_two_classes(y[:, k]) for k in range(y.shape[1])]
            labels = np.where(y.T == 1, 1, -1)
            if self.random_state is None:
                rs = check_random_state(None)
                seeds = [binary_seed(rs) for _ in range(y.shape[1])]
            else:          # MultiOutputClassifier clones the estimator: every column starts from the same state
                seeds = [binary_seed(check_random_state(copy.deepcopy(self.random_state))) for _ in range(y.shape[1])]
            self._multi_output = True
        else:
            self.classes_ = _two_classes(y)
            self._multi_output = False
            if len(self.classes_) == 2:
                labels = np.where(y == self.classes_[1], 1, -1)[None, :]
                seeds = [binary_seed(check_random_state(self.random_state))]
            else:
                labels = np.where(y[None, :] == self.classes_[:, None], 1, -1)
                rs = check_random_state(self.random_state)
                seeds = [binary_seed(np.random.RandomState(s)) for s in rs.randint(MAX_INT, size=len(self.classes_))]
        coef, intercept = _fit_problems(X, labels, seeds, self.device)
        if not (np.isfinite(coef).all() and np.isfinite(intercept).all()):
            raise ValueError("Floating-point under-/overflow occurred. Scaling input data with StandardScaler or "
                             "MinMaxScaler might help.")
        self.coef_, self.intercept_ = coef, intercept
        return self

    def decision_function(self, X):
        x = torch.from_numpy(np.asarray(X, dtype=np.float64)).to(self.device)
        coef = torch.from_numpy(self.coef_).to(self.device)
        scores = (x @ coef.T + torch.from_numpy(self.intercept_).to(self.device)).cpu().numpy()
        return scores.ravel() if scores.shape[1] == 1 and not self._multi_output else scores

    def predict(self, X):
        scores = self.decision_function(X)
        if self._multi_output:
            return np.stack([c[(scores[:, k] > 0).astype(np.intp)] for k, c in enumerate(self.classes_)], axis=1)
        if scores.ndim == 1:
            return self.classes_[(scores > 0).astype(np.intp)]
        return self.classes_[scores.argmax(axis=1)]


class DummyClassifier(object):
    """sklearn.dummy.DummyClassifier() of scikit-learn 0.19.1 (strategy "stratified"): predict draws one
    multinomial(1, class prior) per row and output column, in column order, from random_state."""

    def __init__(self, strategy="stratified", random_state=None):
        if strategy != "stratified":
            raise NotImplementedError("DummyClassifier: only strategy='stratified' is implemented (got %r)" % (strategy,))
        self.strategy, self.random_state = strategy, random_state

    def fit(self, X, y):
        y = np.asarray(y)
        self.output_2d_ = y.ndim == 2
        y = y.reshape(len(y), -1)
        self.classes_, self.class_prior_ = [], []
        for k in range(y.shape[1]):
            classes, inverse = np.unique(y[:, k], return_inverse=True)
            counts = np.bincount(inverse.ravel())
            self.classes_.append(classes)
            self.class_prior_.append(counts / counts.sum())
        return self

    def predict(self, X):
        n = len(X)
        rs = check_random_state(self.random_state)
        cols = [c[rs.multinomial(1, prior, size=n).argmax(axis=1)] for c, prior in zip(self.classes_, self.class_prior_)]
        return np.vstack(cols).T if self.output_2d_ else cols[0]
