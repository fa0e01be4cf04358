"""CPU: the alias-table contract of WeightedNeighborSampler (oracle/alias_sampling.py).  The table invariants on hand-made
rows of every weight kind, alias_law against the integer masses and the stated bound against w / S, the vectorised
oracle against a scalar restatement of build and draw, k-hop against successive calls, the frequencies of 10^6 draws,
and the sampler's argument errors, set_graph cache and model wiring with the oracle standing in for the kernels."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import alias_sampling as al
from oracle.philox import mulhi32

CAP = 1 << 32
F32 = np.float32


def _csr(rows):
    """rows: list of (ids, weights) -> (indptr, indices, w)."""
    indptr = np.concatenate([[0], np.cumsum([len(r[0]) for r in rows])]).astype(np.int64)
    indices = np.concatenate([np.asarray(r[0], np.int32) for r in rows] + [np.zeros(0, np.int32)])
    w = np.concatenate([np.asarray(r[1], F32) for r in rows] + [np.zeros(0, F32)])
    return indptr, indices, w


ROWS = [
    ([1, 2, 3], [1.0, 2.0, 3.0]),                                  # positive
    ([0, 4, 5, 6], [0.0, -0.0, 3.0, 1.0]),                         # zeros
    ([2, 2, 7], [-1.0, 5.0, -3e38]),                               # negative, duplicate ids
    ([3, 8], [np.nan, 2.0]),                                       # NaN
    ([9], [np.inf]),                                               # +inf alone
    ([1, 2, 3, 4], [np.inf, 1.0, np.inf, 1e38]),                   # +inf mixed
    ([5, 6, 7], [1e-45, 1e-40, 1.0]),                              # subnormal
    ([1, 2], [1e38, 1e38]),                                        # 1e38
    ([4, 4, 4, 4, 4], [0.5] * 5),                                  # equal weights, duplicates
    ([10, 10, 3], [1.0, 2.0, 0.25]),                               # self loop (row 10)
    ([], []),                                                      # empty
    ([1, 2, 3], [0.0, np.nan, -2.0]),                              # no eligible entry
    (list(range(11)) * 7, list(np.random.RandomState(0).exponential(1, 77))),
]


def _eligible(w):
    w = np.asarray(w, F32)
    if np.isposinf(w).any():
        return np.isposinf(w), np.where(np.isposinf(w), 1.0, 0.0)
    with np.errstate(invalid="ignore"):
        e = np.isfinite(w) & (w > 0)
    return e, np.where(e, w.astype(np.float64), 0.0)


def test_table_invariants_on_hand_made_rows():
    indptr, indices, w = _csr(ROWS)
    N = len(indptr) - 1
    m = al.masses(indptr, w)
    tab = al.build_table(indptr, indices, w).view(np.uint32)
    for v in range(N):
        a, z = indptr[v], indptr[v + 1]
        d = z - a
        if d == 0:
            continue
        e, wv = _eligible(w[a:z])
        mv = [int(x) for x in m[a:z]]
        rec = tab[a:z]
        assert (rec[:, 3] == 0).all()
        if not e.any():
            assert sum(mv) == 0
            assert (rec[:, 1] == N).all() and (rec[:, 2] == N).all() and (rec[:, 0] == 0).all()
            continue
        assert sum(mv) == d * CAP
        assert all(x >= 1 for x, ok in zip(mv, e) if ok) and all(x == 0 for x, ok in zip(mv, e) if not ok)
        assert (rec[:, 1].view(np.int32) == indices[a:z]).all()
        for b in range(d):                                          # a full bucket aliases itself
            if mv[b] == CAP and rec[b, 0] == 0:
                assert rec[b, 2] == rec[b, 1]
        S = 0.0
        for x in wv[e]:
            S += float(x)
        ne = int(e.sum())
        for x, ok, wj in zip(mv, e, wv):
            if ok:
                assert abs(Fraction(x) - Fraction(float(wj)) * d * CAP / Fraction(S)) <= al.alias_mass_bound(ne, d)


def test_law_equals_the_masses_and_is_within_the_bound():
    rs = np.random.RandomState(1)
    rows = ROWS + [(list(rs.randint(0, 30, 200)), list(np.exp(2 * rs.randn(200)))) for _ in range(5)]
    indptr, indices, w = _csr(rows)
    N = len(indptr) - 1
    m = al.masses(indptr, w)
    tab = al.build_table(indptr, indices, w)
    for v in range(N):
        a, z = indptr[v], indptr[v + 1]
        law, den = al.alias_law(tab, indptr, v)
        e, wv = _eligible(w[a:z])
        if z == a or not e.any():
            assert law == {N: den} or law == {N: 1}
            continue
        want = {}
        for j in range(a, z):
            if m[j]:
                want[int(indices[j])] = want.get(int(indices[j]), 0) + int(m[j])
        assert law == want and den == (z - a) * CAP
        S = sum(Fraction(float(x)) for x in wv[e])
        for u, c in law.items():
            p = sum(Fraction(float(wv[j - a])) for j in range(a, z) if indices[j] == u and e[j - a]) / S
            n_u = sum(1 for j in range(a, z) if indices[j] == u and e[j - a])
            assert abs(Fraction(c, den) - p) <= Fraction(n_u * al.alias_mass_bound(int(e.sum()), z - a)) / den + \
                Fraction(1, 1 << 40)


# ---------------------------------------------------------------- a scalar restatement of build and draw
def _scalar_masses(w):
    d = len(w)
    e, wv = _eligible(w)
    ne = int(e.sum())
    if ne == 0:
        return [0] * d
    S = 0.0
    for j in range(d):
        if e[j]:
            S = S + float(wv[j])
    R = d * CAP - ne
    Rf = float(R)
    b = []
    for j in range(d):
        if e[j]:
            x = min((float(wv[j]) / S) * Rf, Rf)
            b.append(min(int(x), R))
        else:
            b.append(0)
    rem = R - sum(b)
    out, rank, pre = [], 0, 0
    for j in range(d):
        if e[j]:
            if rem >= 0:
                out.append(1 + b[j] + rem // ne + (1 if rank < rem % ne else 0))
            else:
                out.append(1 + b[j] - min(b[j], max(0, -rem - pre)))
            rank += 1
        else:
            out.append(0)
        pre += b[j]
    return out


def _scalar_sweep(m, ids, pad):
    """The same sweep written with explicit queues of lights and heavies."""
    d = len(m)
    if sum(m) == 0:
        return [(0, pad, pad)] * d
    rec = [None] * d
    lights = [i for i in range(d) if m[i] < CAP]
    heavies = [i for i in range(d) if m[i] >= CAP]
    li, hi = 0, 0
    w = m[heavies[0]]
    while hi < len(heavies):
        j = heavies[hi]
        if w > CAP:
            i = lights[li]
            rec[i] = (m[i], ids[i], ids[j])
            w -= CAP - m[i]
            li += 1
        elif w == CAP:
            rec[j] = (0, ids[j], ids[j])
            hi += 1
            w = m[heavies[hi]] if hi < len(heavies) else 0
        else:
            j2 = heavies[hi + 1]
            rec[j] = (w, ids[j], ids[j2])
            w = m[j2] - (CAP - w)
            hi += 1
    assert li == len(lights) and all(r is not None for r in rec)
    return rec


def _scalar_draw(indptr, rec, v, N, seed, counter, t, j):
    from oracle.philox import philox4x32_10, split64
    if not 0 <= v < N or indptr[v + 1] == indptr[v]:
        return N
    d = int(indptr[v + 1] - indptr[v])
    clo, chi = split64(counter)
    r = philox4x32_10(np.array([clo, chi, t, al.STREAM_ALIAS + (j >> 1)], np.uint32),
                      np.array(split64(seed), np.uint32))
    a, b = (int(r[2]), int(r[3])) if j & 1 else (int(r[0]), int(r[1]))
    thr, i, al_ = rec[int(indptr[v]) + int(mulhi32(a, d))]
    return i if b < thr else al_


def test_vectorised_oracle_equals_the_scalar_restatement():
    rs = np.random.RandomState(2)
    rows = ROWS + [(list(rs.randint(0, 30, n)), list(np.exp(3 * rs.randn(n)))) for n in (1, 2, 33, 500)]
    indptr, indices, w = _csr(rows)
    N = len(indptr) - 1
    m = al.masses(indptr, w)
    tab = al.build_table(indptr, indices, w)
    rec = []
    for v in range(N):
        a, z = indptr[v], indptr[v + 1]
        mv = _scalar_masses(w[a:z])
        assert mv == [int(x) for x in m[a:z]], v
        rec += _scalar_sweep(mv, [int(x) for x in indices[a:z]], N)
    t = tab.view(np.uint32)
    assert [(int(a), int(np.uint32(b).view(np.int32)), int(np.uint32(c).view(np.int32))) for a, b, c, _ in t] == \
        [(a, b, c) for a, b, c in rec]
    ids = np.array(list(range(-1, N + 2)) * 3, np.int32)
    got = al.sample(indptr, tab, ids, 5, 77, 9)
    for tt, v in enumerate(ids):
        for j in range(5):
            assert got[tt, j] == _scalar_draw(indptr, rec, int(v), N, 77, 9, tt, j)


def test_khop_equals_successive_calls():
    rs = np.random.RandomState(3)
    rows = [(list(rs.randint(0, 40, n)), list(rs.exponential(1, n))) for n in rs.randint(0, 30, 40)]
    indptr, indices, w = _csr(rows)
    tab = al.build_table(indptr, indices, w)
    seeds = np.array([0, 5, 39, -1, 40, 12], np.int32)
    outs = al.sample_khop(indptr, tab, seeds, [3, 4, 2], 5, 100)
    cur = seeds
    for h, k in enumerate([3, 4, 2]):
        cur = al.sample(indptr, tab, cur, k, 5, 100 + h).reshape(-1)
        assert np.array_equal(outs[h], cur)
    assert len(outs[2]) == 6 * 3 * 4 * 2


def test_frequencies_of_a_million_draws():
    ids_row = [3, 1, 4, 1, 5, 9, 2, 6]
    w = [0.5, 2.0, 0.0, 1.0, 8.0, 1e-30, np.nan, 3.0]
    indptr, indices, wt = _csr([(ids_row, w)])
    tab = al.build_table(indptr, indices, wt)
    n = 1 << 20
    got = al.sample(indptr, tab, np.zeros(n, np.int32), 1, 11, 0).reshape(-1)
    law, den = al.alias_law(tab, indptr, 0)
    cnt = np.bincount(got, minlength=10)
    for u in range(10):
        p = law.get(u, 0) / den
        assert abs(cnt[u] - n * p) <= 5 * np.sqrt(n * p * (1 - p)) + 1e-9, u
    assert cnt[4] == 0 and cnt[2] == 0


# ---------------------------------------------------------------- the sampler, with the oracle standing in for the kernels
@pytest.fixture
def fake_kernels(monkeypatch):
    from graphsage_b200 import ops, neigh_samplers
    builds = []

    def table(indptr, indices, weights):
        if not isinstance(weights, torch.Tensor) or weights.dtype != torch.float32 or weights.dim() != 1:
            raise TypeError("weights must be a 1-D float32 tensor")
        if weights.numel() != indices.numel():
            raise ValueError("weights needs one weight per CSR entry")
        builds.append(1)
        return torch.from_numpy(al.build_table(indptr.numpy(), indices.numpy(), weights.numpy()))

    def sample(indptr, tab, ids, k, seed, counter, counter_dev=None):
        return torch.from_numpy(al.sample(indptr.numpy(), tab.numpy(), ids.numpy(), k, seed, counter))

    def khop(indptr, tab, seeds, fanouts, seed, counter, counter_dev=None):
        return [torch.from_numpy(x) for x in al.sample_khop(indptr.numpy(), tab.numpy(), seeds.numpy(), fanouts,
                                                            seed, counter)]
    monkeypatch.setattr(ops, "csr_alias_table", table)
    monkeypatch.setattr(ops, "sample_alias", sample)
    monkeypatch.setattr(ops, "sample_alias_khop", khop)
    monkeypatch.setattr(ops, "require_cuda", lambda *t: None)
    monkeypatch.setattr(neigh_samplers.ops, "require_cuda", lambda *t: None)
    return builds


def _graph():
    rs = np.random.RandomState(4)
    rows = [(list(rs.randint(0, 30, n)), list(np.exp(rs.randn(n)))) for n in rs.randint(0, 12, 30)]
    indptr, indices, w = _csr(rows)
    return torch.from_numpy(indptr), torch.from_numpy(indices), torch.from_numpy(w)


def test_sampler_argument_errors(fake_kernels):
    import graphsage_b200 as gs
    ip, ix, w = _graph()
    with pytest.raises(TypeError):
        gs.WeightedNeighborSampler(ip, ix, w.double())
    with pytest.raises(ValueError):
        gs.WeightedNeighborSampler(ip, ix, w[:-1].clone())
    with pytest.raises(TypeError):
        gs.WeightedNeighborSampler(ip.int(), ix, w)
    with pytest.raises(TypeError):
        gs.WeightedNeighborSampler(ip, ix.long(), w)


def test_ops_argument_errors_without_a_device():
    from graphsage_b200 import ops
    ip, ix, w = _graph()
    with pytest.raises(RuntimeError):                 # host tensors: the hot path is CUDA-only
        ops.csr_alias_table(ip, ix, w)


def test_set_graph_caches_tables_by_tensor_identity(fake_kernels):
    import graphsage_b200 as gs
    ip, ix, w = _graph()
    w2 = w * 2
    s = gs.WeightedNeighborSampler(ip, ix, w, seed=3)
    t1 = s.table
    s.set_graph(ip, ix, w2)
    assert s.table is not t1 and len(fake_kernels) == 2
    s.set_graph(ip, ix, w)
    assert s.table is t1 and len(fake_kernels) == 2            # swapping back does not rebuild
    w.mul_(1.0)                                                # a new _version: rebuilt; a captured graph may read t1
    s.set_graph(ip, ix, w)
    assert len(fake_kernels) == 3 and s.table is not t1 and len(s._tables) == 3


def test_model_sample_wiring(fake_kernels):
    import graphsage_b200 as gs
    from graphsage_b200.models import SampleAndAggregate
    ip, ix, w = _graph()
    s = gs.WeightedNeighborSampler(ip, ix, w, seed=9)
    infos = [gs.SAGEInfo("node", s, 5, 8), gs.SAGEInfo("node", s, 3, 8)]
    m = SampleAndAggregate.__new__(SampleAndAggregate)
    m.batch_size = 4
    seeds = torch.tensor([0, 7, 29, 30], dtype=torch.int32)
    samples, support = m.sample(seeds, infos)                   # the one-launch path: sample_khop, hop order (3, 5)
    want = al.sample_khop(ip.numpy(), s.table.numpy(), seeds.numpy(), [3, 5], 9, 0)
    assert support == [1, 3, 15] and s.counter == 2
    for g, x in zip(samples[1:], want):
        assert np.array_equal(g.numpy(), x)
    infos = [gs.SAGEInfo("node", s, 70, 8), gs.SAGEInfo("node", s, 3, 8)]   # fanout > 64: one call per hop
    samples, _ = m.sample(seeds, infos)
    want = al.sample_khop(ip.numpy(), s.table.numpy(), seeds.numpy(), [3, 70], 9, 2)
    assert s.counter == 4
    for g, x in zip(samples[1:], want):
        assert np.array_equal(g.reshape(-1).numpy(), x)
