"""Padded-adjacency construction - the input contract of the sampler
(reference graphsage/minibatch.py:227-259, NodeMinibatchIterator.construct_adj / construct_test_adj).

Host-side, start-up-time code (the reference builds it once in numpy too).  networkx-free:
the graph is given as CSR over node indices 0..N-1.

  adj[N+1, max_degree] int32, filled with N; row N is the dummy row; a node with no usable
  neighbours keeps an all-N row; deg > max_degree -> subsample without replacement,
  deg < max_degree -> resample with replacement.
"""
import numpy as np


def _pad_row(nb, max_degree, rng):
    if len(nb) > max_degree:
        return rng.choice(nb, max_degree, replace=False)
    if len(nb) < max_degree:
        return rng.choice(nb, max_degree, replace=True)
    return nb


def construct_adj(indptr, indices, max_degree, skip_node=None, edge_removed=None, node_order=None, rng=None):
    """Train-time table (reference minibatch.py:227-245).

    skip_node[N] bool   : val/test nodes - their rows stay all-N (:232-233)
    edge_removed[nnz] bool : per CSR entry, the edge's `train_removed` flag (:234-236)
    node_order          : iteration order of nodes (decides the RNG call order); default 0..N-1
    rng                 : numpy RandomState; default RandomState(123) (reference seeds 123, minibatch.py:6)
    Returns (adj int32 [N+1, max_degree], deg float64 [N]).
    """
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices)
    n = len(indptr) - 1
    rng = np.random.RandomState(123) if rng is None else rng
    adj = np.full((n + 1, max_degree), n, dtype=np.int32)
    deg = np.zeros((n,), dtype=np.float64)
    order = range(n) if node_order is None else node_order
    for u in order:
        if skip_node is not None and skip_node[u]:
            continue
        lo, hi = indptr[u], indptr[u + 1]
        nb = indices[lo:hi]
        if edge_removed is not None:
            nb = nb[~np.asarray(edge_removed[lo:hi], dtype=bool)]
        deg[u] = len(nb)
        if len(nb) == 0:
            continue
        adj[u, :] = _pad_row(nb, max_degree, rng)
    return adj, deg


def construct_test_adj(indptr, indices, max_degree, node_order=None, rng=None):
    """Test-time table over ALL edges (reference minibatch.py:247-259)."""
    adj, _ = construct_adj(indptr, indices, max_degree, None, None, node_order, rng)
    return adj


def padded_from_csr_fast(indptr, indices, max_degree, seed=123):
    """Vectorised construction with the same distribution (not the same RNG stream) for large
    synthetic graphs: rows with deg >= max_degree keep a uniform random subset without replacement,
    rows with 0 < deg < max_degree are filled by uniform draws with replacement."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int32)
    n = len(indptr) - 1
    rs = np.random.RandomState(seed)
    deg = np.diff(indptr)
    adj = np.full((n + 1, max_degree), n, dtype=np.int32)
    small = np.nonzero((deg > 0) & (deg < max_degree))[0]
    if len(small):
        pos = (rs.random_sample((len(small), max_degree)) * deg[small, None]).astype(np.int64)
        adj[small] = indices[indptr[small, None] + pos]
    big = np.nonzero(deg >= max_degree)[0]
    if len(big):
        # random keys per entry, take the max_degree smallest keys of each row
        rows = np.repeat(big, deg[big])
        ent = np.concatenate([np.arange(indptr[u], indptr[u + 1]) for u in big]) if len(big) < 4096 else \
            (np.arange(deg[big].sum()) - np.repeat(np.cumsum(deg[big]) - deg[big], deg[big]) + np.repeat(indptr[big], deg[big]))
        keys = rs.random_sample(len(ent))
        order = np.lexsort((keys, rows))
        ent, rows = ent[order], rows[order]
        start = np.cumsum(deg[big]) - deg[big]
        rank = np.arange(len(ent)) - np.repeat(start, deg[big])
        keep = rank < max_degree
        adj[rows[keep], rank[keep]] = indices[ent[keep]]
    return adj, deg.astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# Minibatch iterators: the callers that feed the hot path its seed batches (reference graphsage/minibatch.py:8-320).
# Host-side bookkeeping only.  `G` is anything with the networkx-1.11 surface (graph.Graph).  A "feed dict" is a plain
# dict; its keys are `placeholders[name]` when a placeholders mapping is given (as the reference keys by placeholder
# object) and the names themselves otherwise.  All random draws go through `rng` (default: numpy's global legacy
# generator, which the reference seeds with 123 at import, minibatch.py:6) in the reference's call order.
# ---------------------------------------------------------------------------------------------------------------------
class _TableOwner(object):
    """Shared part of both iterators: the padded tables (construct_adj / construct_test_adj) and feed-dict keys."""

    def _setup(self, G, id2idx, placeholders, batch_size, max_degree, rng):
        self.G = G
        self.id2idx = id2idx
        self.placeholders = placeholders
        self.batch_size = batch_size
        self.max_degree = max_degree
        self.batch_num = 0
        self.rng = np.random if rng is None else rng

    def _key(self, name):
        return name if self.placeholders is None else self.placeholders[name]

    def _csr(self):
        from .graph import to_csr
        if getattr(self, "_csr_cache", None) is None:
            self._csr_cache = to_csr(self.G, self.id2idx)
        return self._csr_cache

    def construct_adj(self):
        c = self._csr()
        return construct_adj(c["indptr"], c["indices"], self.max_degree, c["val_or_test"], c["edge_removed"], c["node_order"],
                             self.rng)

    def construct_test_adj(self):
        c = self._csr()
        return construct_test_adj(c["indptr"], c["indices"], self.max_degree, c["node_order"], self.rng)

    def neighbor_csr(self, test=False):
        """(indptr int64 [N+1], indices int32) over node indices: the rows and edges construct_adj (test=False: the train
        graph - val/test nodes have empty rows, train_removed edges are dropped) or construct_test_adj (test=True: every
        edge) samples from, kept whole: no padding, no subsampling.  The input of full_neighbor_embeddings."""
        c = self._csr()
        indptr = np.asarray(c["indptr"], dtype=np.int64)
        indices = np.asarray(c["indices"], dtype=np.int32)
        if test:
            return indptr.copy(), indices.copy()
        n = len(indptr) - 1
        row = np.repeat(np.arange(n), np.diff(indptr))
        keep = ~np.asarray(c["edge_removed"], dtype=bool) & ~np.asarray(c["val_or_test"], dtype=bool)[row]
        out = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(row[keep], minlength=n), out=out[1:])
        return out, indices[keep]

    def _is_train(self, n):
        a = self.G.node[n]
        return not a["test"] and not a["val"]


class NodeMinibatchIterator(_TableOwner):
    """Supervised batches of nodes with label vectors (reference minibatch.py:178-320).

    label_map: node -> class index or multi-hot list; num_classes: width of the one-hot vector for index labels."""

    def __init__(self, G, id2idx, placeholders, label_map, num_classes, batch_size=100, max_degree=25, rng=None, **kwargs):
        self._setup(G, id2idx, placeholders, batch_size, max_degree, rng)
        self.nodes = G.nodes()
        self.label_map = label_map
        self.num_classes = num_classes
        self.adj, self.deg = self.construct_adj()
        self.test_adj = self.construct_test_adj()
        self.val_nodes = [n for n in G.nodes() if G.node[n]["val"]]
        self.test_nodes = [n for n in G.nodes() if G.node[n]["test"]]
        self.no_train_nodes_set = set(self.val_nodes + self.test_nodes)
        # the reference takes a set difference here (:214), so the initial order is CPython's set order
        candidates = set(G.nodes()).difference(self.no_train_nodes_set)
        self.train_nodes = [n for n in candidates if self.deg[id2idx[n]] > 0]   # no nodes with only val/test edges (:216)

    def _make_label_vec(self, node):
        label = self.label_map[node]
        if isinstance(label, list):
            return np.array(label)
        vec = np.zeros((self.num_classes))
        vec[label] = 1
        return vec

    def end(self):
        return self.batch_num * self.batch_size >= len(self.train_nodes)

    def batch_feed_dict(self, batch_nodes, val=False):
        batch = [self.id2idx[n] for n in batch_nodes]
        labels = np.vstack([self._make_label_vec(n) for n in batch_nodes])
        feed = {self._key("batch_size"): len(batch), self._key("batch"): batch, self._key("labels"): labels}
        return feed, labels

    def node_val_feed_dict(self, size=None, test=False):
        nodes = self.test_nodes if test else self.val_nodes
        if size is not None:
            nodes = self.rng.choice(nodes, size, replace=True)
        return self.batch_feed_dict(nodes)

    def incremental_node_val_feed_dict(self, size, iter_num, test=False):
        nodes = self.test_nodes if test else self.val_nodes
        subset = nodes[iter_num * size:min((iter_num + 1) * size, len(nodes))]
        feed, labels = self.batch_feed_dict(subset)
        return feed, labels, (iter_num + 1) * size >= len(nodes), subset

    def num_training_batches(self):
        return len(self.train_nodes) // self.batch_size + 1

    def next_minibatch_feed_dict(self):
        start = self.batch_num * self.batch_size
        self.batch_num += 1
        return self.batch_feed_dict(self.train_nodes[start:min(start + self.batch_size, len(self.train_nodes))])

    def incremental_embed_feed_dict(self, size, iter_num):
        subset = self.nodes[iter_num * size:min((iter_num + 1) * size, len(self.nodes))]
        return self.batch_feed_dict(subset), (iter_num + 1) * size >= len(self.nodes), subset

    def shuffle(self):
        self.train_nodes = self.rng.permutation(self.train_nodes)
        self.batch_num = 0


class EdgeMinibatchIterator(_TableOwner):
    """Unsupervised batches of (node, context) pairs: graph edges or random-walk co-occurrences
    (reference minibatch.py:8-176)."""

    def __init__(self, G, id2idx, placeholders, context_pairs=None, batch_size=100, max_degree=25, n2v_retrain=False,
                 fixed_n2v=False, rng=None, **kwargs):
        self._setup(G, id2idx, placeholders, batch_size, max_degree, rng)
        self.nodes = self.rng.permutation(G.nodes())            # drawn BEFORE the tables (:36-38)
        self.adj, self.deg = self.construct_adj()
        self.test_adj = self.construct_test_adj()
        edges = G.edges() if context_pairs is None else context_pairs
        self.train_edges = self.edges = self.rng.permutation(edges)
        if not n2v_retrain:
            self.train_edges = self._remove_isolated(self.train_edges)
            self.val_edges = [e for e in G.edges() if G[e[0]][e[1]]["train_removed"]]
        elif fixed_n2v:
            self.train_edges = self.val_edges = self._n2v_prune(self.edges)
        else:
            self.train_edges = self.val_edges = self.edges
        self.val_set_size = len(self.val_edges)

    def _n2v_prune(self, edges):
        return [e for e in edges if self._is_train(e[1])]

    def _remove_isolated(self, edge_list):
        """Drop pairs that touch a node with no train-time neighbours, unless an endpoint is a test-only node
        (the reference's condition, :66-68, kept verbatim in meaning: `not test or val`)."""
        kept = []
        self.missing = 0
        node = self.G.node
        for n1, n2 in edge_list:
            if n1 not in node or n2 not in node:
                self.missing += 1
                continue
            lonely = self.deg[self.id2idx[n1]] == 0 or self.deg[self.id2idx[n2]] == 0
            ok1 = (not node[n1]["test"]) or node[n1]["val"]
            ok2 = (not node[n2]["test"]) or node[n2]["val"]
            if lonely and ok1 and ok2:
                continue
            kept.append((n1, n2))
        return kept

    def end(self):
        return self.batch_num * self.batch_size >= len(self.train_edges)

    def batch_feed_dict(self, batch_edges):
        batch1 = [self.id2idx[a] for a, _ in batch_edges]
        batch2 = [self.id2idx[b] for _, b in batch_edges]
        return {self._key("batch_size"): len(batch_edges), self._key("batch1"): batch1, self._key("batch2"): batch2}

    def next_minibatch_feed_dict(self):
        start = self.batch_num * self.batch_size
        self.batch_num += 1
        return self.batch_feed_dict(self.train_edges[start:min(start + self.batch_size, len(self.train_edges))])

    def num_training_batches(self):
        return len(self.train_edges) // self.batch_size + 1

    def val_feed_dict(self, size=None):
        if size is None:
            return self.batch_feed_dict(self.val_edges)
        ind = self.rng.permutation(len(self.val_edges))
        return self.batch_feed_dict([self.val_edges[i] for i in ind[:min(size, len(ind))]])

    def incremental_val_feed_dict(self, size, iter_num):
        sub = self.val_edges[iter_num * size:min((iter_num + 1) * size, len(self.val_edges))]
        return self.batch_feed_dict(sub), (iter_num + 1) * size >= len(self.val_edges), sub

    def incremental_embed_feed_dict(self, size, iter_num):
        sub = self.nodes[iter_num * size:min((iter_num + 1) * size, len(self.nodes))]
        pairs = [(n, n) for n in sub]
        return self.batch_feed_dict(pairs), (iter_num + 1) * size >= len(self.nodes), pairs

    def label_val(self):
        train, val = [], []
        for n1, n2 in self.G.edges():
            (train if self._is_train(n1) and self._is_train(n2) else val).append((n1, n2))
        return train, val

    def shuffle(self):
        self.train_edges = self.rng.permutation(self.train_edges)
        self.nodes = self.rng.permutation(self.nodes)
        self.batch_num = 0
