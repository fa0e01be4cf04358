"""Dataset ingest for the `<prefix>-G.json / -id_map.json / -class_map.json / -feats.npy / -walks.txt` format
(reference graphsage/utils.py:19-104), networkx-free (graph.py).  Start-up-time host code; what the hot path consumes
are the tables built from its result (minibatch.py, gs_build_padded_adj) and the feature matrix.
"""
import json
import os
import random

import numpy as np

from .graph import Graph, node_link_graph

WALK_LEN = 5          # reference utils.py:16
N_WALKS = 50          # reference utils.py:17


def standard_scale(feats, train_ids):
    """sklearn StandardScaler().fit(feats[train_ids]).transform(feats) (reference utils.py:59-65): per-column mean and
    population standard deviation of the TRAIN rows; a zero-variance column is only centred (scale 1)."""
    train = np.asarray(feats)[train_ids].astype(np.float64)
    n = train.shape[0]
    mean = train.mean(axis=0)
    var = train.var(axis=0)
    # a column whose variance is zero or pure rounding noise is only centred (sklearn's _is_constant_feature bound)
    eps = np.finfo(np.float64).eps
    constant = var <= n * eps * var + (n * mean * eps) ** 2
    scale = np.sqrt(var)
    scale[constant] = 1.0
    return (np.asarray(feats, dtype=np.float64) - mean) / scale


def load_data(prefix, normalize=True, load_walks=False, verbose=False):
    """Returns (G, feats, id_map, walks, class_map) with the reference's conventions (utils.py:19-75):
      * node ids are ints when the graph's first node id is an int, else the JSON strings (:22-25)
      * feats is None when `<prefix>-feats.npy` is absent (:27-31)
      * class_map values are lists (multi-label) or ints (:35-41)
      * nodes without both `val` and `test` annotations are removed (:45-49)
      * every edge gets `train_removed` = either endpoint is val/test (:54-60)
      * normalize: StandardScaler fitted on the train rows (:62-68)
      * walks: list of (node, context) pairs read from `<prefix>-walks.txt` (:70-73)"""
    with open(prefix + "-G.json") as fp:
        G = node_link_graph(json.load(fp))
    conversion = (lambda n: int(n)) if isinstance(G.nodes()[0], int) else (lambda n: n)

    feats = np.load(prefix + "-feats.npy") if os.path.exists(prefix + "-feats.npy") else None
    if feats is None and verbose:
        print("No features present.. Only identity features will be used.")
    with open(prefix + "-id_map.json") as fp:
        id_map = {conversion(k): int(v) for k, v in json.load(fp).items()}
    with open(prefix + "-class_map.json") as fp:
        class_map = json.load(fp)
    lab_conversion = (lambda n: n) if isinstance(list(class_map.values())[0], list) else (lambda n: int(n))
    class_map = {conversion(k): lab_conversion(v) for k, v in class_map.items()}

    broken = [n for n in G.nodes() if "val" not in G.node[n] or "test" not in G.node[n]]
    for n in broken:
        G.remove_node(n)
    if verbose:
        print("Removed {:d} nodes that lacked proper annotations".format(len(broken)))

    for u, v in G.edges():
        a, b = G.node[u], G.node[v]
        G[u][v]["train_removed"] = bool(a["val"] or b["val"] or a["test"] or b["test"])

    if normalize and feats is not None:
        train_ids = np.array([id_map[n] for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]])
        feats = standard_scale(feats, train_ids)

    walks = []
    if load_walks:
        with open(prefix + "-walks.txt") as fp:
            for line in fp:
                walks.append(tuple(conversion(t) for t in line.split()))
    return G, feats, id_map, walks, class_map


def run_random_walks(G, nodes, num_walks=N_WALKS, rng=None):
    """Co-occurrence pairs from fixed-length uniform random walks (reference utils.py:77-92): for every start node with
    degree > 0, `num_walks` walks of WALK_LEN steps; every visited node other than the start yields (start, visited).
    `rng` needs `.choice(list)`; default the `random` module, as in the reference."""
    rng = random if rng is None else rng
    pairs = []
    for node in nodes:
        if G.degree(node) == 0:
            continue
        for _ in range(num_walks):
            curr = node
            for _ in range(WALK_LEN):
                nxt = rng.choice(G.neighbors(curr))
                if curr != node:                      # self co-occurrences are useless (utils.py:86-87)
                    pairs.append((node, curr))
                curr = nxt
    return pairs


WALK_CHUNK = 1 << 16  # starts per device call of run_random_walks_device: bounds the device memory a call needs


def run_random_walks_device(G, nodes, num_walks=N_WALKS, seed=123, device=None, counter=0, p=1.0, q=1.0):
    """run_random_walks on the GPU (ops.random_walks, contract oracle/walks.py): the same list of (node, context) tuples
    of node names, with the reference's loop and WALK_LEN, drawn from the seeded Philox stream instead of `random`.
    Row k of the CSR is G.neighbors(node) in order, so neighbour k is what rng.choice's index k would pick.  The starts
    are walked in chunks of WALK_CHUNK, each copied back before the next, so the pairs need not fit in device memory.
    p, q: node2vec's return and in-out parameters (contract oracle/biased_walks.py); p == q == 1 is the uniform walk.
    The rows are sorted for the biased walk once per call, not per chunk."""
    import torch

    from . import ops
    from .graph import to_csr
    names = G.nodes()
    pos = {n: i for i, n in enumerate(names)}
    csr = to_csr(G, pos)
    dev = torch.device("cuda") if device is None else torch.device(device)
    indptr = torch.from_numpy(csr["indptr"]).to(dev)
    indices = torch.from_numpy(csr["indices"]).to(dev)
    starts = np.array([pos[n] for n in nodes], dtype=np.int32)
    ops.check_walk_bias(p, q)
    biased = not (float(p) == 1.0 and float(q) == 1.0)
    sorted_indices = ops.csr_sort_rows(indptr, indices) if biased else None
    pairs = []
    for c0 in range(0, len(starts), WALK_CHUNK):
        chunk = torch.from_numpy(starts[c0:c0 + WALK_CHUNK]).to(dev)
        idx = ops.random_walks(indptr, indices, chunk, num_walks, WALK_LEN, seed, counter, start_offset=c0, p=p, q=q,
                               sorted_indices=sorted_indices).cpu().numpy()
        pairs += [(names[a], names[b]) for a, b in idx.tolist()]
    return pairs


def format_walks(pairs):
    """The `<prefix>-walks.txt` text the reference's script writes (utils.py:103-104): one `start<TAB>context` line per
    pair, no trailing newline."""
    return "\n".join([str(p[0]) + "\t" + str(p[1]) for p in pairs])


USAGE = "usage: python -m graphsage_b200.utils <graph_file> <out_file> [--p P] [--q Q]"


def _parse_main_args(argv):
    """(graph_file, out_file, bias): bias is {} without --p / --q, else {"p": P, "q": Q} (the one not given is 1)."""
    files, bias, k = [], {}, 0
    while k < len(argv):
        a = argv[k]
        name, eq, val = a.partition("=")
        if name in ("--p", "--q"):
            if not eq:
                if k + 1 >= len(argv):
                    raise SystemExit(USAGE)
                val, k = argv[k + 1], k + 1
            try:
                bias[name[2:]] = float(val)
            except ValueError:
                raise SystemExit("%s: %s must be a number (got %r)" % (USAGE, name, val))
        else:
            files.append(a)
        k += 1
    if len(files) != 2:
        raise SystemExit(USAGE)
    if bias:
        bias = {"p": bias.get("p", 1.0), "q": bias.get("q", 1.0)}
        from . import ops
        try:
            ops.check_walk_bias(bias["p"], bias["q"])
        except ValueError as e:
            raise SystemExit("%s: %s" % (USAGE, e))
    return files[0], files[1], bias


def main(argv=None, walker=None):
    """`python -m graphsage_b200.utils <graph_file> <out_file> [--p P] [--q Q]` (reference utils.py:94-104): the walks
    file of the train subgraph (nodes that are neither val nor test), 50 walks of WALK_LEN per node, seed 123 and
    counter 0.  --p / --q make them node2vec's biased walks (either one alone leaves the other at 1).
    walker(G, nodes) -> pairs replaces run_random_walks_device (tests supply pairs without a device); with --p / --q it
    is called as walker(G, nodes, p=P, q=Q)."""
    import sys
    argv = sys.argv[1:] if argv is None else list(argv)
    graph_file, out_file, bias = _parse_main_args(argv)
    with open(graph_file) as fp:
        G = node_link_graph(json.load(fp))
    nodes = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    G = G.subgraph(nodes)
    pairs = (run_random_walks_device if walker is None else walker)(G, nodes, **bias)
    with open(out_file, "w") as fp:
        fp.write(format_walks(pairs))
    return pairs


def write_dataset(prefix, G, feats, id_map, class_map, walks=None):
    """Write a dataset in the same on-disk format (used by tests and synthetic data generators)."""
    nodes = G.nodes()
    pos = {n: i for i, n in enumerate(nodes)}
    data = {"directed": False, "multigraph": False, "graph": {},
            "nodes": [dict(G.node[n], id=n) for n in nodes],
            "links": [dict(G[u][v], source=pos[u], target=pos[v]) for u, v in G.edges()]}
    with open(prefix + "-G.json", "w") as fp:
        json.dump(data, fp)
    with open(prefix + "-id_map.json", "w") as fp:
        json.dump({str(k): int(v) for k, v in id_map.items()}, fp)
    with open(prefix + "-class_map.json", "w") as fp:
        json.dump({str(k): v for k, v in class_map.items()}, fp)
    if feats is not None:
        np.save(prefix + "-feats.npy", np.asarray(feats))
    if walks is not None:
        with open(prefix + "-walks.txt", "w") as fp:
            fp.write("\n".join("%s\t%s" % (a, b) for a, b in walks))


__all__ = ["Graph", "node_link_graph", "load_data", "run_random_walks", "run_random_walks_device", "format_walks",
           "standard_scale", "write_dataset", "WALK_LEN", "N_WALKS"]


if __name__ == "__main__":
    main()
