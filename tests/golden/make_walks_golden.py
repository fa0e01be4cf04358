"""Generate tests/golden/walks.npz - the random-walk co-occurrence pairs - by executing the reference's own
run_random_walks (graphsage/utils.py:77-92) over this project's Graph, with the module's `random` replaced by
oracle.walks.ContractChoice (Python's unseeded stream is unobtainable; the contract is Philox, oracle/walks.py).
The reference module is executed from where it lies with a stub for its networkx import and version check; its
"Done walks" prints are discarded.  Run where the reference lies; nothing from it is copied.

    python tests/golden/make_walks_golden.py

Cases (pairs are stored as positions in the case's node list, uint16):
  script  the toy-ppi slice (toy_ppi.npz): the train subgraph walked from the train nodes, as the reference's
          `python -m graphsage.utils` does (50 walks of WALK_LEN = 5, seed 123, counter 0)
  n2v     the full slice walked from the val/test nodes, as the Node2Vec trainer's second phase does
  hand    string node ids with a self loop, an isolated node and a duplicated start (3 walks, seed 7, counter 5)
"""
import contextlib
import io
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from graphsage_b200.graph import Graph  # noqa: E402
from oracle.walks import ContractChoice  # noqa: E402

REFERENCE_UTILS = "/root/reference/graphsage/utils.py"
WALK_LEN = 5


def reference_utils():
    """The reference's graphsage/utils.py as a namespace, its networkx imports stubbed."""
    nx = types.ModuleType("networkx")
    nx.__version__ = "1.11"
    readwrite = types.ModuleType("networkx.readwrite")
    readwrite.json_graph = types.SimpleNamespace()
    nx.readwrite = readwrite
    saved = {k: sys.modules.get(k) for k in ("networkx", "networkx.readwrite")}
    sys.modules.update({"networkx": nx, "networkx.readwrite": readwrite})
    try:
        ns = {"__name__": "reference_graphsage_utils"}
        with open(REFERENCE_UTILS) as fp:
            exec(compile(fp.read(), REFERENCE_UTILS, "exec"), ns)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    assert ns["WALK_LEN"] == WALK_LEN
    return ns


def reference_walks(ref, G, nodes, num_walks, seed, counter):
    walked = [i for i, n in enumerate(nodes) if G.degree(n) > 0]
    rng = ContractChoice(walked, num_walks, WALK_LEN, seed, counter)
    ref["random"] = rng
    with contextlib.redirect_stdout(io.StringIO()):
        pairs = ref["run_random_walks"](G, nodes, num_walks=num_walks)
    assert rng.done()
    return pairs


def toy_graph():
    """The toy-ppi slice as a Graph, nodes and links in the fixture's order (what node_link_graph builds from it)."""
    d = np.load(os.path.join(HERE, "toy_ppi.npz"))
    G = Graph()
    ids = [int(u) for u in d["ids"]]
    for u, v, t in zip(ids, d["val"], d["test"]):
        G.add_node(u, val=bool(v), test=bool(t))
    for a, b in zip(d["src"], d["dst"]):
        G.add_edge(ids[int(a)], ids[int(b)])
    return G


def hand_graph():
    G = Graph()
    for n in ["a", "b", "c", "d", "e", "lone", "f"]:
        G.add_node(n)
    for u, v in [("a", "b"), ("b", "c"), ("c", "a"), ("c", "c"), ("c", "d"), ("d", "e"), ("e", "e"), ("f", "a")]:
        G.add_edge(u, v)
    nodes = ["c", "lone", "e", "a", "c", "f", "b", "d", "e"]
    return G, nodes


def as_positions(pairs, names):
    pos = {n: i for i, n in enumerate(names)}
    return np.array([[pos[a], pos[b]] for a, b in pairs], dtype=np.uint16).reshape(-1, 2)


def main():
    ref = reference_utils()
    out = {}
    G = toy_graph()
    train = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    sub = G.subgraph(train)
    out["script_pairs"] = as_positions(reference_walks(ref, sub, train, 50, 123, 0), sub.nodes())
    other = [n for n in G.nodes() if G.node[n]["val"] or G.node[n]["test"]]
    out["n2v_pairs"] = as_positions(reference_walks(ref, G, other, 50, 123, 0), G.nodes())
    H, nodes = hand_graph()
    out["hand_pairs"] = as_positions(reference_walks(ref, H, nodes, 3, 7, 5), H.nodes())
    out["hand_names"] = np.array(H.nodes())
    path = os.path.join(HERE, "walks.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
