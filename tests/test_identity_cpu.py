"""CPU: trainable node embeddings (identity_dim > 0) as the reference builds them.

tests/golden/identity.npz holds what the reference's own constructor lines (supervised_models.py:51-67, models.py:229-245)
and its aggregate() produced under the numpy TF shim, with features and without.  The oracle's op sequence on
concat([E, X]) (or on E alone) must reproduce it: embeddings first, dims[0] = d + F, a [N+1, d] table whose dummy row is
an ordinary (non-zero) glorot row."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import torch_ref


@pytest.mark.parametrize("model", ["sup", "unsup"])
@pytest.mark.parametrize("tag", ["feat", "nofeat"])
def test_reference_identity_table_layout_and_forward(model, tag):
    g = load_golden("identity")
    key = "%s_%s_" % (model, tag)
    adj, feats, seeds, fan, d = g["adj"], g["feats"], g["seeds"], [int(x) for x in g["fanout"]], int(g["identity_dim"])
    E = g[key + "embeds"]
    n_rows = adj.shape[0]
    assert E.shape == (n_rows, d)                                  # one row per adjacency row, the dummy row N included
    r = np.sqrt(6.0 / (n_rows + d))                                # glorot-uniform over [N+1, d]
    assert np.abs(E).max() <= r and np.abs(E).max() > 0.5 * r
    assert np.any(E[n_rows - 1] != 0)                              # the dummy row is NOT zero in the embedding columns
    table = np.concatenate([E, feats], axis=1) if tag == "feat" else E
    np.testing.assert_array_equal(g[key + "features"], table)      # concat([embeds, features], axis=1)
    assert int(g[key + "dims"][0]) == d + (feats.shape[1] if tag == "feat" else 0)
    aggs = [{k: torch.from_numpy(g["%sL%d_%s" % (key, li, k)]) for k in ("self_weights", "neigh_weights")}
            for li in range(len(fan))]
    out = torch_ref.forward(torch.from_numpy(adj), torch.from_numpy(table), torch.from_numpy(seeds), fan, aggs, True, "mean",
                            123, 40, normalize=False)
    assert rel_err(out.numpy(), g[key + "out"]) < 1e-5
