"""numpy restatement of the host-table staging (graphsage_b200.HostFeatures.stage: gs_halo_claim over a one-shard table
whose remap is the cache map, gs_host_fetch, gs_host_translate).

Working set: [C cached rows | 1 zero row | staged rows].  Over the id lists in order, every distinct id in [0, N) that is
not cached is staged once, on its first sighting (the device takes slots in whatever order its threads win them; the
rows and the translated lists agree with this order up to that permutation).  Cached ids are never staged; ids outside
[0, N) - the dummy id N included - read the zero row, as gather_clamped does.  So row(translate(id)) of the working set
is table[clamp(id)] for every id.
"""
import numpy as np


def clamp_ids(ids, n_nodes):
    """The table row an id reads: itself in [0, N), else the dummy row N."""
    ids = np.asarray(ids, dtype=np.int64)
    return np.where((ids < 0) | (ids >= n_nodes), n_nodes, ids)


def claim(lists, cache_ids, n_nodes):
    """The staged ids, in first-sighting order over the lists."""
    cached = set(int(x) for x in np.asarray(cache_ids).reshape(-1))
    seen, out = set(), []
    for ids in lists:
        for i in np.asarray(ids).reshape(-1).tolist():
            if 0 <= i < n_nodes and i not in cached and i not in seen:
                seen.add(i)
                out.append(i)
    return np.asarray(out, dtype=np.int64)


def translate(lists, cache_ids, staged, n_nodes):
    """Each list as working-set rows: cache slot, C for an invalid id, or C + 1 + its slot in `staged`."""
    cache_ids = np.asarray(cache_ids, dtype=np.int64).reshape(-1)
    C = len(cache_ids)
    row = {int(x): s for s, x in enumerate(cache_ids.tolist())}
    row.update({int(x): C + 1 + s for s, x in enumerate(np.asarray(staged).reshape(-1).tolist())})
    return [np.asarray([row.get(i, C) if 0 <= i < n_nodes else C for i in np.asarray(ids).reshape(-1).tolist()],
                       dtype=np.int64) for ids in lists]


def working_set(table, cache_ids, staged):
    """[table[cache_ids] | zero row | table[staged]] (table: [N+1, F], its last row zero)."""
    table = np.asarray(table)
    zero = np.zeros((1,) + table.shape[1:], dtype=table.dtype)
    return np.concatenate([table[np.asarray(cache_ids, dtype=np.int64)], zero,
                           table[np.asarray(staged, dtype=np.int64)]])


def stage(table, lists, cache_ids):
    """(working set, translated lists, staged ids) of one step."""
    n_nodes = np.asarray(table).shape[0] - 1
    staged = claim(lists, cache_ids, n_nodes)
    return working_set(table, cache_ids, staged), translate(lists, cache_ids, staged, n_nodes), staged
