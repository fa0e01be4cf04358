"""numpy restatement of gs_host_gather_rows_f32 (HostFeatures.gather_rows_f32): the layer-0 rows of a sampled block set
read from a host table with a device cache, widened to fp32.

    row(id) = cache[cache_slot[id]]   if 0 <= id < N and cache_slot[id] >= 0
            = zero row                if id is outside [0, N) - the dummy id N included (nothing is read)
            = host[id]                otherwise
    out[i, :F] = widen(row(ids[i])),  out[i, F:out_pitch] = 0

widen: fp32 rows as stored; bf16 rows (given as their uint16 bits) exactly; GS_I8ROW byte rows dequantised as every int8
reader does (oracle/int8_rows.py: fl(float(q) * s), the scale read from the row itself).  Duplicate ids read the same
row.  Every step is exact or one IEEE float32 operation, so this gives the device's bytes.
"""
import numpy as np

from oracle import int8_rows


def widen(rows, F, kind):
    """Stored rows -> float32 [n, F].  kind: "f32" (float32 rows), "bf16" (uint16 bit rows) or "i8row" (uint8 rows)."""
    rows = np.asarray(rows)
    if kind == "f32":
        return np.ascontiguousarray(rows[:, :F], dtype=np.float32)
    if kind == "bf16":
        bits = np.ascontiguousarray(rows[:, :F]).astype(np.uint32) << 16
        return bits.view(np.float32)
    if kind == "i8row":
        return int8_rows.dequantize(*int8_rows.unpack(rows, F))
    raise ValueError("kind must be f32, bf16 or i8row")


def gather_rows_f32(host, cache, cache_slot, ids, F, kind, out_pitch=None):
    """fp32 [n, out_pitch] (default out_pitch = round_up(F, 8)).  host: the [N+1, .] stored rows; cache: the cached
    rows (same layout); cache_slot: int [N+1], -1 for an uncached id."""
    host, cache = np.asarray(host), np.asarray(cache)
    n_nodes = host.shape[0] - 1
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    out_pitch = (F + 7) // 8 * 8 if out_pitch is None else int(out_pitch)
    out = np.zeros((len(ids), out_pitch), dtype=np.float32)
    slot = np.asarray(cache_slot, dtype=np.int64).reshape(-1)
    ok = (ids >= 0) & (ids < n_nodes)
    s = slot[np.where(ok, ids, 0)]
    cached, linked = ok & (s >= 0), ok & (s < 0)
    out[linked, :F] = widen(host, F, kind)[ids[linked]]
    if cached.any():
        out[cached, :F] = widen(cache, F, kind)[s[cached]]
    return out


def link_rows(ids, cache_slot, n_nodes):
    """The ids whose rows cross the host link: in [0, N) and uncached (duplicates counted, as the device reads them)."""
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    slot = np.asarray(cache_slot, dtype=np.int64).reshape(-1)
    ok = (ids >= 0) & (ids < n_nodes)
    return ids[ok][slot[ids[ok]] < 0]
