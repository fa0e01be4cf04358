"""CPU restatement of the pooling branch's backward through the fused bf16 kernels (B1 / B2 of include/graphsage_b200.h,
gs_pool_mlp_backward_dp / gs_pool_mlp_backward_dw).

For one hop: X [n*k, K] the gathered rows, pre = X Wm (fp32), b the MLP bias, dhp [n, hidden] the gradient of the
pooled output.  B1 works on 128-row tiles of G = 128 // k whole fanout groups:
  max:  hp = relu(max_j pre_j + b); if hp > 0, count = #{j : fl(pre_j + b) == hp} and
        dpre_j = dhp / count where fl(pre_j + b) == hp, else 0; if hp == 0 every dpre_j = 0
        (TensorFlow's reduce_max gradient, ties split evenly, times the ReLU mask: the bias is added before comparing)
  mean: dpre_j = (dhp / k) * [fl(pre_j + b) > 0]
  dP = bf16(dpre), round to nearest even
  dbm partial of (tile, column) = (sum over even g of s_g) + (sum over odd g of s_g), each stream in increasing g from
        0.0, s_g = the sum of group g's dpre_j in increasing j from 0.0; all in fp32
B2's dbm: the tile partials summed in increasing tile order in groups of 32 tiles, then the group sums in order.

The dP^T tile images B1 writes: image (tile, slice, half) of 128 hidden rows x 128 bytes, swizzled; 16-byte chunk c of
row n sits at n * 128 + ((c ^ (n & 7)) << 4) and holds rows half * 64 + 8c .. + 7 of hidden unit slice * 128 + n.
"""
import numpy as np

DBM_GROUP = 32
MAX_CHUNKS, MIN_BLOCKS_PER_CHUNK = 32, 8


def dw_chunks(n, k):
    """B2's split of the row blocks (64 row slots, two per tile): (blocks, blocks per chunk, chunks).  At most MAX_CHUNKS
    chunks of equal length (the last one shorter), at least MIN_BLOCKS_PER_CHUNK blocks each; the chunk partials of dWm are
    added in chunk order."""
    G = 128 // k
    blocks = 2 * ((n + G - 1) // G)
    per = max(-(-blocks // MAX_CHUNKS), MIN_BLOCKS_PER_CHUNK)
    return blocks, per, -(-blocks // per)


def bf16_round(x):
    """fp32 -> the nearest bf16 value (ties to even), returned as fp32."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def dpre(pre, bias, dhp, k, pool):
    """pre [n*k, hidden] fp32 (the exact products X Wm), bias [hidden], dhp [n, hidden] -> dpre [n*k, hidden] fp32."""
    pre = np.asarray(pre, np.float32)
    n, hid = dhp.shape
    z = (pre.reshape(n, k, hid) + np.asarray(bias, np.float32)[None, None, :]).astype(np.float32)   # fl(pre + b)
    dhp = np.asarray(dhp, np.float32)
    if pool == "mean":
        q = (dhp / np.float32(k)).astype(np.float32)
        out = np.where(z > 0, q[:, None, :], np.float32(0))
    else:
        hp = np.maximum(z.max(axis=1), np.float32(0))
        sel = (z == hp[:, None, :]) & (hp[:, None, :] > 0)
        cnt = sel.sum(axis=1)
        q = np.where(cnt > 0, dhp / np.maximum(cnt, 1).astype(np.float32), np.float32(0)).astype(np.float32)
        out = np.where(sel, q[:, None, :], np.float32(0))
    return out.astype(np.float32).reshape(n * k, hid)


def dbm_partials(dp_rows, n, k):
    """B1's per-(tile, column) sums of dpre [n*k, hidden] -> [n_tiles, hidden] fp32, in the order of the module doc."""
    hid = dp_rows.shape[1]
    G = 128 // k
    n_tiles = (n + G - 1) // G
    g3 = np.asarray(dp_rows, np.float32).reshape(n, k, hid)
    s = np.zeros((n, hid), np.float32)
    for j in range(k):                                   # per-group sums in j order
        s = (s + g3[:, j, :]).astype(np.float32)
    out = np.zeros((n_tiles, hid), np.float32)
    for t in range(n_tiles):
        acc = [np.zeros(hid, np.float32), np.zeros(hid, np.float32)]
        for g in range(G):
            gg = t * G + g
            if gg >= n:
                break
            acc[g & 1] = (acc[g & 1] + s[gg]).astype(np.float32)
        out[t] = (acc[0] + acc[1]).astype(np.float32)
    return out


def dbm_combine(parts):
    """B2's sum of the tile partials [n_tiles, hidden]: groups of DBM_GROUP tiles in order, then the group sums."""
    parts = np.asarray(parts, np.float32)
    groups = []
    for g0 in range(0, parts.shape[0], DBM_GROUP):
        acc = np.zeros(parts.shape[1], np.float32)
        for t in range(g0, min(g0 + DBM_GROUP, parts.shape[0])):
            acc = (acc + parts[t]).astype(np.float32)
        groups.append(acc)
    acc = np.zeros(parts.shape[1], np.float32)
    for g in groups:
        acc = (acc + g).astype(np.float32)
    return acc


def tile_rows(n, k):
    """Row slot -> gathered row (or -1 for padding) of every B1 tile: [n_tiles, 128] int64."""
    G = 128 // k
    n_tiles = (n + G - 1) // G
    slots = np.arange(128)
    rows = np.arange(n_tiles)[:, None] * (G * k) + slots[None, :]
    return np.where((slots[None, :] < G * k) & (rows < n * k), rows, -1)


def dp_images_to_rows(buf, n, k, hidden):
    """B1's output buffer (uint8) -> (dP [n*k, hidden] fp32 from the images, padding slots [n_tiles, 128, hidden] fp32,
    dbm partials [n_tiles, hidden] fp32)."""
    G = 128 // k
    n_tiles = (n + G - 1) // G
    S = hidden // 128
    img = np.asarray(buf, np.uint8)[:n_tiles * hidden * 256].view(np.uint16).reshape(n_tiles, S, 2, 128, 64)
    nn = np.arange(128)[:, None]
    e = np.arange(64)[None, :]
    src = ((e // 8) ^ (nn & 7)) * 8 + (e % 8)            # element of row n that holds slot 8c + i
    vals = np.take_along_axis(img, np.broadcast_to(src, img.shape), axis=-1)      # [t, s, half, n, slot in half]
    full = (vals.astype(np.uint32) << 16).view(np.float32)
    full = full.transpose(0, 2, 4, 1, 3).reshape(n_tiles, 128, hidden)            # [t, slot, hidden]
    rows = tile_rows(n, k)
    dP = np.zeros((n * k, hidden), np.float32)
    valid = rows >= 0
    dP[rows[valid]] = full[valid]
    parts = np.asarray(buf, np.uint8)[n_tiles * hidden * 256:n_tiles * hidden * 260].view(np.float32).reshape(n_tiles, hidden)
    return dP, full, parts


def rows_to_dp_images(dP, n, k):
    """The inverse of dp_images_to_rows: dP [n*k, hidden] fp32 (bf16 values) -> a B1 output buffer (uint8) holding its dP^T
    images and zero dbm partials."""
    hidden = dP.shape[1]
    G = 128 // k
    n_tiles = (n + G - 1) // G
    S = hidden // 128
    full = np.zeros((n_tiles, 128, hidden), np.float32)
    rows = tile_rows(n, k)
    valid = rows >= 0
    full[valid] = np.asarray(dP, np.float32)[rows[valid]]
    bits = (np.ascontiguousarray(full).view(np.uint32) >> 16).astype(np.uint16)
    vals = bits.reshape(n_tiles, 2, 64, S, 128).transpose(0, 3, 1, 4, 2)           # [t, s, half, n, slot in half]
    nn = np.arange(128)[:, None]
    pos = np.arange(64)[None, :]
    slot_at = ((pos // 8) ^ (nn & 7)) * 8 + (pos % 8)     # the slot that element pos of row n holds
    img = np.take_along_axis(vals, np.broadcast_to(slot_at, vals.shape), axis=-1)
    return np.concatenate([img.reshape(-1).view(np.uint8), np.zeros(n_tiles * hidden * 4, np.uint8)])
