"""numpy restatement of the GS_I8ROW feature table (graphsage_b200.Int8Features, gs_quantize_rows_i8; layout in
include/graphsage_b200.h).

A row of F features is a byte array of pitch(F) bytes:

    bytes [0, F)           q_c  int8
    bytes [F, P4)          zero            P4 = round_up(F, 4)
    bytes [P4, P4 + 4)     s    float32, little-endian
    bytes [P4 + 4, pitch)  zero            pitch = round_up(P4 + 4, 16)

quantise:   a = max_c |x_c| (exact);  s = fl(a / 127);  if s == 0 (a == 0, or a so small that a / 127 rounds to zero):
            every q_c = 0;  else q_c = clamp(rint_half_even(fl(x_c / s)), -127, 127).  Non-finite input is refused.
dequantise: deq_c = fl(float(q_c) * s) - the value every kernel reads, so |x_c - deq_c| <= s / 2 plus one rounding.

Every step is one IEEE float32 operation, so these functions give the device's bytes exactly.
"""
import numpy as np


def pitch(F):
    p4 = (int(F) + 3) // 4 * 4
    return (p4 + 4 + 15) // 16 * 16


def quantize(x):
    """float32 [n, F] -> (q int8 [n, F], s float32 [n])."""
    x = np.asarray(x, dtype=np.float32)
    if x.ndim != 2 or x.shape[1] < 1:
        raise ValueError("x must be a 2-D [n, F] array with F >= 1")
    if not np.isfinite(x).all():
        raise ValueError("x has a non-finite value")
    a = np.abs(x).max(axis=1) if x.shape[0] else np.zeros(0, np.float32)
    s = (a / np.float32(127)).astype(np.float32)
    safe = np.where(s == 0, np.float32(1), s).astype(np.float32)
    q = np.clip(np.rint(x / safe[:, None]), -127, 127)          # np.rint: round half to even
    q = np.where(s[:, None] == 0, 0, q).astype(np.int8)
    return q, s


def dequantize(q, s):
    """(q int8 [n, F], s float32 [n]) -> float32 [n, F], one rounding per value."""
    return (np.asarray(q).astype(np.float32) * np.asarray(s, dtype=np.float32)[:, None]).astype(np.float32)


def pack(q, s):
    """(q, s) -> the uint8 [n, pitch(F)] byte rows."""
    q = np.asarray(q, dtype=np.int8)
    n, F = q.shape
    p4 = (F + 3) // 4 * 4
    rows = np.zeros((n, pitch(F)), dtype=np.uint8)
    rows[:, :F] = q.view(np.uint8)
    rows[:, p4:p4 + 4] = np.asarray(s, dtype="<f4").reshape(n, 1).view(np.uint8)
    return rows


def unpack(rows, F):
    """uint8 [n, >= pitch(F)] byte rows -> (q int8 [n, F], s float32 [n])."""
    rows = np.ascontiguousarray(rows, dtype=np.uint8)
    p4 = (int(F) + 3) // 4 * 4
    return rows[:, :F].view(np.int8).copy(), np.ascontiguousarray(rows[:, p4:p4 + 4]).view("<f4").reshape(-1).astype(np.float32)


def quantize_rows(x):
    """float32 [n, F] -> the byte rows gs_quantize_rows_i8 writes."""
    return pack(*quantize(x))
