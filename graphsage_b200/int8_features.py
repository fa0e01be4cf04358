"""An int8 feature table with one fp32 scale per row: a quarter of fp32's bytes per row for layer 0 to read.

Each row is a byte array (GS_I8ROW, include/graphsage_b200.h; numpy restatement in oracle/int8_rows.py)

    bytes [0, F) q_c int8 | zero to P4 = round_up(F, 4) | s fp32 | zero to pitch = round_up(P4 + 4, 16)

quantised by gs_quantize_rows_i8 (s = fl(max_c |x_c| / 127), q_c = clamp(rint(fl(x_c / s)), -127, 127)).  Every kernel
that reads it sees exactly deq_c = fl(float(q_c) * s) and from there computes what it computes on fp32 rows, so a model
over an Int8Features table gives the bits of the same model over the fp32 table `dequantize()`.  The scale lives inside
the row, so a HostFeatures table over int8 rows stages them with its byte copies unchanged.
"""
import numpy as np
import torch

from . import ops

QUANTIZE_CHUNK_BYTES = 256 << 20          # fp32 rows quantised per launch when the table is not on the device


class Int8Features(ops.I8Rows):
    """A [N+1, F] feature table stored as int8 rows with a per-row fp32 scale, usable wherever SampleAndAggregate,
    SupervisedGraphsage and UnsupervisedGraphsage take `features` (rows on a GPU), and as the table of a HostFeatures
    (rows in host memory).

    table  : float [N+1, F] tensor or numpy array (converted to float32); its last row is the all-zero dummy row.  Every
             value must be finite.
    device : where the rows are kept (default: where the table is).  The quantisation runs on a GPU in any case - a table
             that is not on the device is uploaded and quantised in chunks, so it need not fit there.

    .rows is the uint8 [N+1, pitch] byte table, .shape == (N+1, F), .dtype == torch.int8; dequantize() gives the fp32
    table every kernel reads.  Not supported (NotImplementedError): fused_pool=True, the seq aggregator, training dropout,
    identity_dim > 0, node-partitioned tables and distributed=True, and the whole-graph and whole-neighbourhood passes
    (the sampled-block entry points, sampled_minibatch_*, take it)."""

    def __init__(self, table, device=None):
        t = table if torch.is_tensor(table) else torch.from_numpy(np.asarray(table))
        if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError("the table must be a 2-D [N+1, F] array with F >= 1")
        if not t.is_floating_point():
            raise TypeError("Int8Features quantises a floating-point table (got %s)" % t.dtype)
        n, F = int(t.shape[0]), int(t.shape[1])
        rows = torch.empty((n, ops.i8row_pitch(F)), dtype=torch.uint8, device=t.device if device is None else device)
        work = None
        step = max(1, QUANTIZE_CHUNK_BYTES // (4 * F))
        for a in range(0, n, step):
            x = t[a:a + step].to(torch.float32)                  # checked where it is, before any device work
            b = a + x.shape[0]
            if not bool(torch.isfinite(x).all()):
                raise ValueError("the table has a non-finite value in rows [%d, %d)" % (a, b))
            if b == n and bool((x[-1] != 0).any()):
                raise ValueError("the table's last row is the dummy row and must be all zero")
            if work is None:
                work = rows.device if rows.is_cuda else x.device if x.is_cuda else torch.device(
                    "cuda", torch.cuda.current_device())
            x = x.to(work).contiguous()
            if rows.device == work:
                ops.quantize_rows_i8(x, out=rows[a:b])
            else:
                rows[a:b].copy_(ops.quantize_rows_i8(x))
        ops.I8Rows.__init__(self, rows, F)

    @property
    def pitch(self):
        """Bytes per row (ops.i8row_pitch(F))."""
        return self.rows.stride(0)

    def dequantize(self):
        """The fp32 [N+1, F] table the kernels read (deq = fl(float(q) * s)), a view of an [N+1, pad_cols(F)] buffer on
        the rows' device - the twin whose model gives this table's bits."""
        n, F = self.shape
        if self.rows.is_cuda:
            return ops.gather_rows_f32(self, row0=0, n=n)
        q = self.rows[:, :F].view(torch.int8).to(torch.float32)
        s = self.rows[:, (F + 3) // 4 * 4:(F + 3) // 4 * 4 + 4].contiguous().view(torch.float32)
        out = torch.zeros((n, ops.pad_cols(F)), dtype=torch.float32)
        out[:, :F] = q * s                       # one fp32 rounding per value, as on the device
        return out[:, :F]


def is_int8_table(features):
    """Whether `features` is an int8 row table: an Int8Features, or a HostFeatures over one."""
    return not torch.is_tensor(features) and getattr(features, "dtype", None) == torch.int8


def refuse_int8_table(features, what):
    if is_int8_table(features):
        raise NotImplementedError("%s with an int8 (Int8Features) feature table is not implemented" % what)
