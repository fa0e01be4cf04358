"""The Python mirror of the feature gathers' launch arithmetic (graphsage_b200/csrc/gather.cu), the stress cases that
test_zz_gpu_gather_regimes.py runs on them, and the checks that keep both honest: the mirror's constants are the
source's, every case reaches the regimes it is built for on an H100 PCIe (114 SMs) and an H100 SXM (132 SMs), a numpy
emulation of gather_mean_tma2_kernel's CTA schedule passes every tma2 case while each of a set of subtly wrong schedules
fails one, and the vectorised references the GPU file uses equal oracle.numerics, oracle.dropout and oracle.int8_rows.

Every gather kernel grid-strides over its nodes (or rows) with a grid capped at a multiple of the SM count, and the
bulk-copy kernels cap their threads so a thread may own two column slots.  A CTA only handles a second node, and a thread
only its second slot, past those caps, so the case sizes are derived from the SM count and the widths sit on each side
of every cap."""
import os
import re

import numpy as np
import pytest

from oracle import dropout, int8_rows
from oracle import numerics as nu

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "graphsage_b200", "csrc")
SM_COUNTS = (114, 132)   # H100 PCIe, H100 SXM
GS_ERR_INVALID_ARG, GS_ERR_UNSUPPORTED = -1, -3
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1

# ---------------------------------------------------------------- the mirror of the launch arithmetic
GROUP_ROWS = 13            # kGroupRows: rows per group of the two-buffer ring (tma2 and the narrow kernel)
TMA2_THREADS = 160         # gather_mean_tma2_kernel: thread cap; a thread owns up to TMA2_SLOTS float4 columns
TMA2_SLOTS = 2
TMA_THREADS = 192          # gather_mean_tma_kernel (variant 1): column loop of 192 threads
LDG_THREADS = 256          # gather_mean_ldg_kernel<5>
LDG_UNROLL = 5
SCALAR_THREADS = 256       # gather_mean_scalar_kernel
NARROW_THREADS = 192       # gather_mean_narrow_tma2_kernel: one thread per 8 columns, no second slot
SMEM_PER_SM = 224          # KB: CTAs per SM = (224 * 1024) / (smem + 1024)
CTAS_PER_SM = 8            # gather_ctas_per_sm's default; also the LDG and scalar kernels' grid cap
TMA_SMEM_MAX = 200         # KB: variant 1 takes a launch whose (kmax + 1) rows fit
ROWS_SMEM_PER_SM = 220     # KB: gather_rows_tma_kernel's CTAs per SM = (220 * 1024) / (smem + 1024), at most 16
ROWS_TMA_MAX_PER_SM = 16
ROWS_TMA_BATCH = 32        # rows one one-warp gather_rows_tma_kernel CTA moves per pass (its smem: 32 rows)
WARP_GRID_PER_SM = 8       # the one-warp-per-row kernels: 256-thread CTAs, grid capped at sm_count() * 8


def _cdiv(a, b):
    return -(-a // b)


def _ceil32(x):
    return _cdiv(x, 32) * 32


def _per_sm(smem, budget_kb=SMEM_PER_SM, cap=CTAS_PER_SM):
    return min(max(1, (budget_kb * 1024) // (smem + 1024)), cap)


def mean_launch(api, dtype, F, pitch, out_pitch, kmax, aligned, sms, total):
    """The kernel gs_gather_mean (api "mean") or gs_gather_mean_dropout ("drop") launches, with its threads, dynamic
    shared memory, CTAs per SM, grid and column slots (or passes) per thread; or {"refused": code} when the call is
    refused before any launch.  pitch counts elements (bytes for int8), aligned: every pointer 16-byte aligned."""
    if dtype == "bf16":
        f8 = _cdiv(F, 8) * 8
        if not (aligned and pitch % 8 == 0 and out_pitch % 8 == 0 and f8 <= pitch and f8 <= out_pitch
                and f8 // 8 <= NARROW_THREADS):
            return dict(kernel=None, refused=GS_ERR_UNSUPPORTED)
        return _narrow("narrow_bf16", f8 * 2, out_pitch, sms, total)
    if dtype == "i8":
        rb = int8_rows.pitch(F)
        if not (aligned and pitch % 16 == 0 and rb <= pitch and out_pitch % 8 == 0 and out_pitch <= NARROW_THREADS * 8):
            return dict(kernel=None, refused=GS_ERR_UNSUPPORTED)
        return _narrow("narrow_i8", rb, out_pitch, sms, total)
    vec_ok = aligned and pitch % 4 == 0 and out_pitch % 4 == 0 and _cdiv(F, 4) * 4 <= pitch
    ncol4 = out_pitch // 4
    row_bytes = _cdiv(F, 4) * 16
    if not vec_ok:
        grid = min(total, sms * CTAS_PER_SM)
        return dict(kernel="scalar_drop" if api == "drop" else "scalar", threads=SCALAR_THREADS, smem=0,
                    per_sm=CTAS_PER_SM, grid=grid, col_passes=_cdiv(out_pitch, SCALAR_THREADS))
    if ncol4 <= TMA2_SLOTS * TMA2_THREADS:
        smem = 2 * GROUP_ROWS * row_bytes
        threads = min(max(_ceil32(ncol4), 32), TMA2_THREADS)
        per_sm = _per_sm(smem)
        return dict(kernel="tma2_drop" if api == "drop" else "tma2", threads=threads, smem=smem, per_sm=per_sm,
                    grid=min(total, sms * per_sm), col_passes=_cdiv(ncol4, threads), row_bytes=row_bytes)
    if api == "drop":
        return dict(kernel="scalar_drop", threads=SCALAR_THREADS, smem=0, per_sm=CTAS_PER_SM,
                    grid=min(total, sms * CTAS_PER_SM), col_passes=_cdiv(out_pitch, SCALAR_THREADS))
    smem = row_bytes * (kmax + 1)
    if smem <= TMA_SMEM_MAX * 1024:
        threads = min(max(_ceil32(ncol4), 32), TMA_THREADS)
        per_sm = _per_sm(smem)
        return dict(kernel="tma", threads=threads, smem=smem, per_sm=per_sm, grid=min(total, sms * per_sm),
                    col_passes=_cdiv(ncol4, threads))
    threads = min(_ceil32(ncol4), LDG_THREADS)
    return dict(kernel="ldg", threads=threads, smem=0, per_sm=CTAS_PER_SM, grid=min(total, sms * CTAS_PER_SM),
                col_passes=_cdiv(ncol4, threads))


def _narrow(kernel, row_bytes, out_pitch, sms, total):
    threads = max(_ceil32(out_pitch // 8), 32)
    if threads > NARROW_THREADS:
        return dict(kernel=None, refused=GS_ERR_INVALID_ARG)
    smem = 2 * GROUP_ROWS * row_bytes
    per_sm = _per_sm(smem)
    return dict(kernel=kernel, threads=threads, smem=smem, per_sm=per_sm, grid=min(total, sms * per_sm), col_passes=1,
                row_bytes=row_bytes)


def rows_launch(dtype, F, pitch, out_pitch, n, aligned, sms):
    """gs_gather_rows: the TMA kernel (one warp, ROWS_TMA_BATCH rows per pass) or the simple one (a warp per row)."""
    es = 4 if dtype == "f32" else 2
    row_bytes = _cdiv(F * es, 16) * 16
    if (aligned and (pitch * es) % 16 == 0 and (out_pitch * es) % 16 == 0 and row_bytes <= pitch * es
            and row_bytes <= out_pitch * es and row_bytes * ROWS_TMA_BATCH <= TMA_SMEM_MAX * 1024):
        smem = row_bytes * ROWS_TMA_BATCH
        per_sm = _per_sm(smem, ROWS_SMEM_PER_SM, ROWS_TMA_MAX_PER_SM)
        grid = min(_cdiv(n, ROWS_TMA_BATCH), sms * per_sm)
        return dict(kernel="rows_tma", threads=32, smem=smem, per_sm=per_sm, grid=grid,
                    passes=_cdiv(n, grid * ROWS_TMA_BATCH))
    grid = min(_cdiv(n, 8), sms * WARP_GRID_PER_SM)
    return dict(kernel="rows_simple", threads=256, smem=0, per_sm=WARP_GRID_PER_SM, grid=grid, passes=_cdiv(n, grid * 8),
                lane_passes=_cdiv(F, 32))


def rows_f32_launch(dtype, F, pitch, out_pitch, n, aligned, sms):
    """gs_gather_rows_f32: i8row, the vectorised bf16 kernel, or the scalar one (fp32 or bf16); a warp per row."""
    grid = min(_cdiv(n, 8), sms * WARP_GRID_PER_SM)
    if dtype == "i8":
        if not (pitch >= int8_rows.pitch(F) and aligned and pitch % 16 == 0):
            return dict(kernel=None, refused=GS_ERR_INVALID_ARG)
        kernel, lanes = "i8row", _cdiv(out_pitch, 32)
    elif dtype == "bf16" and pitch % 8 == 0 and out_pitch % 8 == 0 and aligned and out_pitch <= pitch:
        kernel, lanes = "vec_bf16", _cdiv(out_pitch // 8, 32)
    else:
        kernel, lanes = "scalar_" + dtype, _cdiv(out_pitch, 32)
    return dict(kernel=kernel, threads=256, smem=0, per_sm=WARP_GRID_PER_SM, grid=grid, passes=_cdiv(n, grid * 8),
                lane_passes=lanes)


# ---------------------------------------------------------------- the source the mirror restates
def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _function(src, name):
    m = re.search(r"^(?:static )?int32_t %s\(.*?^}$" % name, src, re.S | re.M)
    assert m, name
    return m.group(0)


def _has(body, *snippets):
    for s in snippets:
        assert s in body, s


def test_mirror_constants_equal_the_sources():
    src = _source("gather.cu")
    _has(src, "constexpr int kGroupRows = %d;" % GROUP_ROWS,
         "float4 acc[%d];" % TMA2_SLOTS, "for (int q = 0; q < %d; ++q) {" % TMA2_SLOTS,
         "const int c = threadIdx.x + q * blockDim.x;",
         "__launch_bounds__(%d) gather_mean_tma_kernel" % TMA_THREADS,
         "__launch_bounds__(%d) gather_mean_narrow_tma2_kernel" % NARROW_THREADS,
         "const int c = threadIdx.x;                                // this thread's 8-column chunk (ncol8 <= blockDim)",
         "for (int64_t base = (int64_t)blockIdx.x * %d; base < n; base += (int64_t)gridDim.x * %d)"
         % (ROWS_TMA_BATCH, ROWS_TMA_BATCH))
    budget = "(%d * 1024) / (smem2 + 1024)" % SMEM_PER_SM
    cap = 'tuning("gather_ctas_per_sm", %d)' % CTAS_PER_SM
    _has(_function(src, "launch_gather_tma2"), "if (threads > %d) threads = %d;" % ((TMA2_THREADS,) * 2),
         "if (threads < 32) threads = 32;", "(size_t)2 * kGroupRows * row_bytes", budget, cap,
         "if (per_sm < 1) per_sm = 1;", "((F + 3) / 4) * 16")
    _has(_function(src, "launch_gather_narrow"), "GS_REQUIRE(threads <= %d," % NARROW_THREADS,
         "(size_t)2 * kGroupRows * row_bytes", "const int ncol8 = (int)(out_pitch / 8);", budget, cap)
    mean = _function(src, "gs_gather_mean")
    _has(mean, "variant == 2 && ncol4 <= %d * %d" % (TMA2_SLOTS, TMA2_THREADS),
         "variant >= 1 && smem <= %d * 1024" % TMA_SMEM_MAX, "(size_t)row_bytes * (kmax + 1)",
         "(%d * 1024) / (smem + 1024)" % SMEM_PER_SM, 'gs::tuning("gather_ctas_per_sm", %d)' % CTAS_PER_SM,
         "if (threads > %d) threads = %d;" % ((TMA_THREADS,) * 2), "if (threads > %d) threads = %d;" % ((LDG_THREADS,) * 2),
         "gather_mean_ldg_kernel<%d><<<(unsigned)blocks, threads" % LDG_UNROLL,
         "gather_mean_scalar_kernel<false><<<(unsigned)blocks, %d," % SCALAR_THREADS,
         "(int64_t)gs::sm_count() * %d;" % CTAS_PER_SM,
         "pitch % 4 == 0 && out_pitch % 4 == 0 && ((F + 3) / 4) * 4 <= pitch",
         "f8 <= pitch && f8 <= out_pitch && f8 / 8 <= %d" % NARROW_THREADS,
         "rb <= pitch && out_pitch %% 8 == 0 && out_pitch <= %d" % (NARROW_THREADS * 8), "pitch % 16 == 0")
    drop = _function(src, "gs_gather_mean_dropout")
    _has(drop, "vec_ok && ncol4 <= %d * %d" % (TMA2_SLOTS, TMA2_THREADS), "(int64_t)gs::sm_count() * %d;" % CTAS_PER_SM,
         "gather_mean_scalar_kernel<true><<<(unsigned)blocks, %d," % SCALAR_THREADS,
         "pitch % 4 == 0 && out_pitch % 4 == 0 && ((F + 3) / 4) * 4 <= pitch")
    rows = _function(src, "gs_gather_rows")
    _has(rows, "row_bytes * %d <= %d * 1024" % (ROWS_TMA_BATCH, TMA_SMEM_MAX), "(size_t)row_bytes * %d;" % ROWS_TMA_BATCH,
         "(%d * 1024) / (smem + 1024)" % ROWS_SMEM_PER_SM, "if (per_sm > %d) per_sm = %d;" % ((ROWS_TMA_MAX_PER_SM,) * 2),
         "(n + %d) / %d;" % (ROWS_TMA_BATCH - 1, ROWS_TMA_BATCH), "<<<(unsigned)blocks, 32, smem, st>>>",
         "int64_t blocks = (n + 7) / 8;", "(int64_t)gs::sm_count() * %d;" % WARP_GRID_PER_SM,
         "<<<(unsigned)blocks, 256, 0, st>>>")
    f32 = _function(src, "gs_gather_rows_f32")
    _has(f32, "int64_t blocks = (n + 7) / 8;", "(int64_t)gs::sm_count() * %d;" % WARP_GRID_PER_SM,
         "pitch % 8 == 0 && out_pitch % 8 == 0 && gs::aligned16(feats) && gs::aligned16(out) && out_pitch <= pitch",
         "pitch >= gs_i8row_pitch(F) && gs::aligned16(feats) && pitch % 16 == 0")
    assert f32.count("<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>") == 4
    # the one-warp-per-row kernels: 8 warps of a 256-thread CTA
    assert src.count("const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;") >= 4


def test_launch_mirror():
    # the bench's layer-0 call: 5,632 rows of F = 602 at 3 CTAs per SM, about 14 nodes per CTA
    L = mean_launch("mean", "f32", 602, 608, 608, 25, True, 132, 5632)
    assert (L["kernel"], L["threads"], L["smem"], L["per_sm"], L["grid"]) == ("tma2", 160, 62816, 3, 396)
    assert 5632 // L["grid"] == 14
    assert mean_launch("mean", "f32", 50, 56, 56, 13, True, 132, 10**6)["per_sm"] == 8
    assert mean_launch("mean", "f32", 1000, 1000, 1000, 13, True, 132, 10**6)["per_sm"] == 2
    assert mean_launch("mean", "f32", 1280, 1280, 1280, 13, True, 132, 10**6)["per_sm"] == 1
    assert mean_launch("mean", "f32", 1280, 1284, 1284, 38, True, 132, 10)["kernel"] == "tma"
    assert mean_launch("mean", "f32", 2048, 2048, 2048, 24, True, 132, 10)["smem"] == 200 * 1024
    assert mean_launch("mean", "f32", 2048, 2048, 2048, 25, True, 132, 10)["kernel"] == "ldg"
    assert mean_launch("mean", "f32", 1300, 1304, 1304, 38, True, 132, 10)["kernel"] == "tma"
    assert mean_launch("mean", "f32", 1300, 1304, 1304, 39, True, 132, 10)["kernel"] == "ldg"
    assert mean_launch("drop", "f32", 1300, 1304, 1304, 3, True, 132, 10)["kernel"] == "scalar_drop"
    assert mean_launch("mean", "f32", 602, 605, 608, 3, True, 132, 10)["kernel"] == "scalar"
    assert mean_launch("mean", "bf16", 1536, 1536, 1536, 3, True, 132, 10)["threads"] == 192
    assert mean_launch("mean", "bf16", 1536, 1536, 1544, 3, True, 132, 10)["refused"] == GS_ERR_INVALID_ARG
    assert mean_launch("mean", "bf16", 1537, 1544, 1544, 3, True, 132, 10)["refused"] == GS_ERR_UNSUPPORTED
    assert mean_launch("mean", "i8", 1535, 1552, 1544, 3, True, 132, 10)["refused"] == GS_ERR_UNSUPPORTED
    assert rows_launch("f32", 1600, 1600, 1600, 10, True, 132)["kernel"] == "rows_tma"
    assert rows_launch("f32", 1601, 1608, 1608, 10, True, 132)["kernel"] == "rows_simple"
    assert rows_launch("bf16", 3200, 3200, 3200, 10, True, 132)["kernel"] == "rows_tma"
    assert rows_launch("bf16", 3201, 3208, 3208, 10, True, 132)["kernel"] == "rows_simple"
    assert rows_launch("f32", 50, 56, 56, 10**6, True, 132)["per_sm"] == 16
    assert rows_f32_launch("bf16", 300, 304, 312, 10, True, 132)["kernel"] == "scalar_bf16"


# ---------------------------------------------------------------- cases
# A mean case: segments [(n, k)] of one call, run in every (include_self, want_self) mode.  Sizes come from the grid
# cap of the kernel the width selects, so every CTA handles at least three nodes on any SM count.  Segment s takes its
# ids as: 0 random ids with out-of-range ones, 1 a pool of six rows (heavy repeats), 2 row ranges running past the
# table, 3 random ids.
ALL_MODES = ((False, False), (False, True), (True, False), (True, True))
MEAN_CASES = {
    # name: (api, dtype, F, pitch, out_pitch, ks, CTAs per pass over the cap, segment weights, needs)
    "tma2 F50 8/SM k1,12,13,14": ("mean", "f32", 50, 56, 56, (1, 12, 13, 14), 3.3, None,
                                  dict(kernel="tma2", per_sm=8, nodes=3, groups={1, 2}, self_only_k={13},
                                       zero_self_k={13}, flip=True)),
    "tma2 F602 3/SM k25,26,27,129": ("mean", "f32", 602, 608, 608, (25, 26, 27, 129), 3.3, (3, 3, 3, 1),
                                     dict(kernel="tma2", per_sm=3, nodes=3, groups={2, 3, 10}, self_only_k={26},
                                          zero_self_k={26}, flip=True)),
    "tma2 F602 out1280 pad-only slot 2": ("mean", "f32", 602, 608, 1280, (12, 26), 3.3, None,
                                          dict(kernel="tma2", per_sm=3, nodes=3, slot2="pad", self_only_k={26})),
    "tma2 F641 slot 2 one column": ("mean", "f32", 641, 648, 648, (13, 14, 1), 3.3, None,
                                    dict(kernel="tma2", per_sm=3, nodes=3, slot2="one", self_only_k={13})),
    "tma2 F1000 2/SM slot 2": ("mean", "f32", 1000, 1000, 1000, (12, 13, 26, 27), 3.3, None,
                               dict(kernel="tma2", per_sm=2, nodes=3, slot2="full", self_only_k={13, 26},
                                    zero_self_k={13, 26})),
    "tma2 F1280 1/SM slot 2": ("mean", "f32", 1280, 1280, 1280, (13, 129, 1, 26), 3.3, (3, 1, 3, 3),
                               dict(kernel="tma2", per_sm=1, nodes=3, slot2="full", self_only_k={13, 26},
                                    zero_self_k={13, 26})),
    "tma2 interleaved 1-2-3 groups": ("mean", "f32", 64, 64, 64, (1, 14, 27, 12), 3.4, None,
                                      dict(kernel="tma2", per_sm=8, nodes=3, groups={1, 2, 3}, interleave=3,
                                           flip=True)),
    "drop p0.5 F50 k1,13,14,26": ("drop", "f32", 50, 56, 56, (1, 13, 14, 26), 3.3, None,
                                  dict(kernel="tma2_drop", per_sm=8, nodes=3, self_only_k={13, 26},
                                       zero_self_k={13, 26}, flip=True)),
    "drop p0.1 F1000 slot 2": ("drop", "f32", 1000, 1000, 1000, (12, 13, 27), 3.3, None,
                               dict(kernel="tma2_drop", per_sm=2, nodes=3, slot2="full", self_only_k={13})),
    "drop p0.5 F1280 slot 2": ("drop", "f32", 1280, 1280, 1280, (26, 1, 14), 3.3, None,
                               dict(kernel="tma2_drop", per_sm=1, nodes=3, slot2="full", self_only_k={26})),
    "drop p0.5 F641 slot 2 one column": ("drop", "f32", 641, 644, 644, (13, 2), 3.3, None,
                                         dict(kernel="tma2_drop", per_sm=3, nodes=3, slot2="one", self_only_k={13})),
    "tma F1281 out1284 leaves tma2": ("mean", "f32", 1281, 1284, 1284, (38, 5), 3.3, None,
                                      dict(kernel="tma", per_sm=1, nodes=3, col_passes=2)),
    "tma F1300 kmax38": ("mean", "f32", 1300, 1304, 1304, (38, 1, 13), 3.3, (1, 3, 3),
                         dict(kernel="tma", per_sm=1, nodes=3, col_passes=2, ks={1, 38})),
    "tma F2048 kmax24 200KB": ("mean", "f32", 2048, 2048, 2048, (24, 1), 3.3, None,
                               dict(kernel="tma", per_sm=1, nodes=3, col_passes=3, ks={1, 24}, smem=200 * 1024)),
    "ldg F1300 k39": ("mean", "f32", 1300, 1304, 1304, (39, 5, 6, 12), 3.3, (1, 3, 3, 3),
                      dict(kernel="ldg", per_sm=8, nodes=3, col_passes=2, kmod5={4, 0, 1, 2})),
    "ldg F2048 k25": ("mean", "f32", 2048, 2048, 2048, (25, 23, 1, 2), 3.3, (1, 3, 3, 3),
                      dict(kernel="ldg", per_sm=8, nodes=3, col_passes=2, kmod5={0, 3, 1, 2})),
    "scalar F700 pitch701": ("mean", "f32", 700, 701, 704, (3, 13, 1, 7), 3.3, None,
                             dict(kernel="scalar", nodes=3, col_passes=3)),
    "scalar F300 unaligned view": ("mean", "f32", 300, 304, 304, (2, 5), 3.3, None,
                                   dict(kernel="scalar", nodes=3, col_passes=2)),
    "scalar drop p0.5 F520 pitch521": ("drop", "f32", 520, 521, 520, (3, 2), 3.3, None,
                                  dict(kernel="scalar_drop", nodes=3, col_passes=3)),
    "narrow bf16 F1536 192 threads": ("mean", "bf16", 1536, 1536, 1536, (12, 13, 25, 26), 3.3, None,
                                      dict(kernel="narrow_bf16", threads=192, nodes=3, self_only_k={13, 26})),
    "narrow bf16 F50": ("mean", "bf16", 50, 56, 56, (13, 1), 3.3, None,
                        dict(kernel="narrow_bf16", per_sm=8, nodes=3, self_only_k={13})),
    "narrow i8 F1535 192 threads": ("mean", "i8", 1535, 1552, 1536, (25, 26), 3.3, None,
                                    dict(kernel="narrow_i8", threads=192, nodes=3, self_only_k={26})),
}
for _F, _extra in zip(range(601, 608), (0, 16, 48, 0, 16, 48, 0)):
    MEAN_CASES["narrow i8 F%d pitch+%d" % (_F, _extra)] = (
        "mean", "i8", _F, int8_rows.pitch(_F) + _extra, 608, (12, 13, 25, 26), 3.3, None,
        dict(kernel="narrow_i8", per_sm=8, nodes=3, self_only_k={13, 26}))
# (dtype, F, pitch, out_pitch): refused before any launch, with the code each check returns
REFUSALS = {
    "bf16 out1544": ("bf16", 1536, 1536, 1544, GS_ERR_INVALID_ARG, "out_pitch too wide for a narrow-row table"),
    "i8 out1544": ("i8", 1535, 1552, 1544, GS_ERR_UNSUPPORTED, "out_pitch % 8 == 0 and <= 1536"),
}
SITE_RATES = {"p0.5": 0.5, "p0.1": 0.1}


def mean_case(name, sms):
    """The case with sizes for `sms` SMs: a dict with the call's parameters and its segments [(n, k)]."""
    api, dtype, F, pitch, out_pitch, ks, over, weights, need = MEAN_CASES[name]
    aligned = "unaligned" not in name
    cap = mean_launch(api, dtype, F, pitch, out_pitch, max(ks), aligned, sms, 10**12)["grid"]
    total = int(over * cap) + 7
    w = np.ones(len(ks)) if weights is None else np.asarray(weights, float)
    ns = [int(total * x / w.sum()) for x in w]
    ns[0] += total - sum(ns)
    rate = next((v for key, v in SITE_RATES.items() if key in name), 0.0)
    return dict(name=name, api=api, dtype=dtype, F=F, pitch=pitch, out_pitch=out_pitch, aligned=aligned,
                segs=list(zip(ns, ks)), modes=ALL_MODES, rate=rate, need=need, seed=sum(map(ord, name)))


def _self_rows(case, include_self, want_self):
    return 1 if case["dtype"] in ("bf16", "i8") or include_self or want_self else 0


def mean_regimes(case, sms):
    """What the case reaches on `sms` SMs: the launch, nodes per CTA and, for the ring kernels, groups per node, the
    fanouts whose last group holds only the self row, the CTAs whose nodes interleave group counts and the nodes that
    start on the second buffer."""
    segs = case["segs"]
    total = sum(n for n, _ in segs)
    L = mean_launch(case["api"], case["dtype"], case["F"], case["pitch"], case["out_pitch"], max(k for _, k in segs),
                    case["aligned"], sms, total)
    f = dict(L, total=total, nodes=total // L["grid"], ks={k for n, k in segs if n},
             kmod5={k % LDG_UNROLL for n, k in segs if n})
    if L["kernel"] in ("tma2", "tma2_drop"):
        ncol4, t = case["out_pitch"] // 4, L["threads"]
        real = max(0, min(case["F"], ncol4 * 4) - t * 4)
        f["slot2"] = None if ncol4 <= t else "pad" if real == 0 else "one" if real == 1 else \
            "full" if real == (ncol4 - t) * 4 else "part"
    if L["kernel"] in ("tma2", "tma2_drop", "narrow_bf16", "narrow_i8"):
        f.update(groups=set(), self_only_k=set(), zero_self_k=set(), interleave=0, flip=False)
        k_of = np.concatenate([np.full(n, k) for n, k in segs])
        G = L["grid"]
        for mode in case["modes"]:
            sr = _self_rows(case, *mode)
            g = _cdiv(k_of + sr, GROUP_ROWS)
            f["groups"] |= set(g.tolist())
            f["self_only_k" if sr else "zero_self_k"] |= {k for n, k in segs if n and k % GROUP_ROWS == 0}
            mat = np.zeros(_cdiv(total, G) * G, np.int64)        # row t, column b: node t * G + b of CTA b
            mat[:total] = g
            mat = mat.reshape(-1, G)
            starts = np.cumsum(mat, axis=0) - mat                # groups the CTA handled before the node
            f["flip"] |= bool(((mat >= 2) & (starts % 2 == 1)).any())
            f["interleave"] = max(f["interleave"], int(sum((mat == v).any(axis=0) for v in set(g.tolist())).max()))
    return f


def require_mean(case, f):
    """Assert the case reaches its regimes; return a one-line description."""
    need = case["need"]
    for key, want in need.items():
        got = f.get(key)
        if key in ("nodes", "col_passes", "interleave"):
            assert got >= want, (case["name"], key, got, want)
        elif isinstance(want, set):
            assert want <= got, (case["name"], key, got, want)
        else:
            assert got == want, (case["name"], key, got, want)
    desc = "%s: %d threads, %d CTAs/SM, grid %d, %d nodes (>= %d per CTA), %d column pass(es)" % (
        f["kernel"], f["threads"], f["per_sm"], f["grid"], f["total"], f["nodes"], f["col_passes"])
    if "groups" in f:
        desc += ", groups per node %s, self-only last group at k %s, k %% 13 == 0 without self %s, %d group counts " \
                "in one CTA, node on buffer 1: %s" % (sorted(f["groups"]), sorted(f["self_only_k"]),
                                                      sorted(f["zero_self_k"]), f["interleave"], f["flip"])
    if f.get("slot2"):
        desc += ", slot 2: %s" % f["slot2"]
    if f["kernel"] == "ldg":
        desc += ", k %% 5 in %s" % sorted(f["kmod5"])
    return desc


# gs_gather_rows and gs_gather_rows_f32: (api, dtype, F, pitch, out_pitch, passes over one grid's rows, needs)
ROW_CASES = {
    "rows f32 F1600 tma": ("rows", "f32", 1600, 1608, 1608, 3.2, dict(kernel="rows_tma", passes=3)),
    "rows f32 F1601 simple": ("rows", "f32", 1601, 1608, 1608, 3.2, dict(kernel="rows_simple", passes=3)),
    "rows bf16 F3200 tma": ("rows", "bf16", 3200, 3208, 3208, 3.2, dict(kernel="rows_tma", passes=3)),
    "rows bf16 F3201 simple": ("rows", "bf16", 3201, 3208, 3216, 3.2, dict(kernel="rows_simple", passes=3)),
    "rows_f32 bf16 vec F300": ("rows_f32", "bf16", 300, 304, 304, 3.2, dict(kernel="vec_bf16", passes=3, lane_passes=2)),
    "rows_f32 bf16 out>pitch scalar": ("rows_f32", "bf16", 300, 304, 312, 3.2,
                                       dict(kernel="scalar_bf16", passes=3, lane_passes=10)),
    "rows_f32 f32 F301": ("rows_f32", "f32", 301, 304, 320, 3.2, dict(kernel="scalar_f32", passes=3, lane_passes=10)),
    "rows_f32 i8 F601 pitch+16": ("rows_f32", "i8", 601, int8_rows.pitch(601) + 16, 608, 3.2,
                                  dict(kernel="i8row", passes=3, lane_passes=19)),
}


def row_case(name, sms):
    api, dtype, F, pitch, out_pitch, over, need = ROW_CASES[name]
    fn = rows_launch if api == "rows" else rows_f32_launch
    per_pass = fn(dtype, F, pitch, out_pitch, 10**12, True, sms)
    per_pass = per_pass["grid"] * (ROWS_TMA_BATCH if per_pass["kernel"] == "rows_tma" else 8)
    n = int(over * per_pass) // 32 * 32 + 17                      # never a multiple of 32
    return dict(name=name, api=api, dtype=dtype, F=F, pitch=pitch, out_pitch=out_pitch, n=n, need=need,
                seed=sum(map(ord, name)))


def row_regimes(case, sms):
    fn = rows_launch if case["api"] == "rows" else rows_f32_launch
    return dict(fn(case["dtype"], case["F"], case["pitch"], case["out_pitch"], case["n"], True, sms), n=case["n"])


def require_rows(case, f):
    assert case["n"] % 32, case["name"]
    for key, want in case["need"].items():
        assert (f[key] >= want) if key in ("passes", "lane_passes") else (f[key] == want), (case["name"], key, f[key])
    return "%s: grid %d x %d threads, %d rows, %d passes%s" % (
        f["kernel"], f["grid"], f["threads"], f["n"], f["passes"],
        ", %d lane passes" % f["lane_passes"] if "lane_passes" in f else "")


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_every_case_reaches_its_regimes(sms):
    for name in MEAN_CASES:
        c = mean_case(name, sms)
        require_mean(c, mean_regimes(c, sms))
    for name in ROW_CASES:
        c = row_case(name, sms)
        require_rows(c, row_regimes(c, sms))
    for dtype, F, pitch, out_pitch, code, _ in REFUSALS.values():
        assert mean_launch("mean", dtype, F, pitch, out_pitch, 3, True, sms, 10)["refused"] == code
    # every regime row of the issue's table is some case's
    kernels = {mean_regimes(mean_case(n, sms), sms)["kernel"] for n in MEAN_CASES}
    assert kernels == {"tma2", "tma2_drop", "tma", "ldg", "scalar", "scalar_drop", "narrow_bf16", "narrow_i8"}
    per_sm = {mean_regimes(mean_case(n, sms), sms)["per_sm"] for n in MEAN_CASES if n.startswith("tma2")}
    assert per_sm == {8, 3, 2, 1}
    slots = {mean_regimes(mean_case(n, sms), sms).get("slot2") for n in MEAN_CASES}
    assert {"pad", "one", "full"} <= slots
    ks = set().union(*(mean_regimes(mean_case(n, sms), sms)["ks"] for n in MEAN_CASES if n.startswith("tma2")))
    assert {1, 12, 13, 14, 25, 26, 27, 129} <= ks
    mods = set().union(*(mean_regimes(mean_case(n, sms), sms)["kmod5"] for n in MEAN_CASES if n.startswith("ldg")))
    assert mods == {0, 1, 2, 3, 4}


def test_regimes_move_with_the_caps():
    """A CTA cap one larger, or a case sized for fewer SMs, drops a case below its regimes."""
    c = mean_case("tma2 F1280 1/SM slot 2", 114)
    assert mean_regimes(c, 132)["nodes"] == 2
    with pytest.raises(AssertionError):
        require_mean(c, mean_regimes(c, 132))
    c = row_case("rows f32 F1600 tma", 114)
    assert row_regimes(c, 132)["passes"] == 3 and row_regimes(c, 200)["passes"] == 2


# ---------------------------------------------------------------- data and references the GPU file compares against
ID_ROWS, NAN_ROWS, TAIL_ROWS = 2000, 40, 64       # ids read [0, ID_ROWS); then rows no id reads; then the ranges' rows
N_SRC = ID_ROWS + NAN_ROWS + TAIL_ROWS
BAD_IDS = (-1, N_SRC, INT32_MAX, INT32_MIN)


def feature_values(rs, n, F):
    """float32 [n, F] with a row of -0.0, a row of subnormals and mixed tiny values among normal ones."""
    x = rs.randn(n, F).astype(np.float32)
    x[0] = -0.0
    x[1] = rs.choice([1e-45, -1e-45, 1e-40, -2e-39, 5e-39], size=F)
    x[2] = rs.choice([-0.0, 0.0, 1e-44, -1e-38], size=F)
    return x


def make_table(dtype, F, pitch, rs, aligned=True):
    """(values, store): values the fp32 table the kernels read (bf16 widened, int8 dequantised; NaN in the rows no id
    reads), store the device bytes - [N_SRC, pitch] with NaN in
    every pad column and unread row, and for int8 junk bytes past gs_i8row_pitch(F) and a NaN scale in unread rows.
    aligned=False: the rows start one column into the store, so the table's view is not 16-byte aligned."""
    x = feature_values(rs, N_SRC, F)
    unread = slice(ID_ROWS, ID_ROWS + NAN_ROWS)
    if dtype == "i8":
        q = rs.randint(-127, 128, size=(N_SRC, F)).astype(np.int8)
        q[0] = 0
        s = np.exp(rs.uniform(-12, 4, size=N_SRC)).astype(np.float32)
        s[unread] = np.nan
        store = rs.randint(0, 256, size=(N_SRC, pitch)).astype(np.uint8)
        store[:, :int8_rows.pitch(F)] = int8_rows.pack(q, s)
        return int8_rows.dequantize(q, s), store
    x[unread] = np.nan
    c0 = 0 if aligned else 1
    if dtype == "bf16":
        bits = (nu.bf16_rne(x).view(np.uint32) >> 16).astype(np.uint16)
        store = np.full((N_SRC, pitch), 0x7FC0, np.uint16)
        store[:, c0:c0 + F] = bits
        return nu.bf16_widen(bits), store
    store = np.full((N_SRC, pitch), np.nan, np.float32)
    store[:, c0:c0 + F] = x
    return x, store


def segment_ids(rs, s, n, k):
    """(self ids, neighbour ids, (self_row0, neigh_row0) or None) of segment s - see MEAN_CASES."""
    if s % 4 == 2:
        r0 = ID_ROWS + NAN_ROWS
        return np.arange(r0, r0 + n), np.arange(r0 + 5, r0 + 5 + n * k), (r0, r0 + 5)
    if s % 4 == 1:
        pool = rs.choice(ID_ROWS, size=6, replace=False)
        pool[:2] = (0, 1)
        return pool[rs.randint(0, 6, size=n)], pool[rs.randint(0, 6, size=n * k)], None
    sf, nb = rs.randint(0, ID_ROWS, size=n), rs.randint(0, ID_ROWS, size=n * k)
    for a in (sf, nb):
        bad = rs.rand(a.size) < 0.03
        a[bad] = rs.choice(BAD_IDS, size=int(bad.sum()))
        a[:len(BAD_IDS)] = BAD_IDS[:a.size]
    return sf, nb, None


def layout(case):
    """Output row of each segment: segments in reverse order with three unwritten rows between them and after the last."""
    r0, out = 3, []
    for n, _ in reversed(case["segs"]):
        out.append(r0)
        r0 += n + 3
    return out[::-1], r0


def mean_data(case):
    rs = np.random.RandomState(case["seed"])
    values, store = make_table(case["dtype"], case["F"], case["pitch"], rs, case["aligned"])
    segs = []
    out_rows, rows_out = layout(case)
    for s, ((n, k), o) in enumerate(zip(case["segs"], out_rows)):
        sf, nb, ranges = segment_ids(rs, s, n, k)
        site = ((11 + s, 2 * s + 1, case["rate"]), (11 + s, 2 * s + 2, case["rate"])) if case["api"] == "drop" else None
        segs.append(dict(n=n, k=k, sf=sf.astype(np.int32), nb=nb.astype(np.int32), ranges=ranges, out_row0=o,
                         sites=site))
    return dict(values=values, store=store, segs=segs, rows_out=rows_out)


def mean_sum_reference(values, sf, nb, k, neigh_site=None, self_site=None):
    """(sum, self): the fp32 sum of the k neighbour rows in j order (each dropped at position i * k + j by neigh_site)
    and the self rows (dropped at i by self_site) - the operands of numerics.mean_f32, a neighbour column at a time."""
    n = len(sf)
    nb = np.asarray(nb).reshape(n, k)
    acc = np.zeros((n, values.shape[1]), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(k):
            x = nu.gather_clamped(values, nb[:, j])
            if neigh_site is not None:
                x = dropout.apply(x, *neigh_site, pos=np.arange(n, dtype=np.int64) * k + j)
            acc = acc + x
        s = nu.gather_clamped(values, sf)
        if self_site is not None:
            s = dropout.apply(s, *self_site)
    return acc, s


def mean_from_sum(acc, s, k, include_self):
    with np.errstate(over="ignore", invalid="ignore"):
        return ((acc + s) if include_self else acc) / np.float32(k + (1 if include_self else 0))


def expected_outputs(case, data, include_self, want_self, sums):
    """The whole out_mean / out_self buffers as NaN-filled [rows_out, out_pitch] arrays with each segment's rows written:
    the mean (or self row) in the first F columns, +0 in the pad columns."""
    F, op = case["F"], case["out_pitch"]
    om = np.full((data["rows_out"], op), np.nan, np.float32)
    osf = om.copy() if want_self else None
    for sg, (acc, s) in zip(data["segs"], sums):
        if not sg["n"]:
            continue
        rows = slice(sg["out_row0"], sg["out_row0"] + sg["n"])
        om[rows] = 0
        om[rows, :F] = mean_from_sum(acc, s, sg["k"], include_self)
        if want_self:
            osf[rows] = 0
            osf[rows, :F] = s
    return om, osf


def segment_sums(data):
    return [mean_sum_reference(data["values"], sg["sf"], sg["nb"], sg["k"], *(sg["sites"] or (None, None)))
            for sg in data["segs"]]


# ---------------------------------------------------------------- the tma2 CTA schedule, emulated
MUTANTS = ("no_reset", "slot2_skipped", "self_only_group_summed", "self_from_first_row", "stops_after_first_node",
           "reads_prefetch_buffer")


def emulate_tma2(case, data, sms, include_self, want_self, mutant=None):
    """gather_mean_tma2_kernel<DenseRows, false> in numpy, CTA by CTA: the same grid, the per-CTA node sequence
    (r = blockIdx, blockIdx + grid, ...), 13-row groups of the k neighbour rows then the self row through two buffers
    (group t + 1 issued into the other buffer before group t is summed), per-thread accumulators in two column slots,
    the self row taken from the last row of the node's last group.  Returns (out_mean, out_self) as expected_outputs
    lays them out.  `mutant` names a subtly wrong schedule (MUTANTS)."""
    F, op, values = case["F"], case["out_pitch"], data["values"]
    segs = data["segs"]
    total = sum(sg["n"] for sg in segs)
    L = mean_launch("mean", "f32", F, case["pitch"], op, max(sg["k"] for sg in segs), True, sms, total)
    assert L["kernel"] == "tma2"
    G, T, ncol4 = L["grid"], L["threads"], op // 4
    c4 = np.arange(op) // 4
    slot = c4 // T
    in_slot = (slot == 0) | ((slot == 1) & (mutant != "slot2_skipped"))
    sums = in_slot & (c4 * 4 < F)                         # the columns a thread accumulates
    keep = np.arange(op) < F                              # mask_tail
    self_rows = 1 if include_self or want_self else 0
    om = np.full((data["rows_out"], op), np.nan, np.float32)
    osf = om.copy() if want_self else None
    bounds = np.cumsum([0] + [sg["n"] for sg in segs])
    table = np.full((values.shape[0], op), np.nan, np.float32)
    table[:, :F] = values

    def node(r):
        s = int(np.searchsorted(bounds, r, side="right") - 1)
        return segs[s], r - bounds[s]

    def group_rows(r, g):
        sg, i = node(r)
        k = sg["k"]
        first = g * GROUP_ROWS
        cnt = min(GROUP_ROWS, k + self_rows - first)
        ids = [sg["nb"][i * k + jj] if jj < k else sg["sf"][i] for jj in range(first, first + cnt)]
        return table[np.where((np.asarray(ids) < 0) | (np.asarray(ids) >= len(table)), len(table) - 1, ids)]

    with np.errstate(over="ignore", invalid="ignore"):
        for b in range(G):
            items = iter([(r, g) for r in range(b, total, G)
                          for g in range(_cdiv(node(r)[0]["k"] + self_rows, GROUP_ROWS))])
            bufs = [np.full((GROUP_ROWS, op), np.nan, np.float32) for _ in range(2)]

            def issue(buf):
                it = next(items, None)
                if it is None:
                    return False
                rows = group_rows(*it)
                bufs[buf][:len(rows)] = rows
                return True

            buf, have, r, g = 0, issue(0), b, 0
            acc = np.zeros(op, np.float32)
            while have:
                have_next = issue(buf ^ 1)
                sg, i = node(r)
                k = sg["k"]
                rows_total = k + self_rows
                first = g * GROUP_ROWS
                cnt = min(GROUP_ROWS, rows_total - first)
                last = first + cnt >= rows_total
                rows = bufs[buf ^ 1 if mutant == "reads_prefetch_buffer" else buf]
                nn = cnt - self_rows if last else cnt
                if mutant == "self_only_group_summed" and last and cnt == self_rows:
                    nn = cnt
                for j in range(nn):
                    acc[sums] = acc[sums] + rows[j, sums]
                if last:
                    o = sg["out_row0"] + i
                    sv = np.zeros(op, np.float32)
                    if self_rows:
                        sv[sums] = rows[0 if mutant == "self_from_first_row" else cnt - 1, sums]
                    a = (acc + sv) if include_self else acc.copy()
                    a = np.where(keep, a / np.float32(k + (1 if include_self else 0)), np.float32(0))
                    om[o, in_slot] = a[in_slot]
                    if want_self:
                        osf[o, in_slot] = np.where(keep, sv, np.float32(0))[in_slot]
                    if mutant != "no_reset":
                        acc = np.zeros(op, np.float32)
                    r, g = r + G, 0
                    if mutant == "stops_after_first_node":
                        break
                else:
                    g += 1
                buf ^= 1
                have = have_next
    return om, osf


EMULATED = [n for n in MEAN_CASES if n.startswith("tma2")]
EMULATED_MODES = ((True, True), (False, False))


def _emulation_agrees(name, sms, mutant=None):
    c = mean_case(name, sms)
    d = mean_data(c)
    sums = segment_sums(d)
    for mode in EMULATED_MODES:
        om, osf = emulate_tma2(c, d, sms, *mode, mutant=mutant)
        em, es = expected_outputs(c, d, *mode, sums)
        if not (nu.bits_equal(om, em) and (es is None or nu.bits_equal(osf, es))):
            return False
    return True


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("name", EMULATED)
def test_tma2_emulation_passes_the_case(name, sms):
    assert _emulation_agrees(name, sms)


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("mutant", MUTANTS)
def test_every_tma2_mutant_fails_a_case(mutant, sms):
    assert any(not _emulation_agrees(name, sms, mutant) for name in EMULATED), mutant


# ---------------------------------------------------------------- the references against the oracle
def test_mean_reference_equals_the_oracle():
    rs = np.random.RandomState(5)
    for F in (1, 7, 50):
        x = feature_values(rs, 30, F)
        x[3] = 3e38                                        # two of them overflow to +inf
        for k in (1, 3, 14):
            n = 9
            sf = rs.randint(-3, 33, size=n)
            nb = rs.randint(-3, 33, size=n * k)
            for sites in (None, ((7, 3, 0.5), (7, 4, 0.1))):
                acc, s = mean_sum_reference(x, sf, nb, k, *(sites or (None, None)))
                rows = nu.gather_clamped(x, nb)
                srow = nu.gather_clamped(x, sf)
                for inc in (False, True):
                    want = nu.mean_f32(rows, k, srow, inc, *(sites or (None, None)))
                    assert nu.bits_equal(mean_from_sum(acc, s, k, inc), want), (F, k, sites, inc)
                if sites:
                    with np.errstate(over="ignore"):
                        assert nu.bits_equal(s, dropout.apply(srow, *sites[1]))
                else:
                    assert nu.bits_equal(s, srow)


def test_tables_equal_the_oracle():
    rs = np.random.RandomState(6)
    for F in (601, 604, 607):
        for extra in (0, 16, 48):
            pitch = int8_rows.pitch(F) + extra
            values, store = make_table("i8", F, pitch, rs)
            q, s = int8_rows.unpack(store, F)
            read = np.r_[0:ID_ROWS, ID_ROWS + NAN_ROWS:N_SRC]
            assert nu.bits_equal(values[read], int8_rows.dequantize(q, s)[read])
            assert np.isnan(s[ID_ROWS:ID_ROWS + NAN_ROWS]).all()
            assert (store[:, F:(F + 3) // 4 * 4] == 0).all()   # the format's own padding stays zero
    values, store = make_table("bf16", 50, 56, rs)
    assert nu.bits_equal(values[:ID_ROWS], nu.bf16_widen(store[:ID_ROWS, :50]))
    assert (store[:, 50:] == 0x7FC0).all()
    values, store = make_table("f32", 300, 304, rs, aligned=False)
    assert nu.bits_equal(store[:, 1:301], values) and np.isnan(store[:, 0]).all()
