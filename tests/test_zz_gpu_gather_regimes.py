"""GPU: the feature gathers where the rest of the suite never reaches them - CTAs that handle three or more nodes at 8,
3, 2 and 1 CTAs per SM, the second column slot of gather_mean_tma2_kernel (one real column, full, pad only), fanouts at
every edge of the 13-row groups with and without the self row, nodes of 1, 2 and 3 groups interleaved in one CTA, every
kernel at its width limit and the dispatch on each side of it (tma2 / variant 1 / LDG / scalar, the narrow bf16 and
int8 kernels, the TMA and simple row gathers, every gs_gather_rows_f32 kernel), and int8 rows whose last 8-column chunk
straddles the scale or whose pitch is wider than gs_i8row_pitch(F).

Every output is compared bit for bit with an order-exact reference: numerics.mean_f32's operands and order (the fp32
sum in j order, the self row last, one division), oracle.dropout's sites for gs_gather_mean_dropout, oracle.int8_rows'
dequantisation, plain indexing for the row gathers.  Pad columns and rows that no id reads hold NaN, ids include -1,
n_rows, INT32_MAX and INT32_MIN, heavy repeats and row ranges running past the table, and the outputs are NaN-filled
buffers, so a wrong read or a missing write cannot look plausible: pad columns must come back +0 and the rows between
and after the segments' outputs (and columns past F of a row gather) NaN.  Each call runs twice with identical bits.

The cases and the Python mirror of the launches are in test_gather_regimes_cpu.py, which checks the mirror's constants
against the source and that every case reaches its regimes on 114 and 132 SMs; here each case asserts its regimes again
for this GPU's SM count and prints them."""
import numpy as np
import pytest
import torch

import test_gather_regimes_cpu as cs
from oracle import numerics as nu

pytestmark = pytest.mark.gpu

TAIL = 37                                     # floats past the last output row of a mean buffer: must stay NaN


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def nan_buffer(n):
    return torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")


def same_bits(got, want, what):
    """got (a CUDA float32 tensor) equals want (numpy) bit for bit; on a mismatch name where."""
    g = nu.f32_bits(got.cpu().numpy()).reshape(want.shape)
    w = nu.f32_bits(want)
    bad = np.argwhere(g != w)
    if len(bad):
        at = tuple(bad[0])
        pytest.fail("%s: %d of %d elements differ; first at %s: got %08x, want %08x" % (
            what, len(bad), w.size, at, g[at], w[at]))


def device_table(gs, case, store):
    """(pointer, dtype code, the tensor that owns the memory): the store on the device; an unaligned case's table view
    starts one column in."""
    if case["dtype"] == "i8":
        t = dev(store)
        return t.data_ptr(), gs._lib.GS_I8ROW, t
    if case["dtype"] == "bf16":
        t = dev(store.view(np.int16)).view(torch.bfloat16)
        return t.data_ptr(), gs._lib.GS_BF16, t
    t = dev(store)
    return t.data_ptr() + (0 if case["aligned"] else 4), gs._lib.GS_F32, t


def c_segments(gs, data):
    """The ctypes gs_segment array of the case, and the id tensors it points into."""
    keep, segs = [], []
    for sg in data["segs"]:
        if sg["ranges"] is not None:
            segs.append(gs._lib.Segment(0, 0, sg["ranges"][0], sg["ranges"][1], sg["n"], sg["k"], 0, sg["out_row0"]))
            continue
        sf, nb = dev(sg["sf"]), dev(sg["nb"])
        keep += [sf, nb]
        segs.append(gs._lib.Segment(sf.data_ptr(), nb.data_ptr(), 0, 0, sg["n"], sg["k"], 0, sg["out_row0"]))
    return (gs._lib.Segment * len(segs))(*segs), keep


def run_mean(gs, case, data, src, code, arr, include_self, want_self):
    lib = gs._lib.lib()
    size = data["rows_out"] * case["out_pitch"] + TAIL
    om = nan_buffer(size)
    osf = nan_buffer(size) if want_self else None
    nseg = len(data["segs"])
    common = (include_self, 0 if osf is None else osf.data_ptr(), om.data_ptr(), case["out_pitch"],
              gs._lib.stream_ptr())
    if case["api"] == "drop":
        ns = (gs._lib.DropoutSite * nseg)(*[gs._lib.DropoutSite(*sg["sites"][0], 0) for sg in data["segs"]])
        ss = (gs._lib.DropoutSite * nseg)(*[gs._lib.DropoutSite(*sg["sites"][1], 0) for sg in data["segs"]])
        rc = lib.gs_gather_mean_dropout(src, cs.N_SRC, case["F"], case["pitch"], arr, nseg, ns, ss, *common)
    else:
        rc = lib.gs_gather_mean(src, code, cs.N_SRC, case["F"], case["pitch"], arr, nseg, *common)
    gs._lib.check(rc)
    torch.cuda.synchronize()
    return om, osf


def _with_tail(x):
    return np.concatenate([x.reshape(-1), np.full(TAIL, np.nan, np.float32)])


@pytest.mark.parametrize("name", list(cs.MEAN_CASES))
def test_gather_mean_regime(gs, sms, name):
    case = cs.mean_case(name, sms)
    print("\n%d SMs, %s -> %s" % (sms, name, cs.require_mean(case, cs.mean_regimes(case, sms))))
    data = cs.mean_data(case)
    sums = cs.segment_sums(data)
    src, code, owner = device_table(gs, case, data["store"])
    arr, ids = c_segments(gs, data)
    for include_self, want_self in case["modes"]:
        want_m, want_s = cs.expected_outputs(case, data, include_self, want_self, sums)
        first = None
        for rep in range(2):
            om, osf = run_mean(gs, case, data, src, code, arr, int(include_self), want_self)
            what = "%s, include_self=%d want_self=%d, run %d" % (name, include_self, want_self, rep)
            same_bits(om, _with_tail(want_m), what + ": out_mean")
            if want_self:
                same_bits(osf, _with_tail(want_s), what + ": out_self")
            bits = (om.cpu().numpy().view(np.uint32), None if osf is None else osf.cpu().numpy().view(np.uint32))
            if first is None:
                first = bits
            else:
                assert np.array_equal(first[0], bits[0]) and (want_self is False or np.array_equal(first[1], bits[1]))
    del owner, ids


@pytest.mark.parametrize("name", list(cs.REFUSALS))
def test_gather_mean_refusal(gs, sms, name):
    """A narrow-row call past its width is refused with its own code and message before anything is launched."""
    dtype, F, pitch, out_pitch, code, message = cs.REFUSALS[name]
    assert cs.mean_launch("mean", dtype, F, pitch, out_pitch, 3, True, sms, 10)["refused"] == code
    case = dict(dtype=dtype, aligned=True)
    _, store = cs.make_table(dtype, F, pitch, np.random.RandomState(F))
    src, dcode, owner = device_table(gs, case, store)
    ids = dev(np.arange(4 * 3, dtype=np.int32))
    arr = (gs._lib.Segment * 1)(gs._lib.Segment(ids.data_ptr(), ids.data_ptr(), 0, 0, 4, 3, 0, 0))
    om, osf = nan_buffer(4 * out_pitch), nan_buffer(4 * out_pitch)
    lib = gs._lib.lib()
    rc = lib.gs_gather_mean(src, dcode, cs.N_SRC, F, pitch, arr, 1, 1, osf.data_ptr(), om.data_ptr(), out_pitch,
                            gs._lib.stream_ptr())
    msg = lib.gs_last_error_string().decode()
    torch.cuda.synchronize()
    print("\n%s: rc %d, %r" % (name, rc, msg))
    assert rc == code and message in msg, (rc, msg)
    assert torch.isnan(om).all() and torch.isnan(osf).all()
    del owner


def row_data(case):
    rs = np.random.RandomState(case["seed"])
    values, store = cs.make_table(case["dtype"], case["F"], case["pitch"], rs)
    ids = rs.randint(0, cs.ID_ROWS, size=case["n"])
    ids[rs.rand(case["n"]) < 0.5] = rs.randint(0, 6)                      # heavy repeats of a few rows
    bad = rs.rand(case["n"]) < 0.02
    ids[bad] = rs.choice(cs.BAD_IDS, size=int(bad.sum()))
    ids[-len(cs.BAD_IDS):] = cs.BAD_IDS
    return values, store, ids.astype(np.int32)


@pytest.mark.parametrize("name", list(cs.ROW_CASES))
def test_gather_rows_regime(gs, sms, name):
    case = cs.row_case(name, sms)
    print("\n%d SMs, %s -> %s" % (sms, name, cs.require_rows(case, cs.row_regimes(case, sms))))
    values, store, ids = row_data(case)
    n, F, op = case["n"], case["F"], case["out_pitch"]
    _, _, table = device_table(gs, dict(dtype=case["dtype"], aligned=True), store)
    d_ids = dev(ids)
    first = None
    for rep in range(2):
        if case["api"] == "rows":
            # bf16 / fp32 rows copied as they are; the output's pad columns and its rows past n are never written
            dt = torch.float32 if case["dtype"] == "f32" else torch.int16
            back = torch.full((n + 3, op), -1 if dt == torch.int16 else float("nan"), dtype=dt, device="cuda")
            out = back.view(torch.bfloat16) if case["dtype"] == "bf16" else back
            gs.ops.gather_rows(table[:, :F], d_ids, out=out[:n, :F])
            torch.cuda.synchronize()
            got = back.cpu().numpy()
            want = np.full((n + 3, op), -1, np.int16) if case["dtype"] == "bf16" else \
                np.full((n + 3, op), np.nan, np.float32)
            clamped = np.where((ids < 0) | (ids >= cs.N_SRC), cs.N_SRC - 1, ids)
            want[:n, :F] = store[clamped, :F].view(want.dtype)
            bits = got.view(np.uint16 if case["dtype"] == "bf16" else np.uint32)
            bad = np.argwhere(bits != want.view(bits.dtype))
            assert not len(bad), "%s: %d elements differ, first at %s" % (name, len(bad), tuple(bad[0]))
        else:
            back = nan_buffer((n + 3) * op).view(n + 3, op)
            src = gs.ops.I8Rows(table, F) if case["dtype"] == "i8" else table[:, :F]
            gs.ops.gather_rows_f32(src, d_ids, out=back[:n])
            torch.cuda.synchronize()
            want = np.full((n + 3, op), np.nan, np.float32)
            want[:n] = 0
            want[:n, :F] = nu.gather_clamped(values, ids)
            same_bits(back, want, "%s run %d" % (name, rep))
            bits = back.cpu().numpy().view(np.uint32)
        if first is None:
            first = bits.copy()
        else:
            assert np.array_equal(first, bits), name


def test_gather_rows_f32_ranges_past_the_table(gs, sms):
    """gs_gather_rows_f32 by row range (no ids) over three passes, the range running past the table: the rows past it
    read the last row."""
    case = cs.row_case("rows_f32 i8 F601 pitch+16", sms)
    values, store, _ = row_data(case)
    n, F, op = case["n"], case["F"], case["out_pitch"]
    row0 = cs.ID_ROWS + cs.NAN_ROWS
    table = dev(store)
    back = nan_buffer((n + 3) * op).view(n + 3, op)
    gs.ops.gather_rows_f32(gs.ops.I8Rows(table, F), None, row0=row0, n=n, out=back[:n])
    want = np.full((n + 3, op), np.nan, np.float32)
    want[:n] = 0
    want[:n, :F] = nu.gather_clamped(values, np.arange(row0, row0 + n))
    same_bits(back, want, "row range")


def test_every_regime_row_is_run(sms):
    """The kernels the cases above reach on this GPU: every one the dispatch has."""
    got = {cs.mean_regimes(cs.mean_case(n, sms), sms)["kernel"] for n in cs.MEAN_CASES}
    got |= {cs.row_regimes(cs.row_case(n, sms), sms)["kernel"] for n in cs.ROW_CASES}
    assert got == {"tma2", "tma2_drop", "tma", "ldg", "scalar", "scalar_drop", "narrow_bf16", "narrow_i8", "rows_tma",
                   "rows_simple", "vec_bf16", "scalar_bf16", "scalar_f32", "i8row"}
    print("\n%d SMs: %s" % (sms, ", ".join(sorted(got))))
