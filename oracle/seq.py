"""Oracle for the LSTM sequence aggregator (reference graphsage/aggregators.py:363-449) - numpy, fp32 by default (pass
dtype=np.float64 for the error-budget twin).

The cell is TF 1.8's BasicLSTMCell as documented: z = [x, h] @ kernel + bias with gate columns i, j, f, o;
c' = c * sigmoid(f + forget_bias) + sigmoid(i) * tanh(j); h' = tanh(c') * sigmoid(o); forget_bias = 1.0.  dynamic_rnn with
sequence_length freezes the state past the length and outputs zeros there; the aggregator gathers output len - 1.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .aggregate import gather_rows, identity, relu

FORGET_BIAS = 1.0


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def cell_kernel(seed, shape):
    """The LSTM kernel of tests/golden/seq.npz, which stores its seed rather than its [K + H, 4H] values: U(-r, r),
    r = sqrt(6 / (fan_in + fan_out)) (tf.get_variable's default, glorot uniform), fp32, drawn from numpy's legacy
    RandomState(seed), a stream NumPy keeps fixed across releases."""
    r = np.sqrt(6.0 / (shape[0] + shape[1]))
    return np.random.RandomState(int(seed)).uniform(-r, r, size=tuple(int(s) for s in shape)).astype(np.float32)


def seq_lengths(neigh_vecs):
    """aggregators.py:411-414: used = sign(max |x| over features), len = max(1, sum used); -0.0 counts as zero."""
    used = (np.abs(np.asarray(neigh_vecs)).max(axis=2) > 0).astype(np.int64)
    return np.maximum(used.sum(axis=1), 1).astype(np.int32)


def lstm_run(P, Wh, lengths, train=False, dtype=np.float32):
    """The recurrence on the input projection P [n, k, 4H] = X W_x + b: h after len_i steps [n, H]; with train=True also
    the post-activation gates [n, k, 4H] (i, j, f + 1, o), c [n, k, H] and h_{t-1} [n, k, H], zero for t >= len_i."""
    P, Wh = np.asarray(P, dtype), np.asarray(Wh, dtype)
    n, k, G = P.shape
    H = G // 4
    h, c = np.zeros((n, H), dtype), np.zeros((n, H), dtype)
    gates, cs, hp = np.zeros((n, k, G), dtype), np.zeros((n, k, H), dtype), np.zeros((n, k, H), dtype)
    for t in range(k):
        on = (t < lengths)[:, None]
        z = P[:, t] + h @ Wh
        ig, jg = sigmoid(z[:, :H]), np.tanh(z[:, H:2 * H])
        fg, og = sigmoid(z[:, 2 * H:3 * H] + FORGET_BIAS), sigmoid(z[:, 3 * H:])
        cn = c * fg + ig * jg
        hn = np.tanh(cn) * og
        gates[:, t] = np.where(on, np.concatenate([ig, jg, fg, og], axis=1), 0)
        cs[:, t] = np.where(on, cn, 0)
        hp[:, t] = np.where(on, h, 0)
        c, h = np.where(on, cn, c), np.where(on, hn, h)
    return (h, gates, cs, hp) if train else h


def lstm_bptt(dh_last, gates, cs, lengths, Wh, dtype=np.float64):
    """Backpropagation through time of lstm_run: dZ [n, k, 4H], the gradient of the pre-activations z_t (zero for
    t >= len_i), from the gradient dh_last of h after len_i steps."""
    gates, cs, Wh = np.asarray(gates, dtype), np.asarray(cs, dtype), np.asarray(Wh, dtype)
    n, k, G = gates.shape
    H = G // 4
    dZ = np.zeros((n, k, G), dtype)
    dh, dc = np.zeros((n, H), dtype), np.zeros((n, H), dtype)
    last = np.asarray(lengths) - 1
    for t in range(k - 1, -1, -1):
        on = (t < lengths)[:, None]
        d = dh + np.where((t == last)[:, None], np.asarray(dh_last, dtype), 0)
        ig, jg, fg, og = gates[:, t, :H], gates[:, t, H:2 * H], gates[:, t, 2 * H:3 * H], gates[:, t, 3 * H:]
        cp = cs[:, t - 1] if t > 0 else np.zeros((n, H), dtype)
        tc = np.tanh(cs[:, t])
        dct = dc + d * og * (1 - tc * tc)
        z = np.concatenate([dct * jg * ig * (1 - ig), dct * ig * (1 - jg * jg), dct * cp * fg * (1 - fg),
                            d * tc * og * (1 - og)], axis=1)
        z = np.where(on, z, 0)
        dZ[:, t] = z
        dc = np.where(on, dct * fg, 0)
        dh = z @ Wh.T
    return dZ


# ---------------------------------------------------------------- operand-exact references of the recurrence kernels
U = 2.0 ** -24                # fp32 unit roundoff (round to nearest)
TINY = 2.0 ** -149            # spacing of the fp32 subnormals: the absolute error of a rounding that underflows
FLT_MIN = 2.0 ** -126
# CUDA's expf and tanhf are not correctly rounded.  The CUDA C++ Programming Guide (appendix "Mathematical Functions",
# single precision, CUDA 12) gives a maximum error of 2 ulp over the full range for both; x / y and 1 / x are IEEE-rounded
# (0.5 ulp) because the library is built without fast math (-prec-div=true).  An ulp of y is at most 2^-23 |y| = 2 U |y|.
EXPF_ULP, TANHF_ULP = 2, 2
# sigmoid(x) = 1 / (1 + expf(-x)): expf 2 ulp (4 U), the add (U), the division (U), plus 1 U for the second-order terms.
SIGMOID_REL = (2 * EXPF_ULP + 3) * U
TANH_REL = 2 * TANHF_ULP * U


def _rnd(v, e):
    """An fp32 result whose exact value v is known within e from its operands' errors, after its own rounding: one
    more U |computed| <= U (|v| + e), plus TINY for a result that underflows."""
    return v, e + U * (np.abs(v) + e) + TINY


def _mul(a, b):
    (x, ex), (y, ey) = a, b
    return _rnd(x * y, np.abs(x) * ey + np.abs(y) * ex + ex * ey)


def _add(a, b):
    (x, ex), (y, ey) = a, b
    return _rnd(x + y, ex + ey)


def _neg(a):
    return -a[0], a[1]


def _one_minus(a):
    return _add((1.0, 0.0), _neg(a))


def _apply(fn, a):
    """fn in {"sigmoid", "tanh"} of an operand known within e: both have an even derivative that falls with |x|, so
    |fn(x') - fn(x)| <= fn'(max(|x| - e, 0)) e for |x' - x| <= e (mean value theorem); then the function's own relative
    error, and FLT_MIN for a result the device returns as 0 (expf(-x) overflows for x < -88.7, where
    sigmoid(x) < 2^-127)."""
    x, ex = a
    near = np.maximum(np.abs(x) - ex, 0.0)
    if fn == "sigmoid":                                   # sigmoid' = sigmoid(x) sigmoid(-x), no cancellation at large |x|
        with np.errstate(over="ignore"):
            v, slope, rel = sigmoid(x), sigmoid(near) * sigmoid(-near), SIGMOID_REL
    else:                                                 # tanh' = 1 - tanh^2 = 4 e^-2x / (1 + e^-2x)^2 for x >= 0
        q = np.exp(-2.0 * near)
        v, slope, rel = np.tanh(x), 4.0 * q / (1.0 + q) ** 2, TANH_REL
    e = slope * ex
    return v, e + rel * (np.abs(v) + e) + FLT_MIN


def _on_mask(lengths, k):
    """[n, k] bool: step t of sequence i runs.  The kernels clamp len to [0, k]."""
    L = np.clip(np.asarray(lengths, np.int64).reshape(-1), 0, k)
    return np.arange(k)[None, :] < L[:, None], L


def lstm_step_reference(P, Wh, h_prev, c_prev, lengths):
    """Teacher-forced float64 reference of gs_lstm_forward, one step at a time from the kernel's OWN state: step t of
    sequence i is recomputed from P[i, t], the kernel's h_{t-1} (its saved h_prev[i, t]) and the kernel's c_{t-1}
    (c_prev[i, t] = its saved c[i, t - 1], 0 at t = 0).  The error of each step is then local and does not grow with k,
    so one bound holds at every k.  P [n, k, 4H], Wh [H, 4H], h_prev / c_prev [n, k, H] (fp32 values).
    Returns {"gates": (ref, bound) [n, k, 4H], "c": ..., "h": ... [n, k, H]}: h[i, t] is h_t, which the kernel saves as
    h_prev[i, t + 1] (or returns as h_last at t = len - 1).  Past len both are 0: the kernel must write exact zeros.

    The bound, for the kernel's arithmetic on exactly these fp32 operands (u = 2^-24):
      z = P_t + h_{t-1} W_h is an FMA chain over the H hidden units (lstm_forward_kernel: acc = P, then acc =
          fmaf(h_m, w_m, acc)), H roundings: |dz| <= gamma_H (|P| + sum_m |h_m w_m|) <= (H + 1) u S1 (gamma_H =
          H u / (1 - H u), below (H + 1) u for H <= 2^12).
      Each later +, - and * is one rounding, bounded as a separate operation (which also covers any FMA the compiler
          contracts them into): an fp32 result known within e from its operands is within e + u (|v| + e) + 2^-149
          (_rnd; for products |x| e_y + |y| e_x + e_x e_y, for sums e_x + e_y).  The forget gate's z_f + 1 is one add.
      sigmoid(x) = 1 / (1 + expf(-x)) and tanhf: an operand error e moves the value by at most f'(max(|x| - e, 0)) e
          (sigmoid' <= 1/4, tanh' <= 1, both falling with |x|, so saturated gates get tight bounds); then a relative
          error of SIGMOID_REL = 7 u (expf 2 ulp = 4 u, the add and the division 1 u each, 1 u spare) or TANH_REL = 4 u
          (tanhf 2 ulp), and FLT_MIN absolute.
      c_t = c_{t-1} f + i j and h_t = tanh(c_t) o follow by the product and sum rules from the gate bounds.
    """
    P, Wh = np.asarray(P, np.float64), np.asarray(Wh, np.float64)
    n, k, G = P.shape
    H = G // 4
    on, _ = _on_mask(lengths, k)
    P = np.where(on[:, :, None], P, 0.0)                  # rows past len are never read: they may hold anything
    hp, cp = np.asarray(h_prev, np.float64), np.asarray(c_prev, np.float64)
    z = P + hp @ Wh
    ez = (H + 1) * U * (np.abs(P) + np.abs(hp) @ np.abs(Wh))
    part = lambda a, g: a[:, :, g * H:(g + 1) * H]        # noqa: E731
    ig = _apply("sigmoid", (part(z, 0), part(ez, 0)))
    jg = _apply("tanh", (part(z, 1), part(ez, 1)))
    fg = _apply("sigmoid", _add((part(z, 2), part(ez, 2)), (FORGET_BIAS, 0.0)))
    og = _apply("sigmoid", (part(z, 3), part(ez, 3)))
    c = _add(_mul((cp, 0.0), fg), _mul(ig, jg))
    h = _mul(_apply("tanh", c), og)
    gates = tuple(np.concatenate([g[j] for g in (ig, jg, fg, og)], axis=2) for j in (0, 1))
    live = on[:, :, None]
    return {name: (np.where(live, v, 0.0), np.where(live, e, 0.0)) for name, (v, e) in
            (("gates", gates), ("c", c), ("h", h))}


def lstm_bptt_step_reference(dh_last, gates, c, lengths, Wh, dZ):
    """Float64 reference of gs_lstm_backward on its own operands - the forward's saved fp32 gates and c, not an fp64
    trajectory - with dh teacher-forced: the dh_t that step t reads is recomputed as dZ_{t+1} W_h^T from the kernel's OWN
    dZ_{t+1} (dZ [n, k, 4H], the output being checked), so a wrong step cannot hide behind its successor and the dh
    error does not accumulate over t.  dc_t, which the kernel keeps in registers and never writes, is carried.
    dh_last [n, H], gates [n, k, 4H], c [n, k, H], Wh [H, 4H].  Returns (ref, bound) [n, k, 4H], 0 and 0 past len.

    The bound follows lstm_step_reference's rules on the kernel's expressions, in its order of evaluation:
      dh_t = sum over the 4H columns of dz_{t+1} W_h^T, an FMA chain of 4H roundings from +0: <= (4H + 1) u S1 with
          S1 = |dz_{t+1}| |W_h|^T.
      d = dh_t + dh_last (at t = len - 1);  tc = tanhf(c_t) (TANH_REL);  z_o = ((d tc) o)(1 - o);
      dc_t = dc_{t+1} + (d o)(1 - tc tc);  z_i = ((dc_t j) i)(1 - i);  z_j = (dc_t i)(1 - j j);
      z_f = ((dc_t c_{t-1}) f)(1 - f);  dc_{t-1} = dc_t f.
    The dc carry is the only error that accumulates: each step multiplies the carried bound by f <= 1 and adds its own
    roundings, so the bound at step t grows at most linearly in the number of steps after t (len - 1 - t) and no
    faster; it is tracked exactly, step by step, rather than bounded by k.  Where a saturated gate makes a factor
    (1 - i), (1 - j j), (1 - f), (1 - o) exactly 0 the reference is exactly 0 and the bound is O(2^-149).
    """
    gates, c, Wh = np.asarray(gates, np.float64), np.asarray(c, np.float64), np.asarray(Wh, np.float64)
    dZk = np.asarray(dZ, np.float64)
    n, k, G = gates.shape
    H = G // 4
    on, L = _on_mask(lengths, k)
    dhl = np.asarray(dh_last, np.float64)
    dh_in, e_in = np.zeros((n, k, H)), np.zeros((n, k, H))
    if k > 1:
        nxt = np.where(on[:, 1:, None], dZk[:, 1:], 0.0)  # what a kernel with zeros past len multiplies
        dh_in[:, :-1] = nxt @ Wh.T
        e_in[:, :-1] = (4 * H + 1) * U * (np.abs(nxt) @ np.abs(Wh).T)
    ref, bound = np.zeros((n, k, G)), np.zeros((n, k, G))
    dc = (np.zeros((n, H)), np.zeros((n, H)))
    for t in range(k - 1, -1, -1):
        live = on[:, t, None]
        last = (t == L - 1)[:, None]
        d = (dh_in[:, t], e_in[:, t])
        dl = _add(d, (np.where(last, dhl, 0.0), 0.0))
        d = (np.where(last, dl[0], d[0]), np.where(last, dl[1], d[1]))
        ig, jg, fg, og = ((gates[:, t, g * H:(g + 1) * H], 0.0) for g in range(4))
        ct = (c[:, t], 0.0)
        cp = (c[:, t - 1] if t > 0 else np.zeros((n, H)), 0.0)
        tc = _apply("tanh", ct)
        zo = _mul(_mul(_mul(d, tc), og), _one_minus(og))
        dct = _add(dc, _mul(_mul(d, og), _add((1.0, 0.0), _neg(_mul(tc, tc)))))
        zi = _mul(_mul(_mul(dct, jg), ig), _one_minus(ig))
        zj = _mul(_mul(dct, ig), _add((1.0, 0.0), _neg(_mul(jg, jg))))
        zf = _mul(_mul(_mul(dct, cp), fg), _one_minus(fg))
        for g, z in enumerate((zi, zj, zf, zo)):
            ref[:, t, g * H:(g + 1) * H] = np.where(live, z[0], 0.0)
            bound[:, t, g * H:(g + 1) * H] = np.where(live, z[1], 0.0)
        dcn = _mul(dct, fg)
        dc = (np.where(live, dcn[0], dc[0]), np.where(live, dcn[1], dc[1]))
    return ref, bound


def saturated(gates):
    """[..., 4H] bool: where a saved gate sits exactly at a saturation value - sigmoid gates at 0 or 1, the tanh gate
    at +-1 - so that its backward factor i (1 - i), 1 - j j, f (1 - f), o (1 - o) is exactly 0 and dZ must be +-0."""
    g = np.asarray(gates)
    H = g.shape[-1] // 4
    tanh_col = (np.arange(4 * H) // H == 1)
    return np.where(tanh_col, np.abs(g) == 1.0, (g == 0.0) | (g == 1.0))


def bound_ratio(out, ref, bound):
    """max |out - ref| / bound (<= 1 passes).  Where the bound is 0 (rows past len) out must equal ref exactly; a NaN or
    inf in out fails."""
    out = np.asarray(out, np.float64)
    err = np.where(np.isfinite(out), np.abs(out - ref), np.inf)
    if err.size == 0:
        return 0.0
    r = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)
    return float(r.max())


def check_lstm_forward(P, Wh, lengths, h_last, gates, c, h_prev):
    """(ok, worst) for one gs_lstm_forward call with training outputs: every saved row and h_last against
    lstm_step_reference on the kernel's own state.  P [n, k, 4H], gates [n, k, 4H], c / h_prev [n, k, H], h_last [n, H];
    worst maps each output to its largest error / bound."""
    c, h_prev = np.asarray(c, np.float64), np.asarray(h_prev, np.float64)
    n, k, H = c.shape
    c_prev = np.concatenate([np.zeros((n, 1, H)), c[:, :-1]], axis=1)
    r = lstm_step_reference(P, Wh, h_prev, c_prev, lengths)
    on, L = _on_mask(lengths, k)
    hv, hb = r["h"]
    hp_ref, hp_bound = np.zeros((n, k, H)), np.zeros((n, k, H))     # h_prev[t] = h_{t-1}; exactly 0 at t = 0 and past len
    hp_ref[:, 1:], hp_bound[:, 1:] = hv[:, :-1], hb[:, :-1]
    live = on[:, :, None]
    hp_ref, hp_bound = np.where(live, hp_ref, 0.0), np.where(live, hp_bound, 0.0)
    idx = np.maximum(L - 1, 0)
    has = (L > 0)[:, None]
    hl_ref = np.where(has, hv[np.arange(n), idx], 0.0)
    hl_bound = np.where(has, hb[np.arange(n), idx], 0.0)
    worst = {"gates": bound_ratio(gates, *r["gates"]), "c": bound_ratio(c, *r["c"]),
             "h_prev": bound_ratio(h_prev, hp_ref, hp_bound), "h_last": bound_ratio(h_last, hl_ref, hl_bound)}
    return max(worst.values()) <= 1.0, worst


def check_lstm_backward(dh_last, gates, c, lengths, Wh, dZ):
    """(ok, worst) for one gs_lstm_backward call against lstm_bptt_step_reference on its own operands and dZ."""
    ref, bound = lstm_bptt_step_reference(dh_last, gates, c, lengths, Wh, dZ)
    worst = bound_ratio(dZ, ref, bound)
    return worst <= 1.0, worst


def seq_hidden(neigh_vecs, kernel, bias, dtype=np.float32):
    """dynamic_rnn + the gather of output len - 1 (aggregators.py:407-433): h after len_i steps, [n, H]."""
    x = np.asarray(neigh_vecs, dtype)
    n, k, K = x.shape
    kernel, bias = np.asarray(kernel, dtype), np.asarray(bias, dtype)
    P = (x.reshape(n * k, K) @ kernel[:K] + bias).reshape(n, k, -1)
    return lstm_run(P, kernel[K:], seq_lengths(x), dtype=dtype)


def seq_aggregator(self_vecs, neigh_vecs, kernel, cell_bias, neigh_weights, self_weights, concat=False, act=relu,
                   bias=None, dtype=np.float32):
    """aggregators.py:405-449: act(concat_or_add(self @ Ws, h_len @ Wn) (+ bias)); no dropout."""
    h = seq_hidden(neigh_vecs, kernel, cell_bias, dtype)
    from_neighs = h @ np.asarray(neigh_weights, dtype)
    from_self = np.asarray(self_vecs, dtype) @ np.asarray(self_weights, dtype)
    out = np.concatenate([from_self, from_neighs], axis=1) if concat else from_self + from_neighs
    if bias is not None:
        out = out + np.asarray(bias, dtype)
    return act(out)


def aggregate_khop_seq(samples, features, num_samples, support_sizes, batch_size, aggregators, concat, dtype=np.float32):
    """reference models.py:278-330 with SeqAggregator: `aggregators` is one dict per layer with kernel, cell_bias,
    neigh_weights, self_weights (and optionally bias)."""
    hidden = [gather_rows(features, s).astype(dtype) for s in samples]
    L = len(num_samples)
    for layer in range(L):
        act = identity if layer == L - 1 else relu
        a = aggregators[layer]
        nxt = []
        for hop in range(L - layer):
            d = hidden[hop + 1].shape[1]
            neigh = hidden[hop + 1].reshape(batch_size * support_sizes[hop], num_samples[L - hop - 1], d)
            nxt.append(seq_aggregator(hidden[hop], neigh, a["kernel"], a["cell_bias"], a["neigh_weights"],
                                      a["self_weights"], concat, act, a.get("bias"), dtype))
        hidden = nxt
    return hidden[0]


def torch_seq_layer(self_vecs, neigh, kernel, cell_bias, self_weights, neigh_weights, k, concat, last):
    """seq_aggregator as differentiable torch (any dtype / device) for gradient checks; neigh is [n * k, K].  The lengths
    come from the values (not differentiable), as in the reference."""
    import torch
    n, K = self_vecs.shape[0], neigh.shape[1]
    x = neigh.reshape(n, k, K)
    lengths = torch.clamp((x.abs().amax(dim=2) > 0).sum(dim=1), min=1)
    H = kernel.shape[1] // 4
    P = (neigh @ kernel[:K] + cell_bias).reshape(n, k, 4 * H)
    h = torch.zeros(n, H, dtype=neigh.dtype, device=neigh.device)
    c = torch.zeros_like(h)
    for t in range(k):
        on = (t < lengths).unsqueeze(1)
        z = P[:, t] + h @ kernel[K:]
        cn = c * torch.sigmoid(z[:, 2 * H:3 * H] + FORGET_BIAS) + torch.sigmoid(z[:, :H]) * torch.tanh(z[:, H:2 * H])
        hn = torch.tanh(cn) * torch.sigmoid(z[:, 3 * H:])
        c, h = torch.where(on, cn, c), torch.where(on, hn, h)
    fs, fn = self_vecs @ self_weights, h @ neigh_weights
    y = torch.cat([fs, fn], dim=1) if concat else fs + fn
    return y if last else torch.relu(y)
