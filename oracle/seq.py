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
