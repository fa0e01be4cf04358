"""Supervised GraphSAGE trainer: the reference's `python -m graphsage.supervised_train` (graphsage/supervised_train.py)
over this package's kernels.

    python -m graphsage_b200.supervised_train --train_prefix ./example_data/ppi --model graphsage_mean --sigmoid

Same flags (names, types, defaults), model branches, loop, print lines, log directory and stats files as the reference.
Differences:
  * --gpu N selects cuda:N (cuda:0, with one line of output, when N does not exist); CUDA_VISIBLE_DEVICES is not set.
  * time= is the wall time per step between device synchronises at the print steps (train_cli.StepClock): a step here
    returns before the GPU finishes it.
  * Full-size batches replay one CUDA graph (graphed_train_step); print steps and the short last batch of an epoch run
    the eager train_step, which computes the same bits.
  * The samplers and initialisers draw from this package's seeded streams, not TensorFlow's; numpy is seeded with 123
    before the iterator is built, so tables, shuffles and validation draws are the reference's.
  * No TensorBoard summaries (summary_writer); --log_device_placement is accepted and ignored.
"""
import os
import sys
import time

import numpy as np
import torch

from . import inits
from .minibatch import NodeMinibatchIterator
from .models import SAGEInfo
from .neigh_samplers import UniformNeighborSampler
from .supervised_models import SupervisedGraphsage
from .train_cli import StepClock, parse_or_exit, select_device, to_device, train_loop
from .utils import load_data

SEED = 123

# reference supervised_train.py:28-57
FLAGS_SPEC = [
    ("log_device_placement", "boolean", False),
    ("model", "string", "graphsage_mean"),
    ("learning_rate", "float", 0.01),
    ("model_size", "string", "small"),
    ("train_prefix", "string", ""),
    ("epochs", "integer", 10),
    ("dropout", "float", 0.0),
    ("weight_decay", "float", 0.0),
    ("max_degree", "integer", 128),
    ("samples_1", "integer", 25),
    ("samples_2", "integer", 10),
    ("samples_3", "integer", 0),
    ("dim_1", "integer", 128),
    ("dim_2", "integer", 128),
    ("random_context", "boolean", True),
    ("batch_size", "integer", 512),
    ("sigmoid", "boolean", False),
    ("identity_dim", "integer", 0),
    ("base_log_dir", "string", "."),
    ("validate_iter", "integer", 5000),
    ("validate_batch_size", "integer", 256),
    ("gpu", "integer", 1),
    ("print_every", "integer", 5),
    ("max_total_steps", "integer", 10 ** 10),
]

# --model -> (aggregator_type, concat, width multiplier of dim_1 / dim_2)   (supervised_train.py:150-239)
MODELS = {"graphsage_mean": ("mean", True, 1), "gcn": ("gcn", False, 2), "graphsage_seq": ("seq", True, 1),
          "graphsage_maxpool": ("maxpool", True, 1), "graphsage_meanpool": ("meanpool", True, 1)}


def parse_flags(argv=()):
    return parse_or_exit(FLAGS_SPEC, argv)


def _counts(tp, fp, fn):
    """2tp / (2tp + fp + fn), 0 where nothing was true or predicted (sklearn's zero_division default)."""
    den = 2 * tp + fp + fn
    return np.where(den > 0, 2 * tp / np.maximum(den, 1), 0.0)


def calc_f1(y_true, y_pred, sigmoid):
    """(micro F1, macro F1) of sklearn.metrics.f1_score (supervised_train.py:63-70).  sigmoid: multi-label, predictions
    thresholded at > 0.5, every label column counts; else argmax of both, over the labels present in either."""
    y_true, y_pred = np.asarray(y_true), np.asarray(y_pred)
    if sigmoid:
        t, p = y_true > 0.5, y_pred > 0.5
    else:
        a, b = np.argmax(y_true, axis=1), np.argmax(y_pred, axis=1)
        labels = np.union1d(a, b)
        t, p = a[:, None] == labels[None, :], b[:, None] == labels[None, :]
    tp = (t & p).sum(axis=0).astype(np.float64)
    fp = (~t & p).sum(axis=0).astype(np.float64)
    fn = (t & ~p).sum(axis=0).astype(np.float64)
    micro = float(_counts(tp.sum(), fp.sum(), fn.sum()))
    macro = float(_counts(tp, fp, fn).mean()) if len(tp) else 0.0
    return micro, macro


def log_dir(flags):
    """supervised_train.py:81-89 (creates the directory)."""
    d = flags.base_log_dir + "/sup-" + flags.train_prefix.split("/")[-2]
    d += "/{model:s}_{model_size:s}_{lr:0.4f}/".format(model=flags.model, model_size=flags.model_size,
                                                       lr=flags.learning_rate)
    if not os.path.exists(d):
        os.makedirs(d)
    return d


def val_stats_line(cost, f1_mic, f1_mac, duration):
    return "loss={:.5f} f1_micro={:.5f} f1_macro={:.5f} time={:.5f}".format(cost, f1_mic, f1_mac, duration)


def test_stats_line(cost, f1_mic, f1_mac):
    return "loss={:.5f} f1_micro={:.5f} f1_macro={:.5f}".format(cost, f1_mic, f1_mac)


def num_classes_of(class_map):
    first = next(iter(class_map.values()))
    return len(first) if isinstance(first, list) else len(set(class_map.values()))


def build_iterator(train_data, flags):
    """supervised_train.py:124-146 with numpy seeded first (the reference seeds it at import)."""
    G, _, id_map, context, class_map = train_data[:5]
    np.random.seed(SEED)
    return NodeMinibatchIterator(G, id_map, None, class_map, num_classes_of(class_map), batch_size=flags.batch_size,
                                 max_degree=flags.max_degree, context_pairs=context if flags.random_context else None)


def build_model(flags, features, minibatch, num_classes, device):
    """The --model branches of supervised_train.py:150-239.  features: [N+1, F] with the dummy row, or None."""
    if flags.model not in MODELS:
        raise Exception('Error: model name unrecognized.')
    kind, concat, mult = MODELS[flags.model]
    inits.manual_seed(SEED, device)
    sampler = UniformNeighborSampler(torch.from_numpy(minibatch.adj).to(device))
    widths = [(flags.samples_1, mult * flags.dim_1), (flags.samples_2, mult * flags.dim_2)]
    if flags.model == "graphsage_mean":
        if flags.samples_3 != 0:
            widths.append((flags.samples_3, flags.dim_2))
        elif flags.samples_2 == 0:
            widths = widths[:1]
    layer_infos = [SAGEInfo("node", sampler, k, d) for k, d in widths]
    return SupervisedGraphsage(num_classes, {"batch_size": flags.batch_size, "dropout": flags.dropout}, features,
                               sampler.adj_info, minibatch.deg, layer_infos, concat=concat, aggregator_type=kind,
                               model_size=flags.model_size, sigmoid_loss=flags.sigmoid, identity_dim=flags.identity_dim,
                               learning_rate=flags.learning_rate, weight_decay=flags.weight_decay, device=device)


def _eval_batch(model, feed, labels, device):
    """One forward pass at dropout 0: the loss and the predictions from the same logits."""
    with torch.no_grad():
        loss = model.loss(to_device(feed["batch"], np.int32, device), to_device(labels, np.float32, device))
        return loss, model.last_predictions()


def evaluate(model, minibatch, size, flags, device):
    """supervised_train.py:73-79: one sampled validation batch."""
    t = time.time()
    feed, labels = minibatch.node_val_feed_dict(size)
    loss, preds = _eval_batch(model, feed, labels, device)
    mic, mac = calc_f1(labels, preds.cpu().numpy(), flags.sigmoid)
    return float(loss), mic, mac, time.time() - t


def incremental_evaluate(model, minibatch, size, flags, device, test=False):
    """supervised_train.py:91-110: every val (test) node, in batches of `size`."""
    t = time.time()
    losses, preds, labels = [], [], []
    finished, iter_num = False, 0
    while not finished:
        feed, batch_labels, finished, _ = minibatch.incremental_node_val_feed_dict(size, iter_num, test=test)
        loss, p = _eval_batch(model, feed, batch_labels, device)
        losses.append(loss)
        preds.append(p)
        labels.append(batch_labels)
        iter_num += 1
    mic, mac = calc_f1(np.vstack(labels), torch.cat(preds).cpu().numpy(), flags.sigmoid)
    return float(torch.stack(losses).cpu().numpy().mean()), mic, mac, time.time() - t


def train(train_data, flags, device=None):
    """supervised_train.py:122-330.  train_data: load_data's (G, feats, id_map, walks, class_map).  Returns the model."""
    device = select_device(flags.gpu) if device is None else device
    features = train_data[1]
    if features is not None:
        features = np.vstack([features, np.zeros((features.shape[1],))])        # the dummy row (:133-135)
    minibatch = build_iterator(train_data, flags)
    model = build_model(flags, features, minibatch, minibatch.num_classes, device)
    sampler = model.layer_infos[0].neigh_sampler
    adj, test_adj = sampler.adj_info, torch.from_numpy(minibatch.test_adj).to(device)
    replay = model.graphed_train_step(flags.batch_size)
    clock = StepClock(device)
    val, last = {}, {}

    def step(item, it, total_steps, eager):
        feed, labels = item
        if eager:
            loss = model.train_step(to_device(feed["batch"], np.int32, device), to_device(labels, np.float32, device))
            last["labels"], last["preds"] = labels, model.last_predictions()    # before a validation replaces them
            return loss
        return replay(torch.from_numpy(np.asarray(feed["batch"], np.int32)).pin_memory(),
                      torch.from_numpy(np.asarray(labels, np.float32)).pin_memory())

    def validate():
        sampler.set_adj(test_adj)
        if flags.validate_batch_size == -1:
            r = incremental_evaluate(model, minibatch, flags.batch_size, flags, device)
        else:
            r = evaluate(model, minibatch, flags.validate_batch_size, flags, device)
        sampler.set_adj(adj)
        val["cost"], val["mic"], val["mac"], _ = r
        return val["cost"]

    def after(loss, it, total_steps, printing):
        if not printing:
            return
        train_cost = float(loss)
        train_mic, train_mac = calc_f1(last["labels"], last["preds"].cpu().numpy(), flags.sigmoid)
        print("Iter:", '%04d' % it,
              "train_loss=", "{:.5f}".format(train_cost),
              "train_f1_mic=", "{:.5f}".format(train_mic),
              "train_f1_mac=", "{:.5f}".format(train_mac),
              "val_loss=", "{:.5f}".format(val["cost"]),
              "val_f1_mic=", "{:.5f}".format(val["mic"]),
              "val_f1_mac=", "{:.5f}".format(val["mac"]),
              "time=", "{:.5f}".format(clock.avg(total_steps + 1)))

    train_loop(minibatch, flags, step, validate, after)

    print("Optimization Finished!")
    sampler.set_adj(test_adj)
    cost, mic, mac, duration = incremental_evaluate(model, minibatch, flags.batch_size, flags, device)
    print("Full validation stats:",
          "loss=", "{:.5f}".format(cost),
          "f1_micro=", "{:.5f}".format(mic),
          "f1_macro=", "{:.5f}".format(mac),
          "time=", "{:.5f}".format(duration))
    with open(log_dir(flags) + "val_stats.txt", "w") as fp:
        fp.write(val_stats_line(cost, mic, mac, duration))
    print("Writing test set stats to file (don't peak!)")
    cost, mic, mac, duration = incremental_evaluate(model, minibatch, flags.batch_size, flags, device, test=True)
    with open(log_dir(flags) + "test_stats.txt", "w") as fp:
        fp.write(test_stats_line(cost, mic, mac))
    return model


def main(argv=None):
    flags = parse_flags(sys.argv[1:] if argv is None else argv)
    print("Loading training data..")
    train_data = load_data(flags.train_prefix)
    print("Done loading training data..")
    return train(train_data, flags)


if __name__ == "__main__":
    main()
