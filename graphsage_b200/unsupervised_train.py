"""Unsupervised GraphSAGE / Node2Vec trainer: the reference's `python -m graphsage.unsupervised_train`
(graphsage/unsupervised_train.py) over this package's kernels.

    python -m graphsage_b200.unsupervised_train --train_prefix ./example_data/ppi --model graphsage_mean \\
        --max_total_steps 1000 --validate_iter 10

Same flags (names, types, defaults), model branches, loop, print lines (with the two MRR moving averages), log directory
and `val.npy` / `val.txt` embedding files as the reference, and for --model n2v its second phase (walks from the val and
test nodes, `val-test.npy` / `val-test.txt`).  Differences, as in supervised_train: --gpu selects cuda:N (cuda:0 when N
does not exist) without touching CUDA_VISIBLE_DEVICES; time= is wall time per step between device synchronises at the
print steps; full-size batches replay one CUDA graph, print steps and short batches run the eager train_step (same bits);
samplers and initialisers use this package's seeded streams (numpy is seeded with 123 before the iterator); no
TensorBoard summaries; --log_device_placement is accepted and ignored.  The reference's attempt to freeze the train
nodes' context rows in the n2v second phase has no effect there, so every table keeps training here too.
"""
import os
import sys
import time

import numpy as np
import torch

from . import inits
from .minibatch import EdgeMinibatchIterator
from .models import SAGEInfo
from .neigh_samplers import UniformNeighborSampler
from .node2vec import Node2VecModel
from .train_cli import StepClock, parse_or_exit, select_device, to_device, train_loop
from .unsupervised_models import UnsupervisedGraphsage
from .utils import load_data, run_random_walks

SEED = 123

# reference unsupervised_train.py:25-55
FLAGS_SPEC = [
    ("log_device_placement", "boolean", False),
    ("model", "string", "graphsage"),
    ("learning_rate", "float", 0.00001),
    ("model_size", "string", "small"),
    ("train_prefix", "string", ""),
    ("epochs", "integer", 1),
    ("dropout", "float", 0.0),
    ("weight_decay", "float", 0.0),
    ("max_degree", "integer", 100),
    ("samples_1", "integer", 25),
    ("samples_2", "integer", 10),
    ("dim_1", "integer", 128),
    ("dim_2", "integer", 128),
    ("random_context", "boolean", True),
    ("neg_sample_size", "integer", 20),
    ("batch_size", "integer", 512),
    ("n2v_test_epochs", "integer", 1),
    ("identity_dim", "integer", 0),
    ("save_embeddings", "boolean", True),
    ("base_log_dir", "string", "."),
    ("validate_iter", "integer", 5000),
    ("validate_batch_size", "integer", 256),
    ("gpu", "integer", 1),
    ("print_every", "integer", 50),
    ("max_total_steps", "integer", 10 ** 10),
]

# --model -> (aggregator_type, concat, width multiplier of dim_1 / dim_2)   (unsupervised_train.py:152-226)
MODELS = {"graphsage_mean": ("mean", True, 1), "gcn": ("gcn", False, 2), "graphsage_seq": ("seq", True, 1),
          "graphsage_maxpool": ("maxpool", True, 1), "graphsage_meanpool": ("meanpool", True, 1)}


def parse_flags(argv=()):
    return parse_or_exit(FLAGS_SPEC, argv)


def log_dir(flags):
    """unsupervised_train.py:61-69 (creates the directory)."""
    d = flags.base_log_dir + "/unsup-" + flags.train_prefix.split("/")[-2]
    d += "/{model:s}_{model_size:s}_{lr:0.6f}/".format(model=flags.model, model_size=flags.model_size,
                                                       lr=flags.learning_rate)
    if not os.path.exists(d):
        os.makedirs(d)
    return d


def build_iterator(train_data, flags):
    """unsupervised_train.py:132-148 with numpy seeded first (the reference seeds it at import)."""
    G, _, id_map, context = train_data[:4]
    np.random.seed(SEED)
    return EdgeMinibatchIterator(G, id_map, None, batch_size=flags.batch_size, max_degree=flags.max_degree,
                                 context_pairs=context if flags.random_context else None)


def build_model(flags, features, minibatch, device):
    """The --model branches of unsupervised_train.py:152-234.  features: [N+1, F] with the dummy row, or None."""
    if flags.model == "n2v":
        # dict_size = features.shape[0] = N + 1 rows; 2x because graphsage uses concat (:227-232)
        return Node2VecModel({"batch_size": flags.batch_size}, len(minibatch.id2idx) + 1, minibatch.deg,
                             nodevec_dim=2 * flags.dim_1, lr=flags.learning_rate, neg_sample_size=flags.neg_sample_size,
                             seed=SEED, device=device)
    if flags.model not in MODELS:
        raise Exception('Error: model name unrecognized.')
    kind, concat, mult = MODELS[flags.model]
    inits.manual_seed(SEED, device)
    sampler = UniformNeighborSampler(torch.from_numpy(minibatch.adj).to(device))
    layer_infos = [SAGEInfo("node", sampler, flags.samples_1, mult * flags.dim_1),
                   SAGEInfo("node", sampler, flags.samples_2, mult * flags.dim_2)]
    return UnsupervisedGraphsage({"batch_size": flags.batch_size, "dropout": flags.dropout}, features, sampler.adj_info,
                                 minibatch.deg, layer_infos, concat=concat, aggregator_type=kind,
                                 model_size=flags.model_size, identity_dim=flags.identity_dim,
                                 neg_sample_size=flags.neg_sample_size, learning_rate=flags.learning_rate,
                                 weight_decay=flags.weight_decay, seed=SEED, device=device)


def _ids(feed, device):
    return to_device(feed["batch1"], np.int32, device), to_device(feed["batch2"], np.int32, device)


def evaluate(model, minibatch, size, device):
    """unsupervised_train.py:72-77: loss and MRR of one sampled batch of validation edges."""
    t = time.time()
    with torch.no_grad():
        loss = model.loss(*_ids(minibatch.val_feed_dict(size), device))
        mrr = model.mrr()
    return float(loss), float(mrr), time.time() - t


def save_val_embeddings(model, minibatch, size, out_dir, device, mod=""):
    """unsupervised_train.py:94-117: outputs1 of every node, in the iterator's order, first occurrence of each edge[0]
    kept; `<out_dir>val<mod>.npy` and `.txt` (ids joined by newlines)."""
    outputs1 = model.outputs1 if isinstance(model, Node2VecModel) else model.embed
    rows, nodes, seen = [], [], set()
    finished, iter_num = False, 0
    while not finished:
        feed, finished, edges = minibatch.incremental_embed_feed_dict(size, iter_num)
        iter_num += 1
        with torch.no_grad():
            out = outputs1(to_device(feed["batch1"], np.int32, device))
        keep = []
        for i, edge in enumerate(edges):
            if edge[0] not in seen:
                keep.append(i)
                nodes.append(edge[0])
                seen.add(edge[0])
        rows.append(out[torch.as_tensor(keep, dtype=torch.long, device=out.device)])
    if not os.path.exists(out_dir):
        os.makedirs(out_dir)
    np.save(out_dir + "val" + mod + ".npy", torch.cat(rows).cpu().numpy())
    with open(out_dir + "val" + mod + ".txt", "w") as fp:
        fp.write("\n".join(map(str, nodes)))


def train(train_data, flags, device=None):
    """unsupervised_train.py:132-372.  train_data: load_data's (G, feats, id_map, walks, class_map).  Returns the model."""
    device = select_device(flags.gpu) if device is None else device
    G, features, id_map = train_data[:3]
    if features is not None:
        features = np.vstack([features, np.zeros((features.shape[1],))])        # the dummy row (:137-139)
    minibatch = build_iterator(train_data, flags)
    model = build_model(flags, features, minibatch, device)
    sampler = adj = test_adj = None                             # Node2Vec samples no neighbours
    if not isinstance(model, Node2VecModel):
        sampler = model.layer_infos[0].neigh_sampler
        adj, test_adj = sampler.adj_info, torch.from_numpy(minibatch.test_adj).to(device)
    replay = model.graphed_train_step(flags.batch_size)
    clock = StepClock(device)
    st = {"train_ema": None, "val_ema": None}

    def use_adj(table):
        if sampler is not None:
            sampler.set_adj(table)

    def run_step(feed, eager):
        if eager:
            return model.train_step(*_ids(feed, device))
        return replay(torch.from_numpy(np.asarray(feed["batch1"], np.int32)).pin_memory(),
                      torch.from_numpy(np.asarray(feed["batch2"], np.int32)).pin_memory())

    def step(feed, it, total_steps, eager):
        loss = run_step(feed, eager)
        st["train_mrr"] = mrr = model.mrr()                   # a device scalar: the moving average stays on the device
        ema = st["train_ema"]
        st["train_ema"] = mrr.clone() if ema is None else ema - (1 - 0.99) * (ema - mrr)
        return loss

    def validate():
        use_adj(test_adj)
        st["val_cost"], st["val_mrr"], _ = evaluate(model, minibatch, flags.validate_batch_size, device)
        use_adj(adj)
        return st["val_cost"]

    def after(loss, it, total_steps, printing):
        ema = st["val_ema"]
        st["val_ema"] = st["val_mrr"] if ema is None else ema - (1 - 0.99) * (ema - st["val_mrr"])
        if printing:
            print("Iter:", '%04d' % it,
                  "train_loss=", "{:.5f}".format(float(loss)),
                  "train_mrr=", "{:.5f}".format(float(st["train_mrr"])),
                  "train_mrr_ema=", "{:.5f}".format(float(st["train_ema"])),
                  "val_loss=", "{:.5f}".format(st["val_cost"]),
                  "val_mrr=", "{:.5f}".format(st["val_mrr"]),
                  "val_mrr_ema=", "{:.5f}".format(st["val_ema"]),
                  "time=", "{:.5f}".format(clock.avg(total_steps + 1)))

    train_loop(minibatch, flags, step, validate, after)

    print("Optimization Finished!")
    if flags.save_embeddings:
        use_adj(test_adj)
        save_val_embeddings(model, minibatch, flags.validate_batch_size, log_dir(flags), device)
        if flags.model == "n2v":
            nodes = [n for n in G.nodes() if G.node[n]["val"] or G.node[n]["test"]]
            start = time.time()
            pairs = run_random_walks(G, nodes, num_walks=50)
            walk_time = time.time() - start
            test_minibatch = EdgeMinibatchIterator(G, id_map, None, batch_size=flags.batch_size,
                                                   max_degree=flags.max_degree, context_pairs=pairs, n2v_retrain=True,
                                                   fixed_n2v=True)
            start = time.time()
            print("Doing test training for n2v.")
            test_steps = 0
            for _ in range(flags.n2v_test_epochs):
                test_minibatch.shuffle()
                while not test_minibatch.end():
                    feed = test_minibatch.next_minibatch_feed_dict()
                    printing = test_steps % flags.print_every == 0
                    loss = run_step(feed, printing or feed["batch_size"] != flags.batch_size)
                    if printing:
                        print("Iter:", '%04d' % test_steps,
                              "train_loss=", "{:.5f}".format(float(loss)),
                              "train_mrr=", "{:.5f}".format(float(model.mrr())))
                    test_steps += 1
            torch.cuda.synchronize(device)
            train_time = time.time() - start
            save_val_embeddings(model, minibatch, flags.validate_batch_size, log_dir(flags), device, mod="-test")
            print("Total time: ", train_time + walk_time)
            print("Walk time: ", walk_time)
            print("Train time: ", train_time)
    if isinstance(model, Node2VecModel):
        model.neg_sampler.check()
    return model


def main(argv=None):
    flags = parse_flags(sys.argv[1:] if argv is None else argv)
    print("Loading training data..")
    train_data = load_data(flags.train_prefix, load_walks=True)
    print("Done loading training data..")
    return train(train_data, flags)


if __name__ == "__main__":
    main()
