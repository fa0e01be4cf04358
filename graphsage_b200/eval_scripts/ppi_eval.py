"""Logistic-regression evaluation of PPI embeddings (reference eval_scripts/ppi_eval.py): one binary classifier per label
column (MultiOutputClassifier(SGDClassifier(loss="log")), all columns in one GPU launch), then the per-column F1 of the
classifier and of the stratified random baseline.  Run it after unsupervised training; embed_dir 'feat' scores the raw
features instead:

    python -m graphsage_b200.eval_scripts.ppi_eval ../data/ppi unsup-ppi/graphsage_mean_small_0.000010 test
"""
import json
import sys

import numpy as np

from . import device_for, log_counts, micro_f1, parse_args, read_embeddings, scale_pair, split_ids
from ..graph import node_link_graph
from ..linear_model import DummyClassifier, SGDClassifier


def run_regression(train_embeds, train_labels, test_embeds, test_labels, device):
    np.random.seed(1)
    dummy = DummyClassifier()
    dummy.fit(train_embeds, train_labels)
    log = SGDClassifier(loss="log", device=device)
    log.fit(train_embeds, train_labels)
    pred = log.predict(test_embeds)          # the reference predicts once per column; the result is the same
    for i in range(test_labels.shape[1]):
        print("F1 score", micro_f1(test_labels[:, i], pred[:, i]))
    for i in range(test_labels.shape[1]):    # every call draws all columns from the global RandomState
        print("Random baseline F1 score", micro_f1(test_labels[:, i], dummy.predict(test_embeds)[:, i]))


def main(argv=None, device=None):
    args = parse_args("Run evaluation on PPI data.", sys.argv[1:] if argv is None else argv,
                      "Path to directory containing the learned node embeddings. Set to 'feat' for raw features.")
    dataset_dir, data_dir, setting = args.dataset_dir, args.embed_dir, args.setting
    device = device_for(args, device)

    print("Loading data...")
    with open(dataset_dir + "/ppi-G.json") as fp:
        G = node_link_graph(json.load(fp))
    with open(dataset_dir + "/ppi-class_map.json") as fp:
        labels = {int(i): l for i, l in json.load(fp).items()}

    train_ids, test_ids = split_ids(G, setting)
    train_labels = np.array([labels[i] for i in train_ids])
    if train_labels.ndim == 1:
        train_labels = np.expand_dims(train_labels, 1)
    test_labels = np.array([labels[i] for i in test_ids])
    print("running", data_dir)

    if data_dir == "feat":
        print("Using only features..")
        feats = log_counts(np.load(dataset_dir + "/ppi-feats.npy"))
        with open(dataset_dir + "/ppi-id_map.json") as fp:
            feat_id_map = {int(k): v for k, v in json.load(fp).items()}
        train_feats = feats[[feat_id_map[i] for i in train_ids]]
        test_feats = feats[[feat_id_map[i] for i in test_ids]]
        print("Running regression..")
        train_feats, test_feats = scale_pair(train_feats, test_feats)
        run_regression(train_feats, train_labels, test_feats, test_labels, device)
    else:
        embeds, id_map = read_embeddings(data_dir + "/val", int)
        train_embeds = embeds[[id_map[i] for i in train_ids]]
        test_embeds = embeds[[id_map[i] for i in test_ids]]
        print("Running regression..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)


if __name__ == "__main__":
    main()
