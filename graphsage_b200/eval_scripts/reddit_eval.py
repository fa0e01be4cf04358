"""Logistic-regression evaluation of Reddit embeddings (reference eval_scripts/reddit_eval.py): one-vs-rest
SGDClassifier(loss="log") over the subreddit classes on the GPU, then the test, train and stratified random-baseline F1.
embed_dir 'feat' scores the raw features; a directory whose name contains 'n2v' takes the test rows from val-test.npy
and runs a second regression with the features appended.

    python -m graphsage_b200.eval_scripts.reddit_eval ../data/reddit unsup-reddit/graphsage_mean_small_0.000010 test
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
    print("Test scores")
    print(micro_f1(test_labels, log.predict(test_embeds)))
    print("Train scores")
    print(micro_f1(train_labels, log.predict(train_embeds)))
    print("Random baseline")
    print(micro_f1(test_labels, dummy.predict(test_embeds)))


def main(argv=None, device=None):
    args = parse_args("Run evaluation on Reddit data.", sys.argv[1:] if argv is None else argv,
                      "Path to directory containing the learned node embeddings. Set to 'feat' for raw features.")
    dataset_dir, data_dir, setting = args.dataset_dir, args.embed_dir, args.setting
    device = device_for(args, device)

    print("Loading data...")
    with open(dataset_dir + "/reddit-G.json") as fp:
        G = node_link_graph(json.load(fp))
    with open(dataset_dir + "/reddit-class_map.json") as fp:
        labels = json.load(fp)

    train_ids, test_ids = split_ids(G, setting)
    train_labels = [labels[i] for i in train_ids]
    test_labels = [labels[i] for i in test_ids]

    def features():
        with open(dataset_dir + "/reddit-id_map.json") as fp:
            feat_id_map = json.load(fp)
        return feat_id_map

    if data_dir == "feat":
        print("Using only features..")
        feats = log_counts(np.load(dataset_dir + "/reddit-feats.npy"))
        feat_id_map = features()
        train_feats = feats[[feat_id_map[i] for i in train_ids]]
        test_feats = feats[[feat_id_map[i] for i in test_ids]]
        print("Running regression..")
        train_feats, test_feats = scale_pair(train_feats, test_feats)
        run_regression(train_feats, train_labels, test_feats, test_labels, device)

    elif "n2v" in data_dir:
        print("Doing it N2V style.")
        base_embeds, base_id_map = read_embeddings(data_dir + "/val", str)
        tuned_embeds, tuned_id_map = read_embeddings(data_dir + "/val-test", str)
        train_embeds = base_embeds[[base_id_map[i] for i in train_ids]]
        test_embeds = tuned_embeds[[tuned_id_map[i] for i in test_ids]]

        print("Running regression..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)

        feats = np.load(dataset_dir + "/reddit-feats.npy")
        feat_id_map = features()
        train_feats = feats[[feat_id_map[i] for i in train_ids]]
        test_feats = feats[[feat_id_map[i] for i in test_ids]]
        train_embeds, test_embeds = scale_pair(np.hstack([train_feats, train_embeds]), np.hstack([test_feats, test_embeds]))

        print("Running regression with feats..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)
    else:
        embeds, id_map = read_embeddings(data_dir + "/val", str)
        train_embeds = embeds[[id_map[i] for i in train_ids]]
        test_embeds = embeds[[id_map[i] for i in test_ids]]

        print("Running regression..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)


if __name__ == "__main__":
    main()
