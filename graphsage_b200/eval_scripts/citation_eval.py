"""Logistic-regression evaluation of citation-graph embeddings (reference eval_scripts/citation_eval.py): one-vs-rest
SGDClassifier(loss="log") over six subject classes on the GPU, then the F1 of the classifier and of the stratified random
baseline.  The class of a paper comes from <labels_dir>/{CU,DA,DR,NI,GU,IA}.tsv (a header line, then one paper id per
line); --labels_dir defaults to the reference's hard-coded location.  embed_dir 'feat' scores the raw features; a
directory whose name contains 'n2v' takes the test rows from val-test.npy and runs a second regression with the
features appended.

    python -m graphsage_b200.eval_scripts.citation_eval ../data/isi unsup-isi/graphsage_mean_small_0.000010 test
"""
import json
import sys

import numpy as np

from . import device_for, micro_f1, parse_args, read_embeddings, scale_pair, split_ids
from ..graph import node_link_graph
from ..linear_model import DummyClassifier, SGDClassifier

SUBJECTS = ["CU", "DA", "DR", "NI", "GU", "IA"]
LABELS_DIR = "/dfs/scratch0/scisurv/clean"


def get_class_labels(ids, labels_dir=LABELS_DIR):
    class_map = {}
    for i, code in enumerate(SUBJECTS):
        with open("{}/{}.tsv".format(labels_dir, code)) as fp:
            fp.readline()
            for line in fp:
                class_map[int(line.split()[0])] = i
    return [class_map[i] for i in ids]


def run_regression(train_embeds, train_labels, test_embeds, test_labels, device):
    np.random.seed(1)
    dummy = DummyClassifier()
    dummy.fit(train_embeds, train_labels)
    log = SGDClassifier(loss="log", device=device)
    log.fit(train_embeds, train_labels)
    print("F1 score:", micro_f1(test_labels, log.predict(test_embeds)))
    print("Random baseline f1 score:", micro_f1(test_labels, dummy.predict(test_embeds)))


def main(argv=None, device=None):
    args = parse_args("Run evaluation on citation data.", sys.argv[1:] if argv is None else argv,
                      "Path to directory containing the learned node embeddings.",
                      extra=[(("--labels_dir",), dict(default=LABELS_DIR,
                                                      help="Directory of the per-subject <code>.tsv label files."))])
    dataset_dir, data_dir, setting = args.dataset_dir, args.embed_dir, args.setting
    device = device_for(args, device)

    print("Loading data...")
    with open(dataset_dir + "/isi-G.json") as fp:
        G = node_link_graph(json.load(fp))

    train_ids, test_ids = split_ids(G, setting)
    test_labels = get_class_labels(test_ids, args.labels_dir)
    train_labels = get_class_labels(train_ids, args.labels_dir)

    def features():
        feats = np.load(dataset_dir + "/isi-feats.npy")
        with open(dataset_dir + "/isi-id_map.json") as fp:
            feat_id_map = {int(k): v for k, v in json.load(fp).items()}
        return feats[[feat_id_map[i] for i in train_ids]], feats[[feat_id_map[i] for i in test_ids]]

    if data_dir == "feat":
        print("Using only features..")
        train_feats, test_feats = features()
        print("Running regression..")
        run_regression(train_feats, train_labels, test_feats, test_labels, device)

    elif "n2v" in data_dir:
        print("Using n2v vectors.")
        base_embeds, base_id_map = read_embeddings(data_dir + "/val", int)
        tuned_embeds, tuned_id_map = read_embeddings(data_dir + "/val-test", int)
        train_embeds = base_embeds[[base_id_map[i] for i in train_ids]]
        test_embeds = tuned_embeds[[tuned_id_map[i] for i in test_ids]]

        print("Running regression..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)

        train_feats, test_feats = features()
        train_embeds, test_embeds = scale_pair(np.hstack([train_feats, train_embeds]), np.hstack([test_feats, test_embeds]))

        print("Running regression with feats..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)
    else:
        embeds, id_map = read_embeddings(data_dir + "/val", int)
        train_embeds = embeds[[id_map[i] for i in train_ids]]
        test_embeds = embeds[[id_map[i] for i in test_ids]]

        print("Running regression..")
        run_regression(train_embeds, train_labels, test_embeds, test_labels, device)


if __name__ == "__main__":
    main()
