"""The reference's embedding evaluations (eval_scripts/{ppi,reddit,citation}_eval.py) with the logistic classifier on the GPU:

    python -m graphsage_b200.eval_scripts.ppi_eval <dataset_dir> <embed_dir> <setting> [--gpu N]

Each script keeps the reference's positional arguments, file names, branches and print lines; what they share is here.
`main(argv, device=None)` runs a script in-process (device=None: the --gpu choice of the trainers)."""
import argparse

import numpy as np

from .. import utils
from ..supervised_train import calc_f1
from ..train_cli import select_device


def parse_args(description, argv, embed_help, extra=()):
    parser = argparse.ArgumentParser(description)
    parser.add_argument("dataset_dir", help="Path to directory containing the dataset.")
    parser.add_argument("embed_dir", help=embed_help)
    parser.add_argument("setting", help="Either val or test.")
    parser.add_argument("--gpu", type=int, default=0, help="which GPU to use")
    for args, kwargs in extra:
        parser.add_argument(*args, **kwargs)
    return parser.parse_args(argv)


def device_for(args, device):
    return select_device(args.gpu) if device is None else device


def split_ids(G, setting):
    """The train ids (neither val nor test) and the ids whose `setting` flag is set, in graph order."""
    train_ids = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    test_ids = [n for n in G.nodes() if G.node[n][setting]]
    return train_ids, test_ids


def read_embeddings(prefix, conversion):
    """<prefix>.npy and the id of each of its rows from <prefix>.txt -> (embeddings, {id: row})."""
    embeds = np.load(prefix + ".npy")
    id_map = {}
    with open(prefix + ".txt") as fp:
        for i, line in enumerate(fp):
            id_map[conversion(line.strip())] = i
    return embeds, id_map


def log_counts(feats):
    """The reference's log transform of columns 0 and 1 (comment counts and scores) before scaling."""
    feats = np.array(feats, dtype=np.float64)
    feats[:, 0] = np.log(feats[:, 0] + 1.0)
    feats[:, 1] = np.log(feats[:, 1] - min(np.min(feats[:, 1]), -1))
    return feats


def scale_pair(train, test):
    """StandardScaler fitted on the train rows, applied to both (utils.standard_scale)."""
    both = utils.standard_scale(np.vstack([train, test]), np.arange(len(train)))
    return both[:len(train)], both[len(train):]


def micro_f1(y_true, y_pred):
    """f1_score(y_true, y_pred, average="micro") for single-label y (calc_f1 over the labels present in either)."""
    y_true, y_pred = np.asarray(y_true).ravel(), np.asarray(y_pred).ravel()
    labels = np.union1d(y_true, y_pred)
    onehot = lambda y: (y[:, None] == labels[None, :]).astype(np.float64)
    return calc_f1(onehot(y_true), onehot(y_pred), False)[0]
