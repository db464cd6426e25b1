"""Stub of the reference's ``preprocessing`` module for running its unmodified ``Main.py`` on large enclosing
subgraphs: the loaders Main.py dispatches to (Main.py:229-251) return the synthetic ``ml_100k`` split, cut to 2 000
training and 200 test pairs, over the FULL training matrix (so every subgraph has ml_100k*'s size), in the reference's
13-tuple contract (adj_train = CSR float32 with value label+1, preprocessing.py:190-197).  No network, no h5py."""
import numpy as np


def _split(testing=False):
    from igmc_b200.data import make_synthetic_dataset
    ds = make_synthetic_dataset("ml_100k", seed=0)
    tu, tv, tl = [a[:2000] for a in ds["train"]]
    eu, ev, el = [a[:200] for a in ds["test"]]
    half = len(eu) // 2
    cv = ds["class_values"].astype(np.float64)
    # (u_features, v_features, adj_train, train_labels, train_u, train_v, val_labels, val_u, val_v,
    #  test_labels, test_u, test_v, class_values)
    return (None, None, ds["adj_train"], tl, tu, tv, el[:half], eu[:half], ev[:half], el[half:], eu[half:], ev[half:],
            cv)


def create_trainvaltest_split(dataset, seed=1234, testing=False, datasplit_path=None, datasplit_from_file=False,
                              verbose=True, rating_map=None, post_rating_map=None, ratio=1.0):
    return _split(testing)


def load_data_monti(dataset, testing=False, rating_map=None, post_rating_map=None):
    return _split(testing)


def load_official_trainvaltest_split(dataset, testing=False, rating_map=None, post_rating_map=None, ratio=1.0):
    return _split(testing)
