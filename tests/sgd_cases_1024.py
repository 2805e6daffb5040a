"""Seeded 1024-wide inputs for the linear probe at MuDiPath's width: what ``DenseNetEmbedder.image_embedder`` returns
is float32 ``[N, 1024]``, un-normalised, and the reference fits the same ``SGDClassifier`` on it.

``tests/sgd_oracle.py``'s ``fit`` / ``plain_sgd`` / ``predict`` take any width; only its ``embeddings`` is 512 wide.
This module generates the ``[n, 1024]`` cases of ``tests/golden/linear_probe_1024_golden.npz``
(``tests/golden/make_linear_probe_1024_golden.py``).
"""
import numpy as np

from sgd_oracle import LABELS

DIM = 1024


def embeddings(n: int, n_classes: int, seed: int, imbalance: float = 0.0, scale: float = 1.0, shift: float = 0.0):
    """Seeded synthetic ``[n, 1024]`` float32 features around one mean per class and integer class ids, drawn like
    ``sgd_oracle.embeddings`` (legacy ``RandomState``): ``(means[y] + noise) * scale + shift``.  ``imbalance`` > 0
    makes later classes rarer; ``scale`` / ``shift`` give un-normalised, DenseNet-like features."""
    rs = np.random.RandomState(seed)
    p = np.exp(-imbalance * np.arange(n_classes))
    y = rs.choice(n_classes, size=n, p=p / p.sum())
    y[:n_classes] = np.arange(n_classes)               # every class present
    means = rs.standard_normal((n_classes, DIM)) * 0.06
    x = means[y] + rs.standard_normal((n, DIM)) * 0.04
    return (x * scale + shift).astype(np.float32), y


# name: (n_train, n_test, classes, alpha, imbalance, string labels, max_iter, scale, shift).  "c9" is Kather-like
# (nine tissue classes), "c2" an imbalanced binary problem, "unnorm" features at 8x the scale with a positive offset;
# "reset" reaches wscale < 1e-6 with non-zero weights (alpha 1e4), "max_iter" stops at max_iter and "overflow" raises
# at epoch 1.
GOLDEN_CASES = {
    "c9": (450, 96, 9, 1e-3, 0.2, True, 10000, 1.0, 0.0),
    "c2": (240, 64, 2, 1e-4, 0.8, True, 10000, 1.0, 0.0),
    "unnorm": (200, 64, 3, 1e-3, 0.3, False, 10000, 8.0, 0.25),
    "reset": (300, 64, 2, 1e4, 0.0, False, 10000, 1.0, 0.0),
    "max_iter": (300, 64, 4, 1e-1, 0.3, False, 3, 1.0, 0.0),
    "overflow": (100, 16, 3, 1e-4, 0.0, False, 10000, 1e36, 0.0),
}


def golden_case(name: str):
    """``(X_train, y_train, X_test, y_test, alpha, max_iter)`` of a 1024-wide golden case, regenerated from its seed."""
    n, m, c, alpha, imbalance, strings, max_iter, scale, shift = GOLDEN_CASES[name]
    x, y = embeddings(n + m, c, seed=DIM + sum(map(ord, name)), imbalance=imbalance, scale=scale, shift=shift)
    labels = LABELS[:c][y] if strings else y
    return x[:n], labels[:n], x[n:], labels[n:], alpha, max_iter
