"""Seeded float16 / float64 inputs for the linear probe's 64-bit instantiation.

When the reference embeds on a GPU, its ``plip`` and ``clip`` arms return float16 rows: ``clip.load(..., device="cuda")``
keeps OpenAI CLIP's fp16 weights, ``encode_image`` returns half, and ``embedders/plip.py`` L2-normalises the rows in
numpy float16.  scikit-learn fits float16 (and float64) input with its 64-bit ``_plain_sgd``.  This module generates
the cases of ``tests/golden/linear_probe_f64_golden.npz`` (``tests/golden/make_linear_probe_f64_golden.py``).
"""
import numpy as np

from sgd_oracle import LABELS


def embeddings(n: int, n_classes: int, seed: int, dim: int = 512, imbalance: float = 0.0, dtype=np.float16,
               normalise: bool = True, scale: float = 1.0, shift: float = 0.0):
    """Seeded synthetic ``[n, dim]`` features around one mean per class and integer class ids (legacy
    ``RandomState``).  ``normalise``: cast to ``dtype`` first, then divide by the row norms in that dtype, as
    ``embedders/plip.py`` does with float16 ``encode_image`` rows.  Otherwise ``(means[y] + noise) * scale + shift``,
    un-normalised like DenseNet features."""
    rs = np.random.RandomState(seed)
    p = np.exp(-imbalance * np.arange(n_classes))
    y = rs.choice(n_classes, size=n, p=p / p.sum())
    y[:n_classes] = np.arange(n_classes)               # every class present
    means = rs.standard_normal((n_classes, dim)) * 0.06
    x = means[y] + rs.standard_normal((n, dim)) * 0.04
    if normalise:
        x = x.astype(dtype)
        return x / np.linalg.norm(x, axis=1, keepdims=True), y
    return (x * scale + shift).astype(dtype), y


# name: (n_train, n_test, classes, alpha, imbalance, string labels, max_iter, dim, dtype, normalise, scale, shift).
# "c9" is Kather-like (nine tissue classes, float16 unit rows), "c2" a binary benchmark (intercept_ [1]), "unnorm"
# float64 DenseNet-like features at 1024, "reset" reaches wscale < 1e-9 with non-zero weights (alpha 1e8: eta * alpha
# starts near 1), "max_iter" stops at max_iter and "overflow" (float64 rows at 1e200) raises at epoch 1.
GOLDEN_CASES = {
    "c9": (450, 96, 9, 1e-3, 0.2, True, 10000, 512, np.float16, True, 1.0, 0.0),
    "c2": (240, 64, 2, 1e-4, 0.8, True, 10000, 512, np.float16, True, 1.0, 0.0),
    "unnorm": (200, 64, 3, 1e-3, 0.3, False, 10000, 1024, np.float64, False, 8.0, 0.25),
    "reset": (300, 64, 2, 1e8, 0.0, False, 10000, 512, np.float16, True, 1.0, 0.0),
    "max_iter": (300, 64, 4, 1e-1, 0.3, False, 3, 512, np.float16, True, 1.0, 0.0),
    "overflow": (100, 16, 3, 1e-4, 0.0, False, 10000, 512, np.float64, False, 1e200, 0.0),
}


def golden_case(name: str):
    """``(X_train, y_train, X_test, y_test, alpha, max_iter)`` of a 64-bit golden case, regenerated from its seed."""
    n, m, c, alpha, imbalance, strings, max_iter, dim, dtype, normalise, scale, shift = GOLDEN_CASES[name]
    x, y = embeddings(n + m, c, seed=64 + sum(map(ord, name)), dim=dim, imbalance=imbalance, dtype=dtype,
                      normalise=normalise, scale=scale, shift=shift)
    labels = LABELS[:c][y] if strings else y
    return x[:n], labels[:n], x[n:], labels[n:], alpha, max_iter
