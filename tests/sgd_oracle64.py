"""Test oracle for the linear probe's 64-bit instantiation: scikit-learn 1.9.0's ``SGDClassifier(loss="log_loss",
penalty="l2", class_weight="balanced")`` on float16 / float64 input, restated in numpy + ``math`` one sample at a time.

scikit-learn's ``check_array`` widens anything that is not float32 to float64 and fits it with the 64-bit instantiation
of ``_plain_sgd`` (``linear_model/_sgd_fast.pyx.tp``, ``utils/_weight_vector.pyx.tp``).  This module follows it
variable by variable, next to the 32-bit restatement in ``sgd_oracle.py``, whose shuffle, seeds, class weights and loss
it reuses: everything is double, ``dot`` returns ``sum(w * x) * wscale`` unrounded, ``scale`` takes
``max(0, 1 - eta * alpha)`` as is, ``add`` adds ``x * (update / wscale)``, the class weights are not rounded, and
``wscale`` resets below 1e-9.  Sums run in index order (``np.cumsum`` is sequential).  ``plip_b200``'s
``sgd_fit_kernel<double, D>`` is checked against it; nothing here runs on the device.
"""
import math

import numpy as np

from sgd_oracle import (MAX_DLOSS, _seqsum, balanced_weights, gradient, log1pexp, overflow_message, problem_seeds,
                        shuffle_permutation)

RESET_WSCALE_64 = 1e-9       # WeightVector64's reset threshold


def plain_sgd64(X: np.ndarray, y01: np.ndarray, alpha: float, weight_pos: float, weight_neg: float, seed: int,
                max_iter: int = 10000, tol: float = 1e-3, n_iter_no_change: int = 5, stats: dict = None):
    """One binary problem: ``(coef float64 [d], intercept, n_iter, overflow)``.  ``y01`` holds 0 / 1 labels.
    ``stats``, if given, receives ``resets``: the wscale resets that found a non-zero weight vector."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _plain_sgd64(np.asarray(X, np.float64), y01, alpha, weight_pos, weight_neg, seed, max_iter, tol,
                            n_iter_no_change, stats)


def _plain_sgd64(X, y01, alpha, weight_pos, weight_neg, seed, max_iter, tol, n_iter_no_change, stats):
    n, d = X.shape
    w = np.zeros(d)
    wscale, sq_norm, intercept, t = 1.0, 0.0, 0.0, 1.0
    typw = float(np.sqrt(1.0 / np.sqrt(alpha)))
    optimal_init = 1.0 / ((typw / max(1.0, gradient(1.0, -typw))) * alpha)
    cw_pos, cw_neg = float(weight_pos), float(weight_neg)
    sigma = shuffle_permutation(n, seed)
    order = np.arange(n)
    best, no_improvement, resets = math.inf, 0, 0
    epoch = 0
    for epoch in range(max_iter):
        objective = 0.0
        order = order[sigma]
        for idx in order:
            x = X[idx]
            yv = float(y01[idx])
            p = _seqsum(w * x) * wscale + intercept
            eta = 1.0 / (alpha * (optimal_init + t - 1))
            objective += log1pexp(p) - yv * p
            # alpha * ((1 - l1_ratio) * 0.5 * w.norm() ** 2 + l1_ratio * w.l1norm()), l1_ratio = 0
            objective += alpha * (0.5 * math.sqrt(sq_norm) ** 2)
            # sklearn's if / elif clip; Python's max / min also let a NaN through
            dloss = min(max(gradient(yv, p), -MAX_DLOSS), MAX_DLOSS)
            update = -eta * dloss
            update *= cw_pos if yv > 0.0 else cw_neg
            c = max(0.0, 1.0 - eta * alpha)
            wscale *= c
            sq_norm *= c * c
            if wscale < RESET_WSCALE_64:
                resets += bool(np.any(w))
                w = w * wscale
                wscale = 1.0
            if update != 0.0:
                w = w + x * (update / wscale)
                sq_norm = _seqsum(w * w) * (wscale * wscale)
            intercept += update
            t += 1
        if not math.isfinite(intercept) or not np.all(np.isfinite(w)):
            return w, intercept, epoch + 1, True
        mean = objective / n
        no_improvement = no_improvement + 1 if mean > best - tol else 0
        best = min(best, mean)
        if no_improvement >= n_iter_no_change:
            break
    if stats is not None:
        stats["resets"] = stats.get("resets", 0) + resets
    return w * wscale, intercept, epoch + 1, False


def fit64(X: np.ndarray, y, alpha: float, random_state: int = 7, max_iter: int = 10000, tol: float = 1e-3,
          n_iter_no_change: int = 5, stats: dict = None) -> dict:
    """``SGDClassifier(...).fit(X, y)`` on float16 or float64 ``X``: ``classes_``, ``coef_`` float64 ``[C or 1, d]``,
    ``intercept_`` float64 ``[C or 1]`` and ``n_iter_``.  Raises scikit-learn's ``ValueError`` on overflow.
    ``sgd_oracle.predict`` scores the result."""
    X = np.asarray(X).astype(np.float64)
    classes, y_ind = np.unique(np.asarray(y), return_inverse=True)
    C = len(classes)
    cw = balanced_weights(y_ind, C)
    seeds = problem_seeds(C, random_state)
    problems = [(1, cw[1], cw[0])] if C == 2 else [(i, cw[i], 1.0) for i in range(C)]
    coefs, intercepts, n_iter = [], [], 0
    for (pos, wp, wn), seed in zip(problems, seeds):
        coef, b, it, overflow = plain_sgd64(X, (y_ind == pos).astype(np.float64), alpha, wp, wn, seed, max_iter, tol,
                                            n_iter_no_change, stats)
        if overflow:
            raise ValueError(overflow_message(it))
        coefs.append(coef)
        intercepts.append(b)
        n_iter = max(n_iter, it)
    return {"classes_": classes, "coef_": np.stack(coefs), "intercept_": np.array(intercepts, np.float64),
            "n_iter_": n_iter}
