"""Test oracle for the linear probe: scikit-learn 1.9.0's ``SGDClassifier(loss="log_loss", penalty="l2",
class_weight="balanced")`` on float32 input, restated in numpy + ``math`` one sample at a time.

It follows the 32-bit instantiation of ``_plain_sgd`` (``linear_model/_sgd_fast.pyx.tp``) variable by variable:
weights are float32, the scalars (``p``, ``eta``, ``update``, ``wscale``, ``sq_norm``, the objective) are double,
``dot`` / ``add`` multiply float by float and accumulate in double, in index order (``np.cumsum`` is sequential), and
the casts of ``WeightVector32`` are kept (``dot`` and ``norm`` return float, ``add`` and ``scale`` take a float).
``exp`` / ``log`` / ``log1p`` come from ``math`` (the C library sklearn's Cython calls).  ``plip_b200``'s
``sgd_fit_kernel`` is checked against it; nothing here runs on the device.
"""
import math

import numpy as np

MAX_INT = np.iinfo(np.int32).max
RESET_WSCALE = 1e-6          # WeightVector32's reset threshold
MAX_DLOSS = 1e12
F32 = np.float32


def rand_r(state: int):
    """``our_rand_r`` (``utils/_random.pxd``): the new state and the drawn number."""
    if state == 0:
        state = 1
    state ^= (state << 13) & 0xFFFFFFFF
    state ^= state >> 17
    state ^= (state << 5) & 0xFFFFFFFF
    return state, state % (2 ** 31)


def shuffle_permutation(n: int, seed: int) -> np.ndarray:
    """The permutation ``SequentialDataset.shuffle(seed)`` applies to the current order: ``new[i] = old[sigma[i]]``."""
    ind = np.arange(n, dtype=np.int32)
    state = int(seed) & 0xFFFFFFFF
    for i in range(n - 1):
        state, r = rand_r(state)
        j = i + r % (n - i)
        ind[i], ind[j] = ind[j], ind[i]
    return ind


def problem_seeds(n_classes: int, random_state: int):
    """The ``seed`` handed to ``_plain_sgd`` per binary problem (one problem when there are two classes)."""
    def seed_of(rs):
        rs.randint(1, MAX_INT)             # make_dataset's draw
        return int(rs.randint(MAX_INT))
    if n_classes == 2:
        return [seed_of(np.random.RandomState(random_state))]
    seeds = np.random.RandomState(random_state).randint(MAX_INT, size=n_classes)
    return [seed_of(np.random.RandomState(s)) for s in seeds]


def balanced_weights(y_ind: np.ndarray, n_classes: int) -> np.ndarray:
    counts = np.bincount(y_ind, minlength=n_classes).astype(np.float64)
    return float(len(y_ind)) / (n_classes * counts)


def log1pexp(x: float) -> float:
    if x <= -37:
        return math.exp(x)
    if x <= -2:
        return math.log1p(math.exp(x))
    if x <= 18:
        return math.log(1. + math.exp(x))
    if x <= 33.3:
        return x + math.exp(-x)
    return x


def gradient(y: float, p: float) -> float:
    if p > -37:
        e = math.exp(-p)
        return ((1 - y) - y * e) / (1 + e)
    return math.exp(p) - y


def _seqsum(v: np.ndarray) -> float:
    return float(np.cumsum(v.astype(np.float64))[-1])


def plain_sgd(X: np.ndarray, y01: np.ndarray, alpha: float, weight_pos: float, weight_neg: float, seed: int,
              max_iter: int = 10000, tol: float = 1e-3, n_iter_no_change: int = 5, stats: dict = None):
    """One binary problem: ``(coef float32 [d], intercept float, n_iter, overflow)``.  ``y01`` holds 0 / 1 labels.
    ``stats``, if given, receives ``resets``: the wscale resets that found a non-zero weight vector."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _plain_sgd(X, y01, alpha, weight_pos, weight_neg, seed, max_iter, tol, n_iter_no_change, stats)


def _plain_sgd(X, y01, alpha, weight_pos, weight_neg, seed, max_iter, tol, n_iter_no_change, stats):
    n, d = X.shape
    w = np.zeros(d, F32)
    wscale, sq_norm, intercept, t = 1.0, 0.0, 0.0, 1.0
    typw = float(np.sqrt(1.0 / np.sqrt(alpha)))
    optimal_init = 1.0 / ((typw / max(1.0, gradient(1.0, -typw))) * alpha)
    cw_pos, cw_neg = float(F32(weight_pos)), float(F32(weight_neg))   # class_weight is a float local
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
            p = float(F32(_seqsum(w * x) * wscale)) + intercept
            eta = 1.0 / (alpha * (optimal_init + t - 1))
            objective += log1pexp(p) - yv * p
            norm = F32(math.sqrt(sq_norm))
            objective += 0.5 * float(norm * norm) * alpha
            dloss = min(max(gradient(yv, p), -MAX_DLOSS), MAX_DLOSS)
            update = -eta * dloss
            update *= cw_pos if yv > 0.0 else cw_neg
            c = F32(max(0.0, 1.0 - eta * alpha))
            wscale *= float(c)
            sq_norm *= float(c * c)
            if wscale < RESET_WSCALE:
                resets += bool(np.any(w))
                w = w * F32(wscale)
                wscale = 1.0
            if update != 0.0:
                wsf = F32(wscale)
                q = F32(F32(update) / wsf)
                w = (w.astype(np.float64) + x.astype(np.float64) * float(q)).astype(F32)
                sq_norm = _seqsum(w * w) * float(wsf * wsf)
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
    return w * F32(wscale), intercept, epoch + 1, False


def overflow_message(epoch: int) -> str:
    return ("Floating-point under-/overflow occurred at epoch #%d. Scaling input data with StandardScaler or "
            "MinMaxScaler might help." % epoch)


def fit(X: np.ndarray, y, alpha: float, random_state: int = 7, max_iter: int = 10000, tol: float = 1e-3,
        n_iter_no_change: int = 5, stats: dict = None) -> dict:
    """``SGDClassifier(...).fit(X, y)``: ``classes_``, ``coef_`` float32 ``[C or 1, d]``, ``intercept_`` (float32, or
    float64 ``[1]`` for two classes, as sklearn keeps them) and ``n_iter_``.  Raises sklearn's ``ValueError`` on
    overflow."""
    X = np.asarray(X, F32)
    classes, y_ind = np.unique(np.asarray(y), return_inverse=True)
    C = len(classes)
    cw = balanced_weights(y_ind, C)
    seeds = problem_seeds(C, random_state)
    problems = [(1, cw[1], cw[0])] if C == 2 else [(i, cw[i], 1.0) for i in range(C)]
    coefs, intercepts, n_iter = [], [], 0
    for (pos, wp, wn), seed in zip(problems, seeds):
        coef, b, it, overflow = plain_sgd(X, (y_ind == pos).astype(F32), alpha, wp, wn, seed, max_iter, tol,
                                          n_iter_no_change, stats)
        if overflow:
            raise ValueError(overflow_message(it))
        coefs.append(coef)
        intercepts.append(b)
        n_iter = max(n_iter, it)
    intercept = np.array(intercepts, np.float64 if C == 2 else F32)
    return {"classes_": classes, "coef_": np.stack(coefs), "intercept_": intercept, "n_iter_": n_iter}


def predict(model: dict, X: np.ndarray) -> np.ndarray:
    """``decision_function`` in float64 and sklearn's rule: the first arg-max, or ``classes_[1]`` where ``> 0``."""
    scores = np.asarray(X, np.float64) @ model["coef_"].astype(np.float64).T + model["intercept_"].astype(np.float64)
    if scores.shape[1] == 1:
        return model["classes_"][(scores[:, 0] > 0).astype(int)]
    return model["classes_"][np.argmax(scores, axis=1)]


def embeddings(n: int, n_classes: int, seed: int, imbalance: float = 0.0, scale: float = 1.0):
    """Seeded synthetic ``[n, 512]`` float32 embeddings around one mean per class (legacy ``RandomState``, whose
    stream numpy keeps fixed) and integer class ids; ``imbalance`` > 0 makes later classes rarer."""
    rs = np.random.RandomState(seed)
    p = np.exp(-imbalance * np.arange(n_classes))
    y = rs.choice(n_classes, size=n, p=p / p.sum())
    y[:n_classes] = np.arange(n_classes)               # every class present
    means = rs.standard_normal((n_classes, 512)) * 0.06
    x = means[y] + rs.standard_normal((n, 512)) * 0.04
    return (x * scale).astype(F32), y


LABELS = np.array(["adipose", "background", "debris", "lymphocytes", "mucus", "smooth muscle", "normal mucosa",
                   "stroma", "tumour"])

# name: (n_train, n_test, classes, alpha, imbalance, string labels, max_iter, scale).  "reset" reaches
# wscale < 1e-6 with non-zero weights (alpha 1e4: eta * alpha starts near 1); alpha 1 resets an all-zero vector at the
# first sample; "max_iter" stops at max_iter; "overflow" raises at epoch 1.
GOLDEN_CASES = {
    "c2": (240, 64, 2, 1e-4, 0.8, True, 10000, 1.0),
    "c3": (300, 64, 3, 1e-2, 0.5, True, 10000, 1.0),
    "c9": (450, 96, 9, 1e-3, 0.2, True, 10000, 1.0),
    "alpha1": (300, 64, 3, 1.0, 0.3, False, 10000, 1.0),
    "reset": (300, 64, 2, 1e4, 0.0, False, 10000, 1.0),
    "max_iter": (300, 64, 4, 1e-1, 0.3, False, 3, 1.0),
    "overflow": (100, 16, 3, 1e-4, 0.0, False, 10000, 1e36),
}
GOLDEN_SEED = 7


def golden_case(name: str):
    """``(X_train, y_train, X_test, y_test, alpha, max_iter)`` of a golden case, regenerated from its seed."""
    n, m, c, alpha, imbalance, strings, max_iter, scale = GOLDEN_CASES[name]
    x, y = embeddings(n + m, c, seed=sum(map(ord, name)), imbalance=imbalance, scale=scale)
    labels = LABELS[:c][y] if strings else y
    return x[:n], labels[:n], x[n:], labels[n:], alpha, max_iter
