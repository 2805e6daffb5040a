"""Device versions of the reference's similarity heads (``reproducibility/evaluation``).

``ZeroShotClassifier`` (``evaluation/zero_shot/zero_shot.py:10-13``) and ``ImageRetrieval``
(``evaluation/retrieval/retrieval.py:9-17``) take ``[N,512]`` embedding matrices (numpy or torch, host or
device) like the reference; the ``dot`` + ``argmax`` / ``argsort()[-50:][::-1]`` arithmetic runs in the CUDA
similarity kernels (fp32).  The sklearn metrics of the reference (``metrics.py``) are CPU statistics outside the
hot path: pass ``eval_metrics=`` to reuse them; the p@10 / p@50 retrieval metric is restated here because it is a
pure function of the top-k indices.

``LinearProber`` (``evaluation/linear_probing/linear_classifier.py``) fits, on ``[N,512]`` PLIP / CLIP or ``[N,1024]``
MuDiPath (DenseNet-121) features, the reference's
``SGDClassifier(loss="log_loss", penalty="l2", max_iter=10000, class_weight="balanced")`` with scikit-learn 1.9's
algorithm restated on the device (``plip_sgd_fit``): same shuffles, same casts, every one-vs-rest problem at once;
``linear_probe_sweep`` fits a whole alpha sweep in one launch.  The training features' dtype picks the instantiation, as
in scikit-learn: float32 runs the 32-bit one (``plip_sgd_fit``), float16 and float64 the 64-bit one
(``plip_sgd_fit_f64``; the reference's ``plip`` and ``clip`` embedders return float16 rows when they run on a GPU).
"""
from __future__ import annotations

import warnings
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from .engine import (PROBE_DIMS, Engine, linear_decision, linear_decision_f64, probe_widths, sgd_fit, sgd_fit_f64,
                     sgd_shuffle_permutation, similarity_topk)


def _t(x) -> torch.Tensor:
    return x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))


class _Head:
    """Constructible with no arguments like the reference's classes (``zero_shot.py:7-8``, ``retrieval.py:6-7``): the
    similarity kernels need no weights, only a device — the current CUDA device, or that of an ``engine`` if given."""

    def __init__(self, engine: Optional[Engine] = None):
        self.engine = engine

    def _topk(self, query, space, k):
        dev = self.engine.device if self.engine is not None else None
        return similarity_topk(query, space, k, scale=1.0, normalize_query=False, normalize_space=False, device=dev)


class ZeroShotClassifier(_Head):

    def predict(self, image_embeddings, text_embeddings, unique_labels: Sequence) -> List:
        """``[unique_labels[np.argmax(i)] for i in image_embeddings.dot(text_embeddings.T)]`` (zero_shot.py:12-13)."""
        idx, _ = self._topk(_t(image_embeddings), _t(text_embeddings), 1)
        return [unique_labels[i] for i in idx[:, 0].cpu().tolist()]

    def zero_shot_classification(self, image_embeddings, text_embeddings, unique_labels, target_labels,
                                 eval_metrics: Optional[Callable] = None):
        predictions = self.predict(image_embeddings, text_embeddings, unique_labels)
        if eval_metrics is None:
            acc = float(np.mean([p == t for p, t in zip(predictions, target_labels)]))
            train_metrics, test_metrics = {"accuracy": acc}, {"accuracy": acc}
        else:
            test_metrics = eval_metrics(target_labels, predictions)
            train_metrics = eval_metrics(target_labels, predictions)
        test_metrics["split"], train_metrics["split"] = "test", "train"
        return train_metrics, test_metrics


def retrieval_metrics(y_target, y_predictions):
    """``reproducibility/metrics.py:5-15``: fraction of queries whose target is in the top 10 / top 50."""
    p10 = sum(1 for t, p in zip(y_target, y_predictions) if t in list(p[:10]))
    p50 = sum(1 for t, p in zip(y_target, y_predictions) if t in list(p[:50]))
    return {"p@10": p10 / len(y_target), "p@50": p50 / len(y_target)}


class ImageRetrieval(_Head):

    def best_scores(self, image_embeddings, text_embeddings, top_k: int = 50) -> np.ndarray:
        """Per text query, indices of the ``top_k`` most similar images, best first
        (``t.dot(image_embeddings.T).argsort()[-50:][::-1]``, retrieval.py:13-16)."""
        imgs, txt = _t(image_embeddings), _t(text_embeddings)
        k = min(top_k, imgs.shape[0])
        idx, _ = self._topk(txt, imgs, k)
        return idx.cpu().numpy()

    def retrieval(self, image_embeddings, text_embeddings):
        best = self.best_scores(image_embeddings, text_embeddings, 50)
        targets = list(range(0, len(image_embeddings)))
        test_metrics, train_metrics = retrieval_metrics(targets, best), retrieval_metrics(targets, best)
        test_metrics["split"], train_metrics["split"] = "test", "train"
        return train_metrics, test_metrics


# ---- linear probe ------------------------------------------------------------------------------------------------

MAX_INT = np.iinfo(np.int32).max


class ConvergenceWarning(UserWarning):
    """A fit stopped at ``max_iter`` epochs (scikit-learn warns with its own ``ConvergenceWarning`` there)."""


def _device(engine: Optional[Engine]) -> torch.device:
    if engine is not None:
        return engine.device
    if not torch.cuda.is_available():
        raise RuntimeError("plip_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def _embeddings(x, device: torch.device) -> torch.Tensor:
    """float32 ``[n, 512]`` or ``[n, 1024]`` (numpy or torch, host or device) as a contiguous tensor on ``device``.
    Other dtypes raise: scikit-learn runs float64 input through its 64-bit instantiation, which is not restated here."""
    want = f"float32 [n, d] with d = {probe_widths()}"
    if not torch.is_tensor(x):
        x = np.asarray(x)
        if x.dtype != np.float32:
            raise ValueError(f"the embeddings must be {want}, got {x.dtype}")
        x = torch.from_numpy(np.ascontiguousarray(x))
    if x.dtype != torch.float32 or x.dim() != 2 or x.shape[1] not in PROBE_DIMS:
        raise ValueError(f"the embeddings must be {want}, got {x.dtype} {tuple(x.shape)}")
    x = x.to(device).contiguous()
    if x.shape[0] and not bool(torch.isfinite(x).all()):
        kind = "NaN" if bool(torch.isnan(x).any()) else "infinity or a value too large for dtype('float32')"
        raise ValueError(f"Input X contains {kind}.")
    return x


_WIDE = (np.float16, np.float64)          # the dtypes scikit-learn's check_array widens to float64
_NUMPY_DTYPE = {torch.float16: np.dtype(np.float16), torch.float32: np.dtype(np.float32),
                torch.float64: np.dtype(np.float64)}


def _dtype_of(x):
    """``x``'s dtype as numpy names it (``np.asarray``'s for anything that is not an array or a tensor; other torch
    dtypes stay torch dtypes)."""
    if torch.is_tensor(x):
        return _NUMPY_DTYPE.get(x.dtype, x.dtype)
    return x.dtype if isinstance(x, np.ndarray) else np.asarray(x).dtype


def _probe_input(x, device: torch.device) -> torch.Tensor:
    """The probe's features as scikit-learn's ``SGDClassifier`` takes them, as a contiguous tensor on ``device``:
    float32 ``[n, d]`` through ``_embeddings``, float16 or float64 ``[n, d]`` (numpy or torch, host or device) in their
    own dtype, ``d`` 512 or 1024.  Other dtypes raise; non-finite float16 / float64 input raises scikit-learn's message,
    which names ``dtype('float64')``, the dtype it converts both to."""
    dt = _dtype_of(x)
    if dt == np.float32:
        return _embeddings(x, device)
    want = f"float32, float16 or float64 [n, d] with d = {probe_widths()}"
    if dt not in _WIDE:
        raise ValueError(f"the embeddings must be {want}, got {dt}")
    if not torch.is_tensor(x):
        x = torch.from_numpy(np.ascontiguousarray(x))
    if x.dim() != 2 or x.shape[1] not in PROBE_DIMS:
        raise ValueError(f"the embeddings must be {want}, got {dt} {tuple(x.shape)}")
    x = x.to(device).contiguous()
    if x.shape[0] and not bool(torch.isfinite(x).all()):
        kind = "NaN" if bool(torch.isnan(x).any()) else "infinity or a value too large for dtype('float64')"
        raise ValueError(f"Input X contains {kind}.")
    return x


def _problem_seeds(n_classes: int, seed: int) -> List[int]:
    """The ``seed`` scikit-learn hands to ``_plain_sgd`` per binary problem: ``fit_binary`` draws it after
    ``make_dataset``'s draw, from ``RandomState(seed)`` for two classes, else from one ``RandomState`` per class
    seeded by ``RandomState(seed).randint(MAX_INT, size=n_classes)`` (``_fit_multiclass``)."""
    def draw(rs):
        rs.randint(1, MAX_INT)
        return int(rs.randint(MAX_INT))
    if n_classes == 2:
        return [draw(np.random.RandomState(seed))]
    return [draw(np.random.RandomState(s)) for s in np.random.RandomState(seed).randint(MAX_INT, size=n_classes)]


class SGDLinearClassifier:
    """A fitted one-vs-rest logistic regression with ``SGDClassifier``'s attributes: ``classes_``, ``coef_`` float32
    ``[C, d]`` (``[1, d]`` for two classes; ``d`` the width of the training features, 512 or 1024), ``intercept_``
    (float32 ``[C]``, float64 ``[1]`` for two classes, as scikit-learn keeps them), ``n_features_in_`` (``d``),
    ``n_iter_`` and ``alpha``.  A fit on float16 or float64 features keeps scikit-learn's 64-bit attributes: ``coef_``
    float64 ``[C, d]`` or ``[1, d]``, ``intercept_`` float64 ``[C]`` or ``[1]``.  ``decision_function`` / ``predict`` run
    on the device, with numpy's promotion of ``X . coef_.T``: float64 scores when ``X`` or ``coef_`` is float64, float32
    otherwise (float16 ``X`` on a float32 model is widened to float32).  Features of another width raise scikit-learn's
    ``ValueError`` before anything is copied or launched."""

    def __init__(self, classes, coef, intercept, n_iter: int, alpha: float, device: torch.device):
        self.classes_, self.coef_, self.intercept_, self.n_iter_, self.alpha = classes, coef, intercept, n_iter, alpha
        self.n_features_in_ = int(coef.shape[1])
        self.device = device

    def _decide(self, X):
        shape = tuple(X.shape) if hasattr(X, "shape") else np.shape(X)
        if len(shape) == 2 and shape[1] != self.n_features_in_:
            raise ValueError(f"X has {shape[1]} features, but SGDClassifier is expecting {self.n_features_in_} "
                             "features as input.")
        if self.coef_.dtype == np.float32 and _dtype_of(X) == np.float32:
            x = _embeddings(X, self.device)
            coef = torch.from_numpy(self.coef_).to(self.device)
            return linear_decision(x, coef, torch.from_numpy(self.intercept_.astype(np.float64)))
        x = _probe_input(X, self.device)
        b = torch.from_numpy(self.intercept_.astype(np.float64))
        if self.coef_.dtype == np.float32 and x.dtype == torch.float16:        # float16 . float32 -> float32
            return linear_decision(x.to(torch.float32), torch.from_numpy(self.coef_).to(self.device), b)
        coef = torch.from_numpy(self.coef_.astype(np.float64)).to(self.device)
        return linear_decision_f64(x.to(torch.float64), coef, b)

    def decision_function(self, X) -> np.ndarray:
        """``X . coef_.T + intercept_``: ``[n, C]``, or ``[n]`` for two classes; float64 when ``X`` or ``coef_`` is
        float64, else float32."""
        scores = self._decide(X)[0].cpu().numpy()
        return scores[:, 0] if scores.shape[1] == 1 else scores

    def predict(self, X) -> np.ndarray:
        """``classes_`` of the first largest score, or ``classes_[1]`` where the score is ``> 0`` for two classes."""
        return self.classes_[self._decide(X)[1].cpu().numpy()]


def fit_sgd_classifiers(X, y, alphas: Sequence[float], seed: int = 7, max_iter: int = 10000, tol: float = 1e-3,
                        n_iter_no_change: int = 5, engine: Optional[Engine] = None) -> List[SGDLinearClassifier]:
    """``SGDClassifier(random_state=seed, loss="log_loss", alpha=a, penalty="l2", max_iter=max_iter, tol=tol,
    class_weight="balanced").fit(X, y)`` for every ``a`` in ``alphas``, all binary problems in one ``plip_sgd_fit``
    launch.  ``y``: any labels (``classes_ = np.unique(y)``).  ``X``: float32 runs scikit-learn's 32-bit instantiation,
    float16 / float64 its 64-bit one (``plip_sgd_fit_f64``).  A problem whose weights overflow raises scikit-learn's
    ``ValueError`` (the first alpha and class in order)."""
    dev = _device(engine)
    x = _probe_input(X, dev)
    wide = x.dtype != torch.float32
    if wide:
        x = x.to(torch.float64)          # float16 widens exactly: one storage type for the 64-bit kernel
    classes, y_ind = np.unique(np.asarray(y), return_inverse=True)
    n, n_classes = int(x.shape[0]), len(classes)
    if y_ind.shape != (n,):
        raise ValueError(f"{n} samples but {y_ind.size} labels")
    if n_classes < 2:
        raise ValueError(f"The number of classes has to be greater than one; got {n_classes} class")
    counts = np.bincount(y_ind, minlength=n_classes).astype(np.float64)
    cw = float(n) / (n_classes * counts)                       # compute_class_weight("balanced")
    seeds = _problem_seeds(n_classes, seed)
    per_alpha = [(1, cw[1], cw[0], 0)] if n_classes == 2 else [(i, cw[i], 1.0, i) for i in range(n_classes)]
    problems = [(float(a), pc, wp, wn, si) for a in alphas for pc, wp, wn, si in per_alpha]
    sigma = np.stack([sgd_shuffle_permutation(n, s) for s in seeds])
    fit = sgd_fit_f64 if wide else sgd_fit
    coef, intercept, n_iter, overflow = (t.cpu().numpy() for t in fit(x, y_ind, n_classes, problems, sigma,
                                                                       max_iter, tol, n_iter_no_change))
    out, k = [], len(per_alpha)
    for i, a in enumerate(alphas):
        rows = slice(i * k, (i + 1) * k)
        bad = np.flatnonzero(overflow[rows])
        if bad.size:
            raise ValueError("Floating-point under-/overflow occurred at epoch #%d. Scaling input data with "
                             "StandardScaler or MinMaxScaler might help." % int(n_iter[rows][bad[0]]))
        it = int(n_iter[rows].max())
        if max_iter > 1 and it == max_iter:
            warnings.warn("Maximum number of iteration reached before convergence. Consider increasing max_iter to "
                          "improve the fit.", ConvergenceWarning)
        b = intercept[rows] if n_classes == 2 or wide else intercept[rows].astype(np.float32)
        out.append(SGDLinearClassifier(classes, coef[rows].copy(), b.copy(), it, float(a), dev))
    return out


def _encode_labels(train_y, test_y):
    """``LabelEncoder().fit_transform(train_y)`` / ``.transform(test_y)``: indices into the sorted unique labels."""
    classes = np.unique(np.asarray(train_y))
    test = np.asarray(test_y)
    unseen = np.setdiff1d(np.unique(test), classes)
    if unseen.size:
        raise ValueError(f"y contains previously unseen labels: {unseen.tolist()}")
    return np.searchsorted(classes, np.asarray(train_y)), np.searchsorted(classes, test)


def _probe_metrics(clf: SGDLinearClassifier, train_x, train_y, test_x, test_y, eval_metrics):
    test_pred, train_pred = clf.predict(test_x), clf.predict(train_x)
    if eval_metrics is None:
        test_metrics = {"accuracy": float(np.mean(test_pred == test_y))}
        train_metrics = {"accuracy": float(np.mean(train_pred == train_y))}
    else:
        test_metrics = eval_metrics(test_y, test_pred, average_method="macro")
        train_metrics = eval_metrics(train_y, train_pred, average_method="macro")
    test_metrics["split"], train_metrics["split"] = "test", "train"
    return test_metrics, train_metrics


def linear_probe_sweep(train_x, train_y, test_x, test_y, alphas: Sequence[float], seed: int = 7,
                       eval_metrics: Optional[Callable] = None, engine: Optional[Engine] = None):
    """``LinearProber(alpha, seed).train_and_test(...)`` for every alpha of ``alphas`` (the reference's
    ``reproduce.sh`` loop), fitted in one launch: one ``(classifier, (test_metrics, train_metrics))`` per alpha, each
    bit-identical to the single-alpha call."""
    ytr, yte = _encode_labels(train_y, test_y)
    dev = _device(engine)
    xtr, xte = _probe_input(train_x, dev), _probe_input(test_x, dev)
    clfs = fit_sgd_classifiers(xtr, ytr, alphas, seed=seed, max_iter=10000, engine=engine)
    return [(clf, _probe_metrics(clf, xtr, ytr, xte, yte, eval_metrics)) for clf in clfs]


class LinearProber:
    """The reference's ``LinearProber`` (``linear_classifier.py``): labels are encoded as ``LabelEncoder`` does, the
    classifier is fitted on the indices (so its ``classes_`` are ``0..C-1``), and the metrics are accuracy, or
    ``eval_metrics(y, pred, average_method="macro")`` (the reference's ``metrics.eval_metrics``) when given."""

    def __init__(self, alpha: float, seed: int = 7, engine: Optional[Engine] = None):
        self.alpha, self.seed, self.engine = alpha, seed, engine

    def train_and_test(self, train_x, train_y, test_x, test_y, eval_metrics: Optional[Callable] = None):
        return linear_probe_sweep(train_x, train_y, test_x, test_y, [self.alpha], self.seed, eval_metrics,
                                  self.engine)[0]
