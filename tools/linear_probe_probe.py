"""The linear probe on one GPU, on a Kather-shaped synthetic problem: 100 k training and 7 k test rows of float32
[., 512] embeddings (unit-norm, like PLIP's), or with ``--dim 1024`` of [., 1024] features shaped like MuDiPath's
DenseNet-121 ones (un-normalised, non-negative, a positive offset and a scale of a few units), 9 classes, and
``reproduce.sh``'s alphas (1e-4, 1e-3, 1e-2, 1e-1).  Reports the wall time of
``evaluation.linear_probe_sweep`` (all 4 x 9 binary problems in one launch, ending in a device synchronise), the
epochs per alpha, and ns per sample step along the longest problem's chain (the kernel is bound by that dependent
chain, not by a roofline).  When scikit-learn imports, also the host time of the same 4 ``SGDClassifier`` fits,
whether the predictions agree and the fraction of bit-identical ``coef_`` entries.  Prints the card name and power
limit with the numbers.  GPU only.

``--dtype float16`` gives the rows as the reference's ``plip`` / ``clip`` embedders return them on a GPU (float16,
normalised in float16), ``--dtype float64`` as float64; both run scikit-learn's 64-bit instantiation
(``plip_sgd_fit_f64``), and scikit-learn is timed on the same float16 / float64 array.

    python tools/linear_probe_probe.py [out.json] [--dim 1024] [--dtype float16|float64] [--no-sklearn]
"""
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from plip_b200.evaluation import fit_sgd_classifiers, linear_probe_sweep  # noqa: E402
from region_probe import card  # noqa: E402

N_TRAIN, N_TEST, CLASSES = 100_000, 7_000, 9
ALPHAS = [1e-4, 1e-3, 1e-2, 1e-1]


def kather_like(n, seed, dim=512, dtype=np.float32):
    """Embeddings around 9 class means with class sizes as uneven as Kather's (about 2:1).  ``dim`` 512: unit-norm
    rows (float16 rows are normalised in float16, as ``embedders/plip.py`` does).  ``dim`` 1024: DenseNet-like pooled
    features, un-normalised: non-negative around a positive offset of 1 with a spread of about 0.5."""
    rs = np.random.RandomState(seed)
    p = np.linspace(1.0, 2.0, CLASSES)
    y = rs.choice(CLASSES, size=n, p=p / p.sum())
    means = np.random.RandomState(0).standard_normal((CLASSES, dim))
    if dim == 1024:
        x = np.maximum(1.0 + means[y] * 0.1 + rs.standard_normal((n, dim)) * 0.5, 0.0)
        return x.astype(dtype), y
    x = means[y] * 0.05 + rs.standard_normal((n, dim)) * 0.3
    if dtype == np.float16:
        x = x.astype(dtype)
        return x / np.linalg.norm(x, axis=1, keepdims=True), y
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x.astype(dtype), y


def main():
    if not torch.cuda.is_available():
        sys.exit("linear_probe_probe: needs a CUDA device")
    args = sys.argv[1:]
    opts = {"--dim": "512", "--dtype": "float32"}
    for key in opts:
        if key in args:
            opts[key] = args[args.index(key) + 1]
            del args[args.index(key):args.index(key) + 2]
    dim, dtype = int(opts["--dim"]), np.dtype(opts["--dtype"])
    if dtype not in (np.float32, np.float16, np.float64):
        sys.exit("linear_probe_probe: --dtype is float32, float16 or float64")
    out_path = next((a for a in args if not a.startswith("--")), None)
    xtr, ytr = kather_like(N_TRAIN, 1, dim, dtype)
    xte, yte = kather_like(N_TEST, 2, dim, dtype)
    res = {"card": card(), "dim": dim, "dtype": dtype.name, "n_train": N_TRAIN, "n_test": N_TEST, "classes": CLASSES,
           "alphas": ALPHAS}

    fit_sgd_classifiers(xtr[:2000], ytr[:2000], ALPHAS)          # module load, first launches
    dtr, dte = torch.from_numpy(xtr).cuda(), torch.from_numpy(xte).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sweep = linear_probe_sweep(dtr, ytr, dte, yte, ALPHAS)
    torch.cuda.synchronize()
    res["sweep_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    fit_sgd_classifiers(dtr, ytr, ALPHAS)
    torch.cuda.synchronize()
    res["fit_s"] = time.perf_counter() - t0
    epochs = [clf.n_iter_ for clf, _ in sweep]
    res["epochs_per_alpha"] = epochs
    res["ns_per_step_longest_chain"] = res["fit_s"] / (max(epochs) * N_TRAIN) * 1e9
    res["test_accuracy"] = [m[0]["accuracy"] for _, m in sweep]

    if "--no-sklearn" not in sys.argv:
        try:
            from sklearn.linear_model import SGDClassifier
        except ImportError:
            res["sklearn"] = "not installed"
        else:
            sk_s, agree, sk_epochs, dcoef, same = 0.0, [], [], [], []
            for a, (clf, _) in zip(ALPHAS, sweep):
                sk = SGDClassifier(random_state=7, loss="log_loss", alpha=a, penalty="l2", max_iter=10000,
                                   class_weight="balanced")
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    t0 = time.perf_counter()
                    sk.fit(xtr, ytr)
                    sk_s += time.perf_counter() - t0
                sk_epochs.append(int(sk.n_iter_))
                agree.append(float(np.mean(sk.predict(xte) == clf.predict(dte))))
                dcoef.append(float(np.abs(sk.coef_ - clf.coef_).max() / np.abs(sk.coef_).max()))
                same.append(float(np.mean(sk.coef_ == clf.coef_)))
            res["sklearn_fit_s"] = sk_s
            res["sklearn_epochs_per_alpha"] = sk_epochs
            res["prediction_agreement"] = agree
            res["max_abs_dcoef_over_max_coef"] = dcoef
            res["coef_bit_identical_fraction"] = same
    print(json.dumps(res, indent=1))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
