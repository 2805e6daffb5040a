"""Generate tests/golden/linear_probe_f64_golden.npz from the live scikit-learn ``SGDClassifier``:

    python tests/golden/make_linear_probe_f64_golden.py

The 64-bit counterpart of ``make_linear_probe_golden.py``: for every case of ``tests/sgd_cases_f64.GOLDEN_CASES``,
``SGDClassifier(random_state=7, loss="log_loss", alpha=alpha, penalty="l2", max_iter=max_iter,
class_weight="balanced")`` fitted on the case's seeded float16 or float64 features (float16 L2-normalised rows at 512,
as the reference's ``plip`` / ``clip`` embedders return on a GPU, and float64 rows), which scikit-learn runs through
its 64-bit ``_plain_sgd``.  Stored: ``coef_``, ``intercept_``, ``n_iter_``, the test-set predictions,
and the error message for a case that raises.  Inputs are regenerated from their seeds at test time; a checksum of
each case's training matrix is kept so that a change of the generator is caught.
"""
import hashlib
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sgd_cases_f64 import GOLDEN_CASES, golden_case  # noqa: E402
from sgd_oracle import GOLDEN_SEED  # noqa: E402


def main():
    import sklearn
    from sklearn.linear_model import SGDClassifier

    out = {"sklearn_version": np.array(sklearn.__version__)}
    for name in GOLDEN_CASES:
        xtr, ytr, xte, _, alpha, max_iter = golden_case(name)
        out[f"{name}_x_sha256"] = np.array(hashlib.sha256(xtr.tobytes()).hexdigest())
        clf = SGDClassifier(random_state=GOLDEN_SEED, loss="log_loss", alpha=alpha, penalty="l2", max_iter=max_iter,
                            class_weight="balanced")
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                clf.fit(xtr, ytr)
        except ValueError as e:
            out[f"{name}_error"] = np.array(str(e))
            print(name, "raises:", e)
            continue
        out[f"{name}_coef"] = clf.coef_
        out[f"{name}_intercept"] = clf.intercept_
        out[f"{name}_n_iter"] = np.array(clf.n_iter_)
        out[f"{name}_pred"] = clf.predict(xte)
        print(name, xtr.dtype, "classes", len(clf.classes_), "n_iter", clf.n_iter_, "coef", clf.coef_.dtype)
    path = os.path.join(ROOT, "tests", "golden", "linear_probe_f64_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
