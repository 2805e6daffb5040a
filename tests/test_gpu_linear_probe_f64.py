"""The linear probe's 64-bit instantiation on the device (``sgd_fit_kernel<double, D>`` /
``linear_decision_kernel<double, D>``) against scikit-learn 1.9.0's ``SGDClassifier`` on float16 and float64 features
(tests/golden/linear_probe_f64_golden.npz) and its numpy restatement (tests/sgd_oracle64.py ``fit64``), and the
reference's GPU flow end to end: float16 embeddings, normalised in numpy float16 as ``embedders/plip.py`` does, through
``LinearProber.train_and_test``.

Nothing is rounded to float in this instantiation, so the order of the D-term double sums (per lane, then across the
warp, against scikit-learn's index order) and CUDA's exp / log1p against the C library's show in the last bits.
n_iter_ and the predictions must be equal, coef_ / intercept_ within 1e-12 of their largest magnitude."""
import os
import warnings

import numpy as np
import pytest
import torch

import sgd_cases_f64 as K
import sgd_oracle as O
import sgd_oracle64 as O64
from plip_b200 import evaluation as ev
from plip_b200.engine import linear_decision_f64

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "linear_probe_f64_golden.npz")
FITTED = [name for name in K.GOLDEN_CASES if name != "overflow"]
SWEEP = [1e-4, 1e-3, 1e-2, 1e-1]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def _fit(case, alphas=None, x=None):
    xtr, ytr, _, _, alpha, max_iter = case
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ev.ConvergenceWarning)
        return ev.fit_sgd_classifiers(xtr if x is None else x, ytr, alphas or [alpha], seed=O.GOLDEN_SEED,
                                      max_iter=max_iter)


def _close(got, want, what):
    bound = 1e-12 * max(float(np.abs(want).max()), 1e-300)
    err = float(np.abs(got - want).max())
    same = float(np.mean(got == want))
    print(f"{what}: max |delta| {err:.3e} (bound {bound:.3e}), bit-identical {100 * same:.1f} %")
    assert err <= bound, (what, err, bound)


def _same(a, b):
    for x, y in zip(a, b):
        assert x.n_iter_ == y.n_iter_ and x.coef_.dtype == y.coef_.dtype == np.float64
        assert np.array_equal(x.coef_, y.coef_) and np.array_equal(x.intercept_, y.intercept_)


@pytest.mark.parametrize("name", FITTED)
def test_fit_matches_sklearn(golden, name):
    case = K.golden_case(name)
    clf = _fit(case)[0]
    assert clf.n_iter_ == int(golden[f"{name}_n_iter"])
    assert np.array_equal(clf.classes_, np.unique(case[1]))
    for key in ("coef", "intercept"):
        got, want = getattr(clf, f"{key}_"), golden[f"{name}_{key}"]
        assert got.dtype == want.dtype == np.float64 and got.shape == want.shape
        _close(got, want, f"{name} {key}")
    assert np.array_equal(clf.predict(case[2]), golden[f"{name}_pred"])


def test_max_iter_warns():
    xtr, ytr, _, _, alpha, max_iter = K.golden_case("max_iter")
    with pytest.warns(ev.ConvergenceWarning):
        clf = ev.fit_sgd_classifiers(xtr, ytr, [alpha], max_iter=max_iter)[0]
    assert clf.n_iter_ == max_iter and clf.coef_.dtype == np.float64


def test_overflow_raises_sklearns_error(golden):
    xtr, ytr, _, _, alpha, max_iter = K.golden_case("overflow")
    assert xtr.dtype == np.float64
    with pytest.raises(ValueError) as e:
        ev.fit_sgd_classifiers(xtr, ytr, [alpha], max_iter=max_iter)
    assert str(e.value) == str(golden["overflow_error"])


@pytest.mark.parametrize("name", ["c9", "c2"])
def test_float16_equals_its_float64_widening(name):
    case = K.golden_case(name)
    half = _fit(case, SWEEP)
    _same(half, _fit(case, SWEEP, x=case[0].astype(np.float64)))
    _same(half, _fit(case, SWEEP, x=torch.from_numpy(case[0]).cuda()))          # a device float16 tensor
    xte = case[2]
    for clf in half:
        assert np.array_equal(clf.decision_function(xte), clf.decision_function(xte.astype(np.float64)))


@pytest.mark.parametrize("name", ["c9", "c2", "unnorm"])
def test_sweep_is_bit_identical_to_single_fits(name):
    case = K.golden_case(name)
    sweep = _fit(case, SWEEP)
    for alpha, got in zip(SWEEP, sweep):
        assert got.alpha == alpha
        _same([got], _fit(case, [alpha]))


def test_two_runs_are_bit_identical():
    case = K.golden_case("c9")
    _same(_fit(case, SWEEP), _fit(case, SWEEP))


@pytest.mark.parametrize("name", ["unnorm", "reset"])
def test_fit_matches_oracle(name):
    xtr, ytr, xte, _, alpha, max_iter = case = K.golden_case(name)
    want = O64.fit64(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter)
    clf = _fit(case)[0]
    assert clf.n_iter_ == want["n_iter_"]
    _close(clf.coef_, want["coef_"], f"{name} coef vs oracle")
    assert np.array_equal(clf.predict(xte), O.predict(want, xte))


@pytest.mark.parametrize("d", [512, 1024])
@pytest.mark.parametrize("n_out", [1, 3, 9])
def test_decision_kernel_f64(d, n_out):
    g = torch.Generator().manual_seed(200 + n_out + d)
    x = torch.randn(1000, d, generator=g, dtype=torch.float64)
    coef = torch.randn(n_out, d, generator=g, dtype=torch.float64) * 0.05
    b = torch.randn(n_out, generator=g, dtype=torch.float64)
    scores, pred = linear_decision_f64(x.cuda(), coef.cuda(), b.cuda())
    assert scores.dtype == torch.float64 and scores.shape == (1000, n_out)
    xn, wn, bn = x.numpy(), coef.numpy(), b.numpy()
    want = xn @ wn.T + bn
    scale = np.abs(xn) @ np.abs(wn).T + np.abs(bn)                       # sum |x . w| + |b|
    s = scores.cpu().numpy()
    assert np.all(np.abs(s - want) <= 4 * np.finfo(np.float64).eps * scale)     # a few ulp of sum |x . w|
    p = pred.cpu().numpy()
    if n_out == 1:
        assert np.array_equal(p, (s[:, 0] > 0).astype(np.int32))
    else:
        assert np.array_equal(p, np.argmax(s, axis=1))


def test_32_bit_model_on_float64_features_scores_in_float64():
    from sgd_oracle import golden_case
    xtr, ytr, xte, _, alpha, _ = golden_case("c9")
    clf = ev.fit_sgd_classifiers(xtr, ytr, [alpha], seed=O.GOLDEN_SEED)[0]
    assert clf.coef_.dtype == np.float32
    s64 = clf.decision_function(xte.astype(np.float64))
    assert s64.dtype == np.float64
    want = xte.astype(np.float64) @ clf.coef_.astype(np.float64).T + clf.intercept_.astype(np.float64)
    assert np.abs(s64 - want).max() <= 1e-12 * np.abs(want).max()
    assert clf.decision_function(xte).dtype == np.float32                   # float32 x float32 stays as it was
    assert np.array_equal(clf.predict(xte.astype(np.float64)), np.unique(ytr)[np.argmax(want, axis=1)])


def test_reference_gpu_flow_float16_embeddings_end_to_end(engine):
    """``embedders/plip.py`` on a GPU: ``encode_image`` returns float16 rows, which are normalised in numpy float16;
    ``LinearProber(alpha, seed).train_and_test`` then fits scikit-learn's 64-bit instantiation on them."""
    from plip_b200.synthetic import tiles_u8
    emb = engine.encode_images(torch.from_numpy(tiles_u8(96, seed=7)), normalize=False)
    torch.cuda.synchronize()
    x = emb.cpu().numpy().astype(np.float16)
    x = x / np.linalg.norm(x, axis=1, keepdims=True)
    assert x.dtype == np.float16
    names = np.array(["tumour", "stroma", "lymphocytes"])
    y = names[np.argsort(np.argsort(x[:, 0].astype(np.float64))) * 3 // len(x)]
    tr, te = np.arange(len(x)) % 4 != 0, np.arange(len(x)) % 4 == 0
    clf, (test_metrics, train_metrics) = ev.LinearProber(alpha=1e-3, seed=3, engine=engine).train_and_test(
        x[tr], y[tr], x[te], y[te])
    ytr, yte = np.searchsorted(np.unique(y), y[tr]), np.searchsorted(np.unique(y), y[te])
    want = O64.fit64(x[tr], ytr, 1e-3, 3)
    assert clf.n_iter_ == want["n_iter_"] and np.array_equal(clf.classes_, np.arange(3))
    assert clf.coef_.dtype == np.float64 and clf.intercept_.dtype == np.float64
    _close(clf.coef_, want["coef_"], "float16 engine embeddings coef vs oracle")
    _close(clf.intercept_, want["intercept_"], "float16 engine embeddings intercept vs oracle")
    assert test_metrics == {"accuracy": float(np.mean(O.predict(want, x[te]) == yte)), "split": "test"}
    assert train_metrics == {"accuracy": float(np.mean(O.predict(want, x[tr]) == ytr)), "split": "train"}
