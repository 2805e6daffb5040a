"""The linear probe on the device (``plip_sgd_fit`` / ``plip_linear_decision``) against scikit-learn 1.9.0's
``SGDClassifier`` (tests/golden/linear_probe_golden.npz) and its numpy restatement (tests/sgd_oracle.py).

The kernel restates sklearn's arithmetic cast for cast; the only differences allowed are the order of the 512-term
double sums (a warp reduction against sklearn's index-order loop) and CUDA's exp / log1p against the C library's.
So n_iter_ and the predictions must be equal, and coef_ / intercept_ within 1e-5 of their largest magnitude."""
import os
import warnings

import numpy as np
import pytest
import torch

import sgd_oracle as O
from plip_b200 import evaluation as ev
from plip_b200.engine import linear_decision

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "linear_probe_golden.npz")
FITTED = [name for name in O.GOLDEN_CASES if name != "overflow"]
SWEEP = [1e-4, 1e-3, 1e-2, 1e-1]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def _fit(name, alphas=None):
    xtr, ytr, _, _, alpha, max_iter = O.golden_case(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ev.ConvergenceWarning)
        return ev.fit_sgd_classifiers(xtr, ytr, alphas or [alpha], seed=O.GOLDEN_SEED, max_iter=max_iter)


def _close(got, want, what):
    bound = 1e-5 * max(float(np.abs(want).max()), 1e-30)
    err = float(np.abs(got.astype(np.float64) - want.astype(np.float64)).max())
    same = float(np.mean(got == want))
    print(f"{what}: max |delta| {err:.3e} (bound {bound:.3e}), bit-identical {100 * same:.1f} %")
    assert err <= bound, (what, err, bound)


@pytest.mark.parametrize("name", FITTED)
def test_fit_matches_sklearn(golden, name):
    clf = _fit(name)[0]
    _, _, xte, _, _, max_iter = O.golden_case(name)
    assert clf.n_iter_ == int(golden[f"{name}_n_iter"])
    assert np.array_equal(clf.classes_, np.unique(O.golden_case(name)[1]))
    assert clf.coef_.dtype == np.float32 and clf.coef_.shape == golden[f"{name}_coef"].shape
    assert clf.intercept_.dtype == golden[f"{name}_intercept"].dtype
    _close(clf.coef_, golden[f"{name}_coef"], f"{name} coef")
    _close(clf.intercept_, golden[f"{name}_intercept"], f"{name} intercept")
    assert np.array_equal(clf.predict(xte), golden[f"{name}_pred"])


def test_max_iter_warns():
    xtr, ytr, _, _, alpha, max_iter = O.golden_case("max_iter")
    with pytest.warns(ev.ConvergenceWarning):
        clf = ev.fit_sgd_classifiers(xtr, ytr, [alpha], max_iter=max_iter)[0]
    assert clf.n_iter_ == max_iter


def test_overflow_raises_sklearns_error(golden):
    xtr, ytr, _, _, alpha, max_iter = O.golden_case("overflow")
    with pytest.raises(ValueError) as e:
        ev.fit_sgd_classifiers(xtr, ytr, [alpha], max_iter=max_iter)
    assert str(e.value) == str(golden["overflow_error"])


@pytest.mark.parametrize("name", ["c2", "c9"])
def test_sweep_is_bit_identical_to_single_fits(name):
    sweep = _fit(name, SWEEP)
    for alpha, got in zip(SWEEP, sweep):
        one = _fit(name, [alpha])[0]
        assert got.alpha == alpha and got.n_iter_ == one.n_iter_
        assert np.array_equal(got.coef_, one.coef_) and np.array_equal(got.intercept_, one.intercept_)


def test_two_runs_are_bit_identical():
    a, b = _fit("c9", SWEEP), _fit("c9", SWEEP)
    for x, y in zip(a, b):
        assert np.array_equal(x.coef_, y.coef_) and np.array_equal(x.intercept_, y.intercept_)
        assert x.n_iter_ == y.n_iter_


@pytest.mark.parametrize("name", ["c3", "reset"])
def test_fit_matches_oracle(name):
    xtr, ytr, xte, _, alpha, max_iter = O.golden_case(name)
    want = O.fit(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter)
    clf = _fit(name)[0]
    assert clf.n_iter_ == want["n_iter_"]
    _close(clf.coef_, want["coef_"], f"{name} coef vs oracle")
    assert np.array_equal(clf.predict(xte), O.predict(want, xte))


@pytest.mark.parametrize("n_out", [1, 3, 9])
def test_decision_kernel(n_out):
    g = torch.Generator().manual_seed(n_out)
    x = torch.randn(1000, 512, generator=g).cuda()
    coef = torch.randn(n_out, 512, generator=g).cuda() * 0.05
    b = torch.randn(n_out, generator=g, dtype=torch.float64).cuda()
    scores, pred = linear_decision(x, coef, b)
    want = x.double().cpu().numpy() @ coef.double().cpu().numpy().T + b.cpu().numpy()
    s = scores.cpu().numpy()
    assert s.shape == (1000, n_out)
    assert np.abs(s - want).max() <= 2 * np.finfo(np.float32).eps * np.abs(want).max()
    assert np.array_equal(s, want.astype(np.float32))     # one rounding of the double sum
    p = pred.cpu().numpy()
    if n_out == 1:
        assert np.array_equal(p, (s[:, 0] > 0).astype(np.int32))
    else:
        assert np.array_equal(p, np.argmax(s, axis=1))


def test_decision_ties_take_the_lowest_index():
    x = torch.randn(64, 512).cuda()
    row = torch.randn(1, 512) * 0.1
    coef = torch.cat([row * 0.5, row, row, row * 0.5]).cuda()      # classes 1 and 2 tie on every row
    b = torch.zeros(4, dtype=torch.float64).cuda()
    scores, pred = linear_decision(x, coef, b)
    s = scores.cpu().numpy()
    assert np.array_equal(s[:, 1], s[:, 2])
    top = s[:, 1] > s[:, 0]
    assert np.array_equal(pred.cpu().numpy()[top], np.ones(int(top.sum()), np.int32))
    assert np.array_equal(pred.cpu().numpy()[~top], np.zeros(int((~top).sum()), np.int32))


def test_linear_prober_on_engine_embeddings(engine):
    from plip_b200.synthetic import tiles_u8
    emb = engine.encode_images(torch.from_numpy(tiles_u8(96, seed=5)))
    torch.cuda.synchronize()
    x = emb.cpu().numpy()
    names = np.array(["tumour", "stroma", "lymphocytes"])
    y = names[np.argsort(np.argsort(x[:, 0])) * 3 // len(x)]        # classes by the first feature's rank
    tr, te = np.arange(len(x)) % 4 != 0, np.arange(len(x)) % 4 == 0
    clf, (test_metrics, train_metrics) = ev.LinearProber(alpha=1e-3, engine=engine).train_and_test(
        emb[torch.from_numpy(tr).cuda()], y[tr], x[te], y[te])
    ytr = np.searchsorted(np.unique(y), y[tr])
    want = O.fit(x[tr], ytr, 1e-3, 7)
    assert clf.n_iter_ == want["n_iter_"] and np.array_equal(clf.classes_, np.arange(3))
    _close(clf.coef_, want["coef_"], "engine embeddings coef vs oracle")
    yte = np.searchsorted(np.unique(y), y[te])
    assert test_metrics == {"accuracy": float(np.mean(O.predict(want, x[te]) == yte)), "split": "test"}
    assert train_metrics["split"] == "train"
    calls = []
    ev.LinearProber(alpha=1e-3, engine=engine).train_and_test(
        x[tr], y[tr], x[te], y[te], eval_metrics=lambda t, p, average_method: calls.append(average_method) or {})
    assert calls == ["macro", "macro"]
