"""The linear probe on the device at MuDiPath's 1024-wide DenseNet-121 features (the ``D = 1024`` instantiations of
``sgd_fit_kernel`` / ``linear_decision_kernel``) against scikit-learn 1.9.0's ``SGDClassifier``
(tests/golden/linear_probe_1024_golden.npz) and its numpy restatement (tests/sgd_oracle.py), and the reference's
``mudipath`` probe end to end: ``EmbedderFactory`` -> ``image_embedder`` -> ``LinearProber.train_and_test``.

The contract is the 512-wide one (test_gpu_linear_probe.py): the only differences allowed are the order of the
1024-term double sums and CUDA's exp / log1p against the C library's, so n_iter_ and the predictions must be equal,
and coef_ / intercept_ within 1e-5 of their largest magnitude."""
import os
import warnings
from argparse import Namespace

import numpy as np
import pytest
import torch

import sgd_cases_1024 as K
import sgd_oracle as O
from plip_b200 import evaluation as ev
from plip_b200.engine import linear_decision

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "linear_probe_1024_golden.npz")
FITTED = [name for name in K.GOLDEN_CASES if name != "overflow"]
SWEEP = [1e-4, 1e-3, 1e-2, 1e-1]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def _fit(case, alphas=None):
    xtr, ytr, _, _, alpha, max_iter = case
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ev.ConvergenceWarning)
        return ev.fit_sgd_classifiers(xtr, ytr, alphas or [alpha], seed=O.GOLDEN_SEED, max_iter=max_iter)


def _close(got, want, what):
    bound = 1e-5 * max(float(np.abs(want).max()), 1e-30)
    err = float(np.abs(got.astype(np.float64) - want.astype(np.float64)).max())
    same = float(np.mean(got == want))
    print(f"{what}: max |delta| {err:.3e} (bound {bound:.3e}), bit-identical {100 * same:.1f} %")
    assert err <= bound, (what, err, bound)


def _same(a, b):
    for x, y in zip(a, b):
        assert x.n_iter_ == y.n_iter_ and x.n_features_in_ == y.n_features_in_
        assert np.array_equal(x.coef_, y.coef_) and np.array_equal(x.intercept_, y.intercept_)


@pytest.mark.parametrize("name", FITTED)
def test_fit_matches_sklearn(golden, name):
    case = K.golden_case(name)
    clf = _fit(case)[0]
    assert clf.n_iter_ == int(golden[f"{name}_n_iter"])
    assert np.array_equal(clf.classes_, np.unique(case[1]))
    assert clf.coef_.dtype == np.float32 and clf.coef_.shape == golden[f"{name}_coef"].shape
    assert clf.n_features_in_ == 1024
    assert clf.intercept_.dtype == golden[f"{name}_intercept"].dtype
    _close(clf.coef_, golden[f"{name}_coef"], f"{name} coef")
    _close(clf.intercept_, golden[f"{name}_intercept"], f"{name} intercept")
    assert np.array_equal(clf.predict(case[2]), golden[f"{name}_pred"])


def test_max_iter_warns():
    xtr, ytr, _, _, alpha, max_iter = K.golden_case("max_iter")
    with pytest.warns(ev.ConvergenceWarning):
        clf = ev.fit_sgd_classifiers(xtr, ytr, [alpha], max_iter=max_iter)[0]
    assert clf.n_iter_ == max_iter


def test_overflow_raises_sklearns_error(golden):
    xtr, ytr, _, _, alpha, max_iter = K.golden_case("overflow")
    with pytest.raises(ValueError) as e:
        ev.fit_sgd_classifiers(xtr, ytr, [alpha], max_iter=max_iter)
    assert str(e.value) == str(golden["overflow_error"])


@pytest.mark.parametrize("name", ["c2", "c9", "unnorm"])
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
    want = O.fit(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter)
    clf = _fit(case)[0]
    assert clf.n_iter_ == want["n_iter_"]
    _close(clf.coef_, want["coef_"], f"{name} coef vs oracle")
    assert np.array_equal(clf.predict(xte), O.predict(want, xte))


@pytest.mark.parametrize("n_out", [1, 3, 9])
def test_decision_kernel(n_out):
    g = torch.Generator().manual_seed(100 + n_out)
    x = (torch.rand(1000, 1024, generator=g) * 3).cuda()          # non-negative, DenseNet-like
    coef = torch.randn(n_out, 1024, generator=g).cuda() * 0.05
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


def test_512_and_1024_interleaved_equal_alone():
    wide, narrow = K.golden_case("c9"), O.golden_case("c9")
    alone_wide = _fit(wide, SWEEP)
    dec_w = alone_wide[1].decision_function(wide[2])
    alone_narrow = _fit(narrow, SWEEP)
    dec_n = alone_narrow[1].decision_function(narrow[2])
    # the two widths in turn on one stream, twice
    x_w, x_n = torch.from_numpy(wide[0]).cuda(), torch.from_numpy(narrow[0]).cuda()
    runs = [ev.fit_sgd_classifiers(x, y, SWEEP, seed=O.GOLDEN_SEED)
            for _ in range(2) for x, y in ((x_n, narrow[1]), (x_w, wide[1]))]
    for i, run in enumerate(runs):
        _same(run, alone_narrow if i % 2 == 0 else alone_wide)
    assert alone_narrow[0].n_features_in_ == 512 and alone_wide[0].n_features_in_ == 1024
    for _ in range(2):
        assert np.array_equal(runs[0][1].decision_function(narrow[2]), dec_n)
        assert np.array_equal(runs[1][1].decision_function(wide[2]), dec_w)


def test_width_mismatch_raises_sklearns_error():
    wide, narrow = K.golden_case("c2"), O.golden_case("c2")
    clf = _fit(wide)[0]
    msg = "^X has 512 features, but SGDClassifier is expecting 1024 features as input.$"
    with pytest.raises(ValueError, match=msg):
        clf.predict(torch.from_numpy(narrow[2]).cuda())
    with pytest.raises(ValueError, match=msg):     # plip training features, mudipath test features
        ev.LinearProber(alpha=1e-3).train_and_test(wide[0], wide[1], narrow[2], narrow[3])


def test_reference_mudipath_probe_end_to_end(tmp_path, monkeypatch):
    """``linear_probing_evaluation.py --model_name=mudipath``: the factory's DenseNet-121 embeds the train and test
    images, and ``LinearProber(alpha, seed).train_and_test`` fits and scores the probe on the 1024-wide features."""
    import PIL.Image
    import densenet_oracle
    from plip_b200.embedders import DenseNetEmbedder, EmbedderFactory
    ckpt = tmp_path / "densenet121-mh-best-191205-141200.pth"
    sd = densenet_oracle.make_state_dict(0)
    raw = {"features." + k: v for k, v in sd.items() if not k.startswith("classifier.")}
    raw["heads.0.weight"] = torch.zeros(3, 1024)      # the multi-task heads the reference's cleaning drops
    torch.save(raw, ckpt)
    monkeypatch.setenv("PLIP_B200_MTDP", str(ckpt))
    rng = np.random.default_rng(2024)

    def pngs(prefix, sizes):
        paths = []
        for i, (h, w) in enumerate(sizes):
            p = tmp_path / f"{prefix}{i}.png"
            PIL.Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p)
            paths.append(str(p))
        return paths

    # train: mixed sizes (the device Resize(224) + CenterCrop route); test: 224 x 224 (straight to the network)
    train_images = pngs("train", [[(224, 224), (300, 260), (180, 410), (512, 384)][i % 4] for i in range(36)])
    test_images = pngs("test", [(224, 224)] * 12)

    embedder = EmbedderFactory().factory(Namespace(model_name="mudipath", backbone="default"))
    assert isinstance(embedder, DenseNetEmbedder)
    train_x = embedder.image_embedder(train_images)
    test_x = embedder.image_embedder(test_images)
    assert train_x.shape == (36, 1024) and test_x.shape == (12, 1024) and train_x.dtype == np.float32
    names = np.array(["tumour", "stroma", "lymphocytes"])
    edges = np.sort(train_x[:, 0])[[12, 24]]                          # classes by the first feature's tercile
    train_y, test_y = (names[np.searchsorted(edges, v[:, 0], side="right")] for v in (train_x, test_x))
    assert len(np.unique(train_y)) == 3

    clf, (test_metrics, train_metrics) = ev.LinearProber(alpha=1e-3, seed=1).train_and_test(
        train_x, train_y, test_x, test_y)
    classes = np.unique(train_y)
    want = O.fit(train_x, np.searchsorted(classes, train_y), 1e-3, 1)
    assert clf.n_iter_ == want["n_iter_"] and clf.n_features_in_ == 1024
    assert np.array_equal(clf.classes_, np.arange(len(classes)))
    _close(clf.coef_, want["coef_"], "mudipath features coef vs oracle")
    yte = np.searchsorted(classes, test_y)
    assert np.array_equal(clf.predict(test_x), O.predict(want, test_x))
    assert test_metrics == {"accuracy": float(np.mean(O.predict(want, test_x) == yte)), "split": "test"}
    ytr = np.searchsorted(classes, train_y)
    assert train_metrics == {"accuracy": float(np.mean(O.predict(want, train_x) == ytr)), "split": "train"}
