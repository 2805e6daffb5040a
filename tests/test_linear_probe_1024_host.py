"""The linear probe at MuDiPath's 1024-wide DenseNet-121 features, without a GPU: the numpy restatement of
scikit-learn's SGD (tests/sgd_oracle.py) against the 1024-wide golden file and the live library, the width checks of
the C ABI and of the Python layer, and scikit-learn's error for features of the wrong width."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

import sgd_cases_1024 as K
import sgd_oracle as O
from plip_b200 import _lib
from plip_b200 import evaluation as ev
from plip_b200.engine import PROBE_DIMS, sgd_fit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "linear_probe_1024_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def test_golden_inputs_regenerate(golden):
    assert str(golden["sklearn_version"]) == "1.9.0"
    for name in K.GOLDEN_CASES:
        xtr = K.golden_case(name)[0]
        assert xtr.dtype == np.float32 and xtr.shape[1] == 1024
        assert hashlib.sha256(xtr.tobytes()).hexdigest() == str(golden[f"{name}_x_sha256"]), name


def test_unnormalised_case_is_densenet_like():
    x = K.golden_case("unnorm")[0]
    assert x.mean() > 0.2 and np.abs(x).max() > 2       # a positive offset and a scale of a few units, not unit-norm


@pytest.mark.parametrize("name", list(K.GOLDEN_CASES))
def test_oracle_equals_golden_bit_for_bit(golden, name):
    xtr, ytr, xte, _, alpha, max_iter = K.golden_case(name)
    if f"{name}_error" in golden:
        with pytest.raises(ValueError) as e:
            O.fit(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter)
        assert str(e.value) == str(golden[f"{name}_error"])
        return
    stats = {}
    m = O.fit(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter, stats=stats)
    assert m["n_iter_"] == int(golden[f"{name}_n_iter"])
    assert m["coef_"].dtype == np.float32 and m["coef_"].shape[1] == 1024
    assert np.array_equal(m["coef_"], golden[f"{name}_coef"])
    assert m["intercept_"].dtype == golden[f"{name}_intercept"].dtype
    assert np.array_equal(m["intercept_"], golden[f"{name}_intercept"])
    assert np.array_equal(O.predict(m, xte), golden[f"{name}_pred"])
    if name == "reset":
        assert stats["resets"] >= 1          # wscale fell below 1e-6 with non-zero weights
    if name == "max_iter":
        assert m["n_iter_"] == max_iter


@pytest.mark.parametrize("n,classes,alpha,seed,scale,shift", [(160, 2, 3e-4, 0, 1.0, 0.0),
                                                              (180, 5, 3e-2, 11, 4.0, 0.5)])
def test_oracle_equals_live_sklearn(n, classes, alpha, seed, scale, shift):
    sk = pytest.importorskip("sklearn.linear_model")
    x, y = K.embeddings(n, classes, seed=seed + 200, imbalance=0.4, scale=scale, shift=shift)
    m = O.fit(x, y, alpha, seed)
    clf = sk.SGDClassifier(random_state=seed, loss="log_loss", alpha=alpha, penalty="l2", max_iter=10000,
                           class_weight="balanced").fit(x, y)
    assert clf.n_iter_ == m["n_iter_"]
    assert np.array_equal(clf.coef_, m["coef_"]) and np.array_equal(clf.intercept_, m["intercept_"])


# ---- C ABI width checks (all on the host, before any CUDA call) -------------------------------------------------

def _buf(nbytes):
    b = (C.c_char * (nbytes + 64))()
    a = C.addressof(b)
    return b, a + (-a) % 16


def _fit_args(dim, n_classes=2):
    n = 8
    keep = []

    def arr(values, ctype):
        a = (ctype * len(values))(*values)
        keep.append(a)
        return C.cast(a, C.c_void_p)

    bx, x = _buf(n * 2048 * 4)
    bo, out = _buf(1 << 14)
    bw, ws = _buf(1 << 16)
    keep += [bx, bo, bw]
    table = (_lib.SgdProblem * 1)(_lib.SgdProblem(0.01, 1.0, 1.0, 0, 0))
    keep.append(table)
    args = [x, n, dim, arr([0, 1] * (n // 2), C.c_int32), n_classes, table, 1, arr(list(range(n)), C.c_int32), 1, 10,
            1e-3, 5, out, out, out, out, ws, 1 << 16, None]
    return args, keep


def test_sgd_fit_accepts_1024_and_rejects_other_widths():
    L = _lib.lib()
    for dim in PROBE_DIMS:                   # past the width check: the next bad argument is the one reported
        args, keep = _fit_args(dim, n_classes=1)
        assert L.plip_sgd_fit(*args) == -2
        assert "n_classes = 1" in _lib.last_error(), (dim, _lib.last_error())
    for dim in (768, 2048, 256, 0):
        args, keep = _fit_args(dim)
        assert L.plip_sgd_fit(*args) == -2
        err = _lib.last_error()
        assert f"dim = {dim}" in err and "512 or 1024 wide" in err, err


def test_linear_decision_accepts_1024_and_rejects_other_widths():
    L = _lib.lib()
    buf, a = _buf(4 * 2048 * 4)
    assert L.plip_linear_decision(a, 4, 1024, a, a, 0, a, a, None) == -2 and "n_out = 0" in _lib.last_error()
    assert L.plip_linear_decision(a, 0, 1024, a, a, 2, a, a, None) == 0       # nothing to do
    for dim in (768, 2048, 256):
        assert L.plip_linear_decision(a, 4, dim, a, a, 2, a, a, None) == -2
        assert f"dim = {dim}" in _lib.last_error() and "512 or 1024 wide" in _lib.last_error()


def test_python_bindings_name_both_widths():
    with pytest.raises(ValueError, match="CUDA float32 .* 512 or 1024"):
        sgd_fit(torch.zeros(4, 1024), [0, 1, 0, 1], 2, [(0.1, 1, 1.0, 1.0, 0)], np.zeros((1, 4), np.int32))


# ---- LinearProber input handling ----------------------------------------------------------------------------------

def test_embeddings_accept_1024_wide_features():
    cpu = torch.device("cpu")
    assert ev._embeddings(np.zeros((3, 1024), np.float32), cpu).shape == (3, 1024)
    assert ev._embeddings(torch.ones(3, 1024), cpu).shape == (3, 1024)
    for bad in (np.zeros((3, 768), np.float32), np.zeros((3, 2048), np.float32), np.zeros((3, 1024))):
        with pytest.raises(ValueError, match="float32 .* 512 or 1024"):
            ev._embeddings(bad, cpu)
    x = np.zeros((3, 1024), np.float32)
    x[2, 1000] = np.nan
    with pytest.raises(ValueError, match="Input X contains NaN"):
        ev._embeddings(x, cpu)
    x[2, 1000] = -np.inf
    with pytest.raises(ValueError, match="Input X contains infinity"):
        ev._embeddings(x, cpu)


def _classifier(d, n_classes=3):
    # never reaches the device: the width check comes first
    coef = np.zeros((n_classes if n_classes > 2 else 1, d), np.float32)
    return ev.SGDLinearClassifier(np.arange(n_classes), coef, np.zeros(len(coef), np.float32), 1, 1e-3,
                                  torch.device("cuda"))


@pytest.mark.parametrize("fit_d,x_d", [(1024, 512), (512, 1024), (1024, 768)])
def test_width_mismatch_raises_sklearns_error_without_a_gpu(fit_d, x_d):
    clf = _classifier(fit_d)
    assert clf.n_features_in_ == fit_d
    want = f"X has {x_d} features, but SGDClassifier is expecting {fit_d} features as input."
    for X in (np.zeros((3, x_d), np.float32), torch.zeros(3, x_d)):
        for call in (clf.predict, clf.decision_function):
            with pytest.raises(ValueError) as e:
                call(X)
            assert str(e.value) == want


def test_width_mismatch_message_is_live_sklearns():
    sk = pytest.importorskip("sklearn.linear_model")
    x, y = K.embeddings(40, 3, seed=5)
    clf = sk.SGDClassifier(random_state=0, loss="log_loss", max_iter=5, tol=None).fit(x, y)
    with pytest.raises(ValueError) as e:
        clf.predict(np.zeros((3, 512), np.float32))
    with pytest.raises(ValueError) as ours:
        _classifier(1024).predict(np.zeros((3, 512), np.float32))
    assert clf.n_features_in_ == 1024 and str(ours.value) == str(e.value)
