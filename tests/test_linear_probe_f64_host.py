"""The linear probe's 64-bit instantiation (float16 / float64 features) without a GPU: the numpy restatement of
scikit-learn's 64-bit ``_plain_sgd`` (tests/sgd_oracle64.py ``fit64``) against the golden file and the live library, the
argument checks of ``plip_sgd_fit_f64`` / ``plip_linear_decision_f64`` and their bindings, and the dtype routing of
``evaluation`` (which fit and which decision a dtype reaches, and the dtypes of what comes back), with the kernels
replaced by stand-ins that record their calls."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

import sgd_cases_f64 as K
import sgd_oracle as O
import sgd_oracle64 as O64
from plip_b200 import _lib
from plip_b200 import evaluation as ev
from plip_b200.engine import linear_decision_f64, sgd_fit_f64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "linear_probe_f64_golden.npz")
CPU = torch.device("cpu")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def test_golden_inputs_regenerate(golden):
    assert str(golden["sklearn_version"]) == "1.9.0"
    for name, case in K.GOLDEN_CASES.items():
        xtr = K.golden_case(name)[0]
        assert xtr.dtype == case[8] and xtr.shape[1] == case[7]
        assert hashlib.sha256(xtr.tobytes()).hexdigest() == str(golden[f"{name}_x_sha256"]), name
    x = K.golden_case("c9")[0]
    assert x.dtype == np.float16 and np.abs(np.linalg.norm(x.astype(np.float64), axis=1) - 1).max() < 2e-3


@pytest.mark.parametrize("name", list(K.GOLDEN_CASES))
def test_oracle_equals_golden_bit_for_bit(golden, name):
    xtr, ytr, xte, _, alpha, max_iter = K.golden_case(name)
    if f"{name}_error" in golden:
        with pytest.raises(ValueError) as e:
            O64.fit64(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter)
        assert str(e.value) == str(golden[f"{name}_error"])
        return
    stats = {}
    m = O64.fit64(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter, stats=stats)
    assert m["n_iter_"] == int(golden[f"{name}_n_iter"])
    for key in ("coef", "intercept"):
        want = golden[f"{name}_{key}"]
        assert m[f"{key}_"].dtype == want.dtype == np.float64 and m[f"{key}_"].shape == want.shape
        assert np.array_equal(m[f"{key}_"], want), key
    assert np.array_equal(O.predict(m, xte), golden[f"{name}_pred"])
    if name == "c2":
        assert m["coef_"].shape == (1, 512) and m["intercept_"].shape == (1,)
    if name == "reset":
        assert stats["resets"] >= 1          # wscale fell below 1e-9 with non-zero weights
    if name == "max_iter":
        assert m["n_iter_"] == max_iter


@pytest.mark.parametrize("n,classes,alpha,seed,dtype,dim", [(160, 2, 3e-4, 0, np.float16, 512),
                                                            (180, 5, 3e-2, 11, np.float64, 1024)])
def test_oracle_equals_live_sklearn(n, classes, alpha, seed, dtype, dim):
    sk = pytest.importorskip("sklearn.linear_model")
    x, y = K.embeddings(n, classes, seed=seed + 300, dim=dim, imbalance=0.4, dtype=dtype)
    m = O64.fit64(x, y, alpha, seed)
    clf = sk.SGDClassifier(random_state=seed, loss="log_loss", alpha=alpha, penalty="l2", max_iter=10000,
                           class_weight="balanced").fit(x, y)
    assert clf.n_iter_ == m["n_iter_"] and clf.coef_.dtype == np.float64
    assert np.array_equal(clf.coef_, m["coef_"]) and np.array_equal(clf.intercept_, m["intercept_"])


def test_float32_and_64_bit_fits_differ():
    """Casting float16 rows to float32 does not reproduce scikit-learn's fit on them: it is the other instantiation."""
    xtr, ytr, _, _, alpha, _ = K.golden_case("c9")
    wide, narrow = O64.fit64(xtr, ytr, alpha), O.fit(xtr.astype(np.float32), ytr, alpha)
    assert not np.array_equal(wide["coef_"], narrow["coef_"].astype(np.float64))


# ---- C ABI (all on the host, before any CUDA call) -----------------------------------------------------------------

def _buf(nbytes):
    b = (C.c_char * (nbytes + 64))()
    a = C.addressof(b)
    return b, a + (-a) % 16


def _fit_args(**over):
    n = 8
    keep = []

    def arr(values, ctype):
        a = (ctype * len(values))(*values)
        keep.append(a)
        return C.cast(a, C.c_void_p)

    bx, x = _buf(n * 1024 * 8)
    bo, out = _buf(1 << 14)
    bw, ws = _buf(1 << 16)
    keep += [bx, bo, bw]
    problems = over.pop("problems", [(0.01, 1.0, 1.0, 0, 0)])
    table = (_lib.SgdProblem * len(problems))(*[_lib.SgdProblem(*p) for p in problems])
    keep.append(table)
    args = dict(x=x, n=n, dim=512, cls=arr([0, 1] * (n // 2), C.c_int32), n_classes=2, table=table,
                n_problems=len(problems), sigma_rows=arr(list(range(n)), C.c_int32), n_sigma=1, max_iter=10,
                tol=1e-3, n_iter_no_change=5, coef=out, intercept=out, n_iter=out, overflow=out, ws=ws,
                ws_bytes=1 << 16, stream=None)
    args.update(over)
    return list(args.values()), keep


@pytest.mark.parametrize("over,msg", [
    (dict(n=1), "n = 1 samples"),
    (dict(dim=768), "dim = 768; the embeddings must be 512 or 1024 wide"),
    (dict(n_classes=1), "n_classes = 1"),
    (dict(problems=[(0.0, 1.0, 1.0, 0, 0)]), "alpha = 0"),
    (dict(problems=[(0.01, 1.0, 1.0, 2, 0)]), "pos_class = 2"),
    (dict(problems=[(0.01, 1.0, 1.0, 0, 1)]), "sigma_index = 1"),
    (dict(problems=[(0.01, float("inf"), 1.0, 0, 0)]), "weights inf"),
    (dict(max_iter=0), "max_iter = 0"),
    (dict(tol=float("nan")), "tol is NaN"),
    (dict(ws_bytes=100), "workspace of 100 bytes"),
    (dict(x=None), "null argument"),
    (dict(coef=None), "null argument"),
])
def test_sgd_fit_f64_rejects_bad_arguments_before_any_launch(over, msg):
    L = _lib.lib()
    args, keep = _fit_args(**over)
    assert L.plip_sgd_fit_f64(*args) == -2
    err = _lib.last_error()
    assert err.startswith("plip_sgd_fit_f64: ") and msg in err, err


def test_sgd_fit_f64_checks_alignment_and_widths():
    L = _lib.lib()
    for dim in (512, 1024):                  # past the width check: the next bad argument is the one reported
        args, keep = _fit_args(dim=dim, n_classes=1)
        assert L.plip_sgd_fit_f64(*args) == -2 and "n_classes = 1" in _lib.last_error()
    args, keep = _fit_args()
    args[0] += 8
    assert L.plip_sgd_fit_f64(*args) == -2
    assert "x_dev" in _lib.last_error() and "16-byte aligned" in _lib.last_error()


def test_one_workspace_serves_both_precisions():
    """A 40-byte problem entry (double class weights) fits the table section the workspace query reserves."""
    L = _lib.lib()
    for p in (1, 6, 7, 36, 1000):
        b = C.c_uint64(0)
        assert L.plip_sgd_workspace_bytes(100, 1, p, C.byref(b)) == 0
        assert b.value >= 40 * p + 4 * 100 * (1 + 1 + 2 * p)


def test_linear_decision_f64_arguments():
    L = _lib.lib()
    buf, a = _buf(4 * 1024 * 8)
    assert L.plip_linear_decision_f64(a, 4, 256, a, a, 2, a, a, None) == -2
    assert _lib.last_error() == "plip_linear_decision_f64: dim = 256; the embeddings must be 512 or 1024 wide"
    assert L.plip_linear_decision_f64(a, 4, 1024, a, a, 0, a, a, None) == -2 and "n_out = 0" in _lib.last_error()
    assert L.plip_linear_decision_f64(a, 4, 512, None, a, 2, a, a, None) == -2 and "null" in _lib.last_error()
    assert L.plip_linear_decision_f64(a + 8, 4, 512, a, a, 2, a, a, None) == -2 and "aligned" in _lib.last_error()
    assert L.plip_linear_decision_f64(a, 0, 512, a, a, 2, a, a, None) == 0       # nothing to do


def test_python_bindings_want_cuda_float64():
    with pytest.raises(ValueError, match="CUDA float64 .* 512 or 1024"):
        sgd_fit_f64(torch.zeros(4, 512, dtype=torch.float64), [0, 1, 0, 1], 2, [(0.1, 1, 1.0, 1.0, 0)],
                    np.zeros((1, 4), np.int32))
    with pytest.raises(ValueError, match="CUDA float64"):
        linear_decision_f64(torch.zeros(4, 1024), torch.zeros(2, 1024, dtype=torch.float64), torch.zeros(2))


# ---- dtype routing in evaluation ------------------------------------------------------------------------------------

def test_probe_input_keeps_float32_float16_and_float64():
    for x in (np.ones((3, 512), np.float32), torch.ones(3, 1024)):
        assert ev._probe_input(x, CPU).dtype == torch.float32
    for dt, tdt in ((np.float16, torch.float16), (np.float64, torch.float64)):
        for x in (np.ones((3, 512), dt), torch.ones(3, 1024, dtype=tdt)):
            got = ev._probe_input(x, CPU)
            assert got.dtype == tdt and got.is_contiguous() and tuple(got.shape) == tuple(x.shape)
    assert ev._probe_input([[0.5] * 512] * 2, CPU).dtype == torch.float64          # np.asarray's float64


@pytest.mark.parametrize("bad", [np.zeros((3, 512), np.int64), np.zeros((3, 512), bool),
                                 torch.zeros(3, 512, dtype=torch.bfloat16), torch.zeros(3, 512, dtype=torch.int32),
                                 np.zeros((3, 768), np.float16), np.zeros(512, np.float64)])
def test_probe_input_rejects_other_dtypes_and_shapes(bad):
    with pytest.raises(ValueError, match="float32, float16 or float64 .* 512 or 1024"):
        ev._probe_input(bad, CPU)


@pytest.mark.parametrize("dt", [np.float16, np.float64])
def test_non_finite_input_raises_sklearns_message(dt):
    x = np.zeros((3, 512), dt)
    x[1, 7] = np.nan
    with pytest.raises(ValueError, match=r"^Input X contains NaN\.$"):
        ev._probe_input(x, CPU)
    x[1, 7] = -np.inf
    with pytest.raises(ValueError) as e:
        ev._probe_input(torch.from_numpy(x), CPU)
    assert str(e.value) == "Input X contains infinity or a value too large for dtype('float64')."


@pytest.mark.parametrize("dt", [np.float16, np.float64])
def test_non_finite_message_is_live_sklearns(dt):
    sk = pytest.importorskip("sklearn.linear_model")
    x, y = K.embeddings(40, 3, seed=5, dtype=dt)
    x[3, 100] = np.inf
    with pytest.raises(ValueError) as want:
        sk.SGDClassifier(random_state=0, max_iter=5, tol=None).fit(x, y)
    with pytest.raises(ValueError) as got:
        ev._probe_input(x, CPU)
    assert str(got.value) == str(want.value)


class _Calls:
    """Stand-ins for the four kernels' bindings: they record which one ran on what, and return zeros."""

    def __init__(self, monkeypatch):
        self.log = []
        for name, dt in (("sgd_fit", torch.float32), ("sgd_fit_f64", torch.float64)):
            monkeypatch.setattr(ev, name, self._fit(name, dt))
        for name, dt in (("linear_decision", torch.float32), ("linear_decision_f64", torch.float64)):
            monkeypatch.setattr(ev, name, self._decision(name, dt))

    def _fit(self, name, dt):
        def fit(x, class_ids, n_classes, problems, sigma, max_iter, tol, n_iter_no_change):
            self.log.append((name, x.dtype))
            p = len(problems)
            return (torch.zeros(p, x.shape[1], dtype=dt), torch.full((p,), 0.5, dtype=torch.float64),
                    torch.full((p,), 4, dtype=torch.int32), torch.zeros(p, dtype=torch.int32))
        return fit

    def _decision(self, name, dt):
        def decision(x, coef, intercept):
            self.log.append((name, x.dtype, coef.dtype))
            return torch.zeros(x.shape[0], coef.shape[0], dtype=dt), torch.zeros(x.shape[0], dtype=torch.int32)
        return decision


class _Cpu:
    device = CPU


@pytest.mark.parametrize("classes", [2, 3])
def test_fit_routes_by_the_training_dtype(monkeypatch, classes):
    calls = _Calls(monkeypatch)
    y = np.arange(12) % classes
    rows = 1 if classes == 2 else classes
    for x, fit, coef_dt, b_dt in (
            (np.ones((12, 512), np.float32), "sgd_fit", np.float32, np.float64 if classes == 2 else np.float32),
            (np.ones((12, 512), np.float16), "sgd_fit_f64", np.float64, np.float64),
            (torch.ones(12, 1024, dtype=torch.float64), "sgd_fit_f64", np.float64, np.float64)):
        calls.log.clear()
        clf = ev.fit_sgd_classifiers(x, y, [1e-3, 1e-2], engine=_Cpu())[1]
        assert calls.log == [(fit, torch.float64 if fit == "sgd_fit_f64" else torch.float32)]
        assert clf.coef_.dtype == coef_dt and clf.coef_.shape == (rows, x.shape[1])
        assert clf.intercept_.dtype == b_dt and clf.intercept_.shape == (rows,)


def test_decision_follows_numpys_promotion(monkeypatch):
    calls = _Calls(monkeypatch)
    y = np.arange(12) % 3
    m32 = ev.fit_sgd_classifiers(np.ones((12, 512), np.float32), y, [1e-3], engine=_Cpu())[0]
    m64 = ev.fit_sgd_classifiers(np.ones((12, 512), np.float16), y, [1e-3], engine=_Cpu())[0]
    f32, f64 = torch.float32, torch.float64
    for model, X, want, score_dt in (
            (m32, np.ones((2, 512), np.float32), ("linear_decision", f32, f32), np.float32),
            (m32, np.ones((2, 512), np.float16), ("linear_decision", f32, f32), np.float32),   # f16 . f32 -> f32
            (m32, np.ones((2, 512), np.float64), ("linear_decision_f64", f64, f64), np.float64),
            (m64, np.ones((2, 512), np.float32), ("linear_decision_f64", f64, f64), np.float64),
            (m64, torch.ones(2, 512, dtype=torch.float16), ("linear_decision_f64", f64, f64), np.float64),
            (m64, np.ones((2, 512), np.float64), ("linear_decision_f64", f64, f64), np.float64)):
        calls.log.clear()
        assert model.decision_function(X).dtype == score_dt
        assert calls.log == [want]
    with pytest.raises(ValueError, match="got int64"):
        m64.predict(np.ones((2, 512), np.int64))
