"""The linear probe without a GPU: the numpy restatement of scikit-learn's SGD (tests/sgd_oracle.py) against the
golden file and the live library, the library's Fisher-Yates permutation, the argument checks of the C ABI, and the
label / input handling of ``LinearProber``."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

import sgd_oracle as O
from plip_b200 import _lib
from plip_b200 import evaluation as ev
from plip_b200.engine import sgd_fit, sgd_shuffle_permutation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "linear_probe_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def test_golden_inputs_regenerate(golden):
    assert str(golden["sklearn_version"]) == "1.9.0"
    for name in O.GOLDEN_CASES:
        assert hashlib.sha256(O.golden_case(name)[0].tobytes()).hexdigest() == str(golden[f"{name}_x_sha256"]), name


@pytest.mark.parametrize("name", list(O.GOLDEN_CASES))
def test_oracle_equals_golden_bit_for_bit(golden, name):
    xtr, ytr, xte, _, alpha, max_iter = O.golden_case(name)
    if f"{name}_error" in golden:
        with pytest.raises(ValueError) as e:
            O.fit(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter)
        assert str(e.value) == str(golden[f"{name}_error"])
        return
    stats = {}
    m = O.fit(xtr, ytr, alpha, O.GOLDEN_SEED, max_iter=max_iter, stats=stats)
    assert m["n_iter_"] == int(golden[f"{name}_n_iter"])
    assert m["coef_"].dtype == np.float32 and np.array_equal(m["coef_"], golden[f"{name}_coef"])
    assert m["intercept_"].dtype == golden[f"{name}_intercept"].dtype
    assert np.array_equal(m["intercept_"], golden[f"{name}_intercept"])
    assert np.array_equal(O.predict(m, xte), golden[f"{name}_pred"])
    if name == "reset":
        assert stats["resets"] >= 1          # wscale fell below 1e-6 with non-zero weights
    if name == "max_iter":
        assert m["n_iter_"] == max_iter


@pytest.mark.parametrize("n,classes,alpha,seed", [(160, 2, 3e-4, 0), (200, 5, 3e-2, 11)])
def test_oracle_equals_live_sklearn(n, classes, alpha, seed):
    sk = pytest.importorskip("sklearn.linear_model")
    x, y = O.embeddings(n, classes, seed=seed + 100, imbalance=0.4)
    m = O.fit(x, y, alpha, seed)
    clf = sk.SGDClassifier(random_state=seed, loss="log_loss", alpha=alpha, penalty="l2", max_iter=10000,
                           class_weight="balanced").fit(x, y)
    assert clf.n_iter_ == m["n_iter_"]
    assert np.array_equal(clf.coef_, m["coef_"]) and np.array_equal(clf.intercept_, m["intercept_"])


@pytest.mark.parametrize("n,seed", [(1, 5), (2, 9), (7, 0), (7, 1), (300, 123456789), (1000, 2 ** 31 - 2),
                                    (4099, 42)])
def test_shuffle_permutation_is_sklearns(n, seed):
    got = sgd_shuffle_permutation(n, seed)
    assert got.dtype == np.int32 and np.array_equal(got, O.shuffle_permutation(n, seed))
    assert np.array_equal(np.sort(got), np.arange(n))
    if seed == 0:                                  # our_rand_r replaces a zero state by its default, 1
        assert np.array_equal(got, O.shuffle_permutation(n, 1))


def test_shuffle_permutation_is_sklearns_dataset_shuffle():
    ds = pytest.importorskip("sklearn.utils._seq_dataset")
    n = 50
    x = np.zeros((n, 1), np.float32)
    d = ds.ArrayDataset32(x, np.arange(n, dtype=np.float32), np.ones(n, np.float32), seed=1)
    sigma = sgd_shuffle_permutation(n, 77)
    order = np.arange(n)
    for _ in range(3):                             # the same swap sequence every epoch
        d._shuffle_py(77)
        order = order[sigma]
    assert np.array_equal([int(d._next_py()[1]) for _ in range(n)], order)   # y holds the sample index


def test_problem_seeds_follow_sklearn():
    for classes in (2, 3, 9):
        assert ev._problem_seeds(classes, 7) == O.problem_seeds(classes, 7)


# ---- C ABI argument checks (all on the host, before any CUDA call) ----------------------------------------------

def _buf(nbytes):
    b = (C.c_char * (nbytes + 64))()
    a = C.addressof(b)
    return b, a + (-a) % 16


def _fit_args(**over):
    n = over.pop("n", 8)
    keep = []

    def arr(values, ctype):
        a = (ctype * len(values))(*values)
        keep.append(a)
        return C.cast(a, C.c_void_p)

    bx, x = _buf(n * 512 * 4)
    bo, out = _buf(4096)
    bw, ws = _buf(1 << 16)
    keep += [bx, bo, bw]
    problems = over.pop("problems", [(0.01, 1.0, 1.0, 0, 0)])
    table = (_lib.SgdProblem * len(problems))(*[_lib.SgdProblem(*p) for p in problems])
    keep.append(table)
    args = dict(x=x, n=n, dim=512, cls=arr(over.pop("classes", [0, 1] * (n // 2) if n > 1 else [0]), C.c_int32),
                n_classes=2, table=table, n_problems=len(problems),
                sigma_rows=arr(over.pop("sigma", list(range(n))), C.c_int32), n_sigma=1, max_iter=10, tol=1e-3,
                n_iter_no_change=5, coef=out, intercept=out, n_iter=out, overflow=out, ws=ws, ws_bytes=1 << 16,
                stream=None)
    args.update(over)
    return list(args.values()), keep


@pytest.mark.parametrize("over,msg", [
    (dict(n=1), "n = 1"),
    (dict(dim=768), "dim = 768"),
    (dict(n_classes=1), "n_classes = 1"),
    (dict(problems=[(0.0, 1.0, 1.0, 0, 0)]), "alpha = 0"),
    (dict(problems=[(-1e-4, 1.0, 1.0, 0, 0)]), "alpha = -0.0001"),
    (dict(problems=[(float("nan"), 1.0, 1.0, 0, 0)]), "alpha = nan"),
    (dict(problems=[(0.01, 1.0, 1.0, 0, 0), (float("inf"), 1.0, 1.0, 0, 0)]), "problem 1: alpha = inf"),
    (dict(problems=[(0.01, 1.0, 1.0, 2, 0)]), "pos_class = 2"),
    (dict(problems=[(0.01, 1.0, 1.0, 0, 1)]), "sigma_index = 1"),
    (dict(problems=[(0.01, float("inf"), 1.0, 0, 0)]), "weights inf"),
    (dict(classes=[0, 1, 0, 1, 0, 2, 0, 1]), "class id 2 of sample 5"),
    (dict(classes=[0, 1, 0, -1, 0, 1, 0, 1]), "class id -1 of sample 3"),
    (dict(sigma=[0, 1, 2, 3, 8, 5, 6, 7]), "sigma[0][4] = 8"),
    (dict(max_iter=0), "max_iter = 0"),
    (dict(n_iter_no_change=0), "n_iter_no_change = 0"),
    (dict(tol=float("nan")), "tol is NaN"),
    (dict(ws_bytes=100), "workspace of 100 bytes"),
    (dict(x=None), "null argument"),
    (dict(cls=None), "null argument"),
    (dict(table=None), "null argument"),
    (dict(sigma_rows=None), "null argument"),
    (dict(coef=None), "null argument"),
    (dict(ws=None), "null argument"),
])
def test_sgd_fit_rejects_bad_arguments_before_any_launch(over, msg):
    L = _lib.lib()
    args, keep = _fit_args(**over)
    assert L.plip_sgd_fit(*args) == -2
    assert msg in _lib.last_error(), _lib.last_error()


def test_sgd_fit_rejects_unaligned_pointers():
    L = _lib.lib()
    args, keep = _fit_args()
    args[0] += 4
    assert L.plip_sgd_fit(*args) == -2 and "x_dev" in _lib.last_error() and "aligned" in _lib.last_error()


def test_workspace_and_decision_arguments():
    L = _lib.lib()
    b = C.c_uint64(0)
    assert L.plip_sgd_workspace_bytes(100000, 9, 36, C.byref(b)) == 0
    assert b.value >= 4 * 100000 * (1 + 9 + 2 * 36)
    assert L.plip_sgd_workspace_bytes(1, 1, 1, C.byref(b)) == -2 and "n = 1" in _lib.last_error()
    assert L.plip_sgd_workspace_bytes(10, 0, 1, C.byref(b)) == -2
    assert L.plip_sgd_shuffle_permutation(0, 1, None) == -2 and "null" in _lib.last_error()
    buf, a = _buf(4 * 512 * 4)
    assert L.plip_linear_decision(a, 4, 256, a, a, 2, a, a, None) == -2 and "dim = 256" in _lib.last_error()
    assert L.plip_linear_decision(a, 4, 512, a, a, 0, a, a, None) == -2 and "n_out = 0" in _lib.last_error()
    assert L.plip_linear_decision(a, 4, 512, None, a, 2, a, a, None) == -2 and "null" in _lib.last_error()
    assert L.plip_linear_decision(a + 4, 4, 512, a, a, 2, a, a, None) == -2 and "aligned" in _lib.last_error()
    assert L.plip_linear_decision(a, 0, 512, a, a, 2, a, a, None) == 0       # nothing to do


def test_python_bindings_check_inputs_without_a_gpu():
    with pytest.raises(ValueError, match="CUDA float32"):
        sgd_fit(torch.zeros(4, 512), [0, 1, 0, 1], 2, [(0.1, 1, 1.0, 1.0, 0)], np.zeros((1, 4), np.int32))
    with pytest.raises(ValueError, match="outside"):
        sgd_shuffle_permutation(0, 1)


# ---- LinearProber input handling ----------------------------------------------------------------------------------

def test_labels_follow_label_encoder():
    tr, te = ev._encode_labels(["stroma", "tumour", "adipose", "tumour"], ["tumour", "adipose"])
    assert tr.tolist() == [1, 2, 0, 2] and te.tolist() == [2, 0]
    with pytest.raises(ValueError, match="previously unseen labels"):
        ev._encode_labels(["a", "b"], ["a", "c"])
    tr, te = ev._encode_labels(np.array([10, 3, 7]), [3])
    assert tr.tolist() == [2, 0, 1] and te.tolist() == [0]


def test_embeddings_must_be_float32_and_finite():
    cpu = torch.device("cpu")
    assert ev._embeddings(np.zeros((3, 512), np.float32), cpu).shape == (3, 512)
    for bad in (np.zeros((3, 512)), np.zeros((3, 512), np.float16), np.zeros((3, 256), np.float32),
                torch.zeros(3, 512, dtype=torch.float64), np.zeros(512, np.float32)):
        with pytest.raises(ValueError, match="float32"):
            ev._embeddings(bad, cpu)
    x = np.zeros((3, 512), np.float32)
    x[1, 7] = np.nan
    with pytest.raises(ValueError, match="Input X contains NaN"):
        ev._embeddings(x, cpu)
    x[1, 7] = np.inf
    with pytest.raises(ValueError, match="Input X contains infinity"):
        ev._embeddings(x, cpu)
