"""Argument checks of the C entry points that take images or token ids, without a GPU: every bad argument is reported
with the shared message of its input kind, before the handle, and a null handle with valid arguments is reported as
"null engine" (no device is touched).  The ``_hw`` and ``*_outputs`` symbols are checked in ``test_hires_host.py`` and
``test_outputs_host.py``."""
import ctypes as C

import pytest

from plip_b200 import _lib

buf = (C.c_char * 64)()
P = C.cast(buf, C.c_void_p)


def _rejects(rc, fragment):
    assert rc != 0 and fragment in _lib.last_error(), (rc, _lib.last_error())


@pytest.fixture(scope="module")
def L():
    return _lib.lib()


def test_pixel_entry_points(L):
    calls = (  # (pixels, format, n, out) -> rc; null engine
        lambda px, fmt, n, out: L.plip_encode_images(None, px, fmt, n, out, 0, None),
        lambda px, fmt, n, out: L.plip_encode_images_host(None, px, fmt, n, out, 0),
    )
    for f in calls:
        _rejects(f(None, 0, 1, P), "null")
        _rejects(f(P, 0, 1, None), "null")
        _rejects(f(P, 0, 0, P), "positive")
        _rejects(f(P, 0, -3, P), "positive")
        _rejects(f(P, 3, 1, P), "format")
        _rejects(f(P, -1, 1, P), "format")
        for fmt in (0, 1, 2):
            _rejects(f(P, fmt, 1, P), "null engine")


def test_ids_entry_points(L):
    calls = (  # (ids, dtype, n, seq_len, out) -> rc; null engine, no mask
        lambda ids, dt, n, s, out: L.plip_encode_text(None, ids, dt, None, n, s, out, 0, None),
        lambda ids, dt, n, s, out: L.plip_encode_text_prefix(None, ids, dt, None, n, s, s, out, 0, None),
        lambda ids, dt, n, s, out: L.plip_encode_text_host(None, ids, dt, None, n, s, out, 0),
    )
    for f in calls:
        _rejects(f(None, 0, 1, 77, P), "null")
        _rejects(f(P, 0, 1, 77, None), "null")
        _rejects(f(P, 0, 0, 77, P), "positive")
        for s in (0, 78):       # the TF message, host path included
            _rejects(f(P, 0, 1, s, P), "Sequence length must be less than max_position_embeddings")
        _rejects(f(P, 2, 1, 77, P), "dtype")
        for dt in (0, 1):
            for s in (1, 16, 77):
                _rejects(f(P, dt, 1, s, P), "null engine")
    prefix = lambda n, s, p: L.plip_encode_text_prefix(None, P, 0, P, n, s, p, P, 0, None)  # noqa: E731
    _rejects(prefix(1, 77, 0), "prefix_len")
    _rejects(prefix(1, 16, 17), "prefix_len")
    _rejects(prefix(1, 78, 78), "Sequence length")
    _rejects(prefix(1, 16, 1), "null engine")
    _rejects(prefix(1, 77, 77), "null engine")


def test_hidden_states_hook(L):
    def h(tower, x, fmt, n, layers, out):
        return L.plip_dbg_hidden_states(None, tower, x, fmt, None, n, layers, out, None)

    for tower in (2, -1):
        _rejects(h(tower, P, 0, 1, 1, P), "tower")
        _rejects(h(tower, P, 0, 1, 1, P), "out of range")
    for tower in (0, 1):
        _rejects(h(tower, None, 0, 1, 1, P), "null")
        _rejects(h(tower, P, 0, 1, 1, None), "null")
        _rejects(h(tower, P, 0, 0, 1, P), "positive")
        _rejects(h(tower, P, 0, 1, 13, P), "num_layers")
        _rejects(h(tower, P, 0, 1, -1, P), "num_layers")
        for layers in (0, 12):
            _rejects(h(tower, P, 0, 1, layers, P), "null engine")
    _rejects(h(0, P, 3, 1, 1, P), "format")
    _rejects(h(1, P, 2, 1, 1, P), "dtype")
    _rejects(L.plip_dbg_hidden_states_hw(None, P, 0, 1, 224, 224, 13, P, None), "num_layers")
