"""Per-token outputs (``output_hidden_states`` / ``output_attentions``) without a GPU: the CPU oracle against the
live-transformers golden vectors, the HF-style output containers, the Python routing of ``PlipCLIPModel``, and the
argument checks of the new C entry points (no device is touched)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import outputs_oracle as OO
from plip_b200 import _lib
from plip_b200.modeling import BaseModelOutputWithPooling, CLIPOutput, PlipCLIPModel
from plip_b200.synthetic import pixel_values_hw

torch.set_grad_enabled(False)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "outputs_golden.npz")
TOL = 2e-5


@pytest.fixture(scope="module")
def outputs_golden():
    return dict(np.load(GOLDEN, allow_pickle=False))


def _match(got, key, golden):
    ref = torch.from_numpy(golden[key])
    assert got.shape == ref.shape, (key, got.shape, ref.shape)
    assert (got - ref).abs().max().item() < TOL, (key, (got - ref).abs().max().item())


def _check_case(out, key, golden, n_hidden_rows, n_attn_rows, all_hidden):
    S = out["last_hidden_state"].shape[1]
    hr, ar = OO.golden_rows(S, n_hidden_rows), OO.golden_rows(S, n_attn_rows)
    assert len(out["hidden_states"]) == 13 and len(out["attentions"]) == 12
    for l in OO.GOLDEN_HIDDEN_LAYERS:
        h = out["hidden_states"][l]
        _match(h[:, hr] if all_hidden else h[:1, hr], f"{key}_hidden_{l}", golden)
    _match(out["last_hidden_state"][:, hr], f"{key}_last_hidden_state", golden)
    _match(out["pooler_output"], f"{key}_pooler_output", golden)
    for l in OO.GOLDEN_ATTN_LAYERS:
        _match(out["attentions"][l][:, :, ar], f"{key}_attn_{l}", golden)


@pytest.mark.parametrize("key", list(OO.GOLDEN_CASES))
def test_vision_oracle_matches_transformers_golden(outputs_golden, state_dict, key):
    n, size = OO.GOLDEN_CASES[key]
    out = OO.vision_outputs(state_dict, pixel_values_hw(n, size, size), interpolate_pos_encoding=size != 224)
    assert torch.equal(out["last_hidden_state"], out["hidden_states"][12])
    _check_case(out, key, outputs_golden, 5, 1, False)


def test_text_oracle_matches_transformers_golden(outputs_golden, state_dict):
    ids, mask = OO.golden_text_inputs()
    assert (mask == 0).any()
    out = OO.text_outputs(state_dict, ids, mask)
    _check_case(out, "text", outputs_golden, 2, 2, True)
    for a in out["attentions"]:                      # masked keys (causal and padding) are exactly 0
        assert (a.masked_select(~OO.visible_keys(77, mask, True, 3).expand_as(a)) == 0).all()


# ---- output containers ------------------------------------------------------------------------------------------------
def test_output_containers_keys():
    t = torch.zeros(2, 2)
    out = CLIPOutput(logits_per_image=t, logits_per_text=t, text_embeds=t, image_embeds=t)
    assert out.keys() == ("logits_per_image", "logits_per_text", "text_embeds", "image_embeds")  # unchanged
    assert out.vision_model_output is None and out["text_model_output"] is None
    mo = BaseModelOutputWithPooling(last_hidden_state=t, pooler_output=t)
    assert mo.keys() == ("last_hidden_state", "pooler_output") and mo["pooler_output"] is t
    mo = BaseModelOutputWithPooling(last_hidden_state=t, pooler_output=t, attentions=(t,))
    assert mo.keys() == ("last_hidden_state", "pooler_output", "attentions")
    out = CLIPOutput(logits_per_image=t, logits_per_text=t, text_embeds=t, image_embeds=t, vision_model_output=mo)
    assert out.keys()[-1] == "vision_model_output"


class _FakeEngine:
    """Records the calls PlipCLIPModel makes and returns tensors of the shapes the engine returns."""

    def __init__(self):
        self.calls = []

    def _out(self, n, S, D, heads, ohs, oa):
        return {"embeds": torch.ones(n, 512), "pooler_output": torch.zeros(n, D),
                "last_hidden_state": torch.zeros(n, S, D),
                "hidden_states": tuple(torch.zeros(n, S, D) for _ in range(13)) if ohs else None,
                "attentions": tuple(torch.zeros(n, heads, S, S) for _ in range(12)) if oa else None}

    def vision_outputs(self, px, ohs=False, oa=False, ipe=False, normalize=False):
        self.calls.append(("vision_outputs", ohs, oa, ipe, normalize))
        return self._out(px.shape[0], (px.shape[2] // 32) * (px.shape[3] // 32) + 1, 768, 12, ohs, oa)

    def text_outputs(self, ids, mask=None, ohs=False, oa=False, normalize=False):
        self.calls.append(("text_outputs", ohs, oa, normalize))
        return self._out(ids.shape[0], ids.shape[1], 512, 8, ohs, oa)

    def similarity(self, img, txt, normalize_image=True, normalize_text=True):
        return img @ txt.t()


def test_model_routes_flags_through_one_outputs_pass():
    model = PlipCLIPModel.__new__(PlipCLIPModel)
    model.engine = _FakeEngine()
    px, ids = torch.zeros(2, 3, 448, 448), torch.zeros(3, 77, dtype=torch.int64)
    out = model(input_ids=ids, pixel_values=px, output_attentions=True, interpolate_pos_encoding=True)
    assert model.engine.calls == [("vision_outputs", False, True, True, True), ("text_outputs", False, True, True)]
    assert out.keys()[-2:] == ("text_model_output", "vision_model_output")
    assert out.vision_model_output.attentions[0].shape == (2, 12, 197, 197)
    assert out.vision_model_output.hidden_states is None and out.logits_per_image.shape == (2, 3)
    vo = model.vision_model(pixel_values=torch.zeros(1, 3, 224, 224), output_hidden_states=True)
    assert vo.keys() == ("last_hidden_state", "pooler_output", "hidden_states") and len(vo.hidden_states) == 13
    to = model.text_model(input_ids=ids)
    assert to.keys() == ("last_hidden_state", "pooler_output") and to.pooler_output.shape == (3, 512)
    with pytest.raises(ValueError, match="pixel_values"):
        model.vision_model()
    with pytest.raises(ValueError, match="input_ids"):
        model.text_model()


# ---- C entry points: argument checks before any device work -------------------------------------------------------------
def test_tower_outputs_struct_layout():
    assert C.sizeof(_lib.TowerOutputs) == 48
    assert [f for f, _ in _lib.TowerOutputs._fields_] == ["embeds", "pooled", "last_hidden", "hidden", "attn", "normalize"]


def test_c_entry_points_reject_bad_arguments_without_a_device():
    L = _lib.lib()
    buf = (C.c_char * 64)()
    p = C.cast(buf, C.c_void_p)
    some = _lib.TowerOutputs(p, None, None, None, None, 0)
    none = _lib.TowerOutputs(None, None, None, None, None, 1)
    v = lambda *a: L.plip_vision_outputs(*a)  # noqa: E731
    assert v(None, p, 0, 1, 448, 448, C.byref(some), None) != 0 and "null engine" in _lib.last_error()
    assert v(None, p, 0, 1, 16, 448, C.byref(some), None) != 0 and "out of range" in _lib.last_error()
    assert v(None, p, 0, 1, 1056, 224, C.byref(some), None) != 0 and "out of range" in _lib.last_error()
    assert v(None, None, 0, 1, 224, 224, C.byref(some), None) != 0 and "null" in _lib.last_error()
    assert v(None, p, 0, 1, 224, 224, None, None) != 0 and "null" in _lib.last_error()
    assert v(None, p, 0, 0, 224, 224, C.byref(some), None) != 0 and "positive" in _lib.last_error()
    assert v(None, p, 3, 1, 224, 224, C.byref(some), None) != 0 and "format" in _lib.last_error()
    assert v(None, p, 0, 1, 224, 224, C.byref(none), None) != 0 and "no output requested" in _lib.last_error()
    t = lambda *a: L.plip_text_outputs(*a)  # noqa: E731
    assert t(None, p, 0, None, 1, 77, C.byref(some), None) != 0 and "null engine" in _lib.last_error()
    assert t(None, None, 0, None, 1, 77, C.byref(some), None) != 0 and "null" in _lib.last_error()
    assert t(None, p, 0, None, 1, 77, None, None) != 0 and "null" in _lib.last_error()
    assert t(None, p, 0, None, 0, 77, C.byref(some), None) != 0 and "positive" in _lib.last_error()
    assert t(None, p, 0, None, 1, 78, C.byref(some), None) != 0 and "Sequence length" in _lib.last_error()
    assert t(None, p, 0, None, 1, 0, C.byref(some), None) != 0 and "Sequence length" in _lib.last_error()
    assert t(None, p, 2, None, 1, 77, C.byref(some), None) != 0 and "dtype" in _lib.last_error()
    assert t(None, p, 0, None, 1, 77, C.byref(none), None) != 0 and "no output requested" in _lib.last_error()
    a = lambda *x: L.plip_dbg_attention_probs(*x)  # noqa: E731
    assert a(p, 1, 1026, 12, 0, None, p, None) != 0 and "bad shape" in _lib.last_error()
    assert a(p, 1, 0, 12, 0, None, p, None) != 0 and "bad shape" in _lib.last_error()
    assert a(p, 0, 50, 12, 0, None, p, None) != 0 and "bad shape" in _lib.last_error()
    assert a(p, 1, 50, 17, 0, None, p, None) != 0 and "head count" in _lib.last_error()
    assert a(None, 1, 50, 12, 0, None, p, None) != 0 and "null" in _lib.last_error()
    assert a(p, 1, 50, 12, 0, None, None, None) != 0 and "null" in _lib.last_error()
