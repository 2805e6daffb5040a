"""Engine.encode_pair (plip_encode_pair): the text tower on the engine's own stream and workspace at the same time as
the vision tower.  The embeddings must be bit for bit those of encode_images and encode_text, with the same kernels."""
import pytest
import torch

from oracle import synth
from plip_b200._lib import lib
from plip_b200.engine import Engine

pytestmark = pytest.mark.gpu

# kernels of the two tower passes (test_gpu_engine_accounting): vision 67, text 65, + one l2 normalisation each
LAUNCHES = 67 + 65 + 2


@pytest.fixture(scope="module")
def big_engine(state_dict):
    eng = Engine(state_dict, max_micro_batch=1024)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def inputs():
    px = synth.pixel_values(1024, seed=91).to(torch.bfloat16).cuda()
    ids = synth.token_ids(1024, seed=92, full_length=True)[0].cuda()
    return px, ids


def _launches(call):
    before = lib().plip_launch_count()
    out = call()
    torch.cuda.synchronize()
    return out, lib().plip_launch_count() - before


@pytest.mark.parametrize("n", [129, 150, 1024])
def test_encode_pair_equals_the_two_towers(big_engine, inputs, n):
    px, ids = inputs[0][:n], inputs[1][:n]
    want_img = big_engine.encode_images(px, normalize=True)
    want_txt = big_engine.encode_text(ids, normalize=True)
    for _ in range(2):                  # the first call allocates the text workspace and stream
        (img, txt), launches = _launches(lambda: big_engine.encode_pair(px, ids))
        assert torch.equal(img, want_img) and torch.equal(txt, want_txt)
        assert launches == LAUNCHES


def test_encode_pair_masked_uneven_and_pruned(big_engine):
    """Different counts on the two sides, an attention mask, uint8 tiles; and with last-layer pruning."""
    tiles = torch.from_numpy(synth.tiles_u8(200, seed=93)).cuda()
    ids, mask = synth.token_ids(300, seed=94)
    ids, mask = ids.cuda(), mask.cuda()
    img, txt = big_engine.encode_pair(tiles, ids, mask, normalize=False)
    assert torch.equal(img, big_engine.encode_images(tiles))
    assert torch.equal(txt, big_engine.encode_text(ids, mask))
    big_engine.set_last_layer_pruning(True)
    try:
        img, txt = big_engine.encode_pair(tiles, ids, mask)
        assert torch.equal(img, big_engine.encode_images(tiles, normalize=True))
        assert torch.equal(txt, big_engine.encode_text(ids, mask, normalize=True))
    finally:
        big_engine.set_last_layer_pruning(False)


def test_encode_pair_waits_on_the_callers_stream(big_engine, inputs):
    """The inputs are written on a side stream the call's stream waits for, and the outputs are read on that stream
    right after the call, with no device synchronise in between."""
    px, ids = inputs[0][:256], inputs[1][:256]
    want_img, want_txt = big_engine.encode_images(px, normalize=True), big_engine.encode_text(ids, normalize=True)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        px2, ids2 = px.clone(), ids.clone()
    torch.cuda.current_stream().wait_stream(side)
    img, txt = big_engine.encode_pair(px2, ids2)
    img_c, txt_c = img.clone(), txt.clone()
    torch.cuda.synchronize()
    assert torch.equal(img_c, want_img) and torch.equal(txt_c, want_txt)


def test_encode_pair_falls_back_on_small_and_large_batches(engine, inputs):
    """n within the graph-replayed sizes, and n above one micro-batch of the 64-row engine: the two calls."""
    px, ids = inputs
    for n_img, n_txt in ((8, 8), (150, 130)):
        img, txt = engine.encode_pair(px[:n_img], ids[:n_txt])
        assert torch.equal(img, engine.encode_images(px[:n_img], normalize=True))
        assert torch.equal(txt, engine.encode_text(ids[:n_txt], normalize=True))


def test_encode_pair_profile_rows(big_engine, inputs):
    """Profiled, the towers run one after the other: the rows of the two calls."""
    px, ids = inputs[0][:256], inputs[1][:256]

    def rows(call):
        big_engine.profile(True)
        try:
            call()
            return {r["name"]: r["launches"] for r in big_engine.profile_read()}
        finally:
            big_engine.profile(False)
    want = rows(lambda: (big_engine.encode_images(px, normalize=True), big_engine.encode_text(ids, normalize=True)))
    assert rows(lambda: big_engine.encode_pair(px, ids)) == want
