"""Device bilinear resize + crop (``plip_resize_crop_bilinear_u8``) bit-identical to PIL's BILINEAR resize and
torchvision's CenterCrop rounding, and the MuDiPath embedder's device route equal to its host PIL route."""
import numpy as np
import PIL.Image
import pytest
import torch

import densenet_oracle as O

pytestmark = pytest.mark.gpu

# (width, height): odd, 1-pixel, same-size on one axis, upscales, strong shrinks, extreme aspect ratios
SIZES = [(224, 224), (225, 224), (224, 225), (1, 1), (17, 9), (9, 17), (223, 500), (333, 227), (640, 480),
         (1023, 767), (2, 500), (4000, 3000), (6001, 301), (301, 6001), (3000, 5000)]


@pytest.fixture(scope="module")
def engine():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from plip_b200.densenet import DenseNetEngine
    return DenseNetEngine(O.make_state_dict(0), device="cuda:0", max_micro_batch=4)


def test_device_bilinear_bit_identical_to_pil(engine):
    from plip_b200.preprocess import device_resizable, pack_rgb, resize_center_crop_bilinear
    rng = np.random.default_rng(0)
    arrays = []
    for w, h in SIZES:
        assert device_resizable(w, h), (w, h)
        arrays.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    buf, descs = pack_rgb(arrays, crop="round", pinned=True)
    tiles = engine.resize_crop(buf.cuda(), descs).cpu().numpy()
    for (w, h), a, t in zip(SIZES, arrays, tiles):
        ref = np.asarray(resize_center_crop_bilinear(PIL.Image.fromarray(a)))
        assert np.array_equal(t, ref), (w, h, int(np.abs(t.astype(int) - ref).max()))


def test_embedder_device_route_equals_host_route(engine, tmp_path, monkeypatch):
    import plip_b200.embedders as E
    from plip_b200.preprocess import to_uint8_tiles_bilinear
    rng = np.random.default_rng(1)
    arrays = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in [(224, 224), (300, 260), (181, 410),
                                                                           (224, 224), (97, 130), (512, 384)]]
    paths = []
    for i, a in enumerate(arrays):
        p = tmp_path / f"img{i}.png"
        PIL.Image.fromarray(a).save(p)
        paths.append(str(p))
    emb = E.DenseNetEmbedder(engine, None, "mudipath", "default")
    dev = emb.embed_images(paths, batch_size=4)                     # mixed sizes: the device resize
    same = emb.embed_images([arrays[0], arrays[3]])                 # all 224 x 224: straight to the engine
    monkeypatch.setattr(E, "device_resizable", lambda w, h: False)  # every chunk through PIL on the host
    host = emb.embed_images([PIL.Image.fromarray(a) for a in arrays], batch_size=4)
    assert dev.shape == (6, 1024) and dev.dtype == np.float32
    assert np.array_equal(dev, host)
    assert np.array_equal(same, dev[[0, 3]])
    direct = engine.encode_images_host(to_uint8_tiles_bilinear(arrays))
    assert np.array_equal(dev, direct)
