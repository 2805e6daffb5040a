"""Generate tests/golden/train_transform_golden.npz: tiles of the reference's train-time transform, frozen.

Run once in the build container:  python tests/golden/make_train_transform_golden.py

The reference's OpenPath preprocess is ``_train_transform(first_resize, n_px)``
(``reproducibility/embedders/transform.py:18-42``): torchvision's Resize([first_resize], BICUBIC), RandomCrop([224]),
RandomHorizontalFlip(), RandomAffine(10, (0.1, 0.1), (0.8, 1.2), (-15, 15, -15, 15), BILINEAR, fill=127) and
RandomPerspective(0.3, p=0.3, BILINEAR, fill=127) on a PIL image, then ToTensor and Normalize.  The same Compose is
built here from torchvision (the reference is not imported) without the last two steps.  For seeded synthetic images it
stores, per case, the SHA-256 of the 224x224x3 uint8 tile after ``torch.manual_seed(torch_seed)``, its top-left 24x24
patch, and whether RandomPerspective fired.  Inputs are regenerated from the seed at test time (numpy Generator), so
only outputs are stored.  Versions at generation time are recorded in the file."""
import hashlib
import os
import sys

import numpy as np
import PIL
import PIL.Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

CASES = [  # (h, w, image seed, kind, first_resize, torch seed)
    (100, 100, 1, "noise", 512, 0),      # upscale, square
    (300, 224, 2, "stripes", 512, 1),    # upscale, short side 224
    (700, 512, 3, "noise", 512, 2),      # short side exactly 512: no resize
    (512, 512, 4, "stripes", 512, 3),    # exactly first_resize x first_resize
    (900, 1200, 5, "noise", 512, 4),
    (900, 1200, 5, "noise", 512, 5),
    (900, 1200, 6, "stripes", 512, 6),
    (3000, 4000, 7, "noise", 512, 7),
    (250, 3000, 8, "stripes", 512, 8),   # extreme aspect ratios
    (3000, 260, 9, "noise", 512, 9),
    (300, 300, 10, "noise", 224, 10),    # first_resize = 224 on a square: 224 x 224, RandomCrop draws nothing
    (224, 224, 11, "stripes", 224, 11),
    (480, 640, 12, "noise", 512, 12),
    (480, 640, 12, "noise", 512, 13),
    (640, 480, 13, "stripes", 256, 14),
    (1536, 2048, 14, "noise", 512, 15),
]


def make_image(h, w, seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    base = ((xx * 7 + yy * 3 + seed) % 256).astype(np.uint8)
    return np.stack([base, 255 - base, ((xx // 8 + yy // 8) % 2 * 255).astype(np.uint8)], axis=-1)


def train_transform(first_resize):
    """``_train_transform(first_resize, 224)`` without ToTensor / Normalize (the input is already RGB)."""
    import torchvision.transforms as T
    from torchvision.transforms import InterpolationMode
    return T.Compose([
        T.Resize([first_resize], interpolation=InterpolationMode.BICUBIC),
        T.RandomCrop([224]),
        T.RandomHorizontalFlip(),
        T.RandomAffine(degrees=10, translate=(0.1, 0.1), scale=(0.8, 1.2), shear=(-15, 15, -15, 15),
                       interpolation=InterpolationMode.BILINEAR, fill=127),
        T.RandomPerspective(distortion_scale=0.3, p=0.3, interpolation=InterpolationMode.BILINEAR, fill=127),
    ])


def main():
    import torch
    import torchvision
    import torchvision.transforms as T
    fired = []
    get_params = T.RandomPerspective.get_params

    def spy(*a, **k):
        fired.append(True)
        return get_params(*a, **k)

    T.RandomPerspective.get_params = staticmethod(spy)
    shas, patches, persp = [], [], []
    for h, w, seed, kind, first_resize, torch_seed in CASES:
        img = PIL.Image.fromarray(make_image(h, w, seed, kind))
        fired.clear()
        torch.manual_seed(torch_seed)
        tile = np.asarray(train_transform(first_resize)(img))
        assert tile.shape == (224, 224, 3) and tile.dtype == np.uint8
        shas.append(hashlib.sha256(np.ascontiguousarray(tile).tobytes()).hexdigest())
        patches.append(tile[:24, :24].copy())
        persp.append(bool(fired))
    T.RandomPerspective.get_params = get_params
    out = {"cases": np.array([c[:3] + c[4:] for c in CASES], dtype=np.int64),   # h, w, seed, first_resize, torch seed
           "kinds": np.array([c[3] for c in CASES]), "sha256": np.array(shas), "patches": np.stack(patches),
           "perspective": np.array(persp),
           "versions": np.array([f"Pillow {PIL.__version__}", f"torchvision {torchvision.__version__}",
                                 f"torch {torch.__version__}"])}
    path = os.path.join(ROOT, "tests", "golden", "train_transform_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", sum(persp), "of", len(CASES), "with a perspective warp")


if __name__ == "__main__":
    main()
