"""Generate tests/golden/densenet_golden.npz from live torchvision:

    python tests/golden/make_densenet_golden.py

The reference's MuDiPath embedder (``reproducibility/embedders/factory.py:34-47``, ``mudipath.py:125-130``):
torchvision ``densenet121()`` loaded with the seeded synthetic weights of ``tests/densenet_oracle.make_state_dict(0)``,
run as ``F.adaptive_avg_pool2d(model.features(x), (1, 1))`` in eval mode, fp32 on the CPU, on
``Resize(224) + CenterCrop(224) + ToTensor + Normalize`` of a few synthetic RGB sources (one already 224 x 224, one
shrunk, one enlarged).  Stored: the sources (``src<i>``), the uint8 tiles that transform produces before ``ToTensor``,
the ``[n,1024]`` outputs and the sha256 of the weights (``densenet_oracle.checksum``).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import densenet_oracle as O  # noqa: E402

SOURCES = [(224, 224), (240, 233), (120, 170)]   # (height, width)


def source(i, h, w):
    """A synthetic RGB image: plane waves posterised to 16 levels, so that the file compresses well."""
    rng = np.random.default_rng(100 + i)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w, 3))
    for c in range(3):
        for _ in range(4):
            fy, fx, ph = rng.uniform(0.01, 0.12), rng.uniform(0.01, 0.12), rng.uniform(0, 6.3)
            img[..., c] += 30 * np.sin(fy * yy + fx * xx + ph)
    img += 128
    return (np.clip(img, 0, 255).astype(np.uint8) // 16 * 16 + 8).astype(np.uint8)


def main():
    import PIL.Image
    import torch
    import torch.nn.functional as F
    import torchvision
    from torchvision import transforms

    sd = O.make_state_dict(0)
    model = torchvision.models.densenet121()
    model.load_state_dict(sd)
    model.eval()
    crop = transforms.Compose([transforms.Resize(224), transforms.CenterCrop(224)])
    norm = transforms.Compose([transforms.ToTensor(),
                               transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    out = {"weights_sha256": np.array(O.checksum(sd)), "torchvision_version": np.array(torchvision.__version__)}
    tiles, xs = [], []
    for i, (h, w) in enumerate(SOURCES):
        src = source(i, h, w)
        out[f"src{i}"] = src
        tile = crop(PIL.Image.fromarray(src))
        tiles.append(np.asarray(tile))
        xs.append(norm(tile))
    with torch.no_grad():
        y = F.adaptive_avg_pool2d(model.features(torch.stack(xs)), (1, 1)).flatten(1)
    out["tiles"] = np.stack(tiles)
    out["outputs"] = y.numpy().astype(np.float32)
    path = os.path.join(ROOT, "tests", "golden", "densenet_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
