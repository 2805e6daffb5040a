"""The reference's train-time transform (``_train_transform(512, 224)``, the OpenPath preprocess) on one GPU, at a
user-sized batch, against torchvision on PIL on the same host in the same call:

  - device tiles/s: resize + crop (``plip_resize_crop_u8``) and flip / affine / perspective (``plip_warp_tiles_u8``) of
    sources already in device memory, for 1200 x 900 and 2048 x 1536 images, timed with CUDA events (the warp alone
    too);
  - end to end: normalised embeddings/s of ``CLIPEmbedder(model, TrainTransform()).embed_images`` on decoded images
    held in host memory (random draws, packing, upload, resize, warps and the image tower), host clock around a
    device synchronise;
  - the reference's arm: torchvision's Compose with ToTensor and Normalize on PIL images in a ``DataLoader`` with the
    same number of worker processes;
  - host JPEG decode (Pillow) of the same images on the same number of threads, which bounds the end-to-end rate from
    files: decoding stays on the host.

Prints the card name and power limit with the numbers.  Synthetic seeded images and weights.  GPU only.

    python tools/train_transform_probe.py [out.json] [--batch 256] [--threads 8]
"""
import io
import json
import os
import sys
import time
import types

import numpy as np
import PIL.Image
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from densenet_probe import timed  # noqa: E402
from region_probe import card  # noqa: E402

SOURCES = [(1200, 900), (2048, 1536)]


def images(w, h, n, seed=0):
    """n smooth-ish RGB images (noise on a gradient, so JPEG sizes are realistic rather than worst case)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // w), (yy * 255 // h), ((xx + yy) * 127 // (w + h))], -1).astype(np.int16)
    out = []
    for i in range(n):
        noise = rng.integers(-24, 25, (h, w, 3), dtype=np.int16)
        out.append(np.clip(np.roll(base, 37 * i, axis=1) + noise, 0, 255).astype(np.uint8))
    return out


class _TorchvisionArm(torch.utils.data.Dataset):
    def __init__(self, arrays):
        self.arrays = arrays

    def __len__(self):
        return len(self.arrays)

    def __getitem__(self, i):
        import torchvision.transforms as T
        from torchvision.transforms import InterpolationMode as IM
        tf = T.Compose([T.Resize([512], interpolation=IM.BICUBIC), T.RandomCrop([224]), T.RandomHorizontalFlip(),
                        T.RandomAffine(degrees=10, translate=(0.1, 0.1), scale=(0.8, 1.2), shear=(-15, 15, -15, 15),
                                       interpolation=IM.BILINEAR, fill=127),
                        T.RandomPerspective(distortion_scale=0.3, p=0.3, interpolation=IM.BILINEAR, fill=127),
                        T.ToTensor(), T.Normalize((0.48145466, 0.4578275, 0.40821073),
                                                  (0.26862954, 0.26130258, 0.27577711))])
        return tf(PIL.Image.fromarray(self.arrays[i]))


def main():
    if not torch.cuda.is_available():
        sys.exit("train_transform_probe: needs a CUDA device")
    args = sys.argv[1:]
    opt = {k: int(args[args.index(k) + 1]) for k in ("--batch", "--threads") if k in args}
    batch, threads = opt.get("--batch", 256), opt.get("--threads", min(8, os.cpu_count() or 1))
    out_path = next((a for i, a in enumerate(args) if not a.startswith("--") and (i == 0 or not args[i - 1].startswith("--"))), None)
    torch.set_grad_enabled(False)
    from oracle import weights
    from plip_b200.embedders import CLIPEmbedder
    from plip_b200.engine import Engine, resize_crop, warp_tiles
    from plip_b200.preprocess import TrainTransform, decode_rgb, pack_rgb
    res = {"card": card(), "batch": batch, "host_threads": threads, "host_cpus": os.cpu_count()}
    tt = TrainTransform()
    eng = Engine(weights.make_state_dict(0), max_micro_batch=batch)
    model = types.SimpleNamespace(engine=eng, encode_image=eng.encode_images)
    emb = CLIPEmbedder(model, tt, "plip", "synthetic")
    for w, h in SOURCES:
        key = f"{w}x{h}"
        uniq = images(w, h, 16, seed=w)
        arrays = [uniq[i % len(uniq)] for i in range(batch)]
        torch.manual_seed(0)
        t0 = time.perf_counter()
        params = tt.draw([(w, h)] * batch, num_workers=threads, batch_size=batch // threads or 1)
        res[f"{key}_host_draws_per_s"] = batch / (time.perf_counter() - t0)
        res[f"{key}_perspective_share"] = float(params["warp"]["apply_perspective"].mean())
        buf, descs = pack_rgb(arrays, pinned=True, plan=params)
        src = buf.cuda()
        tiles = torch.empty((batch, 224, 224, 3), dtype=torch.uint8, device="cuda")

        def device_route():
            resize_crop(src, descs, out=tiles)
            warp_tiles(tiles, params["warp"], out=tiles)

        t = timed(device_route)
        res[f"{key}_device_tiles_per_s"] = batch / t
        t = timed(lambda: warp_tiles(tiles, params["warp"], out=tiles))
        res[f"{key}_warp_only_tiles_per_s"] = batch / t

        def end_to_end():
            emb.embed_images(arrays, num_workers=threads, batch_size=batch)
            torch.cuda.synchronize()

        end_to_end()
        reps, t0 = 3, time.perf_counter()
        for _ in range(reps):
            end_to_end()
        res[f"{key}_end_to_end_embeddings_per_s"] = reps * batch / (time.perf_counter() - t0)

        n_tv = max(4 * threads, 32)
        dl = torch.utils.data.DataLoader(_TorchvisionArm(arrays[:n_tv]), batch_size=max(1, n_tv // threads),
                                         num_workers=threads, persistent_workers=True)
        for _ in dl:                                    # worker start-up and imports outside the window
            pass
        t0 = time.perf_counter()
        for _ in dl:
            pass
        res[f"{key}_torchvision_images_per_s"] = n_tv / (time.perf_counter() - t0)

        jpegs = []
        for a in uniq:
            b = io.BytesIO()
            PIL.Image.fromarray(a).save(b, format="JPEG", quality=90)
            jpegs.append(b.getvalue())
        files = [io.BytesIO(jpegs[i % len(jpegs)]) for i in range(batch)]
        t0 = time.perf_counter()
        decode_rgb([PIL.Image.open(f) for f in files], threads)
        res[f"{key}_jpeg_decode_per_s"] = batch / (time.perf_counter() - t0)
        res[f"{key}_jpeg_bytes_mean"] = float(np.mean([len(j) for j in jpegs]))
        res[f"{key}_speedup_end_to_end_vs_torchvision"] = (res[f"{key}_end_to_end_embeddings_per_s"]
                                                          / res[f"{key}_torchvision_images_per_s"])
    print(json.dumps(res, indent=1))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
