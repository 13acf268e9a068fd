#!/usr/bin/env python
"""Writes tests/golden/benchmark.npz: encoded benchmark images and the pixel_values the reference's BenchmarkDataset
gives them (dataset_creation/benchmark/benchmark_dataset.py:52-106), for the GPU tests of pigeon_b200.benchmark.
Made with Pillow 12.2.0 over libjpeg-turbo 3.1.

The expected pixels restate the reference per item: `_load_jpg` (`Image.open(f).convert('RGB')`, float32 / 255, first
three channels), `_crop_images` (centred square, `int((h - s) / 2)`), then CLIPProcessor.  transformers 4.23.1 turns the
float crop back into uint8 as `(x * 255).astype(uint8)` before its resize; `oracle.preprocess.clip_preprocess` does the
rest (Pillow-exact bicubic resize to 336, centre crop, normalisation).

Per case k: `name[k]`, `route[k]` ('gpu' for a file the GPU JPEG decoder takes, 'host' for one Pillow decodes),
`size[k]` (H, W) of the decoded image, the file `data[off[k]:off[k+1]]`, and the float32 [3, 336, 336] pixel_values as
`sha{k}` (SHA-256 of their bytes) and `sample{k}` (pixel_values[:, ::17, ::13]).
"""
import hashlib
import io
import os
import sys

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.preprocess import clip_preprocess  # noqa: E402
from pigeon_b200 import synthetic  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "benchmark.npz")


def encode(img: Image.Image, fmt: str, **kw) -> bytes:
    f = io.BytesIO()
    img.save(f, fmt, **kw)
    return f.getvalue()


def cases():
    """(name, route, file bytes): seeded photo-like content at the sizes the crop and the resize must get right."""
    def photo(h, w, seed):
        return Image.fromarray(synthetic.synthetic_photo(h, w, seed))
    out = []
    for k, (h, w) in enumerate([(333, 500), (500, 333), (336, 337), (1, 1), (1, 57), (57, 1), (120, 90), (90, 121),
                                (520, 390)]):
        out.append((f"420 q90 {h}x{w}", "gpu", encode(photo(h, w, k), "JPEG", quality=90, subsampling=2)))
    out.append(("444 q90 241x338", "gpu", encode(photo(241, 338, 20), "JPEG", quality=90, subsampling=0)))
    out.append(("gray q85 350x249", "gpu", encode(photo(350, 249, 21).convert("L"), "JPEG", quality=85)))
    out.append(("420 restart 377x501", "gpu", encode(photo(377, 501, 22), "JPEG", quality=88, restart_marker_blocks=3)))
    out.append(("420 progressive 333x500", "host",
                encode(photo(333, 500, 23), "JPEG", quality=90, progressive=True)))
    out.append(("cmyk q90 120x181", "host", encode(photo(120, 181, 24).convert("CMYK"), "JPEG", quality=90)))
    out.append(("png rgb 143x201", "host", encode(photo(143, 201, 25), "PNG")))
    rgba = photo(70, 111, 26).convert("RGBA")
    rgba.putalpha(Image.fromarray((np.arange(70 * 111) % 256).astype(np.uint8).reshape(70, 111)))
    out.append(("png rgba 70x111", "host", encode(rgba, "PNG")))
    out.append(("png p 101x77", "host", encode(photo(101, 77, 27).convert("P"), "PNG")))
    out.append(("png l 1x40", "host", encode(photo(1, 40, 28).convert("L"), "PNG")))
    out.append(("png l 90x61", "host", encode(photo(90, 61, 29).convert("L"), "PNG")))
    return out


def reference_pixel_values(data: bytes) -> np.ndarray:
    """BenchmarkDataset.__getitem__ restated: _load_jpg, _crop_images, then CLIPProcessor (4.23.1) on the float crop."""
    image = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"), dtype=np.float32) / 255
    image = image[:, :, :3]
    s = np.min(image.shape[:2])
    h_start = int((image.shape[0] - s) / 2)
    w_start = int((image.shape[1] - s) / 2)
    center = image[h_start: h_start + s, w_start:w_start + s]
    u8 = (center * 255).astype(np.uint8)              # transformers 4.23.1 to_pil_image(rescale=True)
    return clip_preprocess(np.ascontiguousarray(u8))


def main():
    cs = cases()
    blobs = [d for _, _, d in cs]
    off = np.concatenate([[0], np.cumsum([len(b) for b in blobs])]).astype(np.int64)
    arrays = dict(name=np.array([n for n, _, _ in cs]), route=np.array([r for _, r, _ in cs]),
                  data=np.frombuffer(b"".join(blobs), dtype=np.uint8), off=off, count=np.int64(len(cs)),
                  size=np.array([Image.open(io.BytesIO(b)).size[::-1] for b in blobs], dtype=np.int64))
    for k, b in enumerate(blobs):
        px = reference_pixel_values(b)
        arrays[f"sha{k}"] = np.frombuffer(hashlib.sha256(px.tobytes()).digest(), dtype=np.uint8)
        arrays[f"sample{k}"] = px[:, ::17, ::13].copy()
    np.savez_compressed(OUT, **arrays)
    print(f"{OUT}: {len(cs)} files, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
