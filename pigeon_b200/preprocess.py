"""GPU replacement of the per-item CPU `CLIPProcessor(images=...)` call (reference
dataset_creation/finetune/embed_dataset.py:17-22, preprocessing/dataset_preprocessing.py:182-204,
dataset_creation/benchmark/benchmark_dataset.py:100-104): raw uint8 RGB images go to the device once (3 B/pixel) and
`pg_preprocess_clip` produces the normalised `pixel_values` there, bit-exact with Pillow BICUBIC + numpy float32.

    proc = ClipImageProcessor()                       # openai/clip-vit-large-patch14-336 settings
    px = proc(images=[pil_or_ndarray, ...], return_tensors='pt')['pixel_values']    # CUDA [n, 3, 336, 336]

Images may also be encoded files (`bytes` / `bytearray` / `memoryview`).  Baseline JPEGs are decoded on the GPU
(pigeon_b200.jpeg, one decode launch sequence per call); every other encoded file (PNG, progressive JPEG, anything the
JPEG parser does not decode) is decoded by Pillow on the host, the reference's own decoder, so the pixels are the same
either way.  `gpu_decoded` / `host_decoded` count the two routes.  A JPEG with corrupt entropy-coded data raises.
`jpeg_multiscan=True` sends progressive and multi-scan JPEGs to the GPU decoder as well (opt-in until it is measured at
least as fast as the host route on progressive photos; DESIGN.md §1).  `png=True` decodes PNGs on the GPU
(pigeon_b200.png); a PNG outside its subset, or whose stream the device refuses, is decoded by Pillow in the same call,
so pixels and exceptions are those of the default route either way.
`square_crop=True` (a keyword of the call) first cuts every decoded image to its centred square, the reference's
`BenchmarkDataset._crop_images` (benchmark_dataset.py:52-66): a strided view of a device image, a slice of a host one.
"""
from __future__ import annotations

import io
from typing import List, Sequence, Union

import numpy as np
import torch

from . import _lib, jpeg
from . import png as _png
from ._lib import PigeonB200Error, check, current_stream_ptr, load

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _to_u8_rgb(img) -> np.ndarray:
    if hasattr(img, "convert") and hasattr(img, "mode"):          # PIL.Image: do_convert_rgb
        if img.mode != "RGB":
            img = img.convert("RGB")
        img = np.asarray(img)
    if isinstance(img, torch.Tensor):
        img = img.cpu().numpy()
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"expected uint8 RGB images of shape (H, W, 3), got {img.dtype} {img.shape}")
    return np.ascontiguousarray(img)


def square_crop_box(h: int, w: int) -> tuple:
    """(h0, w0, s) of the centred square crop `image[h0:h0+s, w0:w0+s]`, with the reference's rounding
    (benchmark_dataset.py:61-64: `int((h - s) / 2)`)."""
    s = min(h, w)
    return int((h - s) / 2), int((w - s) / 2), s


def _square(img):
    """Centred square view of an [H, W, 3] array or tensor (rows keep their stride, pixels stay contiguous)."""
    h0, w0, s = square_crop_box(img.shape[0], img.shape[1])
    return img[h0:h0 + s, w0:w0 + s]


def route_encoded(data, multiscan: bool = False, png: bool = False) -> tuple:
    """('gpu', info) for a file the GPU JPEG decoder takes, ('host', info) for one Pillow decodes on the host (PNG unless
    `png`, progressive JPEG unless `multiscan`, anything else the parser does not decode); ValueError for a JPEG with
    corrupt entropy data.  With `png`, a file with the PNG signature is ('gpu', its pg_png_info) when `png.parse`
    accepts it and ('host', info) otherwise."""
    if png and _png.is_png(data):
        info, _ = _png.parse(data)
        return ("gpu" if info.status == _png.OK else "host"), info
    info, reason = jpeg.parse(data, multiscan)
    if info.status == jpeg.OK:
        return "gpu", info
    if info.status in (jpeg.UNSUPPORTED, jpeg.BAD_HEADER):
        return "host", info
    raise ValueError(f"corrupt JPEG: {reason}")


class ClipImageProcessor:
    """Call-compatible with the way the reference uses `CLIPProcessor` for images: `proc(images=..., return_tensors='pt')`
    returns a dict with 'pixel_values' (here a CUDA tensor).  `dtype=torch.float16` writes the tower's input type directly.
    `jpeg_multiscan=True` decodes encoded progressive and multi-scan JPEGs on the GPU instead of with Pillow, `png=True`
    encoded PNGs (the ones the device refuses are still decoded by Pillow, and counted in `host_decoded`).
    `proc(images, square_crop=True)` cuts each image to its centred square before the resize (BenchmarkDataset)."""

    def __init__(self, size: int = 336, image_mean: Sequence[float] = CLIP_MEAN, image_std: Sequence[float] = CLIP_STD,
                 device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float32,
                 jpeg_multiscan: bool = False, png: bool = False):
        self.size = int(size)
        self.jpeg_multiscan = bool(jpeg_multiscan)
        self.png = bool(png)
        self.mean = np.asarray(image_mean, dtype=np.float64).astype(np.float32)
        self.std = np.asarray(image_std, dtype=np.float64).astype(np.float32)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise PigeonB200Error("ClipImageProcessor runs on a CUDA device only (no CPU path)")
        if dtype not in (torch.float32, torch.float16):
            raise ValueError("dtype must be float32 or float16")
        self.dtype = dtype
        self._lib = load()
        self._ws = None
        self._jpeg = None
        self._png = None
        self.gpu_decoded = 0
        self.host_decoded = 0

    def preprocess_device(self, images_u8: List[torch.Tensor]) -> torch.Tensor:
        """images_u8: CUDA uint8 tensors [H, W, 3] (any sizes, rows may be strided) -> [n, 3, size, size]."""
        n = len(images_u8)
        desc = (_lib.Image * n)()
        for i, t in enumerate(images_u8):
            if not t.is_cuda or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 or t.stride(2) != 1 or t.stride(1) != 3:
                raise ValueError("images must be CUDA uint8 [H, W, 3] tensors with contiguous pixels")
            desc[i] = _lib.Image(t.data_ptr(), t.shape[0], t.shape[1], t.stride(0))
        need = int(self._lib.pg_preprocess_workspace_bytes(desc, n, self.size))
        if need == 0:
            raise PigeonB200Error(f"pg_preprocess_workspace_bytes: {self._lib.pg_last_error().decode()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        out = torch.empty((n, 3, self.size, self.size), dtype=self.dtype, device=self.device)
        check(self._lib.pg_preprocess_clip(desc, n, self.size, self.mean.ctypes.data, self.std.ctypes.data,
                                           self._ws.data_ptr(), self._ws.numel(), out.data_ptr(),
                                           int(self.dtype == torch.float16), current_stream_ptr()), "pg_preprocess_clip")
        return out

    def __call__(self, images=None, return_tensors: str = "pt", square_crop: bool = False, **kwargs):
        if images is None:
            raise ValueError("You have to specify images.")
        if not isinstance(images, (list, tuple)):
            images = [images]
        dev = [None] * len(images)
        gpu_idx, gpu_files, gpu_infos = [], [], []
        png_idx, png_files, png_infos = [], [], []
        for i, img in enumerate(images):
            if isinstance(img, torch.Tensor) and img.is_cuda:
                dev[i] = _square(img) if square_crop else img
                continue
            if isinstance(img, (bytes, bytearray, memoryview)):
                try:
                    route, info = route_encoded(img, self.jpeg_multiscan, self.png)
                except ValueError as e:
                    raise ValueError(f"image {i}: {e}") from None
                if route == "gpu" and isinstance(info, _lib.PngInfo):
                    png_idx.append(i)
                    png_files.append(img)
                    png_infos.append(info)
                    continue
                if route == "gpu":
                    gpu_idx.append(i)
                    gpu_files.append(img)
                    gpu_infos.append(info)
                    continue
                from PIL import Image
                img = Image.open(io.BytesIO(bytes(img)))
                self.host_decoded += 1
            a = _to_u8_rgb(img)
            if square_crop:
                a = np.ascontiguousarray(_square(a))
            dev[i] = torch.from_numpy(a).pin_memory().to(self.device, non_blocking=True)
        if gpu_files:
            if self._jpeg is None:
                self._jpeg = jpeg.JpegDecoder(self.device)
            for i, t in zip(gpu_idx, self._jpeg.decode(gpu_files, gpu_infos)):
                dev[i] = _square(t) if square_crop else t
            self.gpu_decoded += len(gpu_files)
        if png_files:
            if self._png is None:
                self._png = _png.PngDecoder(self.device)
            try:
                decoded = self._png.decode(png_files, png_infos)
            except _png.PngDecodeError as e:
                decoded = e.images
            from PIL import Image
            for i, f, t in zip(png_idx, png_files, decoded):
                if t is None:                                 # refused by the device: Pillow, as without `png`
                    img = Image.open(io.BytesIO(bytes(f)))
                    self.host_decoded += 1
                    a = _to_u8_rgb(img)
                    if square_crop:
                        a = np.ascontiguousarray(_square(a))
                    t = torch.from_numpy(a).pin_memory().to(self.device, non_blocking=True)
                else:
                    self.gpu_decoded += 1
                    if square_crop:
                        t = _square(t)
                dev[i] = t
        return {"pixel_values": self.preprocess_device(dev)}
