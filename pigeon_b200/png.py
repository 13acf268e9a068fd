"""PNG decoding on the GPU (csrc/png.cu), byte-identical to `np.asarray(PIL.Image.open(f).convert('RGB'))` for the
files it decodes: what the reference does on the CPU before every CLIPProcessor call, for the PNGs of user-supplied
benchmark and holdout folders.

    imgs = decode_png([open(p, 'rb').read() for p in paths], 'cuda')      # CUDA uint8 [H, W, 3] views into one arena

The chunks are walked on the host (`parse`); the files of a batch go to the device in one copy and three launches
decode them: inflate (one warp per zlib stream), row unfiltering and the RGB conversion.  Non-interlaced files of every
colour type and bit depth are decoded.  Interlaced files, APNG, IDAT chunks that are not consecutive, CRC errors before
the first IDAT, text above Pillow's limits and images above `PIL.Image.MAX_IMAGE_PIXELS` are refused by `parse`, and a
stream the device does not accept fails its file alone; `PngDecoder.decode` raises `PngDecodeError` naming every such
index and its reason, with the other images of the batch decoded.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, load

OK, UNSUPPORTED, BAD_HEADER, BAD_ZLIB, BAD_DEFLATE, TRUNCATED, TOO_LONG, BAD_FILTER = range(8)
SIGNATURE = b"\x89PNG\r\n\x1a\n"
STATUS_TEXT = {OK: "ok", UNSUPPORTED: "not decoded by this decoder", BAD_HEADER: "not a PNG, or a bad header chunk",
               BAD_ZLIB: "zlib stream: bad header or Adler-32, or bytes after the stream",
               BAD_DEFLATE: "zlib stream: invalid block, code or distance",
               TRUNCATED: "zlib stream: ends early or is shorter than the image",
               TOO_LONG: "zlib stream: more data after the image than the decoder accepts",
               BAD_FILTER: "row filter type above 4"}

Encoded = Union[bytes, bytearray, memoryview]


class PngDecodeError(ValueError):
    """Some files of a batch were not decoded.  `failed` maps each such index to its reason; `images` holds the decoded
    images of the others (None at the failed indices)."""

    def __init__(self, failed: dict, images: list):
        super().__init__("PNG files not decoded: " + "; ".join(f"#{i}: {r}" for i, r in sorted(failed.items())))
        self.failed = failed
        self.images = images


def is_png(data: Encoded) -> bool:
    return bytes(memoryview(data)[:8]) == SIGNATURE


def parse(data: Encoded) -> Tuple[_lib.PngInfo, str]:
    """Host chunk walk of one file: its `pg_png_info` and, when its status is not OK, the reason.  A file of more
    pixels than `PIL.Image.MAX_IMAGE_PIXELS` (read at each call) is UNSUPPORTED, so that Pillow's own warning or error
    applies to it."""
    lib = load()
    buf = bytes(data)
    info = _lib.PngInfo()
    st = lib.pg_png_parse(buf, len(buf), C.byref(info))
    if st != OK:
        return info, lib.pg_last_error().decode()
    from PIL import Image
    limit = Image.MAX_IMAGE_PIXELS
    if limit is not None and info.width * info.height > limit:
        info.status = UNSUPPORTED
        return info, f"{info.width * info.height} pixels > PIL.Image.MAX_IMAGE_PIXELS"
    return info, ""


def _pack(bufs):
    offsets = np.zeros(len(bufs) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(b) for b in bufs])
    return offsets


def decode_host(files: Sequence[Encoded]):
    """The decode of pg_png_decode on the CPU (pg_png_decode_host), for tests: (uint8 [H, W, 3] arrays, None where the
    status is not OK; status per file)."""
    lib = load()
    bufs = [bytes(f) for f in files]
    n = len(bufs)
    infos = [parse(b)[0] for b in bufs]
    info_arr = (_lib.PngInfo * n)(*infos)
    packed = np.frombuffer(b"".join(bufs) or b"\0", dtype=np.uint8)
    offsets = _pack(bufs)
    sizes = [3 * i.width * i.height if i.status == OK else 0 for i in infos]
    rgb = np.zeros(max(sum(sizes), 1), dtype=np.uint8)
    status = np.zeros(n, dtype=np.int32)
    got = lib.pg_png_decode_host(packed.ctypes.data, offsets.ctypes.data, info_arr, n, rgb.ctypes.data,
                                 status.ctypes.data)
    if got != sum(sizes):
        raise PigeonB200Error(f"pg_png_decode_host: {lib.pg_last_error().decode() if got < 0 else got}")
    out, at = [], 0
    for i, s in zip(infos, sizes):
        out.append(rgb[at:at + s].reshape(i.height, i.width, 3).copy() if s else None)
        at += s
    return [o if st == OK else None for o, st in zip(out, status)], status


class PngDecoder:
    """Reusable batch decoder: keeps its device workspace and pinned staging buffer between calls."""

    def __init__(self, device: Union[str, torch.device] = "cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise PigeonB200Error("PngDecoder runs on a CUDA device only (no CPU path)")
        self._lib = load()
        self._ws = None
        self._pinned = None        # staging of the files' bytes; free again once the status has been read back

    def decode(self, files: Sequence[Encoded], infos: Sequence[_lib.PngInfo] = None) -> List[torch.Tensor]:
        """files -> CUDA uint8 [H, W, 3] views into one arena (Pillow's `.convert('RGB')` bytes).  `infos` are the
        `parse` results when the caller already has them.  Raises PngDecodeError (a ValueError) listing every refused
        or failed index; the other files of the batch are still decoded."""
        n = len(files)
        if n == 0:
            return []
        bufs = [memoryview(f).cast("B") for f in files]
        if infos is None:
            parsed = [parse(b) for b in bufs]
            infos = [p[0] for p in parsed]
            reasons = [p[1] for p in parsed]
        else:
            reasons = [STATUS_TEXT.get(i.status, "") for i in infos]
        info_arr = (_lib.PngInfo * n)(*infos)
        offsets = _pack(bufs)
        total = int(offsets[-1])
        if self._pinned is None or self._pinned.numel() < total:
            self._pinned = torch.empty(max(total, 1 << 20), dtype=torch.uint8, pin_memory=True)
        staging = self._pinned.numpy()
        for i, b in enumerate(bufs):
            staging[offsets[i]:offsets[i + 1]] = np.frombuffer(b, dtype=np.uint8)
        sizes = [int(i.height) * int(i.width) * 3 if i.status == OK else 0 for i in infos]
        starts = np.zeros(n + 1, dtype=np.int64)
        starts[1:] = np.cumsum([(s + 255) // 256 * 256 for s in sizes])
        arena = torch.empty(int(starts[-1]), dtype=torch.uint8, device=self.device)
        base = arena.data_ptr()
        desc = (_lib.Image * n)()
        for i, inf in enumerate(infos):
            if inf.status == OK:
                desc[i] = _lib.Image(base + int(starts[i]), inf.height, inf.width, 3 * inf.width)
        need = int(self._lib.pg_png_workspace_bytes(info_arr, n, total))
        if need == 0:
            raise PigeonB200Error(f"pg_png_workspace_bytes: {self._lib.pg_last_error().decode()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        status = torch.empty(n, dtype=torch.int32, device=self.device)
        check(self._lib.pg_png_decode(self._pinned.data_ptr(), offsets.ctypes.data, info_arr, n, desc,
                                      self._ws.data_ptr(), self._ws.numel(), status.data_ptr(), current_stream_ptr()),
              "pg_png_decode")
        st = status.cpu().numpy()                             # synchronises: the pinned buffer is free again
        images = [arena[int(starts[i]):int(starts[i]) + sizes[i]].view(int(infos[i].height), int(infos[i].width), 3)
                  if st[i] == OK else None for i in range(n)]
        failed = {i: (reasons[i] if infos[i].status != OK and reasons[i] else STATUS_TEXT.get(int(s), f"status {int(s)}"))
                  for i, s in enumerate(st) if s != OK}
        if failed:
            raise PngDecodeError(failed, images)
        return images


def decode_png(files: Sequence[Encoded], device: Union[str, torch.device] = "cuda") -> List[torch.Tensor]:
    """One-shot `PngDecoder(device).decode(files)`."""
    return PngDecoder(device).decode(files)
