"""Baseline JPEG decoding on the GPU (csrc/jpeg.cu), byte-identical to `np.asarray(PIL.Image.open(f).convert('RGB'))`
for the files it decodes: what the reference does on the CPU before every CLIPProcessor call
(dataset_creation/finetune/embed_dataset.py:17-22, dataset_creation/benchmark/benchmark_dataset.py:66-79,
pretrain_dataset.py:109-161).

    imgs = decode_jpeg([open(p, 'rb').read() for p in paths], 'cuda')     # CUDA uint8 [H, W, 3] views into one arena

The headers are parsed on the host (`parse`); the compressed bytes of the whole batch go to the device in one copy and
three or four launches decode them (a long entropy-coded segment, such as a photo without restart markers, is decoded
by a whole CTA in self-synchronising chunks).  Files outside the decoded subset (progressive, 12-bit, CMYK,
RGB-transform, other sampling layouts) and corrupt files raise `ValueError` naming every such index and its reason.

With `multiscan=True`, progressive files and sequential files of several scans are decoded too, to the same bytes as
Pillow, when every coefficient is sent and fully refined (what encoders write; libjpeg smooths the blocks of the other
ones, which are refused).  Their scans decode in one launch per dependency level (`scans(data)` lists them).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, load

OK, UNSUPPORTED, BAD_HEADER, BAD_CODE, OVERRUN, UNEXPECTED_MARKER, BAD_RST, NO_EOI = range(8)
MULTISCAN = 1 << 12          # PG_JPEG_MULTISCAN
MAX_SCANS = 256              # PG_JPEG_MAX_SCANS
STATUS_TEXT = {OK: "ok", UNSUPPORTED: "not decoded by this decoder", BAD_HEADER: "truncated or inconsistent header",
               BAD_CODE: "corrupt entropy data: code missing from its Huffman table",
               OVERRUN: "corrupt entropy data: a segment ends before its MCUs",
               UNEXPECTED_MARKER: "corrupt entropy data: marker where data should be",
               BAD_RST: "corrupt entropy data: wrong restart marker", NO_EOI: "corrupt entropy data: no EOI"}

Encoded = Union[bytes, bytearray, memoryview]


class JpegDecodeError(ValueError):
    """Some files of a batch were not decoded.  `failed` maps each such index to its reason; `images` holds the decoded
    images of the others (None at the failed indices)."""

    def __init__(self, failed: dict, images: list):
        super().__init__("JPEG files not decoded: " + "; ".join(f"#{i}: {r}" for i, r in sorted(failed.items())))
        self.failed = failed
        self.images = images


def parse(data: Encoded, multiscan: bool = False) -> Tuple[_lib.JpegInfo, str]:
    """Host marker walk of one file: its `pg_jpeg_info` and, when its status is not OK, the reason.  `multiscan` also
    accepts progressive and multi-scan sequential files (pg_jpeg_parse_multiscan); a single-scan file gets the same
    info either way."""
    lib = load()
    buf = bytes(data)
    info = _lib.JpegInfo()
    fn = lib.pg_jpeg_parse_multiscan if multiscan else lib.pg_jpeg_parse
    st = fn(buf, len(buf), C.byref(info))
    return info, ("" if st == OK else lib.pg_last_error().decode())


def is_multiscan(info: _lib.JpegInfo) -> bool:
    """True for the info of a progressive or multi-scan file (the PG_JPEG_MULTISCAN bit of table_mask)."""
    return bool(info.table_mask & MULTISCAN)


def scans(data: Encoded) -> List[_lib.JpegScan]:
    """The scans of a file that `parse(data, multiscan=True)` accepts, in file order: components, Ss, Se, Ah, Al,
    restart interval, segment count and dependency level.  ValueError with the reason for a refused file."""
    lib = load()
    buf = bytes(data)
    out = (_lib.JpegScan * MAX_SCANS)()
    n = lib.pg_jpeg_scans(buf, len(buf), out, MAX_SCANS)
    if n < 0:
        raise ValueError(lib.pg_last_error().decode())
    return list(out[:n])


def set_schedule(mode: int, chunk_bytes: int = 0) -> None:
    """Huffman-decode kernel of single-scan segments, process-wide (pg_jpeg_set_schedule): 0 = automatic, 1 = one thread
    per segment, 2 = chunked for every segment; `chunk_bytes` > 0 forces the chunk size.  For tests and A/B benchmarks:
    every schedule gives the same bytes."""
    check(load().pg_jpeg_set_schedule(int(mode), int(chunk_bytes)), "pg_jpeg_set_schedule")


def entropy_host(files: Sequence[Encoded], chunk_bytes: int = 0):
    """The entropy decode of single-scan files on the CPU (pg_jpeg_entropy_host): chunk_bytes 0 = one pass per segment,
    > 0 = the chunked decoder at that chunk size, < 0 = at the automatic size.  Returns (int16 coefficient blocks
    [blocks, 64] of the parsed-OK files in order, status per file, synchronisation rounds per file)."""
    lib = load()
    bufs = [bytes(f) for f in files]
    n = len(bufs)
    infos = (_lib.JpegInfo * n)(*[parse(b)[0] for b in bufs])
    packed = np.frombuffer(b"".join(bufs), dtype=np.uint8)
    offsets = np.concatenate([[0], np.cumsum([len(b) for b in bufs])]).astype(np.int64)
    status = np.zeros(n, dtype=np.int32)
    rounds = np.zeros(n, dtype=np.int32)
    nblocks = 0
    for i in infos:
        if i.status == OK:
            three = i.components == 3
            hmax, vmax = (i.h_samp[0], i.v_samp[0]) if three else (1, 1)
            mcus = -(-i.width // (8 * hmax)) * -(-i.height // (8 * vmax))
            nblocks += mcus * (sum(i.h_samp[c] * i.v_samp[c] for c in range(3)) if three else 1)
    coef = np.zeros((nblocks, 64), dtype=np.int16)
    got = lib.pg_jpeg_entropy_host(packed.ctypes.data, offsets.ctypes.data, infos, n, chunk_bytes, coef.ctypes.data,
                                   status.ctypes.data, rounds.ctypes.data)
    if got != nblocks:
        raise PigeonB200Error(f"pg_jpeg_entropy_host: {lib.pg_last_error().decode() if got < 0 else got}")
    return coef, status, rounds


class JpegDecoder:
    """Reusable batch decoder: keeps its device workspace and pinned staging buffer between calls."""

    def __init__(self, device: Union[str, torch.device] = "cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise PigeonB200Error("JpegDecoder runs on a CUDA device only (no CPU path)")
        self._lib = load()
        self._ws = None
        self._pinned = None        # staging of the compressed bytes; free again once the status has been read back

    def decode(self, files: Sequence[Encoded], infos: Sequence[_lib.JpegInfo] = None,
               multiscan: bool = False) -> List[torch.Tensor]:
        """files -> CUDA uint8 [H, W, 3] views into one arena (Pillow's `.convert('RGB')` bytes).  `infos` are the
        `parse` results when the caller already has them (multi-scan infos are decoded whatever `multiscan` says);
        otherwise the files are parsed with `parse(f, multiscan)`.  Raises JpegDecodeError (a ValueError) listing every
        rejected or corrupt index; the other files of the batch are still decoded."""
        n = len(files)
        if n == 0:
            return []
        bufs = [memoryview(f).cast("B") for f in files]
        if infos is None:
            parsed = [parse(b, multiscan) for b in bufs]
            infos = [p[0] for p in parsed]
            reasons = [p[1] for p in parsed]
        else:
            reasons = [STATUS_TEXT.get(i.status, "") for i in infos]
        info_arr = (_lib.JpegInfo * n)(*infos)
        offsets = np.zeros(n + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([len(b) for b in bufs])
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
        need = int(self._lib.pg_jpeg_workspace_bytes(info_arr, n, total))
        if need == 0:
            raise PigeonB200Error(f"pg_jpeg_workspace_bytes: {self._lib.pg_last_error().decode()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        status = torch.empty(n, dtype=torch.int32, device=self.device)
        check(self._lib.pg_jpeg_decode(self._pinned.data_ptr(), offsets.ctypes.data, info_arr, n, desc,
                                       self._ws.data_ptr(), self._ws.numel(), status.data_ptr(), current_stream_ptr()),
              "pg_jpeg_decode")
        st = status.cpu().numpy()                             # synchronises: the pinned buffer is free again
        images = [arena[int(starts[i]):int(starts[i]) + sizes[i]].view(int(infos[i].height), int(infos[i].width), 3)
                  if st[i] == OK else None for i in range(n)]
        failed = {i: (reasons[i] if infos[i].status != OK and reasons[i] else STATUS_TEXT.get(int(s), f"status {int(s)}"))
                  for i, s in enumerate(st) if s != OK}
        if failed:
            raise JpegDecodeError(failed, images)
        return images


def decode_jpeg(files: Sequence[Encoded], device: Union[str, torch.device] = "cuda",
                multiscan: bool = False) -> List[torch.Tensor]:
    """One-shot `JpegDecoder(device).decode(files, multiscan=multiscan)`."""
    return JpegDecoder(device).decode(files, multiscan=multiscan)
