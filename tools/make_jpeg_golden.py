#!/usr/bin/env python
"""Writes tests/golden/jpeg.npz: JPEG files and what Pillow decodes them to (`np.asarray(Image.open(f).convert('RGB'))`),
for the GPU decoder's tests, which must not need Pillow.  Made with Pillow 12.2.0 over libjpeg-turbo 3.1.4.1.

Per case k: `name[k]` describes it, `kind[k]` is 'ok', 'reject' or 'corrupt', `status[k]` the expected PG_JPEG_* status,
`jpg[jpg_off[k]:jpg_off[k+1]]` the file's bytes.  Decoded files and the progressive one have `shape[k]` (H, W, 3) and
either their full pixels `px[px_off[k]:px_off[k+1]]` or, above FULL_PIXELS pixels, `sha{k}` (SHA-256 of the pixels) and
`sample{k}` (pixels[::37, ::23]).
"""
import hashlib
import io
import os
import sys

import numpy as np
from PIL import Image, features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pigeon_b200 import synthetic  # noqa: E402

OK, UNSUPPORTED, BAD_HEADER, BAD_CODE, OVERRUN, BAD_RST, NO_EOI = 0, 1, 2, 3, 4, 6, 7
SUB = {0: "444", 1: "422", 2: "420"}
FULL_PIXELS = 4096          # larger decodes are stored as SHA-256 + samples


def enc(img, **kw):
    f = io.BytesIO()
    Image.fromarray(img).save(f, "JPEG", **kw)
    return f.getvalue()


def smooth(h, w):
    """Gradients and saturated blocks without noise: a large image that compresses small."""
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) // 7) % 256], -1)
    img[h // 4:h // 2, w // 4:w // 2] = 255
    img[h // 2:3 * h // 4, w // 2:3 * w // 4] = 0
    return img.astype(np.uint8)


def segments(b):
    """(marker, start, end) of each marker segment before the first scan."""
    out, p = [], 2
    while True:
        m = b[p + 1]
        L = b[p + 2] << 8 | b[p + 3]
        out.append((m, p, p + 2 + L))
        if m == 0xDA:
            return out
        p += 2 + L


def drop_app0(b):
    for m, s, e in segments(b):
        if m == 0xE0:
            return b[:s] + b[e:]
    return b


def edit_sof(b, off, value):
    for m, s, e in segments(b):
        if m in (0xC0, 0xC1):
            b = bytearray(b)
            b[s + 4 + off] = value
            return bytes(b)
    raise ValueError("no SOF")


def main():
    cases = []

    def ok(name, data):
        cases.append((name, "ok", OK, data))

    for sub in (0, 1, 2):
        tag = SUB[sub]
        for w in range(1, 18):
            for h in (1, 6, 17):
                ok(f"{tag} {h}x{w} q75", enc(synthetic.synthetic_photo(h, w, seed=h * 41 + w), quality=75, subsampling=sub))
        for h in range(1, 18):
            for w in (1, 6, 17):
                ok(f"{tag} {h}x{w} q90", enc(synthetic.synthetic_photo(h, w, seed=h * 43 + w), quality=90, subsampling=sub))
        photo = synthetic.synthetic_photo(41, 53, seed=7 + sub)
        for q in (5, 10, 25, 50, 75, 90, 95, 100):
            ok(f"{tag} photo q{q}", enc(photo, quality=q, subsampling=sub))
        ok(f"{tag} optimize", enc(photo, quality=80, subsampling=sub, optimize=True))
        ok(f"{tag} restart blocks 3", enc(photo, quality=80, subsampling=sub, restart_marker_blocks=3))
        ok(f"{tag} restart rows 1", enc(photo, quality=80, subsampling=sub, restart_marker_rows=1))
        ok(f"{tag} 16-bit qtables", enc(photo, subsampling=sub, qtables=[list(range(1, 65)), [300 + i for i in range(64)]]))
        ok(f"{tag} APPn COM", enc(photo, quality=70, subsampling=sub, comment=b"pigeon", icc_profile=b"\0" * 300,
                                  exif=b"Exif\0\0" + b"\0" * 64))
        rng = np.random.default_rng(100 + sub)
        ok(f"{tag} noise q100", enc(rng.integers(0, 256, (40, 72, 3), dtype=np.uint8), quality=100, subsampling=sub))
        ok(f"{tag} noise q5", enc(rng.integers(0, 256, (40, 72, 3), dtype=np.uint8), quality=5, subsampling=sub))
        for v in (0, 128, 255):
            ok(f"{tag} flat {v}", enc(np.full((24, 40, 3), v, np.uint8), quality=85, subsampling=sub))
        edge = np.zeros((48, 64, 3), np.uint8)
        edge[:, ::2] = 255
        edge[::3, :, 1] = 255
        edge[20:30, 10:50] = (255, 0, 255)
        ok(f"{tag} saturated edges q100", enc(edge, quality=100, subsampling=sub))
        ok(f"{tag} 1x300", enc(synthetic.synthetic_photo(1, 300, seed=3), quality=80, subsampling=sub))
        ok(f"{tag} 300x1", enc(synthetic.synthetic_photo(300, 1, seed=4), quality=80, subsampling=sub))
        ok(f"{tag} 133x251", enc(synthetic.synthetic_photo(133, 251, seed=5), quality=60, subsampling=sub))
    gray = synthetic.synthetic_photo(45, 67, seed=11)[..., 1].copy()
    for q in (5, 75, 100):
        f = io.BytesIO()
        Image.fromarray(gray).save(f, "JPEG", quality=q)
        ok(f"gray q{q}", f.getvalue())
    for h, w in ((1, 1), (1, 17), (17, 1), (9, 13)):
        f = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(gray[:h, :w])).save(f, "JPEG", quality=80)
        ok(f"gray {h}x{w}", f.getvalue())
    f = io.BytesIO()
    Image.fromarray(gray).save(f, "JPEG", quality=80, restart_marker_blocks=2)
    ok("gray restart blocks 2", f.getvalue())
    ok("420 640x640 q90", enc(smooth(640, 640), quality=90, subsampling=2))
    ok("420 4000x3000 q50", enc(smooth(3000, 4000), quality=50, subsampling=2))

    base = enc(synthetic.synthetic_photo(40, 56, seed=31), quality=80, subsampling=2)
    cases.append(("progressive", "reject", UNSUPPORTED, enc(synthetic.synthetic_photo(40, 56, seed=31), quality=80,
                                                             progressive=True)))
    f = io.BytesIO()
    Image.fromarray(synthetic.synthetic_photo(40, 56, seed=32)).convert("CMYK").save(f, "JPEG", quality=80)
    cases.append(("CMYK", "reject", UNSUPPORTED, f.getvalue()))
    for m, s, e in segments(base):
        if m == 0xC0:
            sof = s
    for marker, name in ((0xC3, "SOF3 lossless"), (0xC9, "SOF9 arithmetic")):
        b = bytearray(base)
        b[sof + 1] = marker
        cases.append((name, "reject", UNSUPPORTED, bytes(b)))
    cases.append(("12-bit", "reject", UNSUPPORTED, edit_sof(base, 0, 12)))
    cases.append(("height 0 (DNL)", "reject", UNSUPPORTED, edit_sof(edit_sof(base, 1, 0), 2, 0)))
    cases.append(("4:4:0 sampling", "reject", UNSUPPORTED, edit_sof(base, 7, 0x12)))
    sos = [s for m, s, e in segments(base) if m == 0xDA][0]
    cases.append(("two scans", "reject", UNSUPPORTED, base[:-2] + base[sos:]))
    noj = drop_app0(base)
    cases.append(("Adobe transform 0", "reject", UNSUPPORTED,
                  noj[:2] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + noj[2:]))
    rgb = bytearray(noj)
    for m, s, e in segments(bytes(rgb)):
        if m == 0xC0:
            rgb[s + 10], rgb[s + 13], rgb[s + 16] = ord("R"), ord("G"), ord("B")
        if m == 0xDA:
            rgb[s + 5], rgb[s + 7], rgb[s + 9] = ord("R"), ord("G"), ord("B")
    cases.append(("component ids RGB", "reject", UNSUPPORTED, bytes(rgb)))
    cases.append(("truncated header", "reject", BAD_HEADER, base[:sos - 10]))
    cases.append(("not a JPEG", "reject", BAD_HEADER, b"\x89PNG\r\n\x1a\n" + b"\0" * 32))
    # corrupt entropy-coded data
    scan = sos + 2 + (base[sos + 2] << 8 | base[sos + 3])
    cases.append(("truncated file", "corrupt", NO_EOI, base[:len(base) // 2 + scan // 2]))
    cases.append(("truncated scan + EOI", "corrupt", OVERRUN, base[:scan + 40] + b"\xff\xd9"))
    cases.append(("all-ones code", "corrupt", BAD_CODE, base[:scan] + b"\xff\x00" * 4 + base[scan + 8:]))
    rst = enc(synthetic.synthetic_photo(40, 56, seed=33), quality=80, subsampling=2, restart_marker_blocks=1)
    i = rst.index(b"\xff\xd1")
    cases.append(("wrong RST number", "corrupt", BAD_RST, rst[:i] + b"\xff\xd3" + rst[i + 2:]))

    # One array per field (the files and the full pixels concatenated, with offsets) keeps the archive small: a
    # separate entry per case would cost a zip and an .npy header each.
    n = len(cases)
    out = {"count": np.array(n), "pillow": np.array(Image.__version__),
           "libjpeg_turbo": np.array(str(features.version("libjpeg_turbo"))),
           "name": np.array([c[0] for c in cases]), "kind": np.array([c[1] for c in cases]),
           "status": np.array([c[2] for c in cases], dtype=np.int32), "shape": np.zeros((n, 3), dtype=np.int32)}
    jpg_off, px_off, jpgs, pxs = [0], [0], [], []
    for k, (name, kind, status, data) in enumerate(cases):
        jpgs.append(np.frombuffer(data, dtype=np.uint8))
        jpg_off.append(jpg_off[-1] + len(data))
        px = None
        if kind == "ok" or name == "progressive":          # the progressive file's pixels check the host route
            px = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
            out["shape"][k] = px.shape
            if px.shape[0] * px.shape[1] > FULL_PIXELS:
                out[f"sha{k}"] = np.frombuffer(hashlib.sha256(px.tobytes()).digest(), dtype=np.uint8)
                out[f"sample{k}"] = px[::37, ::23].copy()
                px = None
        if px is not None:
            pxs.append(px.reshape(-1))
        px_off.append(px_off[-1] + (px.size if px is not None else 0))
    out["jpg"] = np.concatenate(jpgs)
    out["jpg_off"] = np.array(jpg_off, dtype=np.int64)
    out["px"] = np.concatenate(pxs)
    out["px_off"] = np.array(px_off, dtype=np.int64)
    path = os.path.join(ROOT, "tests", "golden", "jpeg.npz")
    np.savez_compressed(path, **out)
    print(path, len(cases), "cases", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
