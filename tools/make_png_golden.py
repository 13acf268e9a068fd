#!/usr/bin/env python
"""Writes tests/golden/png.npz: PNG files and what Pillow makes of them (`np.asarray(Image.open(f).convert('RGB'))`, or
the exception it raises), for the GPU decoder's tests.  Made with Pillow 12.2.0 and the zlib of Python's `zlib` module.

Pillow's encoder writes only a few of the layouts a decoder meets, so most files come from the small PNG assembler below
(struct + zlib, plus a DEFLATE writer for streams zlib never emits: a match at distance 32 768, a dynamic block with a
single one-bit distance code).

Per case k: `name[k]` describes it, `kind[k]` is
  'ok'        parsed for the GPU and expected to decode there;
  'host'      refused by the chunk walk (interlaced, APNG, bad CRC, split IDAT runs, ...): Pillow decodes it on the host;
  'fallback'  parsed for the GPU, but its stream or a filter byte is bad: the device must refuse it (`status[k]`, the
              PG_PNG_* the construction implies), and Pillow then decodes it or raises;
  'flip'      a valid file with seeded bit flips: whatever the device does, the output must be Pillow's.
`png[png_off[k]:png_off[k+1]]` holds the file's bytes.  When Pillow decodes it, `shape[k]` is (H, W, 3) and the pixels
are `px[px_off[k]:px_off[k+1]]` or, above FULL_PIXELS pixels, `sha[k]` (SHA-256 of the pixels) and
`sample[sample_off[k]:sample_off[k+1]]` (pixels[::37, ::23], flattened); otherwise `error[k]` is 'Type: message' (object addresses replaced by 0x?).
"""
import hashlib
import io
import os
import re
import struct
import sys
import zlib

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pigeon_b200 import synthetic  # noqa: E402

OK, UNSUPPORTED, BAD_HEADER, BAD_ZLIB, BAD_DEFLATE, TRUNCATED, TOO_LONG, BAD_FILTER = range(8)
FULL_PIXELS = 1024
SIG = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


# ---------------------------------------------------------------------------------------------------------------------
# PNG assembler
# ---------------------------------------------------------------------------------------------------------------------

def chunk(cid: bytes, data: bytes, crc=None) -> bytes:
    c = zlib.crc32(cid + data) & 0xFFFFFFFF if crc is None else crc
    return struct.pack(">I", len(data)) + cid + data + struct.pack(">I", c)


def ihdr(w, h, depth, ct, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ct, 0, 0, interlace))


def png(w, h, depth, ct, stream, pre=(), post=(), split=None, interlace=0):
    """A file: IHDR, the `pre` chunks, the zlib stream in IDAT chunks (one, or the sizes in `split`), `post`, IEND."""
    idat = []
    if split is None:
        idat = [chunk(b"IDAT", stream)]
    else:
        at = 0
        for s in split:
            idat.append(chunk(b"IDAT", stream[at:at + s]))
            at += s
        idat.append(chunk(b"IDAT", stream[at:]))
    return SIG + ihdr(w, h, depth, ct, interlace) + b"".join(pre) + b"".join(idat) + b"".join(post) + chunk(b"IEND", b"")


def samples(rng, h, w, depth, ct, hi=None):
    """Random samples [h, w, channels] below 2**depth (or `hi`), smooth enough to compress."""
    c = CHANNELS[ct]
    top = hi if hi is not None else 1 << depth
    base = rng.integers(0, top, size=(h, 1, c))
    step = rng.choice([-1, 0, 0, 0, 1], size=(h, w, c)).cumsum(1)
    return np.clip(base + step, 0, top - 1).astype(np.int64)


def pack_rows(s, depth):
    """[h, w, c] samples -> list of row byte strings (big-endian 16-bit, MSB-first sub-byte packing)."""
    h, w, c = s.shape
    rows = []
    for r in range(h):
        v = s[r].reshape(-1)
        if depth == 16:
            rows.append(v.astype(">u2").tobytes())
        elif depth == 8:
            rows.append(v.astype(np.uint8).tobytes())
        else:
            per = 8 // depth
            pad = (-len(v)) % per
            v = np.concatenate([v, np.zeros(pad, dtype=np.int64)]).reshape(-1, per)
            shifts = 8 - depth * (np.arange(per) + 1)
            rows.append((v << shifts).sum(1).astype(np.uint8).tobytes())
    return rows


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def filter_rows(rows, bpp, types):
    """Filtered scanlines (filter byte + bytes) with the filter type types[r] on row r."""
    out, prev = [], bytes(len(rows[0]))
    for r, row in enumerate(rows):
        ft = types[r]
        f = bytearray([ft])
        for x in range(len(row)):
            a = row[x - bpp] if x >= bpp else 0
            b = prev[x]
            c = prev[x - bpp] if x >= bpp else 0
            pred = [0, a, b, (a + b) >> 1, paeth(a, b, c)][ft] if ft <= 4 else 0
            f.append((row[x] - pred) & 255)
        out.append(bytes(f))
        prev = row
    return b"".join(out)


def raw_image(rng, h, w, depth, ct, types=None, hi=None):
    s = samples(rng, h, w, depth, ct, hi)
    rows = pack_rows(s, depth)
    bpp = max(1, CHANNELS[ct] * depth // 8)
    return filter_rows(rows, bpp, types if types is not None else [r % 5 for r in range(h)])


def compress(raw, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    return c.compress(raw) + c.flush()


# ---------------------------------------------------------------------------------------------------------------------
# A DEFLATE writer for streams zlib does not emit
# ---------------------------------------------------------------------------------------------------------------------

class BitWriter:
    def __init__(self):
        self.bits, self.n, self.out = 0, 0, bytearray()

    def put(self, v, k):                 # k bits of v, LSB first
        self.bits |= v << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.bits & 255)
            self.bits >>= 8
            self.n -= 8

    def huff(self, code, length):        # a Huffman code, MSB first
        self.put(int(format(code, f"0{length}b")[::-1], 2), length)

    def flush(self):
        if self.n:
            self.out.append(self.bits & 255)
        self.bits = self.n = 0
        return bytes(self.out)


def canonical(lens):
    bl = [0] * 16
    for l in lens:
        if l:
            bl[l] += 1
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1 if b > 1 else 0
        nxt[b] = code
    codes = [0] * len(lens)
    for s, l in enumerate(lens):
        if l:
            codes[s] = nxt[l]
            nxt[l] += 1
    return codes


LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def write_symbols(bw, ops, lit_lens, dist_lens):
    lc, dc = canonical(lit_lens), canonical(dist_lens)
    for op in ops:
        if op[0] == "lit":
            bw.huff(lc[op[1]], lit_lens[op[1]])
            continue
        _, length, dist = op
        i = max(k for k in range(29) if LEN_BASE[k] <= length) if length < 258 else 28
        bw.huff(lc[257 + i], lit_lens[257 + i])
        bw.put(length - LEN_BASE[i], LEN_EXTRA[i])
        j = max(k for k in range(30) if DIST_BASE[k] <= dist)
        bw.huff(dc[j], dist_lens[j])
        bw.put(dist - DIST_BASE[j], DIST_EXTRA[j])
    bw.huff(lc[256], lit_lens[256])


def fixed_block(bw, ops, final):
    bw.put(final, 1)
    bw.put(1, 2)
    write_symbols(bw, ops, FIXED_LIT, FIXED_DIST)


def dynamic_block(bw, ops, lit_lens, dist_lens, final):
    """A dynamic block whose code-length code gives each of the 16 lengths 0..15 a 4-bit code (a complete set)."""
    bw.put(final, 1)
    bw.put(2, 2)
    bw.put(len(lit_lens) - 257, 5)
    bw.put(len(dist_lens) - 1, 5)
    bw.put(19 - 4, 4)
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    for s in order:
        bw.put(4 if s < 16 else 0, 3)
    for l in list(lit_lens) + list(dist_lens):
        bw.huff(l, 4)
    write_symbols(bw, ops, lit_lens, dist_lens)


def zlib_wrap(deflate, raw, cinfo=7):
    cmf = (cinfo << 4) | 8
    flg = 31 - (cmf << 8) % 31
    return bytes([cmf, flg]) + deflate + struct.pack(">I", zlib.adler32(raw))


def ops_for(raw, dist1=False):
    """Literals, or for runs greedy length-258 matches at distance 1."""
    ops, i = [], 0
    while i < len(raw):
        if dist1 and i > 0:
            run = 0
            while i + run < len(raw) and raw[i + run] == raw[i - 1] and run < 258:
                run += 1
            if run >= 3:
                ops.append(("match", run, 1))
                i += run
                continue
        ops.append(("lit", raw[i]))
        i += 1
    return ops


# ---------------------------------------------------------------------------------------------------------------------

def pillow(data):
    try:
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB")), ""
    except Exception as e:  # noqa: BLE001 - the exception is the expected outcome
        return None, re.sub(r"0x[0-9a-fA-F]+", "0x?", f"{type(e).__name__}: {e}")


def picture(h, w, seed):
    """A noisy synthetic photo up to 64 x 64; larger images are gradients with one noisy 32 x 32 patch, so that the
    archive stays small."""
    if h * w <= 4096:
        return synthetic.synthetic_photo(h, w, seed=seed)
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([(xx * 255 // (w - 1)), (yy * 255 // (h - 1)), ((xx + 2 * yy) // 5) % 256], -1).astype(np.uint8)
    img[h // 3:h // 3 + 32, w // 3:w // 3 + 32] = synthetic.synthetic_photo(32, 32, seed=seed)
    return img


def enc(img, mode=None, **kw):
    f = io.BytesIO()
    im = Image.fromarray(img)
    if mode == "1":                   # thresholded, not dithered: flat areas keep the archive small
        im = im.convert("L").convert("1", dither=Image.Dither.NONE)
    elif mode is not None:
        im = im.convert(mode)
    im.save(f, "PNG", **kw)
    return f.getvalue()


def main():
    rng = np.random.default_rng(2026)
    cases = []

    def add(name, kind, data, status=OK):
        cases.append((name, kind, status, data))

    # Pillow-encoded: RGB, RGBA, L, LA, P and 1-bit, at every level and with optimize, 1x1 to 1024x768
    sizes = [(1, 1), (1, 29), (29, 1), (7, 13), (500, 333), (768, 1024)]
    settings = [("level 0", dict(compress_level=0)), ("level 1", dict(compress_level=1)),
                ("level 6", dict(compress_level=6)), ("level 9", dict(compress_level=9)), ("optimize", dict(optimize=True))]
    for h, w in sizes:
        photo = picture(h, w, seed=h * 7 + w)
        big = h * w > 100000
        for mode in ("RGB", "RGBA", "L", "LA", "P", "1"):
            for sname, kw in settings:
                if big and sname not in ("level 6", "optimize"):     # keeps the archive small
                    continue
                if big and mode in ("RGBA", "LA") and sname == "optimize":
                    continue
                src = np.dstack([photo, photo[..., 1]]) if mode in ("RGBA",) else photo
                if mode == "P":
                    data = io.BytesIO()
                    Image.fromarray(photo).quantize(64 if h * w > 16 else 4).save(data, "PNG", **kw)
                    data = data.getvalue()
                elif mode == "RGBA":
                    data = enc(src, **kw)
                else:
                    data = enc(photo, mode if mode != "RGB" else None, **kw)
                add(f"pillow {mode} {h}x{w} {sname}", "ok", data)

    # every colour type and bit depth, each filter type forced on every row and mixed per row
    for ct, depths in ((0, (1, 2, 4, 8, 16)), (2, (8, 16)), (3, (1, 2, 4, 8)), (4, (8, 16)), (6, (8, 16))):
        for d in depths:
            for h, w in ((1, 1), (9, 11), (33, 70)):
                pre = [chunk(b"PLTE", rng.integers(0, 256, 3 << d if d < 8 else 768, dtype=np.uint8).tobytes())] \
                    if ct == 3 else []
                for ftname, types in (("mixed filters", None),) + tuple((f"filter {f}", [f] * h) for f in range(5)):
                    if (h, w) != (33, 70) and ftname != "mixed filters":
                        continue
                    raw = raw_image(rng, h, w, d, ct, types)
                    add(f"ct {ct} depth {d} {h}x{w} {ftname}", "ok", png(w, h, d, ct, compress(raw), pre))

    # zlib strategies and window sizes
    raw = raw_image(rng, 24, 97, 8, 2)
    for sname, st in (("default", zlib.Z_DEFAULT_STRATEGY), ("FILTERED", zlib.Z_FILTERED),
                      ("HUFFMAN_ONLY", zlib.Z_HUFFMAN_ONLY), ("RLE", zlib.Z_RLE), ("FIXED", zlib.Z_FIXED)):
        for lvl in (1, 9):
            add(f"zlib {sname} level {lvl}", "ok", png(97, 24, 8, 2, compress(raw, lvl, strategy=st)))
    for wb in range(9, 16):
        add(f"zlib window bits {wb}", "ok", png(97, 24, 8, 2, compress(raw, 9, wb)))
    # stored blocks past 65 535 bytes, and many stored blocks of a level-0 stream split into 1-byte and empty IDATs
    raw = b"".join(b"\0" + ((np.arange(600) + 3 * r) % 251).astype(np.uint8).tobytes() for r in range(200))
    add("stored blocks 120 KB", "ok", png(150, 200, 8, 6, compress(raw, 0)))
    small = raw_image(rng, 6, 5, 8, 2)
    st = compress(small, 0)
    add("IDAT split into 1-byte and empty chunks", "ok", png(5, 6, 8, 2, st, split=[1, 0, 1, 1, 0, 2, 1] + [1] * 20))
    st = compress(raw_image(rng, 20, 20, 8, 0), 9)
    add("IDAT split inside the zlib header and the Adler-32", "ok",
        png(20, 20, 8, 0, st, split=[1, len(st) - 3, 1]))
    # length-258 matches at distance 1 (a flat image, zlib level 9 and the writer's own run encoder)
    flat = (b"\x00" + b"\x07" * 3000) * 40
    add("length-258 matches at distance 1 (zlib)", "ok", png(1000, 40, 8, 2, compress(flat, 9)))
    bw = BitWriter()
    fixed_block(bw, ops_for(flat, dist1=True), 1)
    add("length-258 matches at distance 1 (fixed block)", "ok", png(1000, 40, 8, 2, zlib_wrap(bw.flush(), flat)))
    # matches at distance exactly 32 768: rows of 128 bytes, the second 256 rows repeat the first 256
    first = raw_image(rng, 8, 127, 8, 0, [int(t) for t in rng.integers(0, 5, 8)]) * 32    # 8 rows, tiled: compressible
    body = first + first
    ops = [("lit", b) for b in first]
    left = len(first)
    while left:
        k = min(258, left)
        if 0 < left - k < 3:
            k = left - 3
        ops.append(("match", k, 32768))
        left -= k
    bw = BitWriter()
    fixed_block(bw, ops, 1)
    add("matches at distance 32768", "ok", png(127, 512, 8, 0, zlib_wrap(bw.flush(), body)))
    # a dynamic block with one one-bit distance code (zlib accepts that incomplete code)
    lit_lens = [9] * 256 + [6] * 28 + [5] * 2
    single = (b"\x00" + b"\x11" * 40 + bytes(range(40))) * 9
    bw = BitWriter()
    dynamic_block(bw, ops_for(single, dist1=True), lit_lens, [1], 1)
    add("dynamic block with a single distance code", "ok", png(80, 9, 8, 0, zlib_wrap(bw.flush(), single)))
    # fixed and stored blocks mixed, not final until the last
    part = raw_image(rng, 12, 30, 8, 2)
    bw = BitWriter()
    fixed_block(bw, ops_for(part[:500]), 0)
    bw.put(0, 1)
    bw.put(0, 2)
    stored = bw.flush()
    mid = part[500:800]
    stored += struct.pack("<HH", len(mid), len(mid) ^ 0xFFFF) + mid
    bw = BitWriter()
    fixed_block(bw, ops_for(part[800:], dist1=True), 1)
    add("fixed, stored and fixed blocks", "ok", png(30, 12, 8, 2, zlib_wrap(stored + bw.flush(), part)))
    # extra decompressed data after the last row
    raw = raw_image(rng, 16, 16, 8, 2)
    add("extra data after the last row", "ok", png(16, 16, 8, 2, compress(raw + b"\x01" * 700)))

    # palette and PLTE quirks, 16-bit rules, tRNS, ignored chunks
    raw = filter_rows([bytes([0, 1, 2, 3, 200, 255])] * 3, 1, [0, 1, 2])
    add("palette index past PLTE", "ok", png(6, 3, 8, 3, compress(raw), [chunk(b"PLTE", bytes(range(9)))]))
    add("palette without PLTE", "ok", png(6, 3, 8, 3, compress(raw)))
    add("palette PLTE after IDAT", "ok", png(6, 3, 8, 3, compress(raw), post=[chunk(b"PLTE", bytes(range(9)))]))
    pl = [chunk(b"PLTE", rng.integers(0, 256, 768, dtype=np.uint8).tobytes())]
    add("palette tRNS one transparent entry", "ok", png(6, 3, 8, 3, compress(raw), pl + [chunk(b"tRNS", b"\xff\x00")]))
    add("palette tRNS alpha per entry", "ok", png(6, 3, 8, 3, compress(raw), pl + [chunk(b"tRNS", b"\x10\x80\xff")]))
    g16 = filter_rows([struct.pack(">6H", 0, 255, 256, 300, 4095, 65535)] * 2, 2, [0, 4])
    add("16-bit grey clips to 255", "ok", png(6, 2, 16, 0, compress(g16)))
    add("16-bit grey with tRNS", "ok", png(6, 2, 16, 0, compress(g16), [chunk(b"tRNS", b"\x01\x2c")]))
    raw = raw_image(rng, 8, 9, 8, 0)
    add("grey tRNS above 255", "ok", png(9, 8, 8, 0, compress(raw), [chunk(b"tRNS", b"\x01\x2c")]))
    add("grey tRNS", "ok", png(9, 8, 8, 0, compress(raw), [chunk(b"tRNS", b"\x00\x10")]))
    raw = raw_image(rng, 8, 9, 1, 0)
    add("1-bit grey tRNS", "ok", png(9, 8, 1, 0, compress(raw), [chunk(b"tRNS", b"\x00\x01")]))
    for d in (8, 16):
        raw = raw_image(rng, 8, 9, d, 2)
        add(f"RGB {d}-bit tRNS", "ok", png(9, 8, d, 2, compress(raw), [chunk(b"tRNS", b"\x00\x10\x01\x20\x00\x30")]))
        add(f"LA {d}-bit with an ignored tRNS", "ok", png(9, 8, d, 4, compress(raw_image(rng, 8, 9, d, 4)),
                                                           [chunk(b"tRNS", b"\x01")]))
    raw = raw_image(rng, 10, 12, 8, 2)
    icc = b"sRGB\x00\x00" + zlib.compress(b"\x00" * 3000)
    ign = [chunk(b"gAMA", struct.pack(">I", 45455)), chunk(b"sRGB", b"\x00"), chunk(b"sBIT", b"\x05\x06\x05"),
           chunk(b"iCCP", icc), chunk(b"cHRM", bytes(32)), chunk(b"pHYs", bytes(9)), chunk(b"tEXt", b"Title\x00a png"),
           chunk(b"zTXt", b"Comment\x00\x00" + zlib.compress(b"text " * 100)),
           chunk(b"iTXt", b"Note\x00\x00\x00en\x00Note\x00plain"),
           chunk(b"iTXt", b"Zip\x00\x01\x00\x00\x00" + zlib.compress("é".encode() * 50)), chunk(b"prVt", b"private")]
    add("gAMA, sRGB, sBIT, iCCP, cHRM, pHYs and text chunks", "ok", png(12, 10, 8, 2, compress(raw), ign,
                                                                         post=[chunk(b"tEXt", b"After\x00idat")]))
    add("no IEND", "ok", png(12, 10, 8, 2, compress(raw))[:-12])

    # host route: refused by the chunk walk
    photo = synthetic.synthetic_photo(20, 24, seed=5)
    good = enc(photo)
    a7 = []
    for x0, y0, dx, dy in ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)):
        sub = photo[y0::dy, x0::dx]
        if sub.size:
            a7.append(b"".join(b"\x00" + r.tobytes() for r in sub))
    add("Adam7 interlaced", "host", png(24, 20, 8, 2, compress(b"".join(a7)), interlace=1), UNSUPPORTED)
    apng = io.BytesIO()
    Image.fromarray(photo).save(apng, "PNG", save_all=True, append_images=[Image.fromarray(photo[::-1].copy())])
    add("APNG", "host", apng.getvalue(), UNSUPPORTED)
    raw = raw_image(rng, 10, 12, 8, 2)
    add("bad CRC in tEXt before IDAT", "host", png(12, 10, 8, 2, compress(raw), [chunk(b"tEXt", b"a\x00b", crc=1)]),
        BAD_HEADER)
    add("bad CRC in IHDR", "host", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 12, 10, 8, 2, 0, 0, 0), crc=7) +
        png(12, 10, 8, 2, compress(raw))[33:], BAD_HEADER)
    st = compress(raw)
    add("IDAT runs split by a tEXt chunk", "host",
        SIG + ihdr(12, 10, 8, 2) + chunk(b"IDAT", st[:20]) + chunk(b"tEXt", b"a\x00b") + chunk(b"IDAT", st[20:]) +
        chunk(b"IEND", b""), UNSUPPORTED)
    add("no IDAT", "host", SIG + ihdr(12, 10, 8, 2) + chunk(b"IEND", b""), BAD_HEADER)
    add("no IHDR", "host", SIG + chunk(b"IDAT", st) + chunk(b"IEND", b""), BAD_HEADER)
    add("bad colour type and depth", "host", png(12, 10, 4, 2, st), BAD_HEADER)
    add("truncated before IDAT", "host", good[:40], BAD_HEADER)
    add("not a PNG", "host", b"GIF89a" + bytes(40), BAD_HEADER)
    add("zTXt above MAX_TEXT_CHUNK", "host",
        png(12, 10, 8, 2, st, [chunk(b"zTXt", b"big\x00\x00" + zlib.compress(b"x" * (1 << 20 | 5)))]), UNSUPPORTED)
    add("palette tRNS without PLTE", "host", png(12, 10, 8, 3, compress(raw_image(rng, 10, 12, 8, 3, hi=4)),
                                                 [chunk(b"tRNS", b"\x00")]), UNSUPPORTED)
    add("short grey tRNS", "host", png(9, 8, 8, 0, compress(raw_image(rng, 8, 9, 8, 0)), [chunk(b"tRNS", b"\x01")]),
        UNSUPPORTED)

    # device fallback: the chunk walk accepts these, the stream or a filter byte does not
    raw = raw_image(rng, 30, 40, 8, 2)
    st = compress(raw)
    add("truncated stream", "fallback", png(40, 30, 8, 2, st[:len(st) // 2]), TRUNCATED)
    add("stream without its Adler-32", "fallback", png(40, 30, 8, 2, st[:-4]), TRUNCATED)
    bad = st[:-4] + struct.pack(">I", (zlib.adler32(raw) + 1) & 0xFFFFFFFF)
    add("bad Adler-32", "fallback", png(40, 30, 8, 2, bad), BAD_ZLIB)
    st2 = compress(raw + b"\x02" * 300)
    add("bad Adler-32 after trailing image data", "fallback",
        png(40, 30, 8, 2, st2[:-4] + struct.pack(">I", 12345)), BAD_ZLIB)
    add("bytes after the zlib stream", "fallback", png(40, 30, 8, 2, st + b"\x00\x01"), BAD_ZLIB)
    add("stream shorter than the image", "fallback", png(40, 31, 8, 2, st), TRUNCATED)
    add("bad zlib header", "fallback", png(40, 30, 8, 2, b"\x78\x00" + st[2:]), BAD_ZLIB)
    add("preset dictionary flag", "fallback", png(40, 30, 8, 2, bytes([0x78, 0xBB]) + st[2:]), BAD_ZLIB)
    add("filter type 5", "fallback", png(40, 30, 8, 2, compress(raw[:121 * 5] + b"\x05" + raw[121 * 5 + 1:])),
        BAD_FILTER)
    add("too much data after the rows", "fallback", png(40, 30, 8, 2, compress(raw + bytes(10000))), TOO_LONG)
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(3, 2)
    add("block type 3", "fallback", png(40, 30, 8, 2, zlib_wrap(bw.flush() + bytes(8), raw)), BAD_DEFLATE)
    small = raw_image(rng, 4, 4, 8, 0)
    bw = BitWriter()
    fixed_block(bw, [("lit", small[0]), ("match", 4, 2)], 1)
    add("distance past the data", "fallback", png(4, 4, 8, 0, zlib_wrap(bw.flush(), small)), BAD_DEFLATE)
    big = raw_image(rng, 20, 300, 8, 0)
    big += big                                  # repeats 6 020 bytes back
    add("distance past the declared window", "fallback", png(300, 40, 8, 0, zlib_wrap(
        compress(big, 9, 15)[2:-4], big, cinfo=0)), BAD_DEFLATE)
    bw = BitWriter()
    dynamic_block(bw, [("lit", b) for b in small], [9] * 256 + [6] * 28 + [5] * 1 + [6], [1], 1)
    add("incomplete literal/length code", "fallback", png(4, 4, 8, 0, zlib_wrap(bw.flush(), small)), BAD_DEFLATE)
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(0, 2)
    add("stored LEN / NLEN mismatch", "fallback",
        png(4, 4, 8, 0, zlib_wrap(bw.flush() + b"\x01\x00\x00\x00" + b"\x00", small)), BAD_DEFLATE)

    # seeded bit flips in the IDAT data of small valid files
    for k in range(48):
        h, w = int(rng.integers(3, 20)), int(rng.integers(3, 20))
        ct = int(rng.choice([0, 2, 6]))
        data = bytearray(png(w, h, 8, ct, compress(raw_image(rng, h, w, 8, ct), int(rng.integers(1, 10)))))
        i0 = data.index(b"IDAT") + 4
        i1 = len(data) - 16
        for _ in range(int(rng.integers(1, 4))):
            p = int(rng.integers(i0, i1))
            data[p] ^= 1 << int(rng.integers(0, 8))
        add(f"bit flips {k}", "flip", bytes(data), -1)

    n = len(cases)
    out = {"count": np.array(n), "pillow": np.array(Image.__version__), "zlib": np.array(zlib.ZLIB_RUNTIME_VERSION),
           "name": np.array([c[0] for c in cases]), "kind": np.array([c[1] for c in cases]),
           "status": np.array([c[2] for c in cases], dtype=np.int32), "shape": np.zeros((n, 3), dtype=np.int32),
           "error": np.array([""] * n, dtype=object)}
    off, px_off, files, pxs, errors = [0], [0], [], [], []
    sha, sample_off, samples_ = np.zeros((n, 32), dtype=np.uint8), [0], []
    for k, (name, kind, status, data) in enumerate(cases):
        files.append(np.frombuffer(data, dtype=np.uint8))
        off.append(off[-1] + len(data))
        px, err = pillow(data)
        errors.append(err)
        if kind == "ok":
            assert px is not None, (name, err)
        if px is not None:
            out["shape"][k] = px.shape
            if px.shape[0] * px.shape[1] > FULL_PIXELS:
                sha[k] = np.frombuffer(hashlib.sha256(px.tobytes()).digest(), dtype=np.uint8)
                sample = px[::37, ::23].reshape(-1)
                samples_.append(sample)
                sample_off.append(sample_off[-1] + sample.size)
                px = None
        if len(sample_off) == k + 1:
            sample_off.append(sample_off[-1])
        if px is not None:
            pxs.append(px.reshape(-1))
        px_off.append(px_off[-1] + (px.size if px is not None else 0))
    out["error"] = np.array(errors)
    out["png"] = np.concatenate(files)
    out["png_off"] = np.array(off, dtype=np.int64)
    out["px"] = np.concatenate(pxs)
    out["px_off"] = np.array(px_off, dtype=np.int64)
    out["sha"] = sha
    out["sample"] = np.concatenate(samples_)
    out["sample_off"] = np.array(sample_off, dtype=np.int64)
    path = os.path.join(ROOT, "tests", "golden", "png.npz")
    np.savez_compressed(path, **out)
    print(path, n, "cases", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
