#!/usr/bin/env python
"""Writes tests/golden/jpeg_multiscan.npz: progressive and multi-scan sequential JPEG files, what Pillow decodes them to,
and their scan scripts, for the tests of the GPU decoder's multi-scan path.  Made with Pillow 12.2.0 over
libjpeg-turbo 3.1.4.1.

Pillow writes the progressive files it can (libjpeg's default script).  Scripts Pillow cannot write come from a lossless
transcoder (test data only): it Huffman-decodes a baseline file's quantised coefficients and re-emits them under the
chosen script with optimal per-scan Huffman tables.  Every transcoded file is checked to decode, in Pillow, to the same
pixels as its source: the coefficients are the same, and a complete progression is not smoothed.

Layout as jpeg.npz (tools/make_jpeg_golden.py): `name`, `kind` ('ok', 'reject', 'corrupt'), `status`, `jpg` / `jpg_off`,
`shape`, and `px` / `px_off` or `sha{k}` + `sample{k}` above FULL_PIXELS pixels; plus `reason[k]`, a substring of the
rejection reason, and, for files the multi-scan parser accepts, the scan script
`scans[scan_off[k]:scan_off[k+1]]`: rows of (components, c0, c1, c2, Ss, Se, Ah, Al, restart interval, segments, level).
"""
import hashlib
import io
import os
import sys

import numpy as np
from PIL import Image, ImageFile, features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pigeon_b200 import synthetic  # noqa: E402

ImageFile.MAXBLOCK = 1 << 24          # Pillow's progressive encoder needs the whole output in its buffer
OK, UNSUPPORTED, BAD_HEADER, BAD_CODE, OVERRUN, MARKER, BAD_RST, NO_EOI = range(8)
FULL_PIXELS = 4096


def enc(img, **kw):
    f = io.BytesIO()
    Image.fromarray(img).save(f, "JPEG", **kw)
    return f.getvalue()


def pixels(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


# ----------------------------------------------------------------------------------------------------------------
# Marker walk and scan description (independent of the library)
# ----------------------------------------------------------------------------------------------------------------

def markers(b):
    """(marker, segment start, segment end, entropy data end) in file order, up to and including EOI."""
    out, p = [], 2
    while p < len(b):
        while b[p + 1] == 0xFF:
            p += 1
        m = b[p + 1]
        if m == 0xD9:
            out.append((m, p, p + 2, p + 2))
            return out
        L = b[p + 2] << 8 | b[p + 3]
        e = p + 2 + L
        if m != 0xDA:
            out.append((m, p, e, e))
            p = e
            continue
        q = e                                   # entropy-coded data runs to the next marker other than RSTn
        while True:
            q = b.index(b"\xff", q)
            if b[q + 1] == 0x00 or 0xD0 <= b[q + 1] <= 0xD7:
                q += 2
                continue
            break
        out.append((m, p, e, q))
        p = q
    return out


def frame(b):
    for m, s, e, _ in markers(b):
        if m in (0xC0, 0xC1, 0xC2):
            nf = b[s + 9]
            comps = [(b[s + 10 + 3 * i], b[s + 11 + 3 * i] >> 4, b[s + 11 + 3 * i] & 15, b[s + 12 + 3 * i]) for i in range(nf)]
            return dict(sof=m, h=b[s + 5] << 8 | b[s + 6], w=b[s + 7] << 8 | b[s + 8], comps=comps)
    raise ValueError("no SOF")


def grid(fr, ncomp_scan, c):
    """Columns and rows of a scan's MCU grid (frame MCUs when interleaved, else the component's blocks)."""
    comps = fr["comps"]
    hmax = max(x[1] for x in comps) if len(comps) == 3 else 1
    vmax = max(x[2] for x in comps) if len(comps) == 3 else 1
    if ncomp_scan > 1:
        return -(-fr["w"] // (8 * hmax)), -(-fr["h"] // (8 * vmax))
    h = comps[c][1] if len(comps) == 3 else 1
    v = comps[c][2] if len(comps) == 3 else 1
    return -(-fr["w"] * h // (8 * hmax)), -(-fr["h"] * v // (8 * vmax))


def describe_scans(b):
    """Rows (components, c0, c1, c2, Ss, Se, Ah, Al, restart interval, segments, level) of every scan."""
    fr = frame(b)
    ids = [c[0] for c in fr["comps"]]
    ri, rows = 0, []
    for m, s, e, q in markers(b):
        if m == 0xDD:
            ri = b[s + 4] << 8 | b[s + 5]
        if m != 0xDA:
            continue
        ns = b[s + 4]
        comps = [ids.index(b[s + 5 + 2 * j]) for j in range(ns)]
        ss, se, a = b[s + 5 + 2 * ns], b[s + 6 + 2 * ns], b[s + 7 + 2 * ns]
        data = b[e:q]
        segs = 1 + sum(1 for i in range(len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7)
        level = 1
        for r in rows:
            if set(r[1:1 + r[0]]) & set(comps) and not (r[4] > se or ss > r[5]):
                level = max(level, r[10] + 1)
        rows.append([ns] + comps + [0] * (3 - ns) + [ss, se, a >> 4, a & 15, ri, segs, level])
    return rows


# ----------------------------------------------------------------------------------------------------------------
# Baseline decoder (quantised coefficients only)
# ----------------------------------------------------------------------------------------------------------------

class Bits:
    def __init__(self, data):
        out, i = bytearray(), 0
        while i < len(data):                    # de-stuff; restart markers are not expected here
            out.append(data[i])
            i += 2 if data[i] == 0xFF else 1
        self.v = int.from_bytes(bytes(out) + b"\0\0\0\0", "big")
        self.n = 8 * (len(out) + 4)
        self.p = 0

    def get(self, k):
        r = (self.v >> (self.n - self.p - k)) & ((1 << k) - 1)
        self.p += k
        return r


def huff_lookup(bits, vals):
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[(length, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return codes


def read_sym(br, t):
    code = 0
    for length in range(1, 17):
        code = code << 1 | br.get(1)
        if (length, code) in t:
            return t[(length, code)]
    raise ValueError("bad code")


def extend(v, s):
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v


def coefficients(b):
    """Quantised coefficients of a baseline single-scan file, zig-zag order: per component [rows, cols, 64] over the
    MCU-padded block grid; plus the frame and the DQT segments."""
    fr = frame(b)
    dc, ac, dqt = {}, {}, []
    for m, s, e, q in markers(b):
        if m == 0xDB:
            dqt.append(b[s:e])
        if m == 0xC4:
            o = s + 4
            while o < e:
                tc, th = b[o] >> 4, b[o] & 15
                bits = list(b[o + 1:o + 17])
                (ac if tc else dc)[th] = huff_lookup(bits, list(b[o + 17:o + 17 + sum(bits)]))
                o += 17 + sum(bits)
        if m == 0xDA:
            ns = b[s + 4]
            sel = [(b[s + 6 + 2 * j] >> 4, b[s + 6 + 2 * j] & 15) for j in range(ns)]
            data = b[e:q]
    comps = fr["comps"]
    n = len(comps)
    samp = [(c[1], c[2]) if n == 3 else (1, 1) for c in comps]
    mx, my = grid(fr, n, 0)
    coef = [np.zeros((my * v, mx * h, 64), np.int32) for h, v in samp]
    br, pred = Bits(data), [0] * n
    for y in range(my):
        for x in range(mx):
            for c in range(n):
                h, v = samp[c]
                for bv in range(v):
                    for bh in range(h):
                        blk = coef[c][y * v + bv, x * h + bh]
                        s = read_sym(br, dc[sel[c][0]])
                        pred[c] += extend(br.get(s), s) if s else 0
                        blk[0] = pred[c]
                        k = 1
                        while k < 64:
                            rs = read_sym(br, ac[sel[c][1]])
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                blk[k] = extend(br.get(s), s)
                                k += 1
                            elif r == 15:
                                k += 16
                            else:
                                break
    return fr, coef, dqt


# ----------------------------------------------------------------------------------------------------------------
# Encoder under any scan script
# ----------------------------------------------------------------------------------------------------------------

def gen_table(freq):
    """ITU T.81 K.2: code lengths of the symbols with nonzero frequency, limited to 16 bits; (bits[16], vals)."""
    syms = [s for s in sorted(freq) if freq[s] > 0]
    f = {s: freq[s] for s in syms}
    f[256] = 1
    size = {s: 0 for s in f}
    nxt = {s: None for s in f}
    while True:
        cand = [s for s in f if f[s] > 0]
        if len(cand) < 2:
            break
        v1 = min(cand, key=lambda s: (f[s], -s))
        cand.remove(v1)
        v2 = min(cand, key=lambda s: (f[s], -s))
        f[v1] += f[v2]
        f[v2] = 0
        size[v1] += 1
        t = v1
        while nxt[t] is not None:
            t = nxt[t]
            size[t] += 1
        nxt[t] = v2
        size[v2] += 1
        t = v2
        while nxt[t] is not None:
            t = nxt[t]
            size[t] += 1
    bits = [0] * 33
    for s, n in size.items():
        if n:
            bits[n] += 1
    for i in range(32, 16, -1):                         # limit code lengths to 16 (K.3)
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                        # drop the reserved code point
    vals = [s for n in range(1, 33) for s in sorted(x for x in size if size[x] == n and x != 256)]
    return bits[1:17], vals


def canonical(bits, vals):
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


def nbits(v):
    return int(abs(v)).bit_length()


def encode_scan(fr, coef, comps, ss, se, ah, al, ri, progressive):
    """Events of one scan: ('d', j, sym) / ('a', j, sym) a DC / AC symbol of scan component j, ('b', value, n) raw
    bits, ('r',) a restart marker."""
    ev = []
    samp = [(c[1], c[2]) if len(fr["comps"]) == 3 else (1, 1) for c in fr["comps"]]
    cols, rows = grid(fr, len(comps), comps[0])
    blocks_of = []                                      # per MCU: [(scan component j, block)]
    for m in range(cols * rows):
        y, x = divmod(m, cols)
        if len(comps) == 1:
            blocks_of.append([(0, coef[comps[0]][y, x])])
        else:
            blocks_of.append([(j, coef[c][y * samp[c][1] + bv, x * samp[c][0] + bh])
                              for j, c in enumerate(comps) for bv in range(samp[c][1]) for bh in range(samp[c][0])])
    st = dict(pred=[0, 0, 0], eobrun=0, be=[])

    def flush_eob():
        if st["eobrun"]:
            n = st["eobrun"].bit_length() - 1
            ev.append(("a", 0, n << 4))
            if n:
                ev.append(("b", st["eobrun"] & ((1 << n) - 1), n))
            st["eobrun"] = 0
        ev.extend(("b", bit, 1) for bit in st["be"])
        st["be"] = []

    def value_bits(v):
        n = nbits(v)
        return ("b", v if v >= 0 else v + (1 << n) - 1, n)

    for m, blocks in enumerate(blocks_of):
        if ri and m and m % ri == 0:
            flush_eob()
            ev.append(("r",))
            st["pred"] = [0, 0, 0]
        for j, blk in blocks:
            if not progressive or (ss == 0 and ah == 0):              # DC (sequential or first)
                v = int(blk[0]) >> al
                d = v - st["pred"][j]
                st["pred"][j] = v
                ev.append(("d", j, nbits(d)))
                if d:
                    ev.append(value_bits(d))
                if progressive:
                    continue
            if progressive and ss == 0:                               # DC refinement
                ev.append(("b", (int(blk[0]) >> al) & 1, 1))
                continue
            if not progressive:                                       # sequential AC
                r = 0
                for k in range(1, 64):
                    v = int(blk[k])
                    if v == 0:
                        r += 1
                        continue
                    while r > 15:
                        ev.append(("a", j, 0xF0))
                        r -= 16
                    ev.append(("a", j, (r << 4) | nbits(v)))
                    ev.append(value_bits(v))
                    r = 0
                if r:
                    ev.append(("a", j, 0))
                continue
            vals = [int(blk[k]) for k in range(64)]
            if ah == 0:                                               # AC first
                r = 0
                for k in range(ss, se + 1):
                    v = vals[k]
                    v = (abs(v) >> al) * (1 if v >= 0 else -1)
                    if v == 0:
                        r += 1
                        continue
                    flush_eob()
                    while r > 15:
                        ev.append(("a", 0, 0xF0))
                        r -= 16
                    ev.append(("a", 0, (r << 4) | nbits(v)))
                    ev.append(value_bits(v))
                    r = 0
                if r:
                    st["eobrun"] += 1
                    if st["eobrun"] == 0x7FFF:
                        flush_eob()
                continue
            absv = [abs(v) >> al for v in vals]                       # AC refinement (jcphuff.c encode_mcu_AC_refine)
            eob = max([k for k in range(ss, se + 1) if absv[k] == 1], default=0)
            r, br = 0, []
            for k in range(ss, se + 1):
                t = absv[k]
                if t == 0:
                    r += 1
                    continue
                while r > 15 and k <= eob:
                    flush_eob()
                    ev.append(("a", 0, 0xF0))
                    r -= 16
                    ev.extend(("b", bit, 1) for bit in br)
                    br = []
                if t > 1:
                    br.append(t & 1)
                    continue
                flush_eob()
                ev.append(("a", 0, (r << 4) | 1))
                ev.append(("b", 1 if vals[k] >= 0 else 0, 1))
                ev.extend(("b", bit, 1) for bit in br)
                br, r = [], 0
            if r > 0 or br:
                st["eobrun"] += 1
                st["be"].extend(br)
                if st["eobrun"] == 0x7FFF or len(st["be"]) > 1000 - 64 + 1:
                    flush_eob()
    flush_eob()
    return ev


def write_jpeg(fr, coef, dqt, script, sof):
    """A JPEG of the coefficients under `script`: a list of (components, Ss, Se, Ah, Al, restart interval or None to
    leave DRI as it is).  Optimal Huffman tables per scan, in a DHT before it."""
    progressive = sof == 0xC2
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    for seg in dqt:
        out += seg
    n = len(fr["comps"])
    out += bytes([0xFF, sof]) + (8 + 3 * n).to_bytes(2, "big") + bytes([8]) + fr["h"].to_bytes(2, "big") + \
        fr["w"].to_bytes(2, "big") + bytes([n])
    for cid, h, v, tq in fr["comps"]:
        out += bytes([cid, h << 4 | v, tq])
    cur_ri = 0
    for comps, ss, se, ah, al, ri in script:
        if ri is not None:
            out += b"\xff\xdd\x00\x04" + ri.to_bytes(2, "big")
            cur_ri = ri
        ev = encode_scan(fr, coef, comps, ss, se, ah, al, cur_ri, progressive)
        keys = sorted({e[:2] for e in ev if e[0] in "da"})      # one table per class and scan component
        freq = {k: {} for k in keys}
        for e in ev:
            if e[0] in "da":
                freq[e[:2]][e[2]] = freq[e[:2]].get(e[2], 0) + 1
        slot = {k: i for i, k in enumerate(sorted(k for k in keys if k[0] == "d"))}
        slot.update({k: i for i, k in enumerate(sorted(k for k in keys if k[0] == "a"))})
        codes = {}
        dht = bytearray()
        for k in keys:
            bits, vals = gen_table(freq[k])
            codes[k] = canonical(bits, vals)
            dht += bytes([(1 if k[0] == "a" else 0) << 4 | slot[k]]) + bytes(bits) + bytes(vals)
        if dht:
            out += b"\xff\xc4" + (len(dht) + 2).to_bytes(2, "big") + dht
        out += b"\xff\xda" + (6 + 2 * len(comps)).to_bytes(2, "big") + bytes([len(comps)])
        for j, c in enumerate(comps):
            td, ta = slot.get(("d", j), 0), slot.get(("a", j), 0)
            out += bytes([fr["comps"][c][0], td << 4 | ta])
        out += bytes([ss, se, ah << 4 | al])
        acc, nacc, data, rst = 0, 0, bytearray(), 0

        def put(v, k):
            nonlocal acc, nacc
            acc = acc << k | v
            nacc += k
            while nacc >= 8:
                byte = (acc >> (nacc - 8)) & 0xFF
                data.append(byte)
                if byte == 0xFF:
                    data.append(0)
                nacc -= 8
            acc &= (1 << nacc) - 1

        def pad():
            if nacc:
                put((1 << (8 - nacc)) - 1, 8 - nacc)
        for e in ev:
            if e[0] == "b":
                if e[2]:
                    put(e[1], e[2])
            elif e[0] == "r":
                pad()
                data += bytes([0xFF, 0xD0 + (rst & 7)])
                rst += 1
            else:
                code, length = codes[e[:2]][e[2]]
                put(code, length)
        pad()
        out += data
    return bytes(out + b"\xff\xd9")


def transcode(src, script, sof=0xC2):
    """`src` (a baseline single-scan file) re-encoded under `script`; Pillow must decode both to the same pixels."""
    fr, coef, dqt = coefficients(src)
    out = write_jpeg(fr, coef, dqt, script, sof)
    assert np.array_equal(pixels(out), pixels(src)), "transcoded file decodes differently"
    return out


DEFAULT = [([0, 1, 2], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([2], 1, 63, 0, 1), ([1], 1, 63, 0, 1), ([0], 6, 63, 0, 2),
           ([0], 1, 63, 2, 1), ([0, 1, 2], 0, 0, 1, 0), ([2], 1, 63, 1, 0), ([1], 1, 63, 1, 0), ([0], 1, 63, 1, 0)]


def script(scans, ri=None):
    return [(c, ss, se, ah, al, ri if i == 0 else None) for i, (c, ss, se, ah, al) in enumerate(scans)]


def patch_sos(b, index, ss=None, se=None, ah=None, al=None):
    """b with the index-th SOS header's Ss / Se / Ah / Al replaced."""
    m = [x for x in markers(b) if x[0] == 0xDA][index]
    ns = b[m[1] + 4]
    o = m[1] + 5 + 2 * ns
    out = bytearray(b)
    a = out[o + 2]
    out[o] = out[o] if ss is None else ss
    out[o + 1] = out[o + 1] if se is None else se
    out[o + 2] = ((a >> 4 if ah is None else ah) << 4) | (a & 15 if al is None else al)
    return bytes(out)


def main():
    cases = []          # (name, kind, status, reason, data)

    def ok(name, data):
        cases.append((name, "ok", OK, "", data))

    photo = synthetic.synthetic_photo(41, 53, seed=7)
    for sub, tag in ((0, "444"), (1, "422"), (2, "420")):
        for w in range(1, 18):
            ok(f"{tag} progressive 7x{w}", enc(synthetic.synthetic_photo(7, w, seed=w), quality=75, subsampling=sub,
                                                progressive=True))
        for h in range(1, 18):
            ok(f"{tag} progressive {h}x9", enc(synthetic.synthetic_photo(h, 9, seed=50 + h), quality=90, subsampling=sub,
                                                progressive=True))
        for q in (5, 25, 50, 75, 90, 95, 100):
            ok(f"{tag} progressive q{q}", enc(photo, quality=q, subsampling=sub, progressive=True))
        ok(f"{tag} progressive restart blocks 3", enc(photo, quality=80, subsampling=sub, progressive=True,
                                                       restart_marker_blocks=3))
        ok(f"{tag} progressive restart rows 1", enc(photo, quality=80, subsampling=sub, progressive=True,
                                                     restart_marker_rows=1))
    gray = synthetic.synthetic_photo(45, 67, seed=11)[..., 1].copy()
    for q in (5, 75, 100):
        ok(f"gray progressive q{q}", enc(gray, quality=q, progressive=True))
    for h, w in ((1, 1), (1, 17), (17, 1), (9, 13)):
        ok(f"gray progressive {h}x{w}", enc(np.ascontiguousarray(gray[:h, :w]), quality=80, progressive=True))
    ok("gray progressive restart blocks 2", enc(gray, quality=80, progressive=True, restart_marker_blocks=2))
    ok("420 progressive 640x640 q90", enc(synthetic.synthetic_photo(640, 640, seed=1000), quality=90, subsampling=2,
                                          progressive=True))
    yy, xx = np.mgrid[0:3000, 0:4000]
    big = np.stack([xx * 255 // 3999, yy * 255 // 2999, (xx + yy) // 7 % 256], -1).astype(np.uint8)
    ok("420 progressive 4000x3000 q50", enc(big, quality=50, subsampling=2, progressive=True))

    # transcoded scripts
    src = {sub: enc(synthetic.synthetic_photo(40, 56, seed=31), quality=80, subsampling=sub) for sub in (0, 1, 2)}
    gsrc = enc(np.ascontiguousarray(gray[:24, :40]), quality=85)
    flat = enc(np.full((48, 64, 3), 90, np.uint8), quality=85, subsampling=2)
    for sub, tag in ((0, "444"), (1, "422"), (2, "420")):
        for order, oname in (([0, 1, 2], "Y Cb Cr"), ([2, 0, 1], "Cr Y Cb")):
            for sof in (0xC0, 0xC1):
                ok(f"{tag} SOF{sof - 0xC0} non-interleaved {oname}",
                   transcode(src[sub], script([([c], 0, 63, 0, 0) for c in order]), sof))
        ok(f"{tag} SOF0 Y then CbCr", transcode(src[sub], script([([0], 0, 63, 0, 0), ([1, 2], 0, 63, 0, 0)]), 0xC0))
        ok(f"{tag} spectral selection", transcode(src[sub], script(
            [([0, 1, 2], 0, 0, 0, 0)] + [([c], a, b, 0, 0) for c in (0, 1, 2) for a, b in ((1, 2), (3, 9), (10, 63))])))
        ok(f"{tag} DC per component", transcode(src[sub], script(
            [([c], 0, 0, 0, 0) for c in (0, 1, 2)] + [([c], 1, 63, 0, 0) for c in (2, 1, 0)])))
        ok(f"{tag} band 10-63 in pieces", transcode(src[sub], script(
            [([0, 1, 2], 0, 0, 0, 1), ([0, 1, 2], 0, 0, 1, 0)] +
            [([c], a, b, 0, 0) for c in (0, 1, 2) for a, b in ((1, 9), (10, 20), (21, 40), (41, 63))])))
        ok(f"{tag} default script restart 2", transcode(src[sub], script(DEFAULT, ri=2)))
    deep = [([0, 1, 2], 0, 0, 0, 13)] + [([0, 1, 2], 0, 0, a + 1, a) for a in range(12, -1, -1)]
    for c in (0, 1, 2):
        deep += [([c], 1, 63, 0, 5)] + [([c], 1, 63, a + 1, a) for a in range(4, -1, -1)]
    ok("420 deep successive approximation", transcode(src[2], script(deep)))
    per_coef = [([0], 0, 0, 0, 1)] + [([0], k, k, 0, 1) for k in range(1, 64)] + [([0], 0, 0, 1, 0)] + \
        [([0], k, k, 1, 0) for k in range(1, 64)]
    ok("gray one scan per coefficient", transcode(gsrc, script(per_coef)))
    ok("420 flat long EOB runs", transcode(flat, script(DEFAULT)))
    ok("420 flat long EOB runs restart 5", transcode(flat, script(DEFAULT, ri=5)))
    dri = [(c, ss, se, ah, al, ri) for (c, ss, se, ah, al), ri in
           zip(DEFAULT, (None, 3, None, 0, None, 7, 1, 0, None, 2))]
    ok("420 DRI changed and removed between scans", transcode(src[2], dri))
    ok("444 component order differs from the frame", transcode(src[0], script(
        [([0, 1, 2], 0, 0, 0, 0), ([2], 1, 63, 0, 0), ([0], 1, 63, 0, 0), ([1], 1, 63, 0, 0)])))

    # refused and corrupt files
    pil = enc(synthetic.synthetic_photo(40, 56, seed=31), quality=80, subsampling=2, progressive=True)

    def rej(name, status, reason, data):
        cases.append((name, "reject", status, reason, data))
    fr, coef, dqt = coefficients(src[2])
    rej("incomplete progression", UNSUPPORTED, "incomplete progression", write_jpeg(fr, coef, dqt, script(DEFAULT[:9]), 0xC2))
    rej("bogus progression: AC before DC", UNSUPPORTED, "before its DC scan",
        write_jpeg(fr, coef, dqt, script([DEFAULT[1], DEFAULT[0]] + DEFAULT[2:]), 0xC2))
    rej("bogus progression: wrong Ah", UNSUPPORTED, "bogus progression",
        write_jpeg(fr, coef, dqt, script(DEFAULT[:5] + [([0], 1, 63, 3, 2)] + DEFAULT[6:]), 0xC2))
    for name, kw in (("DC scan with Se 5", dict(index=0, se=5)), ("Ss > Se", dict(index=1, ss=6, se=5)),
                     ("Se 64", dict(index=2, se=64)), ("Al != Ah - 1", dict(index=5, ah=2, al=0)),
                     ("Al 14", dict(index=0, al=14))):
        rej(f"bad progression: {name}", BAD_HEADER, "bad progression", patch_sos(pil, **kw))
    m = [x for x in markers(pil) if x[0] == 0xDA][1]        # the first AC scan, given two components
    ids = frame(pil)["comps"]
    hdr = b"\xff\xda\x00\x0a\x02" + bytes([ids[0][0], pil[m[1] + 6], ids[1][0], pil[m[1] + 6]]) + pil[m[2] - 3:m[2]]
    rej("bad progression: AC scan of two components", BAD_HEADER, "bad progression", pil[:m[1]] + hdr + pil[m[2]:])
    many = deep[:14] + [([c], k, k, 0, 1) for c in (0, 1, 2) for k in range(1, 64)] + [([0], k, k, 1, 0) for k in range(1, 64)]
    rej("too many scans", UNSUPPORTED, "more than 256 scans", write_jpeg(fr, coef, dqt, script(many), 0xC2))
    cases.append(("truncated progressive file", "corrupt", NO_EOI, "EOI", pil[:len(pil) * 2 // 3]))
    last = [x for x in markers(pil) if x[0] == 0xDA][-1]
    cases.append(("bad code in an AC refinement scan", "corrupt", BAD_CODE, "",
                  pil[:last[2] + 4] + b"\xff\x00" * 8 + pil[last[2] + 20:]))
    first = [x for x in markers(pil) if x[0] == 0xDA][0]
    mid = (first[2] + first[3]) // 2
    mid += pil[mid - 1] == 0xFF
    cases.append(("marker inside a DC scan", "corrupt", BAD_RST, "segments", pil[:mid] + b"\xff\xd0" + pil[mid:]))

    n = len(cases)
    out = {"count": np.array(n), "pillow": np.array(Image.__version__),
           "libjpeg_turbo": np.array(str(features.version("libjpeg_turbo"))),
           "name": np.array([c[0] for c in cases]), "kind": np.array([c[1] for c in cases]),
           "status": np.array([c[2] for c in cases], dtype=np.int32), "reason": np.array([c[3] for c in cases]),
           "shape": np.zeros((n, 3), dtype=np.int32)}
    jpg_off, px_off, scan_off, jpgs, pxs, rows = [0], [0], [0], [], [], []
    for k, (name, kind, status, reason, data) in enumerate(cases):
        jpgs.append(np.frombuffer(data, dtype=np.uint8))
        jpg_off.append(jpg_off[-1] + len(data))
        px = None
        if kind == "ok":
            rows += describe_scans(data)
            px = pixels(data)
            out["shape"][k] = px.shape
            if px.shape[0] * px.shape[1] > FULL_PIXELS:
                out[f"sha{k}"] = np.frombuffer(hashlib.sha256(px.tobytes()).digest(), dtype=np.uint8)
                out[f"sample{k}"] = px[::37, ::23].copy()
                px = None
        scan_off.append(len(rows))
        if px is not None:
            pxs.append(px.reshape(-1))
        px_off.append(px_off[-1] + (px.size if px is not None else 0))
    out["jpg"] = np.concatenate(jpgs)
    out["jpg_off"] = np.array(jpg_off, dtype=np.int64)
    out["px"] = np.concatenate(pxs)
    out["px_off"] = np.array(px_off, dtype=np.int64)
    out["scans"] = np.array(rows, dtype=np.int32)
    out["scan_off"] = np.array(scan_off, dtype=np.int64)
    path = os.path.join(ROOT, "tests", "golden", "jpeg_multiscan.npz")
    np.savez_compressed(path, **out)
    print(path, n, "cases", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
