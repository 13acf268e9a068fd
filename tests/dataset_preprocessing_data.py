"""Synthetic inputs of `pigeon_b200.dataset_preprocessing.preprocess`, shared by tools/make_dataset_preprocessing_golden.py
(which runs the reference's `preprocess` on them) and the tests.

Geocells (lng / lat degrees): a cell with two holes, one of them filled by another cell; a MultiPolygon; two cells that
share an edge vertex for vertex; an overlapping pair; a cell whose first edge lies far from its other edges; cells in
the corners at +-180 / +-90.  Points: strictly inside cells and inside holes, exactly on shared edges and vertices, at sea
(the nearest-cell fallback, including an exact distance tie), at +-180 / +-90, and seeded uniform ones.  Splits have the
columns of the reference's `create_dataset_split` with four views (tiny PNGs), headings 0, 90, 359.999 and values of 360
and more among them.
"""
from __future__ import annotations

import io

import numpy as np

SPLITS = ("train", "val", "test")
MT = ("elevation", "population", "temp_avg", "temp_diff", "prec_avg", "prec_diff")
VIEWS = ("image", "image_2", "image_3", "image_4")
D = 1024


def _sq(x0, y0, x1, y1):
    return [[x0, y0], [x1, y0], [x1, y1], [x0, y1], [x0, y0]]


def cells():
    """Per cell: parts, each a list of rings (shell, then holes), as lists of [lng, lat]."""
    return [
        [[_sq(0, 0, 10, 10), _sq(3, 3, 5, 5)[::-1], _sq(6, 6, 8, 8)[::-1]]],        # 0: two holes
        [[_sq(12, 0, 14, 2)], [_sq(16, 0, 18, 2)]],                                   # 1: MultiPolygon
        [[[[0, 12], [5, 12], [5.5, 14], [5, 16], [0, 16], [0, 12]]]],                  # 2, 3: shared border
        [[[[5, 12], [10, 12], [10, 16], [5, 16], [5.5, 14], [5, 12]]]],
        [[_sq(20, 20, 26, 26)]],                                                      # 4, 5: overlapping
        [[_sq(24, 24, 30, 30)]],
        [[[[-60, -40], [-20, -40], [-20, -10], [-58, -12], [-60, -40]]]],              # 6: far first edge
        [[_sq(170, 80, 180, 90)]],                                                    # 7, 8: corners of the plane
        [[_sq(-180, -90, -170, -80)]],
        [[_sq(3, 3, 5, 5)]],                                                          # 9: fills hole 1 of cell 0
    ]


def wkt(parts) -> str:
    num = lambda v: repr(float(v))
    ring = lambda r: "(" + ", ".join(f"{num(x)} {num(y)}" for x, y in r) + ")"
    poly = lambda p: "(" + ", ".join(ring(r) for r in p) + ")"
    if len(parts) == 1:
        return "POLYGON " + poly(parts[0])
    return "MULTIPOLYGON (" + ", ".join(poly(p) for p in parts) + ")"


def geocell_frame():
    """The geocell CSV as a DataFrame: lng, lat (the mean of the first shell's vertices) and the WKT polygon."""
    import pandas as pd
    cs = cells()
    centre = np.asarray([np.mean(np.asarray(c[0][0][:-1], dtype=np.float64), axis=0) for c in cs])
    return pd.DataFrame(dict(lng=centre[:, 0], lat=centre[:, 1], polygon=[wkt(c) for c in cs]))


SPECIAL = [
    (5, 1), (2, 8), (4, 4), (7, 7), (3, 4), (3, 3), (13, 1), (17, 1.5), (15, 1),       # inside, holes, hole edges
    (5, 12), (5.5, 14), (5.25, 13), (5, 16), (2.5, 12), (0, 14), (10, 14),              # shared vertices and edges
    (25, 25), (24, 24), (26, 26), (22, 22), (28, 28), (-21, -39), (-59, -38),           # overlap, far first edge
    (11, 1), (11, 11), (-5, 50), (40, 0), (-100, 0), (15, 3),                           # at sea; (11, 1) is a tie
    (180, 85), (-180, -85), (175, 90), (-175, -90), (180, 90), (-180, 90), (180, -90), (-180, 0), (0, -90),
]
HEADINGS = [0.0, 90.0, 359.999, 360.0, 450.0, 720.5, 180.0, 270.0]


def inputs(split: str, seed: int) -> dict:
    """The non-image columns of one split, as the reference's create_dataset_split types them."""
    rng = np.random.default_rng(seed)
    k = SPLITS.index(split)
    pts = np.asarray(SPECIAL[k::3] + SPECIAL[3 * (k == 0):][:4], dtype=np.float64)
    rand = np.concatenate([rng.uniform([-65, -45], [35, 30], (10, 2)), rng.uniform([-180, -90], [180, 90], (4, 2))])
    lnglat = np.concatenate([pts, rand])
    n = len(lnglat)
    heading = np.concatenate([HEADINGS, rng.uniform(0, 360, max(n - len(HEADINGS), 0))])[:n]
    out = dict(lng=lnglat[:, 0], lat=lnglat[:, 1], heading=heading,
               index=np.sort(rng.choice(1000, n, replace=False)).astype(np.int64) + 1000 * k,
               labels_climate=rng.integers(0, 28, n).astype(np.int64), labels_month=rng.integers(1, 13, n).astype(np.int64))
    for j, c in enumerate(MT):
        out[c] = rng.normal(j, 1 + j, n)
    return out


def embedding_files(split_inputs: dict, seed: int):
    """`run.py embed`'s files for a split: {split}.npy [n + 2, D] float32 and {split}_indices.npy, the split's index
    values in a shuffled order plus two trailing duplicates (a padded distributed sampler).  Every row is its file
    position repeated with a period-4 pattern, which compresses well."""
    rng = np.random.default_rng(seed)
    idx = split_inputs["index"]
    order = rng.permutation(len(idx))
    indices = np.concatenate([idx[order], idx[order[:2]]]).astype(np.int64)
    rows = np.arange(len(indices), dtype=np.float32)[:, None] * 4 + (np.arange(D) % 4).astype(np.float32)[None, :]
    return rows, indices


def png(seed: int) -> bytes:
    from PIL import Image
    rng = np.random.default_rng(seed)
    f = io.BytesIO()
    Image.fromarray(rng.integers(0, 256, (6, 5, 3), dtype=np.uint8)).save(f, "PNG")
    return f.getvalue()


def raw_split(cols: dict, seed: int):
    """A datasets.Dataset with the reference's raw columns: four encoded views plus `cols`."""
    import datasets
    n = len(cols["lng"])
    data = {v: [{"bytes": png(seed * 100003 + 4 * r + j), "path": None} for r in range(n)] for j, v in enumerate(VIEWS)}
    data.update((k, np.asarray(v).tolist()) for k, v in cols.items())
    feats = {v: datasets.Image() for v in VIEWS}
    for k, v in cols.items():
        v = np.asarray(v)
        value = datasets.Value("int64" if v.dtype.kind == "i" else "float64" if v.dtype == np.float64 else "float32")
        feats[k] = value if v.ndim == 1 else datasets.List(value)
    return datasets.Dataset.from_dict(data, features=datasets.Features(feats))


def raw_dataset(inputs_by_split: dict, seed: int = 0):
    import datasets
    return datasets.DatasetDict({s: raw_split(inputs_by_split[s], seed + k) for k, s in enumerate(SPLITS)})
