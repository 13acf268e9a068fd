"""Labelled training and embedding datasets from raw splits: reference preprocessing/dataset_preprocessing.py
(`preprocess`, :262-332) with the geocell labels located on the GPU.

`preprocess(dataset, geocell_path)` takes the `DatasetDict` the reference's `generate_finetune_dataset` returns (per
split: `image` (and `image_2`..`image_4`), `lng`, `lat`, the six `*_reg` columns named `elevation`, `population`,
`temp_avg`, `temp_diff`, `prec_avg`, `prec_diff`, `index`, `labels_climate`, optionally `heading` and `labels_month`) and
returns the dataset `run.py finetune`, `finetune --embeddings`, `python -m pigeon_b200.prototypes` and
`ProtoRefiner(dataset_path=...)` read, column for column and dtype for dtype as the reference writes it:

- `heading` becomes float64 [4, 2]: sin / cos of the heading plus k * 90 degrees (only when `geocell_path` is
  `config.GEOCELL_PATH`, as in the reference, :281-282);
- `labels` is float64 [lng, lat] and `labels_clf` the int64 geocell: the lowest-index cell that covers the point, else the
  nearest cell (GEOS point-to-segment distance, lowest index on ties), one `CountryIndex.locate` call per split over
  the geocell polygons (csrc/geo_metrics.cu); `lng` and `lat` are dropped;
- with `multi_task`, `labels_multi_task` is float64 [6] of the six regression columns, which are dropped in every case;
- with an `embedder`, the `embedding` column is joined from the `{split}.npy` / `{split}_indices.npy` files `run.py embed`
  writes, with the reference's arithmetic, and the image columns are dropped.

Deviations (DESIGN.md §1): without an embedder the image columns stay encoded instead of becoming `pixel_values` (the
reference's `AutoFeatureExtractor(CLIP_MODEL)` call raises there); the result is then a raw split that `run.py finetune -l`
and `run.py evaluate -l` read from its image files.  Nothing is saved mid-function (the reference writes
`data/hf_landmarks`); the caller saves.  Invalid polygons are located by the crossing rule instead of taking the
`pygeos.GEOSException` path; the lowest covering index wins where cells overlap; no multiprocess `map` is needed.

    python -m pigeon_b200.dataset_preprocessing RAW_DATASET_DIR GEOCELL_CSV OUTPUT_DIR [--embeddings DIR] [--multitask]
"""
from __future__ import annotations

import argparse
import os
import re
from typing import List, Optional, Tuple

import numpy as np

from . import config
from .metrics import CountryIndex, _ring

MULTI_TASK_COLUMNS = ('elevation', 'population', 'temp_avg', 'temp_diff', 'prec_avg', 'prec_diff')   # :176-177, :328
VIEW_COLUMNS = ('image_2', 'image_3', 'image_4')

_TOKEN = re.compile(r"\(|\)|,|[^\s(),]+")


# ------------------------------------------------------------------------------------------------------------- WKT
def parse_wkt(text: str, where: str = "geometry") -> List[List[np.ndarray]]:
    """A WKT POLYGON or MULTIPOLYGON -> parts, each a list of rings (shell first, then holes) as float64 [n, 2] arrays.
    Positions with Z and / or M keep x and y.  Numbers are read with Python's correctly rounded `float()`, as GEOS's
    reader rounds them.  EMPTY, other geometry types, unclosed rings, rings of fewer than 4 positions and non-finite
    coordinates raise ValueError naming `where`."""
    if not isinstance(text, str):
        raise ValueError(f"{where}: expected WKT text (got {type(text).__name__})")
    toks = _TOKEN.findall(text)                    # every character but whitespace is in some token
    kind = toks[0].upper() if toks else ""
    i = 1
    if i < len(toks) and toks[i].upper() in ("Z", "M", "ZM"):
        i += 1
    if kind not in ("POLYGON", "MULTIPOLYGON"):
        raise ValueError(f"{where}: geometry must be a POLYGON or MULTIPOLYGON (got {kind or 'nothing'})")
    if i < len(toks) and toks[i].upper() == "EMPTY":
        raise ValueError(f"{where}: empty geometry")

    def expect(t):
        nonlocal i
        if i >= len(toks) or toks[i] != t:
            got = toks[i] if i < len(toks) else "end of text"
            raise ValueError(f"{where}: malformed WKT: expected {t!r}, got {got!r}")
        i += 1

    def seq(item):                    # '(' item (',' item)* ')'
        expect("(")
        out = [item()]
        while i < len(toks) and toks[i] == ",":
            expect(",")
            out.append(item())
        expect(")")
        return out

    def position():
        nonlocal i
        vals = []
        while i < len(toks) and toks[i] not in ("(", ")", ","):
            try:
                if "_" in toks[i]:
                    raise ValueError
                vals.append(float(toks[i]))
            except ValueError:
                raise ValueError(f"{where}: malformed WKT: {toks[i]!r} is not a number") from None
            i += 1
        if not 2 <= len(vals) <= 4:
            raise ValueError(f"{where}: malformed WKT: a position needs 2 to 4 coordinates (got {len(vals)})")
        return vals[:2]

    ring = lambda: _ring(seq(position), where)
    polygon = lambda: seq(ring)
    parts = [polygon()] if kind == "POLYGON" else seq(polygon)
    if i != len(toks):
        raise ValueError(f"{where}: malformed WKT: unexpected {toks[i]!r} after the geometry")
    return parts


def geometries_to_csr(geoms) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """[parts per geometry] (parse_wkt's output) -> the CSR layout of `metrics.parse_geojson`:
    (verts f64 [V, 2], ring_off i64 [R + 1], part_ring_off i64 [P + 1], geom_part_off i64 [G + 1])."""
    verts, ring_off, part_ring_off, geom_part_off = [], [0], [0], [0]
    for parts in geoms:
        for rings in parts:
            for a in rings:
                verts.append(a)
                ring_off.append(ring_off[-1] + len(a))
            part_ring_off.append(len(ring_off) - 1)
        geom_part_off.append(len(part_ring_off) - 1)
    if not verts:
        raise ValueError("geocells: no polygons")
    i64 = lambda x: np.asarray(x, dtype=np.int64)
    return np.concatenate(verts), i64(ring_off), i64(part_ring_off), i64(geom_part_off)


def parse_geocells(path):
    """The geocell CSV `preprocess` reads (reference load_geocell_df, :48-58: `lng`, `lat` and a WKT `polygon` column;
    a path or a pandas DataFrame) -> ((verts, ring_off, part_ring_off, geom_part_off), lnglat f64 [C, 2])."""
    import pandas as pd
    df = path if isinstance(path, pd.DataFrame) else pd.read_csv(path)
    for col in ('lng', 'lat', 'polygon'):
        if col not in df.columns:
            raise ValueError(f"geocells: missing column {col!r}")
    geoms = [parse_wkt(text, f"geocell row {k}") for k, text in enumerate(df['polygon'].tolist())]
    lnglat = np.ascontiguousarray(df[['lng', 'lat']].to_numpy(dtype=np.float64))
    return geometries_to_csr(geoms), lnglat


def load_geocells(path, device=None) -> Tuple[CountryIndex, np.ndarray]:
    """The geocell CSV -> (its polygons as a device `CountryIndex`, the cells' (lng, lat) float64 [C, 2] in file order,
    which `SuperGuessr(geocells=...)` takes)."""
    csr, lnglat = parse_geocells(path)
    return CountryIndex(*csr, device=device), lnglat


# ---------------------------------------------------------------------------------------------------------- columns
def heading_features(heading) -> np.ndarray:
    """preprocess_heading (:96-114) over a column: degrees -> float64 [N, 4, 2] of (sin, cos) at heading + k pi / 2
    mod 2 pi, k = 0..3, in the reference's operation order (k = 0 is not reduced)."""
    h = np.deg2rad(np.asarray(heading, dtype=np.float64))
    out = np.empty(h.shape + (4, 2), dtype=np.float64)
    out[..., 0, 0], out[..., 0, 1] = np.sin(h), np.cos(h)
    for k in (1, 2, 3):
        a = (h + (k * (np.pi / 2))) % (2 * np.pi)
        out[..., k, 0], out[..., k, 1] = np.sin(a), np.cos(a)
    return out


def multi_task_labels(columns) -> np.ndarray:
    """generate_label_mt (:166-180) over columns: [N, 6] with numpy's dtype for the row's Python scalars (float64
    whenever one column holds floats)."""
    cols = [np.asarray(c) for c in columns]
    dtype = np.float64 if any(c.dtype.kind == 'f' for c in cols) else np.result_type(*cols)
    return np.stack([c.astype(dtype) for c in cols], axis=1)


def join_embeddings(num_samples: int, embeds: np.ndarray, indices: np.ndarray, where: str = "embeddings") -> np.ndarray:
    """The reference's join (:295-304): row i of the split gets `embeds.reshape(-1, D)[argsort(indices.flatten()[:n])][i]`.
    D is taken from the file (the reference hard-codes 1024) and must be config.CLIP_EMBED_DIM."""
    embeds, indices = np.asarray(embeds), np.asarray(indices)
    if embeds.ndim != 2:
        raise ValueError(f"{where}: expected a 2-D [rows, D] embedding array (got shape {embeds.shape})")
    D = embeds.shape[1]
    if D != config.CLIP_EMBED_DIM:
        raise ValueError(f"{where}: embeddings have D = {D}, the model takes config.CLIP_EMBED_DIM = {config.CLIP_EMBED_DIM}")
    flat = indices.reshape(-1)
    if len(flat) < num_samples or len(embeds) < num_samples:
        raise ValueError(f"{where}: {len(embeds)} embeddings and {len(flat)} indices for {num_samples} rows")
    order = np.argsort(flat[:num_samples])
    return embeds.reshape((-1, D))[order]


def _arrow(a: np.ndarray):
    """A numpy array [N, ...] -> a pyarrow column of nested fixed-size lists (the dataset's List(..., length=k))."""
    import pyarrow as pa
    a = np.ascontiguousarray(a)
    arr = pa.array(a.reshape(-1))
    for d in a.shape[:0:-1]:
        arr = pa.FixedSizeListArray.from_arrays(arr, d)
    return arr


def _columns(split, names) -> dict:
    """Scalar columns as stored (the numpy and torch formats would hand out float64 as float32)."""
    table = split.select_columns(list(names)).with_format('arrow')[:]
    return {n: table.column(n).to_numpy() for n in names}


def _set_column(split, name: str, values: np.ndarray):
    """`split` with column `name` set to `values`: in place where it exists (as `map` updates it), appended otherwise."""
    order = list(split.column_names)
    if name in order:
        split = split.remove_columns([name])
    else:
        order.append(name)
    return split.add_column(name, _arrow(values)).select_columns(order)


def _require(dataset, columns, why: str) -> None:
    for split_name, split in dataset.items():
        missing = [c for c in columns if c not in split.column_names]
        if missing:
            raise ValueError(f"split {split_name!r} lacks column(s) {missing} ({why})")


def preprocess(dataset, geocell_path: str, embedder=None, multi_task: bool = False,
               embeddings_dir: str = 'data/landmark_embeddings'):
    """reference preprocess (:262-332) -> a DatasetDict in torch format (see the module docstring).  `embedder` selects
    the embedding branch: its embeddings are the files `run.py embed` wrote to `embeddings_dir` (the reference reads
    the same files; its own embedding call is commented out, :288-289).  A split that lacks a column the reference
    reads or removes raises ValueError before any work is done."""
    import datasets
    heading = geocell_path == config.GEOCELL_PATH                                   # :281
    image_cols = ['image'] + (list(VIEW_COLUMNS) if heading else [])               # :307-309
    _require(dataset, ('lng', 'lat'), 'the geocell labels')
    _require(dataset, MULTI_TASK_COLUMNS, 'the multi-task columns, removed in every case')
    if heading:
        _require(dataset, ('heading',), f'heading features are made under {config.GEOCELL_PATH}')
    if embedder is not None:
        _require(dataset, image_cols, 'the image columns the embedding branch drops')
    index, _ = load_geocells(geocell_path)
    out = {}
    for split_name, split in dataset.items():
        split = split.with_format(None)
        if heading:                                                                 # :282
            split = _set_column(split, 'heading', heading_features(_columns(split, ['heading'])['heading']))
        if embedder is not None:                                                    # :292-311
            where = os.path.join(embeddings_dir, split_name)
            emb = join_embeddings(len(split), np.load(f'{where}.npy'), np.load(f'{where}_indices.npy'), where)
            split = _set_column(split, 'embedding', emb).remove_columns(image_cols)
        c = _columns(split, ['lng', 'lat'])                                         # :320-322
        labels = np.stack([c['lng'].astype(np.float64), c['lat'].astype(np.float64)], axis=1)
        cells, _, _ = index.locate(labels)
        split = _set_column(split, 'labels', labels)
        split = _set_column(split, 'labels_clf', cells.cpu().numpy().astype(np.int64))
        split = split.remove_columns(['lng', 'lat'])
        if multi_task:                                                              # :325-326
            c = _columns(split, MULTI_TASK_COLUMNS)
            split = _set_column(split, 'labels_multi_task', multi_task_labels([c[k] for k in MULTI_TASK_COLUMNS]))
        out[split_name] = split.remove_columns(list(MULTI_TASK_COLUMNS))            # :328-329
    return datasets.DatasetDict(out).with_format('torch')                           # :331


# -------------------------------------------------------------------------------------------------------------- CLI
def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m pigeon_b200.dataset_preprocessing",
                                 description=__doc__.split("\n\n")[0])
    ap.add_argument("raw_dataset_dir", help="DatasetDict saved with save_to_disk (generate_finetune_dataset's output)")
    ap.add_argument("geocell_csv", help=f"geocell CSV (lng, lat, WKT polygon); heading features are made when this is "
                                        f"{config.GEOCELL_PATH!r}")
    ap.add_argument("output_dir")
    ap.add_argument("--embeddings", default=None, metavar="DIR",
                    help="join the embeddings `run.py embed` wrote to DIR and drop the image columns")
    ap.add_argument("--multitask", action="store_true", help="add labels_multi_task")
    return ap


def main(argv: Optional[List[str]] = None) -> None:
    from datasets import DatasetDict
    a = build_parser().parse_args(argv)
    dataset = DatasetDict.load_from_disk(a.raw_dataset_dir)
    kw = {} if a.embeddings is None else dict(embedder=True, embeddings_dir=a.embeddings)
    preprocess(dataset, a.geocell_csv, multi_task=a.multitask, **kw).save_to_disk(a.output_dir)


if __name__ == "__main__":
    main()
