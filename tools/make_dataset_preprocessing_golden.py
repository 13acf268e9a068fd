"""Generate tests/golden/dataset_preprocessing.npz by running the UNMODIFIED reference
preprocessing/dataset_preprocessing.py (`preprocess`) on the synthetic geocells and raw splits of
tests/dataset_preprocessing_data.py.

Authoring-time only: it needs the reference checkout (PIGEON_REFERENCE, default /root/reference) and is never run by tests.
Around the unmodified module:
  - oracle/reference_shim.py provides its `config`;
  - `geopandas` and `shapely` are stub modules built on tests/metrics_oracle.py's exact point location and GEOS
    point-to-segment distance: `shapely.wkt.loads` returns the oracle geometry of the WKT text the data module wrote,
    `sindex.query(point, predicate='covered_by')` the covering cells in ascending order, `sindex.nearest(point)` the
    nearest cell (lowest index on ties);
  - `pygeos` provides only `GEOSException`, `preprocessing.embed` only a no-op `embed_images` (`accelerate` is not
    installed);
  - `transformers.AutoFeatureExtractor` is a stand-in whose `pixel_values` are one zero per image, so that the
    no-embedder branch, which raises in every transformers release, runs to its end; that column is not recorded;
  - `datasets` maps run in one process (num_proc forced to None).
Each configuration runs in a scratch directory holding the geocell CSV (at config.GEOCELL_PATH, or elsewhere to skip the
heading features) and the `data/landmark_embeddings/{split}.npy` / `{split}_indices.npy` files.

    python tools/make_dataset_preprocessing_golden.py
"""
from __future__ import annotations

import contextlib
import importlib.util
import io
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "dataset_preprocessing.npz")

# name, geocell path (None = config.GEOCELL_PATH), embedding branch, multi_task
CONFIGS = [("emb", None, True, False), ("emb_mt", None, True, True), ("raw", None, False, False),
           ("raw_mt", None, False, True), ("emb_other", "data/other_cells.csv", True, False)]


def stubs(geoms_by_wkt):
    import torch

    class Pt:
        def __init__(self, x, y):
            self.x, self.y = float(x), float(y)

    class SIndex:
        def __init__(self, geoms):
            self.geoms = geoms

        def query(self, p, predicate=None):
            assert predicate == "covered_by"
            return np.asarray([q for q, g in enumerate(self.geoms) if g.locate(p.x, p.y)[0]], dtype=np.int64)

        def nearest(self, p):
            d = [g.distance(p.x, p.y) for g in self.geoms]
            return np.asarray([[0], [int(np.argmin(d))]], dtype=np.int64)

    class GeoDataFrame:
        def __init__(self, df, geometry=None, crs=None):
            self.df = df.df if isinstance(df, GeoDataFrame) else df
            self.geometry = geometry if isinstance(geometry, str) else None

        def set_geometry(self, col):
            self.geometry = col
            return self

        @property
        def index(self):
            return self.df.index

        @property
        def sindex(self):
            assert self.geometry == "polygon"
            return SIndex(list(self.df["polygon"]))

    gpd = types.ModuleType("geopandas")
    gpd.GeoDataFrame = GeoDataFrame
    gpd.points_from_xy = lambda x, y, crs=None: [Pt(a, b) for a, b in zip(x, y)]
    shp = types.ModuleType("shapely")
    shp.__path__ = []
    geo = types.ModuleType("shapely.geometry")
    geo.Point = Pt
    wkt = types.ModuleType("shapely.wkt")
    wkt.loads = lambda text: geoms_by_wkt[text]
    shp.geometry, shp.wkt = geo, wkt
    pygeos = types.ModuleType("pygeos")
    pygeos.GEOSException = type("GEOSException", (Exception,), {})
    embed = types.ModuleType("preprocessing.embed")
    embed.embed_images = lambda *a, **kw: None

    class AutoFeatureExtractor:
        def __init__(self, *a, **kw):
            pass

        def __call__(self, images, return_tensors=None):
            return {"pixel_values": torch.zeros(len(images), 1)}

    import transformers
    transformers.AutoFeatureExtractor = AutoFeatureExtractor
    return {"geopandas": gpd, "geopandas.geodataframe": gpd, "shapely": shp, "shapely.geometry": geo,
            "shapely.wkt": wkt, "pygeos": pygeos, "preprocessing.embed": embed}


def single_process():
    import datasets
    for cls in (datasets.Dataset, datasets.DatasetDict):
        real = cls.map

        def map_(self, *a, _real=real, **kw):
            kw["num_proc"] = None
            return _real(self, *a, **kw)
        cls.map = map_


def column(split, name):
    """A column as stored (arrow), as a numpy array; `pixel_values` and images are not recorded."""
    col = split.with_format("arrow")[:].column(name)
    return np.asarray(col.to_pylist()) if col.type.num_fields or str(col.type).startswith(("list", "fixed")) \
        else col.to_numpy()


def main():
    import datasets
    import metrics_oracle as mo
    import dataset_preprocessing_data as data
    from oracle import reference_shim
    reference_shim.install()
    cfg = sys.modules["config"]
    frame = data.geocell_frame()
    geoms = [mo.Geometry([[np.asarray(r, dtype=np.float64) for r in p] for p in c]) for c in data.cells()]
    sys.modules.update(stubs(dict(zip(frame["polygon"], geoms))))
    single_process()
    datasets.disable_progress_bars()
    spec = importlib.util.spec_from_file_location("ref_dp", os.path.join(reference_shim.REF, "preprocessing",
                                                                         "dataset_preprocessing.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)

    inputs = {s: data.inputs(s, 10 + k) for k, s in enumerate(data.SPLITS)}
    files = {s: data.embedding_files(inputs[s], 20 + k) for k, s in enumerate(data.SPLITS)}
    out = {"geocells_csv": np.frombuffer(frame.to_csv(index=False).encode(), dtype=np.uint8)}
    for s in data.SPLITS:
        for k, v in inputs[s].items():
            out[f"in/{s}/{k}"] = np.asarray(v)
        out[f"in/{s}/embeds"], out[f"in/{s}/indices"] = files[s]
    cwd = os.getcwd()
    for name, path, emb, mt in CONFIGS:
        path = path or cfg.GEOCELL_PATH
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                os.makedirs(os.path.dirname(path), exist_ok=True)
                frame.to_csv(path, index=False)
                os.makedirs("data/landmark_embeddings")
                for s in data.SPLITS:
                    np.save(f"data/landmark_embeddings/{s}.npy", files[s][0])
                    np.save(f"data/landmark_embeddings/{s}_indices.npy", files[s][1])
                dataset = data.raw_dataset(inputs)
                with contextlib.redirect_stdout(io.StringIO()):
                    res = ref.preprocess(dataset, path, embedder=object() if emb else None, multi_task=mt)
            finally:
                os.chdir(cwd)
        out[f"{name}/args"] = np.asarray([path == cfg.GEOCELL_PATH, emb, mt])
        for s in data.SPLITS:
            split = res[s]
            cols = [c for c in split.column_names if c != "pixel_values"]
            out[f"{name}/{s}/columns"] = np.asarray(cols)
            row = split.with_format("torch")[:2]
            out[f"{name}/{s}/torch_dtypes"] = np.asarray([str(row[c].dtype) if hasattr(row[c], "dtype") else "-"
                                                           for c in cols])
            for c in cols:
                if not c.startswith("image"):
                    out[f"{name}/{s}/{c}"] = column(split, c)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
