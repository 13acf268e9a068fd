"""Generate tests/golden/prototypes.npz by running the UNMODIFIED reference `ProtoDataset`
(dataset_creation/prototype/prototype.py) with scikit-learn's OPTICS on seeded synthetic geocells.

Authoring-time only: it needs the reference checkout (PIGEON_REFERENCE, default /root/reference) and is never run by tests.
Around the unmodified module:
  - oracle/reference_shim.py provides its `config` and `preprocessing` (haversine_matrix_np);
  - `geopandas` is a stub module (only the reference's __main__ uses it) and `pandarallel` a stub whose `initialize` does
    nothing, with `DataFrameGroupBy.parallel_apply` set to `apply`: cells are clustered one after another;
  - `DatasetDict` in the module is a stand-in whose 'train' split returns a torch tensor for `['labels_clf']`, as the
    datasets 2.x the reference pins did (datasets 4 returns a Column without `.numpy()`);
  - the run happens in a scratch directory with a `tmp/` subdirectory for its `np.save('tmp/clusters_100.npy')`;
  - `OPTICS.fit_predict` is wrapped to record sklearn's ordering_, core_distances_, reachability_ and predecessor_ per cell.
Version drift: the reference's env.yml pins scikit-learn 1.1.1; the arrays here come from the installed version (stored
in the file).  Whether the two differ on this path is unverified.

    python tools/make_prototype_golden.py
"""
from __future__ import annotations

import importlib.util
import io
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "prototypes.npz")


def _cell(rng, n, kind):
    if kind == "identical":
        return np.tile(rng.uniform([-5, 40], [5, 50]), (n, 1))
    if kind == "noise":
        return rng.uniform([-1, 45], [1, 47], (n, 2))
    centres = rng.uniform([-3, 42], [3, 48], (5, 2))
    x = centres[rng.integers(0, 5, n)] + rng.normal(0, 0.02 if kind == "separated" else 0.05, (n, 2))
    if kind == "dups":
        x[rng.integers(0, n, n // 5)] = x[rng.integers(0, n, 1)]
    return x


# (name, min_samples, xi, seed, [(geocell, n, kind)], use labels_clf, sample)
SCENARIOS = [
    ("m100", 100, 0.1, 1, [(0, 1, "clusters"), (2, 99, "clusters"), (3, 100, "clusters"), (4, 101, "separated"),
                           (6, 600, "dups"), (7, 150, "identical"), (9, 400, "noise"), (11, 2000, "separated")], False, None),
    ("m3", 3, 0.15, 2, [(0, 1, "clusters"), (1, 2, "clusters"), (3, 3, "clusters"), (4, 4, "clusters"),
                        (5, 300, "dups"), (8, 40, "identical"), (10, 250, "noise"), (12, 700, "separated")], False, None),
    ("clf_sample", 100, 0.1, 3, [(0, 500, "separated"), (1, 30, "clusters"), (2, 900, "dups"), (5, 300, "noise")],
     True, 1500),
]


def frame(seed, cells, use_clf):
    """Synthetic metadata: train rows interleaved across cells, plus a few 'val' rows the reference drops."""
    import pandas as pd
    rng = np.random.default_rng(seed)
    pts = [_cell(rng, n, kind) for _, n, kind in cells]
    cell = np.concatenate([np.full(n, c) for c, n, _ in cells])
    xy = np.concatenate(pts)
    perm = rng.permutation(len(xy))
    df = pd.DataFrame(dict(lng=xy[perm, 0], lat=xy[perm, 1], selection="train"))
    if not use_clf:
        df["geocell_idx"] = cell[perm]
    val = pd.DataFrame(dict(lng=rng.uniform(0, 1, 7), lat=rng.uniform(0, 1, 7), selection="val"))
    if not use_clf:
        val["geocell_idx"] = 0
    at = rng.integers(0, len(df), 7)
    parts, last = [], 0
    for k, a in enumerate(np.sort(at)):
        parts += [df.iloc[last:a], val.iloc[k:k + 1]]
        last = a
    parts.append(df.iloc[last:])
    return pd.concat(parts, ignore_index=True), cell[perm]


def load_reference():
    from oracle import reference_shim
    reference_shim.install()
    sys.modules.setdefault("geopandas", types.ModuleType("geopandas"))
    pl = types.ModuleType("pandarallel")
    pl.pandarallel = types.SimpleNamespace(initialize=lambda **kw: None)
    sys.modules["pandarallel"] = pl
    from pandas.core.groupby.generic import DataFrameGroupBy
    DataFrameGroupBy.parallel_apply = DataFrameGroupBy.apply
    path = os.path.join(reference_shim.REF, "dataset_creation", "prototype", "prototype.py")
    spec = importlib.util.spec_from_file_location("reference_prototype", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import sklearn
    import torch
    from sklearn.cluster import OPTICS
    ref = load_reference()
    record = []
    real_fit_predict = OPTICS.fit_predict

    def fit_predict(self, X, y=None):
        labels = real_fit_predict(self, X, y)
        record.append((len(X), self.ordering_.copy(), self.core_distances_.copy(), self.reachability_.copy(),
                       self.predecessor_.copy(), labels.copy()))
        return labels
    OPTICS.fit_predict = fit_predict

    out = dict(sklearn_version=np.array(sklearn.__version__), scenarios=np.array([s[0] for s in SCENARIOS]))
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "tmp"))
        os.chdir(tmp)
        try:
            for name, m, xi, seed, cells, use_clf, sample in SCENARIOS:
                df, clf = frame(seed, cells, use_clf)
                train = {"labels_clf": torch.from_numpy(clf.astype(np.int64))}
                ref.DatasetDict = types.SimpleNamespace(load_from_disk=lambda p, t=train: {"train": t})
                record.clear()
                ds = ref.ProtoDataset(df, "embeddings", "protos.csv", cluster_args=(m, xi), sample=sample)
                if sample:
                    np.random.seed(seed)
                ds.generate()
                csv = open("protos.csv", "rb").read()
                g = ds.df
                out[f"{name}/lnglat"] = df[["lng", "lat"]].to_numpy()
                out[f"{name}/selection_train"] = (df["selection"] == "train").to_numpy()
                out[f"{name}/cells"] = clf if use_clf else df["geocell_idx"].to_numpy()
                out[f"{name}/args"] = np.array([m, xi, seed, int(use_clf), sample or 0], dtype=np.float64)
                out[f"{name}/csv"] = np.frombuffer(csv, dtype=np.uint8)
                out[f"{name}/frame_index"] = g.index.to_numpy()
                out[f"{name}/frame_cell"] = g["geocell_idx"].to_numpy()
                out[f"{name}/labels"] = g["cluster"].to_numpy().astype(np.int64)
                # sklearn's arrays per clustered cell, in groupby order, concatenated
                sizes = np.array([r[0] for r in record], dtype=np.int64)
                out[f"{name}/fit_sizes"] = sizes
                for k, key in enumerate(("ordering", "core", "reach", "pred", "fit_labels")):
                    out[f"{name}/{key}"] = np.concatenate([r[k + 1] for r in record]) if record else np.zeros(0)
                print(name, len(g), "points,", len(record), "cells through OPTICS,", csv.count(b"\n") - 1, "prototypes")
        finally:
            os.chdir(old)
            OPTICS.fit_predict = real_fit_predict
    buf = io.BytesIO()
    np.savez_compressed(buf, **out)
    open(OUT, "wb").write(buf.getvalue())
    print(OUT, len(buf.getvalue()), "bytes")


if __name__ == "__main__":
    main()
