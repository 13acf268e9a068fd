"""Prototype table builder: reference dataset_creation/prototype/prototype.py (`ProtoDataset`) with its per-geocell
OPTICS-xi clustering on the GPU (`pg_optics_xi`, csrc/optics.cu).

`ProtoDataset(...).generate()` writes the CSV (geocell_idx, cluster, lng, lat, count, indices) that
`ProtoRefiner(proto_path=..., dataset_path=...)` loads.  The clustering of all geocells is one `pg_optics_xi` call; its
labels equal `OPTICS(min_samples, xi=xi, metric='precomputed').fit_predict(D)` per cell, D being the reference's fp64
haversine matrix (prototype.py:121-133).  Deliberate deviations (DESIGN.md §1): no `tmp/clusters_100.npy` side file,
no pandarallel, labels map back by position instead of the reference's per-row frame scan, and min_samples < 2 is
rejected rather than read as a fraction of the cell.

    python -m pigeon_b200.prototypes METADATA_CSV EMBEDDING_DATASET_DIR OUTPUT_CSV [--min-samples 100] [--xi 0.1]
                                     [--sample N]
"""
from __future__ import annotations

import argparse
from typing import List, Optional, Tuple

import numpy as np

from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr

DEFAULT_CLUSTER_ARGS = (100, 0.1)   # prototype.py:35; PIGEON's own setting is (3, 0.15)


def group_by_cell(cells) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Stable CSR grouping of points by cell id -> (order, cell_ids, cell_off): points order[cell_off[c]:cell_off[c+1]]
    belong to cell_ids[c] (ascending), in their original relative order."""
    cells = np.asarray(cells)
    order = np.argsort(cells, kind="stable")
    cell_ids, counts = np.unique(cells[order], return_counts=True)
    cell_off = np.zeros(len(cell_ids) + 1, dtype=np.int64)
    np.cumsum(counts, out=cell_off[1:])
    return order, cell_ids, cell_off


def optics_xi_csr(lnglat, cell_off, min_samples: int, xi: float, return_graph: bool = False):
    """OPTICS-xi labels of points already grouped by cell (lnglat [N, 2] degrees, cell c = rows cell_off[c]:cell_off[c+1])
    -> labels int64 [N] (cell-local; -1 = noise; 0 everywhere in a cell of fewer than min_samples points).  With
    return_graph, also a dict of sklearn's per-cell arrays at the cell's rows: ordering, core, reach, pred."""
    import torch
    lnglat = np.ascontiguousarray(np.asarray(lnglat, dtype=np.float64).reshape(-1, 2))
    cell_off = np.ascontiguousarray(np.asarray(cell_off, dtype=np.int64))
    N, C = lnglat.shape[0], len(cell_off) - 1
    if C < 0 or cell_off[0] != 0 or cell_off[-1] != N or np.any(np.diff(cell_off) < 0):
        raise PigeonB200Error("optics_xi: cell_off must rise from 0 to the number of points")
    if not np.isfinite(lnglat).all():
        raise PigeonB200Error("optics_xi: coordinates must be finite")
    if int(min_samples) != min_samples or min_samples < 2:
        raise PigeonB200Error(f"optics_xi: min_samples must be an integer >= 2 (got {min_samples})")
    if not torch.cuda.is_available():
        raise PigeonB200Error("optics_xi needs a CUDA device (there is no CPU path)")
    lib = load()
    dev = torch.device("cuda", torch.cuda.current_device())
    x = torch.from_numpy(lnglat).to(dev)
    off = torch.from_numpy(cell_off).to(dev)
    labels = torch.empty(N, dtype=torch.int32, device=dev)
    graph = None
    if return_graph:
        graph = dict(ordering=torch.empty(N, dtype=torch.int64, device=dev), core=torch.empty(N, dtype=torch.float64, device=dev),
                     reach=torch.empty(N, dtype=torch.float64, device=dev), pred=torch.empty(N, dtype=torch.int64, device=dev))
    ws = torch.empty(max(int(lib.pg_optics_workspace_bytes(N, C)), 1), dtype=torch.uint8, device=dev)
    max_cell = int(np.diff(cell_off).max()) if C > 0 else 0
    g = graph or {}
    check(lib.pg_optics_xi(ptr(x), N, ptr(off), C, max_cell, int(min_samples), float(xi), ptr(ws), ws.numel(), ptr(labels),
                           ptr(g.get("ordering")), ptr(g.get("reach")), ptr(g.get("core")), ptr(g.get("pred")),
                           current_stream_ptr()), "pg_optics_xi")
    out = labels.cpu().numpy().astype(np.int64)
    if return_graph:
        return out, {k: v.cpu().numpy() for k, v in graph.items()}
    return out


def optics_xi(lnglat, cells, min_samples: int = DEFAULT_CLUSTER_ARGS[0], xi: float = DEFAULT_CLUSTER_ARGS[1],
              return_graph: bool = False):
    """Per-cell OPTICS-xi of points with cell id `cells` [N] (any order; grouped stably on the host) -> labels int64 [N]
    in the caller's point order.  With return_graph, also (graph, order, cell_off): sklearn's arrays in grouped order
    (see optics_xi_csr), the grouping permutation and the CSR offsets."""
    lnglat = np.asarray(lnglat, dtype=np.float64).reshape(-1, 2)
    order, _, cell_off = group_by_cell(cells)
    res = optics_xi_csr(lnglat[order], cell_off, min_samples, xi, return_graph)
    grouped, graph = res if return_graph else (res, None)
    labels = np.empty_like(grouped)
    labels[order] = grouped
    return (labels, graph, order, cell_off) if return_graph else labels


def write_prototypes(df, output_file: str) -> None:
    """prototype.py:79-92 on a frame that already holds 'cluster': per-(cell, cluster) mean lng/lat, count and the frame
    index labels of its members, noise dropped, to_csv(index=False)."""
    centroids = df.groupby(['geocell_idx', 'cluster']).agg(lng=('lng', 'mean'), lat=('lat', 'mean'), count=('lng', len),
                                                           indices=('lng', lambda s: s.index.values.tolist()))
    centroids = centroids.reset_index(drop=False)
    centroids = centroids.loc[centroids['cluster'] != -1].copy()
    centroids.to_csv(output_file, index=False)


def cluster_column(df, min_samples: int, xi: float, clusterer=None) -> np.ndarray:
    """The reference's 'cluster' column (prototype.py:71-77): each row's label within its geocell slice, the slices
    taken in groupby('geocell_idx') order with rows in frame order.  `clusterer(lnglat, cell_off)` -> grouped labels
    defaults to the GPU (optics_xi_csr)."""
    keys = df['geocell_idx'].to_numpy()
    order, _, cell_off = group_by_cell(keys)
    lnglat = df[['lng', 'lat']].to_numpy(dtype=np.float64)[order]
    grouped = clusterer(lnglat, cell_off) if clusterer else optics_xi_csr(lnglat, cell_off, min_samples, xi)
    labels = np.empty(len(keys), dtype=np.int64)
    labels[order] = grouped
    return labels


class ProtoDataset:
    def __init__(self, df, embedding_path: str, output_file: str,
                 cluster_args: Tuple[float, float] = DEFAULT_CLUSTER_ARGS, sample: Optional[int] = None):
        """prototype.py:38-68: the train rows of `df`, clustered per geocell with OPTICS(min_samples, xi) into the
        prototype CSV `output_file`.  Without a 'geocell_idx' column the cells come from the embedding dataset's
        'labels_clf'.  `sample` draws df.sample(sample) from numpy's global RNG, as the reference does."""
        from datasets import DatasetDict
        m, xi = cluster_args
        if int(m) != m or m < 2:
            raise PigeonB200Error(f"ProtoDataset: min_samples must be an integer >= 2 (got {m})")
        if not 0.0 < xi < 1.0:
            raise PigeonB200Error(f"ProtoDataset: xi must lie in (0, 1) (got {xi})")
        self.df = df[df['selection'] == 'train'].copy().reset_index(drop=True)
        self.embeddings = DatasetDict.load_from_disk(embedding_path)['train']
        self.output = output_file
        self.cluster_args = cluster_args
        self._sample = sample
        if 'geocell_idx' not in self.df.columns:
            self.df['labels_clf'] = np.nan
            train_cell_idx = np.asarray(self.embeddings.with_format('numpy')['labels_clf'])
            self.df.loc[self.df['selection'] == 'train', 'geocell_idx'] = train_cell_idx

    def generate(self, clusterer=None) -> None:
        """prototype.py:70-92: sample, cluster every geocell (one pg_optics_xi call), aggregate, write the CSV."""
        if self._sample:
            self.df = self.df.sample(self._sample).copy()
        m, xi = self.cluster_args
        self.df['cluster'] = cluster_column(self.df, int(m), float(xi), clusterer)
        write_prototypes(self.df, self.output)


def main(argv: Optional[List[str]] = None) -> None:
    """prototype.py:167-171 with the paths and cluster arguments on the command line."""
    import pandas as pd
    ap = argparse.ArgumentParser(prog="python -m pigeon_b200.prototypes", description=__doc__.split("\n\n")[0])
    ap.add_argument("metadata_csv")
    ap.add_argument("embedding_dataset_dir")
    ap.add_argument("output_csv")
    ap.add_argument("--min-samples", type=int, default=DEFAULT_CLUSTER_ARGS[0])
    ap.add_argument("--xi", type=float, default=DEFAULT_CLUSTER_ARGS[1])
    ap.add_argument("--sample", type=int, default=None)
    a = ap.parse_args(argv)
    ProtoDataset(pd.read_csv(a.metadata_csv), a.embedding_dataset_dir, a.output_csv, (a.min_samples, a.xi),
                 a.sample).generate()


if __name__ == "__main__":
    main()
