"""pg_optics_xi (csrc/optics.cu) against the numpy restatement of reference prototype.py + sklearn OPTICS-xi
(tests/optics_oracle.py), per cell: ordering, predecessor and labels exactly; core and reachability within 4 ulp of the
distance (CUDA's fp64 sin/asin are not glibc's) plus one quantum of np.around(x, 15), since a distance a few ulp from a
rounding boundary of around() lands on the neighbouring multiple of 1e-15; inf exactly."""
import numpy as np
import pytest
import torch

import optics_oracle as O
from pigeon_b200 import PigeonB200Error, prototypes as P
from pigeon_b200._lib import check, current_stream_ptr, load, ptr

pytestmark = pytest.mark.gpu

SMEM_POINTS = 2800   # optics.cu: larger cells keep their per-point state in the workspace


def _cell(rng, n, kind="clusters"):
    if kind == "identical":
        return np.tile(rng.uniform([-5, 40], [5, 50]), (n, 1))
    if kind == "noise":
        return rng.uniform([-1, 45], [1, 47], (n, 2))
    centres = rng.uniform([-3, 42], [3, 48], (6, 2))
    x = centres[rng.integers(0, 6, n)] + rng.normal(0, 0.03, (n, 2))
    if n > 40 and kind == "dups":
        x[rng.integers(0, n, n // 4)] = x[rng.integers(0, n, 1)]
    return x


def _close(g, r):
    """|g - r| <= 4 ulp(r) + 1e-15 (one quantum of np.around(., 15))."""
    return np.abs(g - r) <= 4 * np.spacing(r) + 1e-15


def _check_cell(x, m, xi, labels, graph, lo, hi):
    ref = O.optics_xi(x, m, xi)
    assert np.array_equal(labels[lo:hi], ref["labels"])
    if ref["ordering"] is None:
        assert np.all(graph["ordering"][lo:hi] == -1) and np.all(graph["pred"][lo:hi] == -1)
        return ref
    assert np.array_equal(graph["ordering"][lo:hi], ref["ordering"])
    assert np.array_equal(graph["pred"][lo:hi], ref["pred"])
    for k in ("core", "reach"):
        g, r = graph[k][lo:hi], ref[k]
        assert np.array_equal(np.isinf(g), np.isinf(r)), k
        fin = np.isfinite(r)
        assert _close(g[fin], r[fin]).all(), k
    return ref


@pytest.mark.parametrize("m,xi", [(100, 0.1), (3, 0.15)])
def test_cells_match_oracle(m, xi):
    rng = np.random.default_rng(7 + m)
    specs = [(0, "clusters"), (1, "clusters"), (m - 1, "clusters"), (m, "clusters"), (m + 1, "clusters"),
             (400, "dups"), (700, "noise"), (300, "identical"), (1500, "clusters")]
    cells = [_cell(rng, n, kind) for n, kind in specs]
    off = np.cumsum([0] + [len(c) for c in cells])
    x = np.concatenate(cells)
    labels, graph = P.optics_xi_csr(x, off, m, xi, return_graph=True)
    for c, cx in enumerate(cells):
        _check_cell(cx, m, xi, labels, graph, off[c], off[c + 1])


def test_one_launch_equals_one_cell_at_a_time():
    rng = np.random.default_rng(3)
    sizes = list(rng.integers(0, 6000, 14)) + [0, 6000, 1, 99, 100, 2800, 2801]
    cells = [_cell(rng, int(n), "dups" if i % 3 == 0 else "clusters") for i, n in enumerate(sizes)]
    off = np.cumsum([0] + [len(c) for c in cells])
    labels, graph = P.optics_xi_csr(np.concatenate(cells), off, 100, 0.1, return_graph=True)
    for c, cx in enumerate(cells):
        one, g1 = P.optics_xi_csr(cx, [0, len(cx)], 100, 0.1, return_graph=True)
        assert np.array_equal(labels[off[c]:off[c + 1]], one)
        for k in g1:
            assert np.array_equal(graph[k][off[c]:off[c + 1]], g1[k], equal_nan=True), k


def test_cell_above_shared_memory_threshold():
    n = 20000
    assert n > SMEM_POINTS, f"a {n}-point cell must take the workspace path (threshold {SMEM_POINTS} points)"
    x = _cell(np.random.default_rng(11), n, "dups")
    labels, graph = P.optics_xi_csr(x, [0, n], 100, 0.1, return_graph=True)
    ref = _check_cell(x, 100, 0.1, labels, graph, 0, n)
    assert len(set(ref["labels"].tolist())) > 1


def test_two_runs_bit_identical_and_point_order():
    rng = np.random.default_rng(5)
    x = np.concatenate([_cell(rng, n) for n in (900, 3000, 50, 4000)])
    cells = np.repeat([4, 2, 9, 7], [900, 3000, 50, 4000])
    perm = rng.permutation(len(x))
    a = P.optics_xi(x[perm], cells[perm], 100, 0.1, return_graph=True)
    b = P.optics_xi(x[perm], cells[perm], 100, 0.1, return_graph=True)
    assert np.array_equal(a[0], b[0])
    for k in a[1]:
        assert a[1][k].tobytes() == b[1][k].tobytes()
    # per-point labels equal the cell-by-cell result in the caller's order
    for c in (4, 2, 9, 7):
        sel = cells[perm] == c
        assert np.array_equal(a[0][sel], P.optics_xi_csr(x[perm][sel], [0, int(sel.sum())], 100, 0.1))


def test_bad_arguments():
    lib = load()
    dev = torch.device("cuda")
    x = torch.zeros(4, 2, dtype=torch.float64, device=dev)
    off = torch.tensor([0, 4], dtype=torch.int64, device=dev)
    lab = torch.empty(4, dtype=torch.int32, device=dev)
    need = int(lib.pg_optics_workspace_bytes(4, 1))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)

    def call(m=2, xi=0.1, wsb=need):
        return lib.pg_optics_xi(ptr(x), 4, ptr(off), 1, 4, m, xi, ptr(ws), wsb, ptr(lab), None, None, None, None,
                                current_stream_ptr())
    assert call() == 0
    for kw in (dict(m=1), dict(m=0), dict(xi=0.0), dict(xi=1.0), dict(xi=float("nan")), dict(wsb=need - 1)):
        assert call(**kw) != 0 and lib.pg_last_error(), kw
    with pytest.raises(PigeonB200Error):
        check(call(m=1), "pg_optics_xi")
    with pytest.raises(PigeonB200Error, match="finite"):
        P.optics_xi(np.array([[0.0, np.nan], [1.0, 2.0]]), [0, 0], 2, 0.1)
    with pytest.raises(PigeonB200Error, match="min_samples"):
        P.optics_xi(np.zeros((3, 2)), [0, 0, 0], 1, 0.1)
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", ["m100", "m3", "clf_sample"])
def test_generate_writes_reference_csv_and_loads_into_refiner(name, tmp_path):
    """ProtoDataset.generate() on the GPU writes the CSV the unmodified reference wrote (tests/golden/prototypes.npz),
    and ProtoRefiner(proto_path=..., dataset_path=...) loads it and runs forward."""
    import os

    import pandas as pd
    from datasets import Dataset, DatasetDict

    from pigeon_b200 import ProtoRefiner
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prototypes.npz"))
    m, xi, seed, use_clf, sample = g[f"{name}/args"]
    xy, sel = g[f"{name}/lnglat"], g[f"{name}/selection_train"]
    df = pd.DataFrame(dict(lng=xy[:, 0], lat=xy[:, 1], selection=np.where(sel, "train", "val")))
    if not use_clf:
        df["geocell_idx"] = g[f"{name}/cells"]
    n_train, D = int(sel.sum()), 1024
    rng = np.random.default_rng(0)
    clf = g[f"{name}/cells"] if use_clf else np.zeros(n_train, np.int64)
    DatasetDict(train=Dataset.from_dict({"labels_clf": clf.tolist(),
                                         "embedding": rng.standard_normal((n_train, D)).astype(np.float32).tolist(),
                                         "labels": xy[sel].astype(np.float32).tolist()})).save_to_disk(str(tmp_path / "emb"))
    out = tmp_path / "protos.csv"
    if sample:
        np.random.seed(int(seed))
    P.ProtoDataset(df, str(tmp_path / "emb"), str(out), (int(m), float(xi)), int(sample) or None).generate()
    assert out.read_bytes() == g[f"{name}/csv"].tobytes()

    protos = pd.read_csv(out)
    cells = np.unique(protos["geocell_idx"].astype(int))
    refiner = ProtoRefiner(topk=1, max_refinement=1000, temperature=1.6, proto_path=str(out),
                           dataset_path=str(tmp_path / "emb")).eval()
    B = 3
    cand = torch.tensor(np.resize(cells, (B, 1)), dtype=torch.int64)
    _, ll, cell = refiner(torch.randn(B, D), initial_preds=torch.zeros(B, 2), candidate_cells=cand,
                          candidate_probs=torch.ones(B, 1))
    torch.cuda.synchronize()
    assert cell.cpu().tolist() == cand[:, 0].tolist() and torch.isfinite(ll).all()
