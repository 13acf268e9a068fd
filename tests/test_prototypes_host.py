"""Prototype builder on the CPU: the numpy OPTICS-xi oracle (tests/optics_oracle.py) against scikit-learn's arrays recorded
from the unmodified reference ProtoDataset (tests/golden/prototypes.npz, tools/make_prototype_golden.py), the decision
margins that make the GPU's exact comparison meaningful, and the host side of pigeon_b200.prototypes (CSR grouping,
aggregation, CSV) reproducing the reference's CSV byte for byte from the recorded labels."""
import os

import numpy as np
import pytest

import optics_oracle as O
from pigeon_b200 import PigeonB200Error, prototypes as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prototypes.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _scenario(g, name):
    m, xi, seed, use_clf, sample = g[f"{name}/args"]
    train_xy = g[f"{name}/lnglat"][g[f"{name}/selection_train"]]
    idx, cell = g[f"{name}/frame_index"], g[f"{name}/frame_cell"]
    return dict(m=int(m), xi=float(xi), seed=int(seed), use_clf=bool(use_clf), sample=int(sample) or None,
                xy=train_xy[idx], cell=cell, labels=g[f"{name}/labels"])


def _cells(s):
    """The reference's slices: groupby('geocell_idx') order, rows in frame order."""
    order, ids, off = P.group_by_cell(s["cell"])
    return [(ids[c], order[off[c]:off[c + 1]]) for c in range(len(ids))]


SCENARIOS = ["m100", "m3", "clf_sample"]


@pytest.mark.parametrize("name", SCENARIOS)
def test_oracle_equals_sklearn_exactly(golden, name):
    s = _scenario(golden, name)
    sizes, k, fit = golden[f"{name}/fit_sizes"], 0, 0
    for _, rows in _cells(s):
        ref = O.optics_xi(s["xy"][rows], s["m"], s["xi"])
        assert np.array_equal(ref["labels"], s["labels"][rows])
        if len(rows) < s["m"]:
            assert np.all(ref["labels"] == 0)
            continue
        n = sizes[fit]
        assert n == len(rows)
        sl = slice(k, k + n)
        for key in ("ordering", "core", "reach", "pred"):
            assert np.array_equal(ref[key], golden[f"{name}/{key}"][sl]), key
        assert np.array_equal(ref["labels"], golden[f"{name}/fit_labels"][sl])
        k, fit = k + n, fit + 1
    assert fit == len(sizes)


@pytest.mark.parametrize("name", SCENARIOS)
def test_decision_margins(golden, name):
    s = _scenario(golden, name)
    for cell, rows in _cells(s):
        ref = O.optics_xi(s["xy"][rows], s["m"], s["xi"])
        assert ref["order_gap"] >= 1e-12, (cell, ref["order_gap"])
        assert ref["xi_gap"] >= 1e-12, (cell, ref["xi_gap"])


def _train_frame(golden, name, s):
    import pandas as pd
    xy, sel = golden[f"{name}/lnglat"], golden[f"{name}/selection_train"]
    df = pd.DataFrame(dict(lng=xy[:, 0], lat=xy[:, 1], selection=np.where(sel, "train", "val")))
    if not s["use_clf"]:
        df["geocell_idx"] = golden[f"{name}/cells"]
    return df


@pytest.mark.parametrize("name", SCENARIOS)
def test_generate_reproduces_reference_csv(golden, name, tmp_path):
    from datasets import Dataset, DatasetDict
    s = _scenario(golden, name)
    clf = golden[f"{name}/cells"] if s["use_clf"] else np.zeros(1, np.int64)
    DatasetDict(train=Dataset.from_dict({"labels_clf": clf.tolist()})).save_to_disk(str(tmp_path / "emb"))
    ds = P.ProtoDataset(_train_frame(golden, name, s), str(tmp_path / "emb"), str(tmp_path / "protos.csv"),
                        (s["m"], s["xi"]), s["sample"])
    order, _, off = P.group_by_cell(s["cell"])

    def clusterer(lnglat, cell_off):   # the golden labels in place of the GPU, after checking what it was handed
        assert np.array_equal(cell_off, off)
        assert np.array_equal(lnglat, s["xy"][order])
        return s["labels"][order]
    if s["sample"]:
        np.random.seed(s["seed"])
    ds.generate(clusterer=clusterer)
    assert np.array_equal(ds.df.index.to_numpy(), golden[f"{name}/frame_index"])
    assert (tmp_path / "protos.csv").read_bytes() == golden[f"{name}/csv"].tobytes()


def test_group_by_cell_is_stable():
    order, ids, off = P.group_by_cell([7, 2, 7, 7, 2, 5])
    assert order.tolist() == [1, 4, 5, 0, 2, 3] and ids.tolist() == [2, 5, 7] and off.tolist() == [0, 2, 3, 6]


def test_rejects_bad_arguments_without_a_device():
    with pytest.raises(PigeonB200Error, match="min_samples"):
        P.optics_xi_csr(np.zeros((3, 2)), [0, 3], 1, 0.1)
    with pytest.raises(PigeonB200Error, match="finite"):
        P.optics_xi_csr(np.array([[0.0, np.inf]]), [0, 1], 2, 0.1)
    with pytest.raises(PigeonB200Error, match="cell_off"):
        P.optics_xi_csr(np.zeros((3, 2)), [0, 2], 2, 0.1)


def test_cli_parses_reference_arguments(monkeypatch):
    seen = {}

    class Fake:
        def __init__(self, df, emb, out, args, sample):
            seen.update(emb=emb, out=out, args=args, sample=sample, rows=len(df))

        def generate(self):
            seen["generated"] = True
    import pandas as pd
    monkeypatch.setattr(P, "ProtoDataset", Fake)
    monkeypatch.setattr(pd, "read_csv", lambda p: pd.DataFrame(dict(lng=[0.0], lat=[0.0], selection=["train"])))
    P.main(["meta.csv", "embdir", "out.csv", "--min-samples", "3", "--xi", "0.15", "--sample", "10"])
    assert seen == dict(emb="embdir", out="out.csv", args=(3, 0.15), sample=10, rows=1, generated=True)
