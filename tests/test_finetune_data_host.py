"""Host side of building the fine-tuning dataset from the metadata CSV: `finetune_data.generate_finetune_dataset` equals
the unmodified reference's splits (tests/golden/finetune_dataset.npz) column for column, dtype for dtype and value for
value; `sample` is drawn from torch's seed; a CSV that lacks a column, or would need GeoAugmentor, raises before any path
is built; and `run.py` routes each form (no -l in every mode, several -l directories, -s, -t, -m, --yfcc, --landmarks)
to the right calls and save paths.  No GPU: every GPU stage is replaced by a recorder here."""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

datasets = pytest.importorskip("datasets")
pd = pytest.importorskip("pandas")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import finetune_dataset_data as data  # noqa: E402

from pigeon_b200 import config, finetune_data  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "finetune_dataset.npz"))


@pytest.fixture(autouse=True)
def _rows_without_torchvision(monkeypatch):
    """datasets' torch formatter imports torchvision.io.VideoReader whenever torchvision is loaded (an earlier test's
    transformers import loads it), and this torchvision has none: format the rows as a process without it does."""
    monkeypatch.delitem(sys.modules, "torchvision", raising=False)


def _build(case, tmp_path, **kw):
    csv = data.write_csv(case, str(tmp_path / f"{case}.csv"))
    kw.setdefault("geo_augment", data.geo_augment(case))
    return finetune_data.generate_finetune_dataset(metadata_path=csv, image_path=data.IMAGE_FOLDER, **kw)


def _record(split) -> dict:
    out = {"columns": split.column_names, "features": {k: repr(v) for k, v in split.features.items()}}
    table = split.with_format("arrow")[:]
    for name, feature in split.features.items():
        col = table.column(name)
        out[name] = (np.array([v["path"] for v in col.to_pylist()]) if isinstance(feature, datasets.Image)
                     else col.to_numpy())
    return out


@pytest.mark.parametrize("case", [c for c in data.CASES if c not in data.FAILING])
def test_splits_equal_the_reference(tmp_path, case):
    ds = _build(case, tmp_path)
    assert list(ds) == ["train", "val", "test"]
    for s in ds:
        got, key = _record(ds[s]), f"{case}/{s}"
        assert got["columns"] == GOLDEN[f"{key}/columns"].tolist()
        assert got["features"] == json.loads(str(GOLDEN[f"{key}/features"]))
        for name in got["columns"]:
            want = GOLDEN[f"{key}/{name}"]
            assert got[name].dtype == want.dtype, (key, name)
            np.testing.assert_array_equal(got[name], want, err_msg=f"{key}/{name}")
    total = sum(len(ds[s]) for s in ds)
    assert total == sum(sel in ("train", "val", "test") for sel in data.SELECTIONS)      # the holdout row is left out


def test_image_and_image_idx_is_a_panorama(tmp_path):
    """`image_idx` counts as an image column, so `image` with `image_idx` takes the panorama branch: the reference then
    fails (it joins the integer ids), and here the missing views are named before any work."""
    assert str(GOLDEN["image_and_idx/error"]) == "TypeError"
    with pytest.raises(ValueError, match=r"image_2.*image_3.*image_4"):
        _build("image_and_idx", tmp_path)
    ds = _build("idx_panorama", tmp_path)
    assert "image_idx" not in ds["train"].column_names and "image_4" in ds["train"].column_names


def test_sample_repeats_under_manual_seed(tmp_path):
    def drawn(seed):
        torch.manual_seed(seed)
        ds = _build("panorama", tmp_path, sample=7)
        return {s: ds[s].with_format("arrow")[:].column("index").to_numpy().tolist() for s in ds}

    a, b, c = drawn(5), drawn(5), drawn(6)
    assert a == b and a != c
    frame = data.frame("panorama")
    for s, idx in a.items():
        assert all(frame["selection"][i] == s for i in idx)                   # `index` is the CSV row's label
    assert sum(len(v) for v in a.values()) <= 7
    torch.manual_seed(5)
    ds = _build("panorama", tmp_path, sample="7")                              # run.py passes -s as a string
    assert {s: ds[s].with_format("arrow")[:].column("index").to_numpy().tolist() for s in ds} == a


def test_sampled_splits_join_their_own_embeddings(tmp_path):
    """The drawn rows keep their CSV order, so `preprocess`'s join (row i takes `embeds[argsort(indices)][i]`) of the
    files the embedding pass writes in row order gives every row its own embedding."""
    from pigeon_b200.dataset_preprocessing import join_embeddings
    for seed in range(4):
        torch.manual_seed(seed)
        ds = _build("panorama", tmp_path, sample=8)
        for s in ds:
            index = ds[s].with_format("arrow")[:].column("index").to_numpy()
            assert index.tolist() == sorted(index.tolist())
            embeds = np.repeat(index[:, None].astype(np.float32), config.CLIP_EMBED_DIM, axis=1)   # row = its index
            joined = join_embeddings(len(index), embeds, index.copy())
            assert joined[:, 0].tolist() == index.tolist()


def test_empty_split_keeps_column_types(tmp_path):
    for case in ("panorama", "single", "idx"):
        frame = data.frame(case)
        frame[frame["selection"] != "test"].to_csv(tmp_path / "m.csv", index=False)
        ds = finetune_data.generate_finetune_dataset(geo_augment=data.geo_augment(case),
                                                     metadata_path=str(tmp_path / "m.csv"), image_path="x")
        assert len(ds["test"]) == 0 and ds["test"].features == ds["train"].features, case


def test_missing_columns_raise_before_any_work(tmp_path, monkeypatch):
    def fail(*a, **kw):
        raise AssertionError("work started")

    monkeypatch.setattr(finetune_data, "create_dataset_split", fail)
    monkeypatch.setattr(finetune_data, "path", SimpleNamespace(join=fail))
    frame = data.frame("panorama")
    for drop, named in ((["temp_avg_reg"], "temp_avg_reg"), (["climate"], "climate or climate_zone"),
                        (["image_3"], "image_3"), (["selection"], "selection"), (["lat"], "lat")):
        frame.drop(columns=drop).to_csv(tmp_path / "m.csv", index=False)
        with pytest.raises(ValueError, match=named):
            finetune_data.generate_finetune_dataset(metadata_path=str(tmp_path / "m.csv"), image_path="x")
    frame = data.frame("single")
    frame.drop(columns=["prec_diff_reg", "climate", "climate_zone"]).to_csv(tmp_path / "m.csv", index=False)
    with pytest.raises(ValueError, match=r"GeoAugmentor.*prec_diff_reg.*climate or climate_zone"):
        finetune_data.generate_finetune_dataset(metadata_path=str(tmp_path / "m.csv"), image_path="x")
    frame.to_csv(tmp_path / "m.csv", index=False)                  # everything there, but nothing to say it is augmented
    with pytest.raises(ValueError, match="geo_augment=False"):
        finetune_data.generate_finetune_dataset(metadata_path=str(tmp_path / "m.csv"), image_path="x")
    frame.rename(columns={"image": "image_url"}).to_csv(tmp_path / "m.csv", index=False)
    with pytest.raises(ValueError, match="'image'"):
        finetune_data.generate_finetune_dataset(geo_augment=False, metadata_path=str(tmp_path / "m.csv"), image_path="x")


def test_unknown_climate_name_raises(tmp_path):
    frame = data.frame("panorama")
    frame.loc[3, "climate"] = "Lunar"
    frame.to_csv(tmp_path / "m.csv", index=False)
    with pytest.raises(ValueError, match="Lunar"):
        finetune_data.generate_finetune_dataset(metadata_path=str(tmp_path / "m.csv"), image_path="x")


def test_config_paths_are_the_references():
    assert config.METADATA_PATH == "data/data_duels.csv"
    assert config.METADATA_PATH_YFCC == "data/data_yfcc_augmented_non_contaminated.csv"
    assert config.METADATA_PATH_LANDMARKS == "data/data_landmarks_aug.csv"
    assert config.IMAGE_PATH_LANDMARKS == "data/benchmarks/google_landmark/jpgs"


# ------------------------------------------------------------------------------------------------------------ run.py
def _labelled_split(n, seed):
    """A split as `preprocess` leaves it without an embedder: encoded views and the label columns."""
    rng = np.random.default_rng(seed)
    views = ("image", "image_2", "image_3", "image_4")
    cols = {v: [{"bytes": b"\xff\xd8", "path": None}] * n for v in views}
    cols.update(labels=rng.uniform(-50, 50, (n, 2)).tolist(), labels_clf=rng.integers(0, 9, n).tolist(),
                index=list(range(seed * 100, seed * 100 + n)))
    feats = datasets.Features({**{v: datasets.Image() for v in views}, "labels": datasets.List(datasets.Value("float64")),
                               "labels_clf": datasets.Value("int64"), "index": datasets.Value("int64")})
    return datasets.Dataset.from_dict(cols, features=feats)


class Recorder:
    """Stand-ins for every stage `run.main` calls, recording their arguments."""

    def __init__(self, monkeypatch, tmp_path):
        import run
        from pigeon_b200 import dataset_preprocessing, training
        self.calls = []
        monkeypatch.chdir(tmp_path)
        for name in ("METADATA_PATH", "METADATA_PATH_YFCC", "METADATA_PATH_LANDMARKS", "IMAGE_PATH", "IMAGE_PATH_YFCC",
                     "IMAGE_PATH_LANDMARKS"):
            monkeypatch.setattr(config, name, name.lower())
        self.raw = datasets.DatasetDict(train=_labelled_split(5, 1), val=_labelled_split(3, 2), test=_labelled_split(2, 3))
        self.generated = datasets.DatasetDict(                                 # what the builder hands `preprocess`
            {k: v.add_column("heading", [90.0] * len(v)) for k, v in self.raw.items()})
        rec = self.calls.append

        def generate(**kw):
            rec(("generate", kw))
            return self.generated

        def preprocess(dataset, geocells, embedder=None, multi_task=False, **kw):
            rec(("preprocess", dict(dataset=dataset, geocells=geocells, embedder=embedder, multi_task=multi_task, **kw)))
            assert dataset is self.generated
            out = datasets.DatasetDict(dict(self.raw))
            real_save = out.save_to_disk
            out.save_to_disk = lambda p: (rec(("save", p)), real_save(os.path.join(str(tmp_path), "saved")))[0]
            return out

        monkeypatch.setattr(finetune_data, "generate_finetune_dataset", generate)
        monkeypatch.setattr(dataset_preprocessing, "preprocess", preprocess)
        monkeypatch.setattr(run, "CLIPEmbedding", lambda *a, **kw: ("embedder", a, kw))
        monkeypatch.setattr(run, "embed_images", lambda m, splits, **kw: rec(("embed_images", m, splits, kw)))
        monkeypatch.setattr(run, "evaluate", lambda name, split, yfcc, landmarks=False, **kw:
                            rec(("evaluate", name, split, dict(kw, yfcc=yfcc, landmarks=landmarks))))
        monkeypatch.setattr(training, "finetune_model", lambda name, ds, **kw: rec(("finetune_model", name, ds, kw)))
        monkeypatch.setattr(training, "finetune_on_embeddings", lambda ds, **kw: rec(("finetune_on_embeddings", ds, kw)))

    def of(self, kind):
        return [c[1:] if len(c) > 2 else c[1] for c in self.calls if c[0] == kind]

    def kinds(self):
        return [c[0] for c in self.calls]


@pytest.mark.parametrize("flags, metadata, images, geocells, saved", [
    ([], "metadata_path", "image_path", config.GEOCELL_PATH, "data/hf_new_VIT"),
    (["-s", "40"], "metadata_path", "image_path", config.GEOCELL_PATH, "data/hf_dataset_40"),
    (["--yfcc"], "metadata_path_yfcc", "image_path_yfcc", config.GEOCELL_PATH_YFCC, config.DATASET_PATH_YFCC),
    (["--landmarks"], "metadata_path_landmarks", "image_path_landmarks", config.GEOCELL_PATH,
     config.DATASET_PATH_LANDMARKS),
    (["--yfcc", "--landmarks", "-s", "3"], "metadata_path_landmarks", "image_path_landmarks", config.GEOCELL_PATH_YFCC,
     config.DATASET_PATH_LANDMARKS),
])
@pytest.mark.parametrize("mode", ["finetune", "embed", "evaluate"])
def test_run_without_load_generates_preprocesses_and_saves(tmp_path, monkeypatch, mode, flags, metadata, images,
                                                            geocells, saved):
    import run
    from pigeon_b200 import benchmark, loops
    r = Recorder(monkeypatch, tmp_path)
    multi = mode != "evaluate"
    argv = [mode, "model.pt", *flags] + (["-m"] if multi else []) + (["-b", "base.pt"] if mode == "evaluate" else [])
    run.main(argv)
    sample = flags[flags.index("-s") + 1] if "-s" in flags else None
    assert r.of("generate") == [dict(sample=sample, metadata_path=metadata, image_path=images)]
    (pre,) = r.of("preprocess")
    assert pre["geocells"] == geocells and pre["multi_task"] is multi
    assert r.of("save") == [saved]
    yfcc = "--yfcc" in flags
    if mode == "embed":
        assert r.kinds() == ["generate", "embed_images", "preprocess", "save", "finetune_on_embeddings"]
        (model, splits, kw), = r.of("embed_images")
        assert model == ("embedder", ("model.pt",), dict(load_checkpoint=True, panorama=not yfcc))
        assert kw == dict(save_dir="data/landmark_embeddings", collate_fn=loops.encoded_image_collate)
        assert pre["embedder"] is True and pre["embeddings_dir"] == "data/landmark_embeddings"
        (ds, kw), = r.of("finetune_on_embeddings")
        assert sorted(ds) == ["test", "train", "val"]
        assert kw == dict(multi_task=True, heading=False, yfcc=yfcc, metrics=None)
    else:
        assert pre["embedder"] is None
    if mode == "finetune":
        (name, ds, kw), = r.of("finetune_model")
        assert name == "model.pt" and all(isinstance(v, benchmark.EncodedRows) for v in ds.values())
        assert len(ds["train"]) == 5 and kw["collate_fn"] is loops.encoded_eval_collate and kw["multi_task"] is True
    if mode == "evaluate":
        (name, split, kw), = r.of("evaluate")
        assert isinstance(split, benchmark.EvalDataset) and len(split) == 3               # val
        assert kw["base_model"] == "base.pt" and kw["yfcc"] is yfcc and kw["landmarks"] is ("--landmarks" in flags)


def test_run_embed_reads_only_image_and_index(tmp_path, monkeypatch):
    import run
    r = Recorder(monkeypatch, tmp_path)
    run.main(["embed", "clip.pt"])
    (_, splits, _), = r.of("embed_images")
    assert sorted(splits) == ["test", "train", "val"]
    for s, split in splits.items():
        assert split.column_names == ["image", "index"] and not split.features["image"].decode
        assert split[0]["image"]["bytes"] == b"\xff\xd8" and split[0]["index"] == r.raw[s].select_columns(["index"])[0]["index"]


def test_run_evaluate_test_flag(tmp_path, monkeypatch):
    import run
    r = Recorder(monkeypatch, tmp_path)
    run.main(["evaluate", "head.pt", "-b", "base.pt", "-t"])
    run.main(["evaluate", "head.pt", "-b", "base.pt", "-t", "--yfcc"])
    run.main(["evaluate", "head.pt", "-b", "base.pt"])
    assert [len(c[1]) for c in r.of("evaluate")] == [2, 2, 3]                            # test, test, val
    r.raw.save_to_disk(str(tmp_path / "d"))
    for flags in ([], ["-t"]):                                    # with -l the choice is today's: test when there is one
        run.main(["evaluate", "head.pt", "-b", "base.pt", "-l", str(tmp_path / "d"), *flags])
        assert len(r.of("evaluate")[-1][1]) == 2
    assert r.kinds().count("generate") == 3


def test_run_load_several_concatenates_train(tmp_path, monkeypatch):
    import run
    from pigeon_b200 import benchmark
    r = Recorder(monkeypatch, tmp_path)
    a = datasets.DatasetDict(train=_labelled_split(4, 1), val=_labelled_split(3, 2), test=_labelled_split(2, 3))
    b = datasets.DatasetDict(train=_labelled_split(6, 4), val=_labelled_split(5, 5), test=_labelled_split(7, 6))
    a.save_to_disk(str(tmp_path / "a"))
    b.save_to_disk(str(tmp_path / "b"))
    run.main(["finetune", config.CLIP_MODEL, "-l", f"{tmp_path / 'a'},{tmp_path / 'b'}", "-m"])
    (_, ds, kw), = r.of("finetune_model")
    assert sorted(ds) == ["test", "train", "val"] and all(isinstance(v, benchmark.EncodedRows) for v in ds.values())
    assert len(ds["train"]) == 10 and len(ds["val"]) == 3 and len(ds["test"]) == 2
    assert [int(ds["train"][i]["labels_clf"]) for i in range(10)] == \
        list(a["train"]["labels_clf"]) + list(b["train"]["labels_clf"])
    assert [int(ds["val"][i]["labels_clf"]) for i in range(3)] == list(a["val"]["labels_clf"])
    run.main(["finetune", "-", "-l", f"{tmp_path / 'b'},{tmp_path / 'a'}", "--embeddings"])
    (ds, _), = r.of("finetune_on_embeddings")
    assert len(ds["train"]) == 10 and np.asarray(ds["val"]["index"]).tolist() == list(b["val"]["index"])
    run.main(["evaluate", "head.pt", "-b", "base.pt", "-l", f"{tmp_path / 'a'},{tmp_path / 'b'}"])
    assert len(r.of("evaluate")[-1][1]) == 2                                               # the first dataset's test
    run.main(["embed", "clip.pt", "-l", f"{tmp_path / 'a'},{tmp_path / 'b'}"])
    (_, splits, _), = r.of("embed_images")
    assert len(splits["train"]) == 10 and len(splits["val"]) == 3
    assert "generate" not in r.kinds() and "save" not in r.kinds()


def test_run_single_load_and_pretrain_routing_unchanged(tmp_path, monkeypatch):
    import run
    r = Recorder(monkeypatch, tmp_path)
    with pytest.raises(NotImplementedError, match="-l"):
        run.main(["pretrain", config.CLIP_MODEL])
    r.raw.save_to_disk(str(tmp_path / "d"))
    run.main(["embed", "clip.pt", "-l", str(tmp_path / "d"), "-s", "2"])
    assert r.kinds() == ["embed_images"] and len(r.of("embed_images")[0][1]["train"]) == 5
    args = run.build_parser().parse_args(["evaluate", "h", "-s", "12", "-t"])
    assert args.sample == "12" and args.test
    args = run.build_parser().parse_args(["finetune", "h"])
    assert args.sample is None and not args.test and args.load is None


def test_run_checks_preprocess_columns_before_embedding(tmp_path, monkeypatch):
    """`preprocess` needs `heading` under config.GEOCELL_PATH and, in embed mode, `image_2`..`image_4` there: a CSV
    without them fails before the embedding pass, and before anything is saved."""
    import run
    r = Recorder(monkeypatch, tmp_path)
    r.generated = datasets.DatasetDict({k: v.remove_columns(["image_3"]) for k, v in r.generated.items()})
    with pytest.raises(ValueError, match=r"image_3.*embed mode"):
        run.main(["embed", "clip.pt"])
    r.generated = datasets.DatasetDict({k: v.remove_columns(["heading"]) for k, v in r.generated.items()})
    for mode in (["embed", "clip.pt"], ["finetune", config.CLIP_MODEL], ["evaluate", "h", "-b", "b"]):
        with pytest.raises(ValueError, match="heading"):
            run.main(mode)
    assert r.kinds() == ["generate"] * 4
    run.main(["embed", "clip.pt", "--yfcc"])                          # neither is needed under GEOCELL_PATH_YFCC
    assert r.kinds()[4:] == ["generate", "embed_images", "preprocess", "save", "finetune_on_embeddings"]


def test_run_finetune_embeddings_needs_load(tmp_path, monkeypatch):
    import run
    r = Recorder(monkeypatch, tmp_path)
    with pytest.raises(ValueError, match="--embeddings needs -l"):
        run.main(["finetune", "-", "--embeddings"])
    assert r.calls == []
