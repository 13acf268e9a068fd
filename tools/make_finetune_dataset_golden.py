"""Generate tests/golden/finetune_dataset.npz: the splits the UNMODIFIED reference `generate_finetune_dataset`
(dataset_creation/finetune/finetune_dataset.py) builds from the synthetic CSVs of tests/finetune_dataset_data.py, for
pigeon_b200.finetune_data.

The reference module is loaded through oracle/reference_shim.py, with a `preprocessing.GeoAugmentor` stub that fails if
it is called (cases with a `geo_area` column are read with geo_augment=True, which must not augment them; the others with
geo_augment=False).  Image folder: tests/finetune_dataset_data.IMAGE_FOLDER, a relative name; nothing is read from it.

Stored (only data), per case and split:
  {case}/{split}/columns    column names in order
  {case}/{split}/features   JSON {column: repr of its datasets feature}
  {case}/{split}/{column}   the values: image columns as their path strings, the others as stored (arrow -> numpy)
  {case}/error              for a case the reference fails on, the exception's class name

    python tools/make_finetune_dataset_golden.py
"""
from __future__ import annotations

import importlib.util
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "finetune_dataset.npz")


class GeoAugmentorStub:
    def __init__(self, *a, **kw):
        raise AssertionError("GeoAugmentor called: the golden cases must not need augmentation")


def reference_module():
    from oracle import reference_shim
    reference_shim.install()
    sys.modules["preprocessing"].GeoAugmentor = GeoAugmentorStub
    path = os.path.join(reference_shim.REF, "dataset_creation", "finetune", "finetune_dataset.py")
    spec = importlib.util.spec_from_file_location("_ref_finetune_dataset", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def split_record(split) -> dict:
    """{key suffix: array} of one split (see the module docstring)."""
    import datasets
    out = {"columns": np.array(split.column_names),
           "features": np.array(json.dumps({k: repr(v) for k, v in split.features.items()}))}
    table = split.with_format("arrow")[:]
    for name, feature in split.features.items():
        col = table.column(name)
        if isinstance(feature, datasets.Image):
            out[name] = np.array([v["path"] for v in col.to_pylist()])
        else:
            out[name] = col.to_numpy()
    return out


def main():
    import finetune_dataset_data as data
    ref = reference_module()
    arrays = {}
    with tempfile.TemporaryDirectory() as tmp:
        for case in data.CASES:
            csv = data.write_csv(case, os.path.join(tmp, f"{case}.csv"))
            try:
                ds = ref.generate_finetune_dataset(geo_augment=data.geo_augment(case), metadata_path=csv,
                                                   image_path=data.IMAGE_FOLDER)
            except Exception as e:                      # noqa: BLE001 — the failing cases record what the reference raised
                assert case in data.FAILING, (case, e)
                arrays[f"{case}/error"] = np.array(type(e).__name__)
                continue
            assert case not in data.FAILING, case
            for split in ds:
                for k, v in split_record(ds[split]).items():
                    arrays[f"{case}/{split}/{k}"] = v
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}: {len(arrays)} arrays")


if __name__ == "__main__":
    main()
