"""The raw fine-tuning dataset from the metadata CSV and the image folder: reference
dataset_creation/finetune/finetune_dataset.py (`generate_finetune_dataset`, :97-150, and `create_dataset_split`, :39-95).

`generate_finetune_dataset(sample, geo_augment, metadata_path, image_path)` returns the `DatasetDict` (`train`, `val`,
`test`) that `dataset_preprocessing.preprocess` takes, column for column and dtype for dtype as the reference builds it.
Per split, in this order:

- `image`: the image file of each row, an `Image()` feature holding its path (nothing is read or decoded here);
- `lng`, `lat`, and `elevation`, `population`, `temp_avg`, `temp_diff`, `prec_avg`, `prec_diff` from the `*_reg` columns;
- `index`: the pandas index of the CSV row, int64;
- `labels_climate`: `climate`, replaced by `climate_zone` when the CSV has both; names are mapped through CLIMATE_DICT;
- `heading` and `labels_month` (from `month`) when the CSV has them;
- `image_2`, `image_3`, `image_4` for panoramas, `Image()` features like `image`.

Image columns are the columns whose name contains `image`.  With one such column the dataset holds single images: the
file is `{image_idx}.jpg` when that column is `image_idx`, else the `image` value, joined to `image_path`.  With several
the dataset holds panoramas and every one of them is joined to `image_path`; `image_idx` contains `image`, so a CSV with
both `image` and `image_idx` is a panorama, as in the reference, and needs `image_2`..`image_4`.  Rows go to the split
their `selection` names, in CSV order; rows of any other `selection` are left out.

Deviations (DESIGN.md §1):
- `sample` rows are drawn with a generator seeded from `torch.initial_seed()` (the reference's `DataFrame.sample` is
  unseeded), so `torch.manual_seed` repeats a run and a different seed draws different rows.  The drawn rows keep their
  CSV order (the reference keeps the order of the draw, which, unseeded, carries no meaning): every split's `index`
  then ascends, which the embedding join of `preprocess` (`embeds[argsort(indices)]`, row by row) relies on.
- `GeoAugmentor` (GADM areas, climate, elevation and population rasters) is not available: with `geo_augment` and no
  `geo_area` column this raises ValueError instead of augmenting.  A CSV that already carries the `*_reg` and climate
  columns is read with `geo_augment=False`.
- A column the split builder reads that the CSV lacks raises ValueError before any path is built (the reference stops
  later with a KeyError or AttributeError).  A split with no rows is returned empty, with the other splits' column
  types (the reference's climate check raises IndexError on it).
"""
from __future__ import annotations

from os import path
from typing import List, Optional

import numpy as np

from . import config

SPLITS = ('train', 'val', 'test')
VALUE_COLUMNS = ('elevation', 'population', 'temp_avg', 'temp_diff', 'prec_avg', 'prec_diff')   # from `{name}_reg`
VIEW_COLUMNS = ('image_2', 'image_3', 'image_4')

# Köppen-Geiger climate names -> class ids (reference finetune_dataset.py:8-37)
CLIMATE_DICT = {
    'Arid, desert, cold': 0,
    'Arid, desert, hot': 1,
    'Arid, steppe, cold': 2,
    'Arid, steppe, hot': 3,
    'Cold, dry summer, cold summer': 4,
    'Cold, dry summer, hot summer': 5,
    'Cold, dry summer, warm summer': 6,
    'Cold, dry winter, cold summer': 7,
    'Cold, dry winter, hot summer': 8,
    'Cold, dry winter, warm summer': 9,
    'Cold, no dry season, cold summer': 10,
    'Cold, no dry season, hot summer': 11,
    'Cold, no dry season, very cold winter': 12,
    'Cold, no dry season, warm summer': 13,
    'Polar, frost': 14,
    'Polar, tundra': 15,
    'Temperate, dry summer, cold summer': 16,
    'Temperate, dry summer, hot summer': 17,
    'Temperate, dry summer, warm summer': 18,
    'Temperate, dry winter, cold summer': 19,
    'Temperate, dry winter, hot summer': 20,
    'Temperate, dry winter, warm summer': 21,
    'Temperate, no dry season, cold summer': 22,
    'Temperate, no dry season, hot summer': 23,
    'Temperate, no dry season, warm summer': 24,
    'Tropical, monsoon': 25,
    'Tropical, rainforest': 26,
    'Tropical, savannah': 27,
}


def image_columns(columns) -> List[str]:
    """The CSV's image columns: every column whose name contains `image` (finetune_dataset.py:116)."""
    return [c for c in columns if 'image' in c]


def missing_columns(columns) -> List[str]:
    """The columns `generate_finetune_dataset` and the split builder read that `columns` lacks, in reading order."""
    cols = list(columns)
    images = image_columns(cols)
    if images == ['image_idx']:
        need = []
    elif len(images) == 1:
        need = ['image']
    else:                                                           # a panorama (also with no image column at all)
        need = ['image_path' if 'image_path' in cols else 'image', *VIEW_COLUMNS]
    need += ['selection', 'lng', 'lat', *(f'{c}_reg' for c in VALUE_COLUMNS)]
    missing = [c for c in need if c not in cols]
    if 'climate' not in cols and 'climate_zone' not in cols:
        missing.append('climate or climate_zone')
    return missing


def _climate_labels(values: np.ndarray) -> np.ndarray:
    """finetune_dataset.py:72-73: names (the first value decides) become CLIMATE_DICT ids, numbers stay as they are.  An
    empty column of names becomes an empty int64 column, the type the other splits' ids get."""
    if len(values) == 0:
        values = np.asarray(values)
        return values if values.dtype.kind in 'biuf' else values.astype(np.int64)
    if not isinstance(values[0], str):
        return values
    unknown = sorted({v for v in values if v not in CLIMATE_DICT}, key=str)
    if unknown:
        raise ValueError(f'climate names not in CLIMATE_DICT: {unknown[:5]}')
    return np.array([CLIMATE_DICT[v] for v in values])


def create_dataset_split(df, panorama: bool = False):
    """One split (finetune_dataset.py:39-95) from the rows of `df`, whose image columns already hold full paths."""
    from datasets import Dataset, Image
    image_col = 'image_path' if 'image_path' in df.columns else 'image'
    columns = {'image': df[image_col].tolist(), 'lng': df['lng'].values, 'lat': df['lat'].values}
    for name in VALUE_COLUMNS:
        columns[name] = df[f'{name}_reg'].values
    columns['index'] = df.index.values
    climate = 'climate_zone' if 'climate_zone' in df.columns else 'climate'
    columns['labels_climate'] = _climate_labels(df[climate].values)
    if 'heading' in df.columns:
        columns['heading'] = df['heading'].values
    if 'month' in df.columns:
        columns['labels_month'] = df['month'].values
    views = VIEW_COLUMNS if panorama else ()
    for name in views:
        columns[name] = df[name].tolist()
    split = Dataset.from_dict(columns)
    for name in ('image', *views):
        split = split.cast_column(name, Image())
    return split


def generate_finetune_dataset(sample: Optional[int] = None, geo_augment: bool = True,
                              metadata_path: str = config.METADATA_PATH, image_path: str = config.IMAGE_PATH):
    """reference generate_finetune_dataset (finetune_dataset.py:97-150) -> DatasetDict(train, val, test); see the module
    docstring.  `sample`: how many rows to draw (seeded from torch.initial_seed()), None for all.

    The image columns hold paths, not bytes.  `DatasetDict.save_to_disk` embeds the bytes of every file they name (it
    writes with `embed_local_files`), so a saved split that keeps its image columns no longer needs the folder; either
    way the later steps read the files through `loops.read_encoded`."""
    import pandas as pd
    import torch
    from datasets import DatasetDict
    df = pd.read_csv(metadata_path)
    missing = missing_columns(df.columns)
    if geo_augment and 'geo_area' not in df.columns:
        raise ValueError(f'{metadata_path}: has no geo_area column, so the reference would add the geographic columns '
                         f'with GeoAugmentor, which is not available here; missing *_reg / climate columns: '
                         f'{[c for c in missing if c.endswith("_reg") or c.startswith("climate")]}.  Pass '
                         f'geo_augment=False to read a CSV that already has them.')
    if missing:
        raise ValueError(f'{metadata_path}: missing column(s) {missing}')

    images = image_columns(df.columns)
    panorama = len(images) != 1
    if images == ['image_idx']:
        df['image_path'] = [path.join(image_path, f'{v}.jpg') for v in df['image_idx'].tolist()]
    else:
        for col in (images if panorama else ['image']):
            df[col] = [path.join(image_path, v) for v in df[col].tolist()]

    if sample is not None:
        rng = np.random.default_rng(torch.initial_seed())
        df = df.sample(int(sample), random_state=rng).sort_index()

    return DatasetDict({s: create_dataset_split(df.loc[df['selection'] == s], panorama=panorama) for s in SPLITS})
