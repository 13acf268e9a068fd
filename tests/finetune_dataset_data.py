"""Synthetic metadata CSVs for `pigeon_b200.finetune_data.generate_finetune_dataset`, shared by
tools/make_finetune_dataset_golden.py (which runs the reference's builder on them) and the tests.

Every case has rows in each split and one row whose `selection` is none of them, and every image column named `image*`:

- `panorama`: `image`..`image_4`, string climates, `heading` and `month`, a `geo_area` column (read with geo_augment);
- `single`: `image` only, integer `climate` and string `climate_zone` together (the zone wins), integer `*_reg` values;
- `idx`: `image_idx` only (files `{image_idx}.jpg`), integer `climate_zone`, `heading` with a NaN;
- `idx_panorama`: `image`, `image_idx` (strings) and `image_2`..`image_4`: a panorama, every image column joined;
- `image_and_idx`: `image` and integer `image_idx` and nothing else: a panorama without its other views, which fails.

Cases without `geo_area` are read with geo_augment=False.
"""
from __future__ import annotations

import numpy as np

from pigeon_b200.finetune_data import CLIMATE_DICT

IMAGE_FOLDER = 'images'
SELECTIONS = ['train', 'val', 'train', 'test', 'holdout', 'train', 'val', 'test', 'train', 'test', 'train']
CASES = ('panorama', 'single', 'idx', 'idx_panorama', 'image_and_idx')
FAILING = ('image_and_idx',)


def frame(case: str, seed: int = 0):
    """The metadata DataFrame of `case`."""
    import pandas as pd
    rng = np.random.default_rng(seed + CASES.index(case))
    n = len(SELECTIONS)
    names = sorted(CLIMATE_DICT)
    cols = {}
    if case in ('panorama', 'idx_panorama', 'single', 'image_and_idx'):
        cols['image'] = [f'r{i}_0.{"png" if i % 3 == 0 else "jpg"}' for i in range(n)]
    if case == 'idx':
        cols['image_idx'] = (rng.permutation(900)[:n] + 100).tolist()
    if case == 'idx_panorama':
        cols['image_idx'] = [f'x{i}' for i in range(n)]
    if case == 'image_and_idx':
        cols['image_idx'] = list(range(n))
    if case in ('panorama', 'idx_panorama'):
        for v in (2, 3, 4):
            cols[f'image_{v}'] = [f'r{i}_{v - 1}.jpg' for i in range(n)]
    cols['lng'] = rng.uniform(-180, 180, n)
    cols['lat'] = rng.uniform(-90, 90, n)
    for j, c in enumerate(('elevation', 'population', 'temp_avg', 'temp_diff', 'prec_avg', 'prec_diff')):
        if case == 'single':
            cols[f'{c}_reg'] = rng.integers(-5, 50, n)
        else:
            cols[f'{c}_reg'] = rng.normal(j, 1 + j, n)
    if case in ('panorama', 'image_and_idx'):
        cols['climate'] = [names[k] for k in rng.integers(0, len(names), n)]
    if case == 'single':
        cols['climate'] = rng.integers(0, 28, n)
        cols['climate_zone'] = [names[k] for k in rng.integers(0, len(names), n)]
    if case in ('idx', 'idx_panorama'):
        cols['climate_zone'] = rng.integers(0, 28, n)
    if case in ('panorama', 'idx'):
        heading = rng.uniform(0, 360, n)
        if case == 'idx':
            heading[5] = np.nan
        cols['heading'] = heading
    if case in ('panorama', 'idx_panorama'):
        cols['month'] = rng.integers(1, 13, n)
    cols['selection'] = SELECTIONS
    if case == 'panorama':
        cols['geo_area'] = [f'Area {i % 4}' for i in range(n)]
    return pd.DataFrame(cols)


def geo_augment(case: str) -> bool:
    return 'geo_area' in frame(case).columns


def write_csv(case: str, where: str) -> str:
    frame(case).to_csv(where, index=False)
    return where
