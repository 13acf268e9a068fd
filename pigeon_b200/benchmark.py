"""The reference's evaluation datasets (dataset_creation/benchmark/): `BenchmarkDataset` (IM2GPS, IM2GPS3k, YFCC4k,
YFCC26k, GWS15k, ...: a metadata CSV and an image folder named in config.BENCHMARKS) and `EvalDataset` (raw holdout
splits with encoded `image`, `image_2`..`image_4` columns).

Indexing either one by an int or a slice gives the reference's items, with `pixel_values` made on the GPU
(`ClipImageProcessor`; benchmark images are cut to their centred square first, as `_crop_images` does).  That per-item
path is for parity.  `evaluate_model` takes the batched route instead:

    rows = dataset.encoded()                       # items are file references + labels, no I/O
    evaluate_model(model, rows, metrics, collate_fn=loops.encoded_eval_collate, processor=ClipImageProcessor())

The collate reads each row's files on the DataLoader workers; the main process turns a whole batch into pixel_values
with one processor call (one JPEG decode and one pre-processing launch sequence; files the JPEG parser does not take
are decoded by Pillow on the host).  `training.train_model` takes the same pair for fine-tuning on raw splits, whose
rows then also carry the auxiliary label columns their split has (`loops.LABEL_COLUMNS`).

The reference detours through float32 (`np.asarray(image, dtype=np.float32) / 255` before CLIPProcessor, whose
`to_pil_image` multiplies by 255 and truncates to uint8 again): that round trip is the identity on all 256 values, so
the uint8 pixels go to the pre-processor unchanged.
"""
from __future__ import annotations

import json
from typing import Any, Dict, List

import datasets
import numpy as np
import pandas as pd
import torch

from . import config
from .loops import LABEL_COLUMNS, read_encoded

_processor = None


def _clip_processor():
    """The processor behind per-item indexing (the reference's module-level CLIPProcessor), made on first use."""
    global _processor
    if _processor is None:
        from .preprocess import ClipImageProcessor
        _processor = ClipImageProcessor()
    return _processor


class EncodedRows(torch.utils.data.Dataset):
    """Rows of a BenchmarkDataset or EvalDataset as file references plus labels, for `loops.encoded_eval_collate`.
    String keys ('labels', 'labels_clf', columns) go to the dataset, as evaluate_model reads them."""

    def __init__(self, dataset):
        self.dataset = dataset

    def __len__(self) -> int:
        return len(self.dataset)

    def __getitem__(self, index):
        if isinstance(index, str):
            return self.dataset[index]
        return self.dataset.encoded_row(int(index))

    @property
    def panorama(self) -> bool:
        return self.dataset.panorama


class BenchmarkDataset(datasets.Dataset):
    """reference benchmark_dataset.py:14-106."""

    __getitems__ = None        # datasets.Dataset batches DataLoader reads; items here are read one index at a time

    def __init__(self, name: str):
        with open(config.BENCHMARKS, 'r') as f:
            benchmarks = json.load(f)

        assert name in benchmarks.keys(), f'Benchmark {name} is not a valid benchmark. Specify the \
            metadata and image paths in a JSON file and configure it in config under "BENCHMARKS".'

        self.name = name
        self._benchmark = benchmarks[name]
        self.df = pd.read_csv(self._benchmark['meta'])

    def __len__(self) -> int:
        return len(self.df.index)

    def __iter__(self):
        return (self[i] for i in range(len(self)))

    def __repr__(self) -> str:
        return f'BenchmarkDataset(name={self.name!r}, num_rows={len(self)})'

    @property
    def panorama(self):
        return False

    @property
    def multi_task(self):
        return False

    def image_path(self, filename: str) -> str:
        """The reference's string concatenation (benchmark_dataset.py:78), not os.path.join."""
        return self._benchmark['images'] + filename

    def encoded_row(self, index: int) -> Dict[str, Any]:
        sample = self.df.iloc[index]
        return {'images': [{'bytes': None, 'path': self.image_path(sample['image'])}], 'square_crop': True,
                'labels': np.asarray(sample[['lng', 'lat']], dtype=np.float64),
                'labels_clf': np.int64(sample['geocell_idx_yfcc'])}

    def encoded(self) -> EncodedRows:
        return EncodedRows(self)

    def __getitem__(self, index: Any) -> Dict:
        if type(index) == str:
            if index == 'labels':
                return self.df[['lng', 'lat']].values

            elif index == 'labels_clf':
                return self.df['geocell_idx_yfcc'].values

            else:
                return self.df[index]

        row = self.encoded_row(index)
        files = [read_encoded(im) for im in row['images']]
        model_inputs = {'pixel_values': _clip_processor()(images=files, square_crop=True)['pixel_values']}
        model_inputs['labels'] = torch.from_numpy(row['labels'])
        model_inputs['labels_clf'] = torch.tensor(row['labels_clf'])
        return model_inputs


class EvalDataset(datasets.Dataset):
    """reference eval_dataset.py:12-94: pixel_values of the one or four views (`image`, `image_2`..`image_4`) made on
    the fly, four views concatenated on the channel axis ([.., 12, 336, 336]) as `extract_features` does."""

    __getitems__ = None

    def __init__(self, data: datasets.Dataset):
        self.streetview_data = data
        self.views = ['image'] + ([f'image_{i}' for i in range(2, 5)] if 'image_2' in data.column_names else [])
        enc = data
        for col in self.views:
            if isinstance(data.features[col], datasets.Image):
                enc = enc.cast_column(col, datasets.Image(decode=False))
        self._encoded = enc

    def __len__(self) -> int:
        return len(self.streetview_data)

    def __iter__(self):
        return (self[i] for i in range(len(self)))

    def __repr__(self) -> str:
        return f'EvalDataset(views={len(self.views)}, num_rows={len(self)})'

    @property
    def panorama(self) -> bool:
        return len(self.views) == 4

    def encoded_row(self, index: int) -> Dict[str, Any]:
        """The row's encoded views and every one of `loops.LABEL_COLUMNS` the split has."""
        sample = self._encoded[index]
        row = {'images': [sample[c] for c in self.views], 'square_crop': False}
        row.update((k, sample[k]) for k in LABEL_COLUMNS if k in sample)
        return row

    def encoded(self) -> EncodedRows:
        return EncodedRows(self)

    def _pixel_values(self, rows: List[List[Dict[str, Any]]]) -> torch.Tensor:
        """rows: per view, the encoded values of n rows -> [n, 3 * views, 336, 336] on the GPU."""
        n = len(rows[0])
        files = [read_encoded(rows[v][r]) for r in range(n) for v in range(len(self.views))]
        px = _clip_processor()(images=files)['pixel_values']
        return px.view(n, 3 * len(self.views), px.shape[2], px.shape[3])

    def __getitem__(self, index: Any) -> Dict:
        if type(index) == int:
            sample = self._encoded[index]
            pixel_values = self._pixel_values([[sample[c]] for c in self.views])
        elif type(index) == slice:
            sample = self._encoded[index]
            pixel_values = self._pixel_values([sample[c] for c in self.views])
        else:
            return self.streetview_data[index]
        sample = {key: value for key, value in sample.items() if 'image' not in key}
        sample['pixel_values'] = pixel_values
        return sample

    @classmethod
    def transform(cls, dataset: datasets.DatasetDict) -> datasets.DatasetDict:
        if type(dataset) == datasets.DatasetDict:
            return datasets.DatasetDict(
                train=cls(dataset['train']),
                val=cls(dataset['val']),
                test=cls(dataset['test'])
            )

        return cls(dataset)
