"""The reference's CLIP pretraining data (dataset_creation/pretrain/): `PretrainDataset` (StreetView metadata CSV with
`o`, `v` and `l` sources) and `PretrainDatasetYFCC`, read from their metadata CSV and image folders, with captions
synthesised as the reference does.

An item is `(encoded file, crop window, fill, caption)`: the file stays encoded, and the window says which rectangle
of it the reference's crop keeps (`preprocess.CropWindow`, which may extend past the image: torchvision's CenterCrop
pads).  `ClipImageProcessor(images=files, windows=..., fills=...)` decodes, crops and pre-processes a batch on the GPU,
bit-identical to the reference's Pillow path, which `item_pil` restates for tests.

Captions draw from Python's `random`, as the reference's do, so with the same `random` state and the same order of
calls they are the reference's captions.  The reference trains with `dataloader_num_workers=0`: every item is made in
the main process in sampler order.  Here DataLoader workers may read the files (`read`, which draws nothing), and the
captions of a batch are drawn in the main process, in sampler order, when the training loop asks for that batch
(`pretrain_encoded_batches`).

    dataset = PretrainDataset.generate(metadata_csv, auxiliary=False)      # DatasetDict of train, val, test
    pretrain_files('openai/clip-vit-large-patch14-336', metadata_csv)      # what `run.py pretrain -l META.csv` runs
"""
from __future__ import annotations

import functools
import io
import json
import random
from typing import Any, List, Optional, Tuple

import numpy as np
import pandas as pd
import torch
from torch.utils.data import BatchSampler, DataLoader

from . import config
from .preprocess import CropWindow
from .pretrain import CLIPCollator, CLIPPretrainer

MONTHS = dict(enumerate(['January', 'February', 'March', 'April', 'May', 'June', 'July', 'August', 'September',
                         'October', 'November', 'December']))

# Countries whose name takes "the" in a StreetView caption (pretrain_dataset.py:36-57)
THE_LIST = ['Bahamas', 'British Virgin Islands', 'Cayman Islands', 'Cocos Islands', 'Comoros', 'Cook Islands',
            'Falkland Islands', 'Faroe Islands', 'French Southern Territories', 'Maldives', 'Marshall Islands',
            'Netherlands', 'Northern Mariana Islands', 'Paracel Islands', 'Philippines', 'Pitcairn Islands', 'Seychelles',
            'Solomon Islands', 'Spratly Islands', 'Turks and Caicos Islands', 'United Arab Emirates', 'United States']

# The same for YFCC captions, and the names the YFCC metadata truncates (pretrain_dataset_yfcc.py:21-56)
PLURALS = ['Bahamas', 'British Virgin Islands', 'Caspian Sea', 'Cayman Islands', 'Central African Republic',
           'Cocos Islands', 'Cook Islands', 'Democratic Republic of the Congo', 'Dominican Republic', 'Falkland Islands',
           'Faroe Islands', 'Isle of Man', 'Maldives', 'Netherlands', 'Northern Mariana Islands', 'Philippines',
           'Republic of the Congo', 'Seychelles', 'Solomon Islands', 'Turks and Caicos Islands', 'United Arab Emirates',
           'United Kingdom', 'United States', 'United States Minor Outlying Isl', 'Vatican City', 'Virgin Islands, U.S.',
           'Western Sahara']
RENAMING = {'South Georgia and the South Sand': 'South Georgia and the South Sandwich Islands',
            'United States Minor Outlying Isl': 'United States Minor Outlying Islands'}

L_STRIP = 512                   # an `l` panorama is cut into 5 column strips of this width
L_CROP = int(192.53436408909982 * 2)   # CenterCrop(192.53...*2): torchvision truncates the size to 385
V_CROP = 596

# Modes whose zero pixel is black in RGB: what padding adds to a file in that mode before `convert('RGB')`.  A `P`
# file's padding is its palette entry 0; any other mode (CMYK, YCbCr, ...) is cropped by Pillow on the host.
BLACK_MODES = frozenset({'1', 'L', 'LA', 'La', 'I', 'I;16', 'I;16L', 'I;16B', 'I;16N', 'F', 'RGB', 'RGBA', 'RGBa',
                         'RGBX'})


def _valid(value: Any) -> bool:
    """The reference's `_is_valid`: a string, or a number that is not NaN."""
    return type(value) == str or np.isnan(value) == False      # noqa: E721,E712  (the reference's exact test)


def center_crop_origin(width: int, height: int, size: int) -> Tuple[int, int]:
    """(x0, y0) of torchvision's `center_crop(img, size)` on a width x height image, in the image's coordinates: the
    padding (left/top `(size - dim) // 2`) comes first, then `int(round((dim - size) / 2.0))` of the padded image."""
    pad_l = (size - width) // 2 if size > width else 0
    pad_t = (size - height) // 2 if size > height else 0
    w = width + (pad_l + (size - width + 1) // 2 if size > width else 0)
    h = height + (pad_t + (size - height + 1) // 2 if size > height else 0)
    if (size > width or size > height) and w == size and h == size:
        return -pad_l, -pad_t
    return int(round((w - size) / 2.0)) - pad_l, int(round((h - size) / 2.0)) - pad_t


def square_crop_box(width: int, height: int) -> Tuple[int, int, int, int]:
    """(x0, y0, x1, y1) that `image.crop` keeps of the reference's float box in `_crop_resize`
    (pretrain_dataset_yfcc.py:163-170): Pillow 12's `Image._crop` rounds each coordinate half to even, so an odd
    difference between width and height can give a box one pixel narrower or wider than it is tall."""
    d = min(width, height)
    box = ((width - d) / 2, (height - d) / 2, (width + d) / 2, (height + d) / 2)
    x0, y0, x1, y1 = (int(round(v)) for v in box)
    return x0, y0, x1, y1


def header(data: bytes):
    """Pillow's view of an encoded file without decoding it: (width, height, mode, fill), where fill is the RGB that
    padding in the file's own mode becomes after `convert('RGB')`, or None when that is not a known constant."""
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        w, h = im.size
        mode = im.mode
        fill = None
        if mode in BLACK_MODES:
            fill = (0, 0, 0)
        elif mode == 'P' and im.palette is not None and im.palette.rawmode in ('RGB', 'RGBA', 'RGBX'):
            p = bytes(im.palette.palette)
            if len(p) >= 3:
                fill = (p[0], p[1], p[2])
    return w, h, mode, fill


def _read(path: str) -> bytes:
    with open(path, 'rb') as f:
        return f.read()


class _PretrainBase(torch.utils.data.Dataset):
    """What both datasets share: items, the host PIL path, and the contrastive accuracy."""

    collator: Optional['FilesCollator'] = None          # processor + tokenizer for `accuracy` (set by pretrain_files)

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop('collator', None)                     # DataLoader workers only read files: no CUDA objects
        return state

    def locate(self, index: int) -> Tuple[str, str, int]:
        raise NotImplementedError

    def caption(self, index: int) -> str:
        raise NotImplementedError

    def _check(self, index: int) -> int:
        index = int(index)
        if not 0 <= index < len(self):
            raise IndexError(f'index {index} out of range for {len(self)} items')
        return index

    def window(self, index: int, data: bytes) -> Tuple[CropWindow, Optional[tuple]]:
        """The crop window and fill of item `index`, whose file holds `data` (read from its header only)."""
        kind, col = self.locate(index)[1:]
        w, h, _, fill = header(data)
        if kind == 'o':
            return CropWindow(0, 0, w, h), (0, 0, 0)
        if kind == 'l':                                    # convert('RGB') first: the padding is black
            left = min(col * L_STRIP, w)
            sw = min(w, left + L_STRIP) - left
            if sw <= 0:
                raise ValueError(f'item {index}: panorama of width {w} has no strip {col}')
            x0, y0 = center_crop_origin(sw, h, L_CROP)
            return CropWindow(x0, y0, L_CROP, L_CROP, clip=(left, 0, sw, h)), (0, 0, 0)
        if kind == 'v':
            x0, y0 = center_crop_origin(w, h, V_CROP)
            return CropWindow(x0, y0, V_CROP, V_CROP), fill
        x0, y0, x1, y1 = square_crop_box(w, h)              # YFCC
        return CropWindow(x0, y0, x1 - x0, y1 - y0), (0, 0, 0)

    def read(self, index: int) -> Tuple[bytes, CropWindow, Optional[tuple]]:
        """(file bytes, window, fill) of item `index`.  Draws nothing from `random`: DataLoader workers may call it."""
        index = self._check(index)
        data = _read(self.locate(index)[0])
        return (data,) + self.window(index, data)

    def __getitem__(self, index: int) -> Tuple[bytes, CropWindow, Optional[tuple], str]:
        """(encoded file, crop window, fill, caption): the reference's (image, caption) before decoding."""
        data, window, fill = self.read(index)
        return data, window, fill, self.caption(index)

    def item_pil(self, index: int):
        """The reference's (PIL image, caption) of item `index`, with Pillow on the host.  For tests."""
        from PIL import Image
        index = self._check(index)
        path, kind, col = self.locate(index)
        image = Image.open(path)
        if kind == 'l':
            image = Image.fromarray(np.asarray(image.convert('RGB'))[:, col * L_STRIP:(col + 1) * L_STRIP])
            x0, y0 = center_crop_origin(image.width, image.height, L_CROP)
            image = image.crop((x0, y0, x0 + L_CROP, y0 + L_CROP))      # Pillow pads outside the image with 0
        elif kind == 'v':
            x0, y0 = center_crop_origin(image.width, image.height, V_CROP)
            image = image.crop((x0, y0, x0 + V_CROP, y0 + V_CROP))
        elif kind == 'yfcc':
            image = image.crop(square_crop_box(image.width, image.height))
        return image, self.caption(index)

    def accuracy(self, model: Any, batch_size: int, trials: int = 30) -> float:
        """Monte-Carlo contrastive top-1: over `trials` consecutive batches of `batch_size` items from index 0, the share
        of images whose highest-scoring caption in the batch is their own.  The reference's `accuracy` raises (it
        unpacks three values from two-item tuples); this is its evident intent.  Trials that would run past the end
        of the dataset are dropped; with none left the result is NaN."""
        if self.collator is None:
            raise ValueError('accuracy needs a FilesCollator in `.collator` (processor and tokenizer)')
        trials = min(int(trials), len(self) // int(batch_size))
        if trials <= 0:
            return float('nan')
        dev = model.logit_scale.device
        hits = torch.zeros((), dtype=torch.float64, device=dev)
        was_training = model.training
        model.eval()
        with torch.no_grad():
            for t in range(trials):
                batch = self.collator([self[t * batch_size + i] for i in range(batch_size)])
                out = model(input_ids=batch['input_ids'].to(dev), pixel_values=batch['pixel_values'].to(dev),
                            attention_mask=batch['attention_mask'].to(dev), return_loss=True)
                pred = out.logits_per_image.softmax(dim=1).argmax(dim=1)
                hits += (pred == torch.arange(batch_size, device=dev)).double().sum() / batch_size
        if was_training:
            model.train()
        return float(hits) / trials


class PretrainDataset(_PretrainBase):
    """reference pretrain_dataset.py:59-330.  `image_path` / `image_path_2` replace config.IMAGE_PATH / IMAGE_PATH_2
    (the folders of `o` and `l` files; `v` files are absolute paths in the CSV)."""

    def __init__(self, split: str, metadata: str = config.PRETRAIN_METADATA_PATH, auxiliary: bool = True,
                 image_path: str = config.IMAGE_PATH, image_path_2: str = config.IMAGE_PATH_2):
        assert split in ['train', 'val', 'test']
        df = pd.read_csv(metadata)
        self.df = df[df['selection'] == split].reset_index(drop=True)
        self.auxiliary = auxiliary
        self.image_path, self.image_path_2 = image_path, image_path_2
        self.image_columns = [c for c in self.df.columns if 'image' in c]
        src = self.df['source'].str
        self.cutoff_1 = int(src.startswith('o').sum()) * 4
        self.cutoff_2 = int(src.startswith('v').sum()) + self.cutoff_1
        self.cutoff_3 = int(src.startswith('l').sum()) * 5 + self.cutoff_2
        print(f"Initialized {split} dataset with {'no' if auxiliary == False else ''} auxiliary data.")   # noqa: E712

    def __len__(self) -> int:
        return self.cutoff_3

    def _convert_to_row_index(self, index: int) -> Tuple[int, int]:
        """Dataset index -> (row, image column): four per `o` row, then one per `v` row, then five per `l` row.  Rows
        are taken in CSV order, whatever their source: the reference's mapping assumes the CSV lists them so."""
        if index < self.cutoff_1:
            return index // 4, index % 4
        if index < self.cutoff_2:
            return self.cutoff_1 // 4 + (index - self.cutoff_1), 0
        return self.cutoff_1 // 4 + (self.cutoff_2 - self.cutoff_1) + (index - self.cutoff_2) // 5, \
            (index - self.cutoff_2) % 5

    def locate(self, index: int) -> Tuple[str, str, int]:
        """(file path, source kind 'o' / 'l' / 'v', image column) of item `index`; no I/O."""
        row, col = self._convert_to_row_index(self._check(index))
        s = self.df.iloc[row]
        if s.source.startswith('o'):
            return self.image_path + '/' + s[self.image_columns[col]], 'o', col
        if s.source.startswith('l'):
            return self.image_path_2 + '/' + s['image'], 'l', col
        if s.source.startswith('v'):
            return s['image'], 'v', col
        raise Exception(f'Invalid image source: {s.source}')

    def caption(self, index: int) -> str:
        """The reference's `_select_caption` for item `index` (pretrain_dataset.py:171-244): the same `random.random()`
        calls in the same order, and one `random.shuffle`."""
        row, col = self._convert_to_row_index(self._check(index))
        s = self.df.iloc[row]
        offset = col * 90 if s.source.startswith('o') else (col * 72 if s.source.startswith('l') else 0)
        country = s.country_name
        if country == 'United States Of America':
            country = 'United States'
        country = f'the {country}' if country in THE_LIST else country
        region = f'in the region of {s.geo_area} ' if _valid(s.geo_area) and random.random() > 0.4 else ''
        town = f'close to the town of {s.town} ' if _valid(s.town) and random.random() > 0.6 else ''
        climate = f' This location has {s.climate_zone.lower()}.' \
            if _valid(s.climate_zone) and random.random() > 0.6 else ''
        if random.random() > 0.3 or climate == '' or self.auxiliary == False:     # noqa: E712
            location = f'A Street View photo {town}{region}in {country}.'
            if self.auxiliary == False:                                            # noqa: E712
                return location
        else:
            location = ''
        driving = ''
        if _valid(s.driving_right) and climate == '' and random.random() > 0.7:
            driving = f" In this location, people drive on the {'right' if s.driving_right else 'left'} side of the road."
        compass = ''
        if _valid(s.heading) and random.random() > 0.7:
            d = (s.heading + offset) % 360
            compass = ' This photo is facing ' + ('north' if d <= 45 or d > 315 else 'east' if d <= 135 else
                                                  'south' if d <= 225 else 'west') + '.'
        month = f' The photo was taken in {MONTHS[s.month]}.' if _valid(s.month) and random.random() > 0.7 else ''
        others = [climate, driving, compass, month]
        random.shuffle(others)
        return ''.join([location] + others).strip()

    @classmethod
    def generate(cls, metadata: str = config.PRETRAIN_METADATA_PATH, auxiliary: bool = True, **kw):
        """train, val and test splits of `metadata` as a DatasetDict (pretrain_dataset.py:279-297)."""
        from datasets import DatasetDict
        return DatasetDict(train=cls('train', metadata, auxiliary, **kw), val=cls('val', metadata, auxiliary, **kw),
                           test=cls('test', metadata, auxiliary, **kw))


class PretrainDatasetYFCC(_PretrainBase):
    """reference pretrain_dataset_yfcc.py:58-251.  `image_path` replaces config.IMAGE_PATH_YFCC and `driving_side` the
    JSON file of config.DRIVING_SIDE_PATH ({country: 'left' / 'right'}).  `image_size` is kept for the signature; the
    reference does not resize either."""

    def __init__(self, split: str, metadata: str = config.PRETRAIN_METADATA_PATH_YFCC, auxiliary: bool = True,
                 shuffle: bool = True, image_size: int = 336, image_path: str = config.IMAGE_PATH_YFCC,
                 driving_side: str = config.DRIVING_SIDE_PATH):
        assert split in ['train', 'val', 'test']
        df = pd.read_csv(metadata)
        df = df[df['selection'] == split]
        if shuffle:
            df = df.sample(frac=1.0, random_state=330)
        self.df = df.reset_index(drop=True)
        self.auxiliary, self.shuffled, self.image_size = auxiliary, shuffle, image_size
        self.image_path = image_path
        with open(driving_side) as f:
            self.driving_side = json.load(f)
        print(f"Initialized {'shuffled ' if shuffle else ''}{split} YFCC dataset with "
              f"{'no ' if auxiliary == False else ''}auxiliary data.")                # noqa: E712

    def __len__(self) -> int:
        return len(self.df.index)

    def locate(self, index: int) -> Tuple[str, str, int]:
        return self.image_path + '/' + self.df.iloc[self._check(index)]['image'], 'yfcc', 0

    def caption(self, index: int) -> str:
        """The reference's `_select_caption` (pretrain_dataset_yfcc.py:97-152)."""
        s = self.df.iloc[self._check(index)]
        country = s.country_name
        if country == 'United States Of America':
            country = 'United States'
        shown = RENAMING.get(country, country)
        shown = f'the {shown}' if country in PLURALS else shown
        region = f'in the region of {s.geo_area} ' if _valid(s.geo_area) and random.random() > 0.0 else ''
        town = f'close to the town of {s.town} ' if _valid(s.town) and random.random() > 0.0 else ''
        climate = f' This location has a {s.climate_zone.lower()} climate.' \
            if _valid(s.climate_zone) and random.random() > 0.55 else ''
        if random.random() > 0.2 or climate == '' or self.auxiliary == False:     # noqa: E712
            location = f'A photo I took {town}{region}in {shown}.'
            if self.auxiliary == False:                                            # noqa: E712
                return location
        else:
            location = ''
        driving = ''
        if country in self.driving_side and climate == '' and random.random() > 0.8:
            driving = f' In this location, people drive on the {self.driving_side[country]} side of the road.'
        others = [climate, driving]
        random.shuffle(others)
        return ''.join([location] + others).strip()

    @classmethod
    def generate(cls, metadata: str = config.PRETRAIN_METADATA_PATH_YFCC, auxiliary: bool = True, **kw):
        """train, val and test splits of `metadata` as a DatasetDict (pretrain_dataset_yfcc.py:200-218)."""
        from datasets import DatasetDict
        return DatasetDict(train=cls('train', metadata, auxiliary, **kw), val=cls('val', metadata, auxiliary, **kw),
                           test=cls('test', metadata, auxiliary, **kw))


def generate(metadata: str = config.PRETRAIN_METADATA_PATH, auxiliary: bool = True, yfcc: bool = False, **kw):
    """`PretrainDatasetYFCC.generate` with `yfcc`, else `PretrainDataset.generate` (run.py:106-110)."""
    return (PretrainDatasetYFCC if yfcc else PretrainDataset).generate(metadata, auxiliary, **kw)


# ---------------------------------------------------------------------------------------------------- batches
class FilesCollator:
    """The reference's `collate_fn` (train_modes.py:22-28) for items of these datasets: captions tokenised on the host
    (`tokenizer(captions, truncation=True)`, then `CLIPCollator` pads to the longest), files decoded, cropped and
    pre-processed on the GPU in one processor call.  `num_workers` is the DataLoader workers that read files during
    training."""

    def __init__(self, processor, tokenizer, num_workers: int = 0):
        self.processor, self.tokenizer, self.num_workers = processor, tokenizer, int(num_workers)
        self.text = CLIPCollator(pad_token_id=tokenizer.pad_token_id)

    def tokens(self, captions: List[str]) -> dict:
        """input_ids / attention_mask [n, longest] int64 on the host: CLIPProcessor(text, padding=True, truncation=True)."""
        enc = self.tokenizer(list(captions), truncation=True)
        rows = [{'input_ids': i, 'attention_mask': m, 'pixel_values': torch.empty(0)}
                for i, m in zip(enc['input_ids'], enc['attention_mask'])]
        out = self.text(rows)
        del out['pixel_values']
        return out

    def pixels(self, files, windows, fills) -> torch.Tensor:
        return self.processor(images=list(files), windows=list(windows), fills=list(fills))['pixel_values']

    def __call__(self, items) -> dict:
        files, windows, fills, captions = zip(*items)
        out = self.tokens(captions)
        out['pixel_values'] = self.pixels(files, windows, fills)
        return out


def read_batch(dataset: _PretrainBase, indices: List[int]) -> tuple:
    """collate_fn of the DataLoader workers: (indices, files, windows, fills) of a batch.  Each file is read once per
    batch, so the five strips of an `l` panorama share one bytes object, which the processor decodes once."""
    cache, files, windows, fills = {}, [], [], []
    for i in indices:
        path = dataset.locate(i)[0]
        if path not in cache:
            cache[path] = _read(path)
        files.append(cache[path])
        w, f = dataset.window(i, cache[path])
        windows.append(w)
        fills.append(f)
    return list(indices), files, windows, fills


class _Indices(torch.utils.data.Dataset):
    def __init__(self, n: int):
        self.n = n

    def __len__(self) -> int:
        return self.n

    def __getitem__(self, i: int) -> int:
        return int(i)


def pretrain_encoded_batches(loader: DataLoader, dataset: _PretrainBase, collator: FilesCollator):
    """The batches of `loader` (collate_fn=read_batch) as the trainer's batches: input_ids, attention_mask and
    pixel_values on the device.  As `loops.encoded_batches`, each batch's decode and pre-processing run on a side stream
    while the current stream still runs the work queued before the batch was asked for; the current stream waits on
    the side stream before the batch is handed out, and its tensors are recorded as used there.

    A batch's captions are drawn here, in the main process and in the loader's order, when the batch is asked for:
    the `random` calls come in the order the reference's single-process loader makes them."""
    dev = collator.processor.device
    main = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(main)
    for indices, files, windows, fills in loader:
        out = collator.tokens([dataset.caption(i) for i in indices])
        with torch.cuda.stream(side):
            for k in ('input_ids', 'attention_mask'):
                out[k] = out[k].pin_memory().to(dev, non_blocking=True)
            out['pixel_values'] = collator.pixels(files, windows, fills)
        main.wait_stream(side)
        for v in out.values():
            v.record_stream(main)
        yield out


class _EncodedLoader:
    """What `CLIPPretrainer.train` iterates: the drop-last batches of `sampler`, through `pretrain_encoded_batches`."""

    def __init__(self, dataset, sampler, batch_size: int, collator: FilesCollator):
        self.dataset, self.sampler, self.batch_size, self.collator = dataset, sampler, batch_size, collator

    def __len__(self) -> int:
        return len(self.sampler) // self.batch_size

    def __iter__(self):
        batches = list(BatchSampler(self.sampler, self.batch_size, drop_last=True))   # after the trainer's set_epoch
        loader = DataLoader(_Indices(len(self.dataset)), batch_sampler=batches, num_workers=self.collator.num_workers,
                            collate_fn=functools.partial(read_batch, self.dataset))
        return pretrain_encoded_batches(loader, self.dataset, self.collator)


class FilesPretrainer(CLIPPretrainer):
    """`CLIPPretrainer` on a PretrainDataset or PretrainDatasetYFCC, with a `FilesCollator` as its `data_collator`:
    training batches come through `pretrain_encoded_batches` (files read on `collator.num_workers` workers, the GPU
    work of batch i+1 under step i); evaluation batches through the collator in the main process, as before."""

    def get_train_dataloader(self):
        sampler = self._sampler(self.train_dataset, True)
        return _EncodedLoader(self.train_dataset, sampler, self.batch_size, self.data_collator), sampler


def pretrain_files(model: Any, metadata: str, yfcc: bool = False, auxiliary: bool = False, resume: bool = False,
                   num_workers: int = 0, tokenizer: str = config.CLIP_TOKENIZER_PATH, png: bool = False,
                   jpeg_multiscan: bool = False, train_args=None, **dataset_kw):
    """`run.py pretrain NAME -l META.csv`: the reference's run.py:106-110 and train_modes.pretrain on the datasets of
    `metadata`, with CLIPTokenizer loaded from the local directory `tokenizer`.  Returns the trained model."""
    from transformers import CLIPTokenizer

    from .clip_model import CLIPModel
    from .preprocess import ClipImageProcessor
    from .training import pretrain
    if train_args is None:
        train_args = config.PRETAIN_ARGS_YFCC if yfcc else config.PRETAIN_ARGS
    if isinstance(model, str):
        model = CLIPModel.from_pretrained(model)
    elif not isinstance(model, CLIPModel):
        model = CLIPModel.from_hf(model)
    dataset = generate(metadata, auxiliary, yfcc, **dataset_kw)
    processor = ClipImageProcessor(size=model.vision_dims.image_size, png=png, jpeg_multiscan=jpeg_multiscan)
    collator = FilesCollator(processor, CLIPTokenizer.from_pretrained(tokenizer), num_workers)
    for split in dataset.values():
        split.collator = collator
    return pretrain(model, dataset, train_args, resume=resume, data_collator=collator, trainer_cls=FilesPretrainer)
