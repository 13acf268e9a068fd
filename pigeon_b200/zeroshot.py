"""Zero-shot caption scoring with a `CLIPModel` (e.g. a StreetCLIP-style checkpoint): images against captions such as
"a Street View photo in Kenya".

The reference imports `get_caption_probabilities` and `zero_shot_accuracy` from `evaluation/zeroshot.py`
(evaluation/__init__.py:3) but never shipped that module, so only the names are the reference's; the signatures below are
this library's.  The arithmetic is HF CLIPModel's: `logits_per_image.softmax(dim=1)` over the captions, top-1 by first
argmax — what `PretrainDataset.accuracy` (dataset_creation/pretrain/pretrain_dataset.py:299-330) computes — read from
`pg_clip_logits`.
"""
from __future__ import annotations

from typing import Optional, Sequence, Union

import torch
from torch import Tensor

from .clip_text import check_sequence_length


def _features(model, pixel_values: Tensor, input_ids: Tensor, attention_mask: Optional[Tensor]):
    check_sequence_length(input_ids.shape[-1], model.text_dims.max_positions)
    return model.get_image_features(pixel_values), model.get_text_features(input_ids, attention_mask)


@torch.no_grad()
def get_caption_probabilities(model, pixel_values: Tensor, input_ids: Tensor,
                              attention_mask: Optional[Tensor] = None) -> Tensor:
    """model: `pigeon_b200.CLIPModel` on CUDA; pixel_values [Ni, 3, H, W] (as `CLIPProcessor(images=...)` makes them);
    input_ids / attention_mask [Nt, S] (as `CLIPProcessor(text=..., padding=True)` makes them)
    -> f32 [Ni, Nt]: per image, the softmax over the captions of logits_per_image."""
    img, txt = _features(model, pixel_values, input_ids, attention_mask)
    return model.logits(img, txt, per_text=False, probs=True)["probs"]


@torch.no_grad()
def zero_shot_accuracy(model, pixel_values: Tensor, input_ids: Tensor, labels: Union[Tensor, Sequence[int]],
                       attention_mask: Optional[Tensor] = None) -> float:
    """Top-1 accuracy of zero-shot classification: image i is right when its most probable caption (first argmax of
    logits_per_image[i]) is labels[i], an index into the captions."""
    img, txt = _features(model, pixel_values, input_ids, attention_mask)
    pred = model.logits(img, txt, per_text=False, pred=True)["pred"]
    labels = torch.as_tensor(labels, dtype=torch.int64).to(pred.device)
    if labels.shape != pred.shape:
        raise ValueError(f"labels {tuple(labels.shape)} do not match {pred.shape[0]} images")
    return float((pred == labels).double().mean())
