"""CLIPEmbedding — the reference's CLIP ViT-L/14-336 image embedder (models/clip_embedder.py) with the H100 tower behind it.

Same constructor arguments (`model_name, device='cuda', load_checkpoint=False, panorama=False`), same call
(`embedder(image) -> Tensor[N, hidden]`), same result: the mean over ALL tokens of `last_hidden_state`
(reference :63-65) — computed by the fused CUDA path, never trainable, never on the CPU.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from .config import CLIP_MODEL
from .model_utils import load_state_dict
from .super_guessr import as_tower


class CLIPEmbedding(torch.nn.Module):
    def __init__(self, model_name: str, device: str = 'cuda', load_checkpoint: bool = False, panorama: bool = False,
                 clip_model=None, processor=None):
        """Reference arguments (:11-23) plus two keyword extensions for offline use — the reference pulls `CLIP_MODEL`
        and its processor from the hub (:25-26): `clip_model` (a `CLIPVisionTower` or a HF `CLIPVisionModel` to wrap) and
        `processor` (any callable with the `CLIPProcessor(images=..., return_tensors='pt')` convention; by default the GPU
        pre-processor of `pigeon_b200.preprocess`, whose output is bit-identical, built on first use)."""
        super().__init__()
        if clip_model is None:
            from transformers import CLIPVisionModel
            clip_model = CLIPVisionModel.from_pretrained(CLIP_MODEL)
        tower = as_tower(clip_model)
        if load_checkpoint:                                   # :29-32, keys are stored under 'base_model.'
            load_state_dict(tower.base_model, torch.load(model_name, map_location='cuda'), embedder=True)
            print('Loaded embedder from checkpoint:', model_name)
        self.device = device
        self.panorama = panorama
        self.processor = processor
        self.clip_model = tower.to(device) if isinstance(device, str) else tower.cuda(device)     # :34-37
        self.eval()

    def _pixels(self, image) -> Tensor:
        """Pre-processed tensors pass through; anything else (PIL images, uint8 arrays, lists of them) goes through the
        processor (:48-56)."""
        if isinstance(image, Tensor):
            return image
        if self.processor is None:
            from .preprocess import ClipImageProcessor
            self.processor = ClipImageProcessor(size=self.clip_model.dims.image_size,
                                                device=next(self.clip_model.parameters()).device, dtype=torch.float16)
        return self.processor(images=image, return_tensors='pt')['pixel_values']

    @torch.no_grad()
    def _get_embedding(self, image) -> Tensor:
        pixels = self._pixels(image)
        pixels = pixels.to(self.device) if isinstance(self.device, str) else pixels.cuda(self.device)
        return self.clip_model.embed(pixels)                  # tower forward + token mean in one pass (:63-65)

    def forward(self, image) -> Tensor:
        return self._get_embedding(image)
