"""pigeon_b200 — H100-native (sm_90a) implementation of PIGEON's image-geolocation inference hot path.

    CLIPEmbedding  (reference models/clip_embedder.py)   ViT-L/14-336 forward + token mean
    SuperGuessr    (reference models/super_guessr.py)    geocell head: Linear + softmax + argmax + top-k (+ CE loss)
    ProtoRefiner   (reference models/proto_refiner.py)   prototype retrieval refinement
    train_model, AdamW (reference training/train_eval_loop.py:164-253)   fine-tune step: head and tower backward
    ClipImageProcessor (the reference's CLIPProcessor call sites)        image pre-processing on the GPU
    CLIPModel, CLIPTextTower (HF CLIPModel as training/train_modes.py:30-64 uses it)   text tower + image-text logits
    get_caption_probabilities, zero_shot_accuracy (names evaluation/__init__.py:3 imports)   zero-shot caption scoring

Host code is Python/PyTorch plumbing over a C-ABI CUDA library (include/pigeon_b200.h); see DESIGN.md.
"""
from ._lib import PigeonB200Error  # noqa: F401
from .model_utils import ModelOutput, load_state_dict  # noqa: F401
from .vit_engine import VitDims, VitEngine  # noqa: F401


def __getattr__(name):  # lazy: these import pandas / transformers-sized dependencies
    if name in ("SuperGuessr", "CLIPVisionTower"):
        from . import super_guessr
        return getattr(super_guessr, name)
    if name == "ProtoRefiner":
        from .proto_refiner import ProtoRefiner
        return ProtoRefiner
    if name == "CLIPEmbedding":
        from .clip_embedder import CLIPEmbedding
        return CLIPEmbedding
    if name in ("train_model", "AdamW", "finetune_model", "finetune_on_embeddings"):
        from . import training
        return getattr(training, name)
    if name in ("CLIPTextTower", "TextDims", "TextEngine"):
        from . import clip_text
        return getattr(clip_text, name)
    if name in ("CLIPModel", "CLIPOutput"):
        from . import clip_model
        return getattr(clip_model, name)
    if name in ("get_caption_probabilities", "zero_shot_accuracy"):
        from . import zeroshot
        return getattr(zeroshot, name)
    if name == "ClipImageProcessor":
        from .preprocess import ClipImageProcessor
        return ClipImageProcessor
    raise AttributeError(name)
