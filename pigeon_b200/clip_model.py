"""CLIPModel — HF `CLIPModel`'s forward (transformers 4.23.1 modeling_clip.py) on the GPU: the dual encoder that reference
training/train_modes.py:30-64 pretrains into StreetCLIP and that `PretrainDataset.accuracy`
(dataset_creation/pretrain/pretrain_dataset.py:299-330, pretrain_dataset_yfcc.py:220-246) scores with
`model(**clip_processor(text=captions, images=images), return_loss=True).logits_per_image.softmax(1).argmax(1)`.

Parameter names are HF's (`text_model.*`, `vision_model.*`, `visual_projection.weight`, `text_projection.weight`,
`logit_scale`), so CLIPModel checkpoints load by name.

`forward_train` + `backward` is one contrastive training step (the gradient of `clip_loss` for every parameter);
`pretrain.CLIPPretrainer` is the HF Trainer loop around it (schedule, clipping, HF AdamW, checkpoints).

    image features = visual_projection(post_layernorm(last_hidden_state[:, 0]))      (CLS row; pg_vit_forward_cls)
    text features  = text_projection(pooled)                                          (pg_text_forward)
    logits_per_text = normalise(text) @ normalise(image)^T * exp(logit_scale), logits_per_image = its transpose,
    loss = mean of the two cross-entropies against arange                             (pg_clip_logits)
The projections run the geocell head's error-compensated fp16 split GEMM (fp32-faithful, pg_clip_project).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
from torch import Tensor, nn
from torch.nn.parameter import Parameter

from . import _versions, ops
from ._lib import PigeonB200Error
from ._lib import check, current_stream_ptr, load, ptr
from .clip_text import CLIPTextTower, TextDims, check_sequence_length
from .encoder import linear
from .super_guessr import CLIPVisionTower
from .vit_engine import VitDims
from .vit_train import put_grad

LOGIT_SCALE_INIT = math.log(1 / 0.07)   # CLIPConfig.logit_scale_init_value (2.6592)


@dataclass
class CLIPOutput:
    """The fields of HF `CLIPOutput` that the forward computes (text_embeds / image_embeds are L2-normalised, as HF's)."""
    loss: Optional[Tensor] = None
    logits_per_image: Optional[Tensor] = None
    logits_per_text: Optional[Tensor] = None
    text_embeds: Optional[Tensor] = None
    image_embeds: Optional[Tensor] = None

    def __getitem__(self, key):
        return getattr(self, key)


class CLIPModel(nn.Module):
    def __init__(self, text_dims: TextDims = TextDims(), vision_dims: VitDims = VitDims(), projection_dim: int = 768):
        super().__init__()
        self.text_dims, self.vision_dims, self.projection_dim = text_dims, vision_dims, projection_dim
        # The towers own the kernels; their parameter trees are registered here under HF's names.
        self._towers = (CLIPTextTower(text_dims), CLIPVisionTower(vision_dims))
        self.text_model = self._towers[0].text_model
        self.vision_model = self._towers[1].vision_model
        self.visual_projection = linear(projection_dim, vision_dims.hidden, bias=False)
        self.text_projection = linear(projection_dim, text_dims.hidden, bias=False)
        self.logit_scale = Parameter(torch.tensor(LOGIT_SCALE_INIT))
        self._packed = {}
        self.max_train_views = 64    # activation arena of the vision tower's training step (about 0.52 GB per ViT-L/14-336 view)
        self._pend = None

    @property
    def text_tower(self) -> CLIPTextTower:
        return self._towers[0]

    @property
    def vision_tower(self) -> CLIPVisionTower:
        return self._towers[1]

    def _apply(self, fn, *args, **kwargs):
        # .to() / .cuda() move the shared parameters; the towers' engines repack from them lazily
        super()._apply(fn, *args, **kwargs)
        for t in self._towers:
            t._engine, t._packed_version = None, None
        self._packed = {}
        return self

    @classmethod
    def from_hf(cls, hf_model) -> "CLIPModel":
        """Build from a HuggingFace CLIPModel instance (weights copied by name)."""
        cfg = hf_model.config
        model = cls(TextDims.from_hf_config(cfg.text_config), VitDims.from_hf_config(cfg.vision_config),
                    projection_dim=cfg.projection_dim)
        sd = {k: v for k, v in hf_model.state_dict().items() if "position_ids" not in k}
        missing, unexpected = model.load_state_dict(sd, strict=False)
        if missing or unexpected:
            raise PigeonB200Error(f"cannot map HF weights: missing={missing} unexpected={unexpected}")
        return model

    def hf_config_dict(self) -> dict:
        """The `config.json` of an HF CLIPModel with this geometry (quick-GELU towers; BOS / EOS are the last two ids, as in
        CLIP's tokenizer, so HF pools the first EOS row where this model pools the first row of the largest id)."""
        t, v = self.text_dims, self.vision_dims
        return dict(
            architectures=["CLIPModel"], model_type="clip", projection_dim=self.projection_dim,
            logit_scale_init_value=LOGIT_SCALE_INIT, initializer_factor=1.0,
            text_config=dict(model_type="clip_text_model", vocab_size=t.vocab, max_position_embeddings=t.max_positions,
                             hidden_size=t.hidden, num_attention_heads=t.heads, intermediate_size=t.intermediate,
                             num_hidden_layers=t.layers, layer_norm_eps=t.ln_eps, hidden_act="quick_gelu",
                             projection_dim=self.projection_dim, pad_token_id=1, bos_token_id=t.vocab - 2,
                             eos_token_id=t.vocab - 1),
            vision_config=dict(model_type="clip_vision_model", image_size=v.image_size, patch_size=v.patch_size,
                               hidden_size=v.hidden, num_attention_heads=v.heads, intermediate_size=v.intermediate,
                               num_hidden_layers=v.layers, layer_norm_eps=v.ln_eps, hidden_act="quick_gelu",
                               projection_dim=self.projection_dim, num_channels=3))

    def save_pretrained(self, directory: str) -> None:
        """`pytorch_model.bin` (HF parameter names, fp32 on the CPU) and `config.json`: a directory that
        `transformers.CLIPModel.from_pretrained` and `CLIPModel.from_pretrained` both load."""
        import json
        import os
        os.makedirs(directory, exist_ok=True)
        torch.save({k: v.detach().cpu().clone() for k, v in self.state_dict().items()},
                   os.path.join(directory, "pytorch_model.bin"))
        with open(os.path.join(directory, "config.json"), "w") as f:
            json.dump(self.hf_config_dict(), f, indent=2, sort_keys=True)

    @classmethod
    def from_pretrained(cls, name_or_path: str) -> "CLIPModel":
        """A directory with `config.json` and `pytorch_model.bin` (written by `save_pretrained`, an HF Trainer checkpoint or
        `transformers.CLIPModel.save_pretrained(..., safe_serialization=False)`), else an HF model name or a directory
        that `transformers.CLIPModel.from_pretrained` loads (through `from_hf`).  The model stays on the CPU."""
        import json
        import os
        from types import SimpleNamespace
        cfg_path, bin_path = os.path.join(name_or_path, "config.json"), os.path.join(name_or_path, "pytorch_model.bin")
        if not (os.path.isfile(cfg_path) and os.path.isfile(bin_path)):
            from transformers import CLIPModel as HFCLIPModel
            return cls.from_hf(HFCLIPModel.from_pretrained(name_or_path))
        with open(cfg_path) as f:
            cfg = json.load(f)
        model = cls(TextDims.from_hf_config(SimpleNamespace(**{"layer_norm_eps": 1e-5, **cfg["text_config"]})),
                    VitDims.from_hf_config(SimpleNamespace(**{"layer_norm_eps": 1e-5, **cfg["vision_config"]})),
                    projection_dim=cfg["projection_dim"])
        sd = torch.load(bin_path, map_location="cpu", weights_only=True)
        sd = {k: v for k, v in sd.items() if "position_ids" not in k}
        missing, unexpected = model.load_state_dict(sd, strict=False)
        if missing or unexpected:
            raise PigeonB200Error(f"cannot map checkpoint weights: missing={missing} unexpected={unexpected}")
        return model

    # ------------------------------------------------------------------------------------------ kernels
    def _packed_projection(self, name: str) -> Tensor:
        w = getattr(self, name).weight
        key = (w.data_ptr(), w._version, _versions.get(w))
        hit = self._packed.get(name)
        if hit is None or hit[0] != key:
            hit = (key, ops.head_pack_weight(w.detach()))
            self._packed[name] = hit
        return hit[1]

    def _check_cuda(self):
        if not self.logit_scale.is_cuda:
            raise PigeonB200Error("CLIPModel is on the CPU: move the model with .to('cuda') — the H100 path has no CPU "
                                  "implementation")

    @torch.no_grad()
    def get_text_features(self, input_ids: Tensor, attention_mask: Optional[Tensor] = None) -> Tensor:
        """text_projection(pooler_output) f32 [n, projection_dim] (not normalised, as HF's)."""
        self._check_cuda()
        pooled = self.text_tower.pooled(input_ids, attention_mask)
        return ops.clip_project(pooled, self._packed_projection("text_projection"))

    @torch.no_grad()
    def get_image_features(self, pixel_values: Tensor) -> Tensor:
        """visual_projection(post_layernorm(last_hidden_state[:, 0])) f32 [n, projection_dim] (not normalised, as HF's)."""
        self._check_cuda()
        _, cls = self.vision_tower.engine().forward_cls(pixel_values)
        post = self.vision_model.post_layernorm
        return ops.clip_project(cls, self._packed_projection("visual_projection"), post.weight.detach(),
                                post.bias.detach(), self.vision_dims.ln_eps)

    def logits(self, image_features: Tensor, text_features: Tensor, **want) -> dict:
        """`ops.clip_logits` at this model's logit_scale (features need not be normalised)."""
        return ops.clip_logits(image_features, text_features, float(self.logit_scale.detach()), **want)

    @torch.no_grad()
    def forward(self, input_ids: Tensor = None, pixel_values: Tensor = None, attention_mask: Tensor = None,
                return_loss: bool = False) -> CLIPOutput:
        """HF CLIPModel.forward: the reference's `model(**inputs)` with inputs from `CLIPProcessor(text=..., images=...)`
        (input_ids, attention_mask, pixel_values) and `return_loss=True`."""
        if input_ids is None or pixel_values is None:
            raise ValueError("CLIPModel.forward needs both input_ids and pixel_values")
        check_sequence_length(input_ids.shape[-1], self.text_dims.max_positions)
        if return_loss and input_ids.shape[0] != pixel_values.shape[0]:
            raise ValueError(f"the contrastive loss needs as many images as captions (got {pixel_values.shape[0]} images, "
                             f"{input_ids.shape[0]} captions)")
        image_features = self.get_image_features(pixel_values)
        text_features = self.get_text_features(input_ids, attention_mask)
        out = self.logits(image_features, text_features, per_text=True, loss=bool(return_loss))
        # HF returns the normalised embeds; the logits above normalise inside the kernel
        return CLIPOutput(loss=out.get("loss"), logits_per_image=out["logits_per_image"],
                          logits_per_text=out["logits_per_text"],
                          text_embeds=text_features / text_features.norm(p=2, dim=-1, keepdim=True),
                          image_embeds=image_features / image_features.norm(p=2, dim=-1, keepdim=True))

    # ------------------------------------------------------------------------------------------ training step
    def _trainers(self):
        from .clip_train import TextTrainer
        from .vit_train import TowerTrainer
        tr = getattr(self, "_vision_trainer", None)
        if tr is None or tr.tower is not self.vision_tower or tr.max_views != self.max_train_views:
            tr = self._vision_trainer = TowerTrainer(self.vision_tower, max_views=self.max_train_views)
        tt = getattr(self, "_text_trainer", None)
        if tt is None or tt.tower is not self.text_tower:
            tt = self._text_trainer = TextTrainer(self.text_tower)
        return tr, tt

    def forward_train(self, input_ids: Tensor, pixel_values: Tensor, attention_mask: Optional[Tensor] = None) -> CLIPOutput:
        """One contrastive step of HF CLIPModel (`model(input_ids, pixel_values, attention_mask, return_loss=True)` then
        `loss.backward()`, as the HF Trainer of reference training/train_modes.py:30-64 runs it): the forward, the loss
        `clip_loss(logits_per_text)` over n images and n captions, and every parameter gradient, kept pending in fp32
        buffers until `backward()` publishes them.  The vision tower follows `TowerTrainer`'s freeze rules; every text-tower
        parameter must be trainable.  n <= max_train_views (one activation arena; no chunking)."""
        self._check_cuda()
        if input_ids is None or pixel_values is None:
            raise ValueError("CLIPModel.forward_train needs both input_ids and pixel_values")
        if input_ids.dim() != 2:
            raise ValueError(f"input_ids must be [batch, sequence], got {tuple(input_ids.shape)}")
        n, S = input_ids.shape
        check_sequence_length(S, self.text_dims.max_positions)
        if pixel_values.shape[0] != n:
            raise ValueError(f"the contrastive loss needs as many images as captions (got {pixel_values.shape[0]} images, "
                             f"{n} captions)")
        if attention_mask is not None and tuple(attention_mask.shape) != (n, S):
            raise ValueError(f"attention_mask {tuple(attention_mask.shape)} does not match input_ids {(n, S)}")
        tr, tt = self._trainers()
        if n > tr.max_views:
            raise PigeonB200Error(f"{n} image-caption pairs exceed max_views={tr.max_views} of the training arena (a "
                                  f"contrastive batch is not split into chunks)")
        if n == 0:
            raise ValueError("forward_train needs at least one image-caption pair")
        tt.check_trainable()
        tr.layout()                                                      # raises if a block is only partly trainable
        dev = self.logit_scale.device
        vis_trains = tr.any_trainable()
        post = self.vision_model.post_layernorm
        eps = self.vision_dims.ln_eps
        Wv, Wt = self.visual_projection.weight, self.text_projection.weight
        lib = load()
        stream = current_stream_ptr()
        with torch.no_grad():
            # forward: CLS rows -> post_layernorm -> visual_projection; pooled text row -> text_projection
            px = pixel_values.to(dev)
            if px.dtype not in (torch.float16, torch.float32):
                px = px.float()
            tr.forward(px)
            cls = tr.cls_rows()
            pv = ops.layernorm_f32(cls, post.weight.detach(), post.bias.detach(), eps)
            img = ops.clip_project(pv, self._packed_projection("visual_projection"))
            pooled = tt.forward(input_ids.to(dev), None if attention_mask is None else attention_mask.to(dev))
            txt = ops.clip_project(pooled, self._packed_projection("text_projection"))
            out = ops.clip_loss_grad(img, txt, self.logit_scale)

            # backward: projections (pg_head_backward, no bias), post_layernorm, then both towers
            pend = {}

            def grad_buf(p):
                if not p.requires_grad:
                    return None
                pend[p] = torch.zeros_like(p, dtype=torch.float32)
                return pend[p]

            d_pv = torch.empty_like(pv)
            d_pooled = torch.empty_like(pooled)
            check(lib.pg_head_backward(ptr(out["d_image_embeds"]), ptr(pv), ptr(Wv.detach()), n, Wv.shape[0], Wv.shape[1], 1,
                                       ptr(grad_buf(Wv)), None, ptr(d_pv), stream), "pg_head_backward")
            check(lib.pg_head_backward(ptr(out["d_text_embeds"]), ptr(pooled), ptr(Wt.detach()), n, Wt.shape[0], Wt.shape[1],
                                       1, ptr(grad_buf(Wt)), None, ptr(d_pooled), stream), "pg_head_backward")
            if self.logit_scale.requires_grad:
                pend[self.logit_scale] = out["d_logit_scale"]
            dg, db = grad_buf(post.weight), grad_buf(post.bias)
            if (dg is None) != (db is None):
                raise PigeonB200Error("post_layernorm weight and bias must be trainable or frozen together")
            if vis_trains:
                d_cls = torch.empty_like(cls)
                check(lib.pg_layernorm_backward(ptr(d_pv), ptr(cls), ptr(post.weight.detach()), ptr(d_cls), 0, ptr(dg), ptr(db),
                                                None, n, cls.shape[1], eps, stream), "pg_layernorm_backward")
                tr.backward_cls(d_cls)
            elif dg is not None:
                scratch = torch.empty_like(cls)
                check(lib.pg_layernorm_backward(ptr(d_pv), ptr(cls), ptr(post.weight.detach()), ptr(scratch), 0, ptr(dg),
                                                ptr(db), None, n, cls.shape[1], eps, stream), "pg_layernorm_backward")
            tt.backward(d_pooled)
        self._pend = (pend, vis_trains)
        return CLIPOutput(loss=out["loss"], logits_per_image=out["logits_per_image"], logits_per_text=out["logits_per_text"],
                          text_embeds=txt / txt.norm(p=2, dim=-1, keepdim=True),
                          image_embeds=img / img.norm(p=2, dim=-1, keepdim=True))

    @torch.no_grad()
    def backward(self, loss: Optional[Tensor] = None) -> None:
        """Publish the gradients of the last `forward_train` into `.grad` under the HF names, adding to any gradient already
        there (gradient accumulation), like `SuperGuessr.backward`.  `loss` is accepted for the `loss.backward()` shape of
        the call and not used."""
        if self._pend is None:
            raise PigeonB200Error("backward() needs a preceding forward_train()")
        pend, vis_trains = self._pend
        self._pend = None
        for p, g in pend.items():
            put_grad(p, g.reshape(p.shape))
        if vis_trains:
            self._vision_trainer.finalize(1)
        self._text_trainer.finalize()
