"""SuperGuessr — geocell classification model, H100 execution behind the reference's interface.

Mirror of reference models/super_guessr.py (same constructor arguments, `forward(...)` keyword names,
`ModelOutput` / serving tuple, `load_state`, `lla_geocells`, `cell_layer`, `num_cells`).  The arithmetic
of the inference branch (:386-466) and of the classification loss (:468-474) runs in the sm_90a kernels
of libpigeon_b200.so; there is no PyTorch/CPU fallback for it.
"""
from __future__ import annotations

import ctypes as C
import math
from types import SimpleNamespace
from typing import Optional

import pandas as pd
import torch
from torch import Tensor, nn
from torch.nn.parameter import Parameter

from . import _lib, _versions, ops
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr
from .config import (CLIP_EMBED_DIM, CLIP_PRETRAINED_HEAD, CLIP_PRETRAINED_HEAD_YFCC, GEOCELL_PATH, GEOCELL_PATH_YFCC,
                     LABEL_SMOOTHING_CONSTANT)
from .encoder import EncoderTower, Holder, encoder_holder, norm
from .model_utils import ModelOutput, TopK
from .vit_engine import VitDims, VitEngine

NUM_MULTI_TASK_VARIABLES = 6   # super_guessr.py:16-25
REGRESSION_LOSS_SCALING = 8
NUM_CLIMATES = 28
CLIMATE_LOSS_SCALING = 2
NUM_MONTHS = 12
MONTHS_LOSS_SCALING = 1
NUM_ATTENTION_HEADS = 16


class PositionalEncoder(nn.Module):
    """reference models/layers/positional_encoder.py: the sinusoidal table of the PyTorch transformer tutorial,
    pos_encoding [max_len, 1, dim] (a Parameter without gradient, so checkpoints carry it), and the dropout after the add.
    Its forward runs inside pg_view_attn_forward, where sample n of the batch gets row n on all four views, as the
    reference's `pos_encoding[:token_embedding.size(0)]` with batch_first inputs does."""

    def __init__(self, dim_model: int, dropout_p: float = 0.1, max_len: int = 1000):
        super().__init__()
        self.dropout = nn.Dropout(dropout_p)
        positions = torch.arange(0, max_len, dtype=torch.float).view(-1, 1)
        division = torch.exp(torch.arange(0, dim_model, 2).float() * (-math.log(10000.0)) / dim_model)
        table = torch.zeros(max_len, dim_model)
        table[:, 0::2] = torch.sin(positions * division)
        table[:, 1::2] = torch.cos(positions * division)
        self.pos_encoding = Parameter(table.unsqueeze(1), requires_grad=False)


class CLIPVisionTower(EncoderTower, nn.Module):
    """Drop-in for HF `CLIPVisionModel` on the path the reference uses (models/clip_embedder.py:26,63;
    evaluation/evaluate.py:36; models/super_guessr.py:137-160,395-398): same parameter names
    (`vision_model.embeddings...`, `vision_model.pre_layrnorm`, `vision_model.encoder.layers.N....`), `.config`,
    `.base_model`, `.vision_model.encoder.layers`, and `tower(pixel_values=...)` -> `.last_hidden_state`.
    fp32 master parameters live here; the fp16 kernel layouts are (re)packed lazily by `VitEngine`."""
    ENGINE, PASS_LIMIT = VitEngine, "max_views_per_pass"

    def __init__(self, dims: VitDims = VitDims(), name_or_path: str = ""):
        super().__init__()
        self.dims = dims
        self.config = SimpleNamespace(hidden_size=dims.hidden, intermediate_size=dims.intermediate,
                                      num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                                      image_size=dims.image_size, patch_size=dims.patch_size,
                                      layer_norm_eps=dims.ln_eps, _name_or_path=name_or_path)
        vm = Holder()
        emb = Holder()
        emb.class_embedding = Parameter(torch.zeros(dims.hidden))
        pe = Holder()
        pe.weight = Parameter(torch.zeros(dims.hidden, 3, dims.patch_size, dims.patch_size))
        emb.patch_embedding = pe
        pos = Holder()
        pos.weight = Parameter(torch.zeros(dims.tokens, dims.hidden))
        emb.position_embedding = pos
        vm.embeddings = emb
        vm.pre_layrnorm = norm(dims.hidden)  # [sic] HF spelling
        vm.encoder = encoder_holder(dims.hidden, dims.intermediate, dims.layers)
        vm.post_layernorm = norm(dims.hidden)  # present in HF checkpoints; unused by PIGEON (pooler_output)
        self.vision_model = vm
        self.max_views_per_pass = 256
        self.fold_layernorm = True   # LayerNorm applied in the GEMM epilogues (False = LayerNorm kernels; A/B switch)

    # HF: `CLIPVisionModel.base_model` is the model itself
    @property
    def base_model(self):
        return self

    @classmethod
    def from_hf(cls, hf_model) -> "CLIPVisionTower":
        """Build from a HuggingFace CLIPVisionModel / CLIPVisionTransformer instance (weights copied by name)."""
        cfg = hf_model.config
        tower = cls(VitDims.from_hf_config(cfg), name_or_path=getattr(cfg, "_name_or_path", ""))
        sd = {k if k.startswith("vision_model.") else "vision_model." + k: v for k, v in hf_model.state_dict().items()
              if "position_ids" not in k}
        missing, unexpected = tower.load_state_dict(sd, strict=False)
        if unexpected or any("post_layernorm" not in m for m in missing):
            raise PigeonB200Error(f"cannot map HF weights: missing={missing} unexpected={unexpected}")
        return tower

    def _repack_groups(self):
        """The "embeddings" group: patch / class / position embeddings and pre-LayerNorm."""
        vm = self.vision_model
        return list(vm.embeddings.parameters()) + list(vm.pre_layrnorm.parameters()), vm.encoder.layers

    def _engine_kwargs(self) -> dict:
        return {"fold_layernorm": bool(self.fold_layernorm)}

    @torch.no_grad()
    def embed(self, pixel_values: Tensor) -> Tensor:
        """Token mean of last_hidden_state, fused path (last_hidden_state is not returned)."""
        return self.engine().forward(pixel_values)

    @torch.no_grad()
    def forward(self, pixel_values: Tensor = None, **kwargs):
        emb, hidden = self.engine().forward(pixel_values, return_hidden=True)
        return SimpleNamespace(last_hidden_state=hidden, pooler_output=None, token_mean=emb)


def as_tower(base_model) -> Optional[CLIPVisionTower]:
    if base_model is None or isinstance(base_model, CLIPVisionTower):
        return base_model
    if hasattr(base_model, "config") and hasattr(base_model, "state_dict"):
        return CLIPVisionTower.from_hf(base_model)
    raise PigeonB200Error(f"unsupported base_model type {type(base_model).__name__}")


class SuperGuessr(nn.Module):
    def __init__(self, base_model: nn.Module, panorama: bool = False, hierarchical: bool = False,
                 should_smooth_labels: bool = False, multi_task: bool = False, heading: bool = False,
                 yfcc: bool = False, serving: bool = False, freeze_base: bool = False,
                 num_candidates: int = 5, embed_dim: int = CLIP_EMBED_DIM, **kwargs):
        """Same arguments as reference models/super_guessr.py:31-34.  `base_model` may be a `CLIPVisionTower`, a
        HuggingFace `CLIPVisionModel` (converted by name) or None (the model then runs on `embedding`).

        Extension (keyword-only): `geocells=` a (C, 2) array/tensor of (lng, lat) instead of reading the CSV."""
        super().__init__()
        geocells = kwargs.pop("geocells", None)
        if len(kwargs) > 0:
            print(f'Not using keyword arguments: {list(kwargs.keys())}')  # :67-68
        if heading and not panorama:
            raise NotImplementedError("heading features for single images are outside the H100 hot path")
        if hierarchical and heading:
            raise NotImplementedError("hierarchical=True with heading=True: the reference pads the attention width to "
                                      "input_dim + 14 and its cell layer then rejects the wider CLS row "
                                      "(super_guessr.py:90-98,420-433)")

        self.base_model = as_tower(base_model)
        self.panorama = panorama
        self.hidden_size = embed_dim
        self.serving = serving
        self.should_smooth_labels = should_smooth_labels
        self.multi_task = multi_task
        self.heading = heading
        self.yfcc = yfcc
        self.freeze_base = freeze_base
        self.hierarchical = hierarchical
        self.num_candidates = num_candidates

        self._set_hidden_size()
        if geocells is not None:
            # (.clone() keeps the strides of e.g. a Fortran-ordered numpy array: the kernels index it row-major)
            self.lla_geocells = Parameter(torch.as_tensor(geocells, dtype=torch.float64).contiguous().clone(),
                                          requires_grad=False)
        else:
            self.lla_geocells = self.load_geocells(GEOCELL_PATH_YFCC if self.yfcc else GEOCELL_PATH)
        self.num_cells = self.lla_geocells.size(0)
        self.input_dim = self.hidden_size   # panorama + heading leaves the input unchanged (:279-280)

        if self.hierarchical:                                                   # :94-103
            print('Number of attention heads:', NUM_ATTENTION_HEADS)
            self.pos_encoder = PositionalEncoder(self.input_dim)
            self.self_attn = nn.MultiheadAttention(self.input_dim, NUM_ATTENTION_HEADS, dropout=0.1, batch_first=True)
            self.relu = nn.ReLU()
        self.cell_layer = nn.Linear(self.input_dim, self.num_cells)
        self.softmax = nn.Softmax(dim=-1)
        if self.multi_task:
            print('Model is multi-task.')
            self.multi_task_head = nn.Linear(self.hidden_size, NUM_MULTI_TASK_VARIABLES)
            self.loss_fnc_mt = nn.MSELoss(reduction='mean')
            self.climate_layer = nn.Linear(self.input_dim, NUM_CLIMATES)
            self.loss_fnc_climate = nn.CrossEntropyLoss()
            if not self.yfcc:
                self.month_layer = nn.Linear(self.input_dim, NUM_MONTHS)
                self.loss_fnc_month = nn.CrossEntropyLoss()
        self._freeze_params()
        self.loss_fnc = nn.CrossEntropyLoss()
        self._w3 = None
        self._w3_key = None
        self._attn_packs = {}
        self._attn_state = None
        self.last_pooled = None
        print(f'Initialized SuperGuessr classification model with {self.num_cells} geocells.')

    # ---------------------------------------------------------------------------------- setup (reference :133-174)
    def _set_hidden_size(self):
        if self.base_model is not None:
            self.hidden_size = self.base_model.config.hidden_size
            self.mode = 'transformer'

    def _freeze_params(self):
        """reference :146-160: a frozen base model trains nothing in the tower; an unfrozen CLIP tower outside serving starts
        from the pretrained head checkpoint and trains only its last encoder layer."""
        tower = self.base_model
        if tower is None:
            return
        if self.freeze_base:
            tower.requires_grad_(False)
            return
        if self.serving or 'clip-vit' not in tower.config._name_or_path:
            return
        checkpoint = CLIP_PRETRAINED_HEAD_YFCC if self.yfcc else CLIP_PRETRAINED_HEAD
        self.load_state(checkpoint)
        print(f'Initialized model parameters from model: {checkpoint}')
        for layer in tower.vision_model.encoder.layers[:-1]:
            layer.requires_grad_(False)

    def load_geocells(self, path: str) -> Tensor:
        geo_df = pd.read_csv(path)
        lla_coords = torch.tensor(geo_df[['lng', 'lat']].values).contiguous()   # pandas hands out column-major blocks
        return Parameter(data=lla_coords, requires_grad=False)

    def load_state(self, path: str):
        """reference :222-238 — checkpoint entries are copied into the same-named entries of this module; a name this module
        does not have is reported on stdout and skipped (shape mismatches raise, as copy_ does)."""
        mine = self.state_dict()
        for key, value in torch.load(path, map_location=torch.device('cuda')).items():
            target = mine.get(key)
            if target is None:
                print(f'Parameter {key} not in model\'s state.')
            else:
                target.copy_(value.data if isinstance(value, Parameter) else value)
        if self.base_model is not None:
            self.base_model._weights_changed()

    def _assert_requirements(self, pixel_values=None, embedding=None, heading=None):
        if self.training and self.heading:
            assert heading is not None, 'If model is in heading mode, headings must be supplied during training.'
        if self.base_model is not None:
            assert pixel_values is not None, 'Parameter "pixel_values" must be supplied if model has a base model.'
        else:
            assert embedding is not None, 'Parameter "embedding" must be supplied if model does not have a base model.'

    # ---------------------------------------------------------------------------------- device plumbing
    def _device(self) -> torch.device:
        dev = self.cell_layer.weight.device
        if dev.type != 'cuda':
            raise PigeonB200Error("SuperGuessr is on the CPU: call .to('cuda') — the H100 path has no CPU implementation")
        return dev

    def _packed_head(self) -> Tensor:
        w = self.cell_layer.weight
        key = (w.data_ptr(), w._version, _versions.get(w))
        if self._w3 is None or self._w3_key != key:
            self._w3 = ops.head_pack_weight(w.detach())
            self._w3_key = key
        return self._w3

    # ---------------------------------------------------------------------------------- hierarchical head (:94-103, :414-433)
    def _hierarchical(self) -> bool:
        return self.hierarchical and self.panorama

    def _packed_attn(self):
        """fp16 split copies of in_proj_weight and out_proj.weight, repacked whenever the weights change (same key as
        `_packed_head`: torch's version counter plus the raw-pointer updates the optimizers record)."""
        out = []
        for w in (self.self_attn.in_proj_weight, self.self_attn.out_proj.weight):
            key = (w.data_ptr(), w._version, _versions.get(w))
            hit = self._attn_packs.get(id(w))
            if hit is None or hit[0] != key:
                hit = self._attn_packs[id(w)] = (key, ops.head_pack_weight(w.detach()))
            out.append(hit[1])
        return out

    def _attn_params(self):
        sa = self.self_attn
        return [sa.in_proj_weight, sa.in_proj_bias, sa.out_proj.weight, sa.out_proj.bias]

    def _draw_dropout_rng(self):
        """(seed, offset) of this forward's dropout masks, drawn once from torch's default generator in training mode, so
        torch.manual_seed reproduces a run; evaluation draws nothing (no dropout)."""
        if not self.training:
            return 0, 0
        seed, offset = torch.randint(0, 2 ** 62, (2,)).tolist()
        return seed, offset

    def _attn_forward(self, emb: Tensor, n0: int, rng) -> Tensor:
        """View self-attention of the panorama emb f32 [n, 4, E] (samples n0.. of the batch) -> the CLS row f32 [n, E];
        keeps what the backward needs in `self._attn_state`."""
        sa = self.self_attn
        p_x, p_attn = (float(self.pos_encoder.dropout.p), float(sa.dropout)) if self.training else (0.0, 0.0)
        w_in3, w_out3 = self._packed_attn()
        a = ops.view_attention_forward(emb, self.pos_encoder.pos_encoding.data, w_in3,
                                       sa.in_proj_bias.detach().float().contiguous(), w_out3,
                                       sa.out_proj.bias.detach().float().contiguous(), NUM_ATTENTION_HEADS, n0, p_x, p_attn,
                                       *rng)
        self._attn_state = dict(saved=a["saved"], n0=n0, p_x=p_x, p_attn=p_attn, seed=rng[0], offset=rng[1])
        return a["cls"]

    def _attn_backward(self, dcls: Tensor, grads, accumulate: bool) -> Tensor:
        st = self._attn_state
        return ops.view_attention_backward(dcls, st["saved"], self.self_attn.in_proj_weight, self.self_attn.out_proj.weight,
                                           NUM_ATTENTION_HEADS, st["n0"], st["p_x"], st["p_attn"], st["seed"], st["offset"],
                                           grads=grads, accumulate=accumulate)

    def _classification_loss(self, logits: Tensor, labels: Optional[Tensor], labels_clf: Tensor,
                             want_grad: bool = False, grad_scale: float = 1.0) -> Tensor:
        """reference :456,468-474 on the GPU (pg_head_loss); with `want_grad` also d loss / d logits (pg_head_loss_grad),
        kept in `self._saved_dlogits` for `backward()`."""
        B, Cc = logits.shape
        dev = logits.device
        per = torch.empty(B, dtype=torch.float64, device=dev)
        out = torch.empty(1, dtype=torch.float64, device=dev)
        dlog = torch.empty((B, Cc), dtype=torch.float32, device=dev) if want_grad else None
        lib = load()

        def run(mode, idx=None, soft=None, lab=None, cells=None, smoothing=0.0):
            if want_grad:
                check(lib.pg_head_loss_grad(ptr(logits), B, Cc, mode, ptr(idx), ptr(soft), ptr(lab), ptr(cells), smoothing,
                                            float(grad_scale), ptr(per), ptr(out), ptr(dlog), current_stream_ptr()),
                      "pg_head_loss_grad")
            else:
                check(lib.pg_head_loss(ptr(logits), B, Cc, mode, ptr(idx), ptr(soft), ptr(lab), ptr(cells), smoothing,
                                       ptr(per), ptr(out), current_stream_ptr()), "pg_head_loss")

        self._saved_dlogits = dlog
        if self.should_smooth_labels:
            lab = labels.to(device=dev, dtype=torch.float64).contiguous()
            run(2, lab=lab, cells=self.lla_geocells.data, smoothing=float(LABEL_SMOOTHING_CONSTANT))
            return out[0]                                    # float64, like the reference's promoted soft-target CE
        if labels_clf.dim() == 0:                            # _to_one_hot (:298-313)
            labels_clf = labels_clf.reshape(1).expand(B)
        if labels_clf.dim() == 1:
            run(0, idx=labels_clf.to(device=dev, dtype=torch.int64).contiguous())
        else:
            run(1, soft=labels_clf.to(device=dev, dtype=torch.float32).contiguous())
        return out[0].to(torch.float32)

    # ---------------------------------------------------------------------------------- fine-tune step (head only)
    def _trainable_outside_head(self):
        head = {id(self.cell_layer.weight), id(self.cell_layer.bias)}
        return [n for n, p in self.named_parameters() if p.requires_grad and id(p) not in head]

    def _forward_train_tower(self, pixel_values: Tensor, labels: Optional[Tensor], labels_clf: Tensor,
                             labels_multi_task=None, labels_climate=None, labels_month=None) -> ModelOutput:
        """Training-mode forward when tower parameters require grad (reference freeze policy :159-160): the batch is
        processed in chunks that fit the activation arena; each chunk runs tower forward -> head -> loss -> head
        backward -> tower backward, and gradients accumulate in pending buffers that `backward()` publishes (after the
        DDP-style all-reduce).  Numerically the sum over chunks of the mean-loss gradient = the full-batch gradient."""
        from .vit_train import TowerTrainer
        dev = self._device()
        if getattr(self, "_trainer", None) is None or self._trainer.tower is not self.base_model:
            self._trainer = TowerTrainer(self.base_model, max_views=getattr(self, "max_train_views", 64))
        tr = self._trainer
        tr.layout()                                            # raises if a block is only partly trainable
        V = 4 if self.panorama else 1
        B = pixel_values.size(0)
        s = self.base_model.dims.image_size
        px = pixel_values.reshape((B * V, 3, s, s))
        if labels_clf is None:
            raise AttributeError("'NoneType' object has no attribute 'dim' (labels_clf is required unless serving=True)")
        if labels_clf.dim() == 0:
            labels_clf = labels_clf.reshape(1).expand(B)
        step = max(1, tr.max_views // V)
        w, b = self.cell_layer.weight, self.cell_layer.bias
        Cc, D = w.shape
        head_trains = w.requires_grad
        hier = self._hierarchical()
        # the self_attn gradients ride in the head's flat buffer, so one all-reduce averages both
        attn_sizes = [p.numel() for p in self._attn_params()] if hier else []
        flat = torch.zeros(Cc * D + Cc + sum(attn_sizes), dtype=torch.float32, device=dev)
        attn_grads = list(torch.split(flat[Cc * D + Cc:], attn_sizes)) if hier else None
        rng = self._draw_dropout_rng() if hier else None
        lib = load()
        from . import dist as pdist
        pdist_world = pdist.world_size()
        outs, loss_total = [], None
        mt_out, mt_loss, mt_grads = [], [0, 0, 0], None
        with torch.no_grad():
            for lo in range(0, B, step):
                hi = min(B, lo + step)
                n = hi - lo
                emb = tr.forward(px[lo * V:hi * V].to(dev, non_blocking=True)).reshape(n, V, D)
                # the PE row of a sample is its index in the whole batch (lo + i), so chunks see what the whole batch sees
                head_in = self._attn_forward(emb.contiguous(), lo, rng).unsqueeze(1) if hier else emb.contiguous()
                h = ops.head_forward(head_in, self._packed_head(), b.detach().float().contiguous(),
                                     self.lla_geocells.data, self.num_candidates)
                loss = self._classification_loss(h["logits"], None if labels is None else labels[lo:hi], labels_clf[lo:hi],
                                                 want_grad=True, grad_scale=n / B)
                dlog, self._saved_dlogits = self._saved_dlogits, None
                dpooled = torch.empty((n, D), dtype=torch.float32, device=dev)
                check(lib.pg_head_backward(ptr(dlog), ptr(h["pooled"]), ptr(w.detach()), n, Cc, D, 1,
                                           ptr(flat) if head_trains else None, ptr(flat[Cc * D:]) if head_trains else None,
                                           ptr(dpooled), current_stream_ptr()), "pg_head_backward")
                if self.multi_task:
                    sl = lambda t: None if t is None else t[lo:hi]
                    mt = self._multi_task(h["pooled"], sl(labels_multi_task), sl(labels_climate), sl(labels_month), dev, True,
                                          weight=n / B)
                    mt_out.append(mt[:3])
                    for i in range(3):
                        mt_loss[i] = mt_loss[i] + mt[3 + i] * (n / B)
                    dpooled += mt[6]
                    mt_grads = mt[7] if mt_grads is None else [a + b_ for a, b_ in zip(mt_grads, mt[7])]
                if hier:                                                                  # backward of the view attention
                    d_emb = self._attn_backward(dpooled, attn_grads, accumulate=True).reshape(n * V, D)
                else:
                    d_emb = (dpooled / V).repeat_interleave(V, dim=0) if V > 1 else dpooled  # backward of the view mean
                # last chunk under torch.distributed: the gradient all-reduce rides behind this backward, bucket by bucket
                tr.backward(d_emb, overlap_world=pdist_world if hi == B else 1)
                part = loss.double() * (n / B)
                loss_total = part if loss_total is None else loss_total + part
                outs.append((h, emb))
        self._pend_head = flat
        self._pend_mt = mt_grads
        cat = lambda k: torch.cat([h[k] for h, _ in outs])
        embedding = torch.cat([e for _, e in outs])
        loss_clf = loss_total if self.should_smooth_labels else loss_total.to(torch.float32)
        # what the refiner gets: the view mean, or None when the head read the attention's CLS row (the refiner then
        # averages the raw views itself, proto_refiner.py:138-139)
        self.last_pooled = None if hier else cat("pooled")
        preds_mt = preds_climate = preds_month = None
        loss = loss_clf
        if self.multi_task:
            mcat = lambda i: None if mt_out[0][i] is None else torch.cat([m[i] for m in mt_out])
            preds_mt, preds_climate, preds_month = mcat(0), mcat(1), mcat(2)
            loss = loss_clf + mt_loss[0] + mt_loss[1] + mt_loss[2]
        return ModelOutput(loss, loss_clf, mt_loss[0], mt_loss[1], mt_loss[2], cat("pred_lnglat"), cat("pred_cell"), preds_mt,
                           preds_climate, preds_month, TopK(cat("topk_val"), cat("topk_idx")),
                           embedding if self.panorama else embedding[:, 0])

    def backward(self, loss: Optional[Tensor] = None, grad_scale: float = 1.0) -> None:
        """What `accelerator.backward(output.loss)` does in reference training/train_eval_loop.py:216 for the
        parameters this path trains: accumulates d loss / d cell_layer.{weight,bias} into `.grad` (pg_head_backward).
        Under torch.distributed the micro-batch gradient is all-reduced and averaged first, like DDP (:192)."""
        from . import dist as pdist
        if getattr(self, "_pend_head", None) is not None:
            # tower fine-tune path: forward() already ran forward + backward chunk by chunk; publish the gradients
            world = pdist.world_size()
            flat = self._pend_head
            self._pend_head = None
            if world > 1:
                torch.distributed.all_reduce(flat)
                flat.mul_(1.0 / world)
            w, b = self.cell_layer.weight, self.cell_layer.bias
            Cc, D = w.shape
            if w.requires_grad:
                if w.grad is None:
                    w.grad, b.grad = flat[: Cc * D].view(Cc, D), flat[Cc * D:Cc * D + Cc]
                else:
                    w.grad.add_(flat[: Cc * D].view(Cc, D))
                    b.grad.add_(flat[Cc * D:Cc * D + Cc])
            if self._hierarchical():
                self._publish_attn_grads(flat[Cc * D + Cc:])
            self._trainer.finalize(world)
            self._publish_mt_grads(getattr(self, "_pend_mt", None), world)
            self._pend_mt = None
            return
        if getattr(self, "_saved_dlogits", None) is None or getattr(self, "_head_in", None) is None:
            raise PigeonB200Error("backward() needs a preceding training-mode forward with labels")
        if self._hierarchical():
            self._backward_hierarchical(grad_scale)
            return
        w, b = self.cell_layer.weight, self.cell_layer.bias
        dlog, pooled = self._saved_dlogits, self._head_in
        B, Cc = dlog.shape
        D = pooled.shape[1]
        if grad_scale != 1.0:
            dlog = dlog * grad_scale
        lib = load()
        world = pdist.world_size()
        fresh = w.grad is None
        if fresh:                                             # one flat buffer -> one all-reduce for weight and bias
            flat = torch.empty(Cc * D + Cc, dtype=torch.float32, device=dlog.device)
            w.grad, b.grad = flat[: Cc * D].view(Cc, D), flat[Cc * D:]
            self._flat_grad = flat
        if world > 1:
            scratch = torch.empty(Cc * D + Cc, dtype=torch.float32, device=dlog.device)
            check(lib.pg_head_backward(ptr(dlog), ptr(pooled), None, B, Cc, D, 0, ptr(scratch), ptr(scratch[Cc * D:]), None,
                                       current_stream_ptr()), "pg_head_backward")
            torch.distributed.all_reduce(scratch)
            if fresh:
                self._flat_grad.copy_(scratch).mul_(1.0 / world)
            else:
                w.grad.add_(scratch[: Cc * D].view(Cc, D), alpha=1.0 / world)
                b.grad.add_(scratch[Cc * D:], alpha=1.0 / world)
        else:
            check(lib.pg_head_backward(ptr(dlog), ptr(pooled), None, B, Cc, D, 0 if fresh else 1, ptr(w.grad), ptr(b.grad),
                                       None, current_stream_ptr()), "pg_head_backward")
        self._saved_dlogits = None
        self._publish_mt_grads(getattr(self, "_saved_mt", None), world)
        self._saved_mt = None

    def _backward_hierarchical(self, grad_scale: float) -> None:
        """backward() of the hierarchical head on embeddings: cell_layer, the auxiliary heads' d output, then the view
        attention; the cell_layer and self_attn gradients share one flat buffer (one all-reduce under torch.distributed)."""
        from . import dist as pdist
        w, b = self.cell_layer.weight, self.cell_layer.bias
        dlog, cls = self._saved_dlogits, self._head_in
        if grad_scale != 1.0:
            dlog = dlog * grad_scale
        B, Cc = dlog.shape
        D = cls.shape[1]
        sizes = [Cc * D, Cc] + [p.numel() for p in self._attn_params()]
        flat = torch.empty(sum(sizes), dtype=torch.float32, device=dlog.device)
        gw, gb, *attn_grads = torch.split(flat, sizes)
        dcls = torch.empty((B, D), dtype=torch.float32, device=dlog.device)
        check(load().pg_head_backward(ptr(dlog), ptr(cls), ptr(w.detach()), B, Cc, D, 0, ptr(gw), ptr(gb), ptr(dcls),
                                      current_stream_ptr()), "pg_head_backward")
        if self._saved_mt_dx is not None:
            dcls += self._saved_mt_dx * grad_scale
        self._attn_backward(dcls, attn_grads, accumulate=False)
        world = pdist.world_size()
        if world > 1:
            torch.distributed.all_reduce(flat)
            flat.mul_(1.0 / world)
        if w.requires_grad:
            w.grad = gw.view(Cc, D).clone() if w.grad is None else w.grad.add_(gw.view(Cc, D))
            b.grad = gb.clone() if b.grad is None else b.grad.add_(gb)
        self._publish_attn_grads(flat[Cc * D + Cc:])
        self._saved_dlogits = None
        self._saved_mt_dx = None
        self._publish_mt_grads(getattr(self, "_saved_mt", None), world)
        self._saved_mt = None

    def _publish_attn_grads(self, flat: Tensor) -> None:
        """Accumulates the (already averaged) self_attn gradients held in `flat` into `.grad`."""
        for p, g in zip(self._attn_params(), torch.split(flat, [p.numel() for p in self._attn_params()])):
            if p.requires_grad:
                p.grad = g.view_as(p).clone() if p.grad is None else p.grad.add_(g.view_as(p))

    # ---------------------------------------------------------------------------------- multi-task heads (:315-348)
    _MT_HEADS = ("multi_task_head", "climate_layer", "month_layer")

    def _mt_params(self):
        return [p for n in self._MT_HEADS if hasattr(self, n) for p in getattr(self, n).parameters() if p.requires_grad]

    def _multi_task(self, output: Tensor, labels_multi_task, labels_climate, labels_month, dev, want_grad: bool,
                    weight: float = 1.0):
        """The three auxiliary Linear heads and their losses — thin PyTorch on the GPU, not a kernel target.  With
        `want_grad`, torch autograd also returns d(weight * their losses) / d pooled and their parameter gradients."""
        with (torch.enable_grad() if want_grad else torch.no_grad()):
            x = output.detach().requires_grad_(want_grad)
            preds_mt = self.multi_task_head(x)
            preds_climate = self.climate_layer(x)
            preds_month = None if self.yfcc else self.month_layer(x)
            loss_reg = loss_climate = loss_month = 0
            if not self.serving:
                loss_reg = self.loss_fnc_mt(preds_mt, labels_multi_task.to(dev)) * REGRESSION_LOSS_SCALING
                loss_climate = self.loss_fnc_climate(preds_climate, labels_climate.to(dev, torch.float32)) * CLIMATE_LOSS_SCALING
                if not self.yfcc:
                    loss_month = self.loss_fnc_month(preds_month, labels_month.to(dev)) * MONTHS_LOSS_SCALING
            dx, pgrads = None, None
            if want_grad:
                params = self._mt_params()
                g = torch.autograd.grad((loss_reg + loss_climate + loss_month) * weight, [x] + params)
                dx, pgrads = g[0], list(g[1:])
        det = lambda t: t.detach() if isinstance(t, Tensor) else t
        return (det(preds_mt), det(preds_climate), det(preds_month), det(loss_reg), det(loss_climate), det(loss_month),
                dx, pgrads)

    def _publish_mt_grads(self, pgrads, world: int) -> None:
        """Auxiliary-head gradients of this backward: averaged across ranks like DDP, then accumulated into `.grad`."""
        if not pgrads:
            return
        if world > 1:
            flat = torch.cat([g.reshape(-1) for g in pgrads])
            torch.distributed.all_reduce(flat)
            flat.mul_(1.0 / world)
            out, o = [], 0
            for g in pgrads:
                out.append(flat[o:o + g.numel()].view_as(g))
                o += g.numel()
            pgrads = out
        for p, g in zip(self._mt_params(), pgrads):
            p.grad = g.clone() if p.grad is None else p.grad.add_(g)

    # ---------------------------------------------------------------------------------- forward (reference :350-483)
    def forward(self, pixel_values: Tensor = None, embedding: Tensor = None, heading: Tensor = None,
                labels: Tensor = None, labels_clf: Tensor = None, labels_multi_task: Tensor = None,
                labels_climate: Tensor = None, labels_month: Tensor = None, index: Tensor = None) -> ModelOutput:
        self._assert_requirements(pixel_values, embedding, heading)
        want_grad = self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if want_grad:
            tower_trains = self.base_model is not None and any(p.requires_grad for p in self.base_model.parameters())
            stray = [n for n in self._trainable_outside_head()
                     if not n.startswith("base_model.") and n.split(".")[0] not in self._MT_HEADS + ("self_attn",)]
            if stray:
                raise NotImplementedError(f"no backward for trainable parameters {stray[:3]}")
            if tower_trains:
                return self._forward_train_tower(pixel_values, labels, labels_clf, labels_multi_task, labels_climate,
                                                 labels_month)
        dev = self._device()
        with torch.no_grad():
            # host -> device (reference _move_to_cuda, :193-217)
            # host pixel_values stay on the host here: VitEngine overlaps their H2D copy with compute, chunk by chunk
            if embedding is not None:
                embedding = embedding.to(dev, non_blocking=True)

            num_samples = None
            if self.panorama and pixel_values is not None:                      # :386-388
                num_samples = pixel_values.size(0)
                s = self.base_model.dims.image_size if self.base_model is not None else 336
                pixel_values = pixel_values.reshape((num_samples * 4, 3, s, s))

            if self.base_model is not None and pixel_values is not None:        # :391-405
                if pixel_values.dim() > 4:
                    pixel_values = pixel_values.squeeze(1)
                embedding = self.base_model.embed(pixel_values)                 # ViT + token mean, fused
                if self.panorama:
                    embedding = embedding.reshape((num_samples, 4, -1))

            layer_input = embedding.to(torch.float32)
            if self.panorama:                                                   # :437
                head_in = layer_input if layer_input.dim() == 3 else layer_input.unsqueeze(1)
            elif layer_input.dim() == 3 and layer_input.size(1) == 4:           # :440-441
                head_in = layer_input[:, 0].unsqueeze(1)
            else:
                head_in = layer_input.unsqueeze(1) if layer_input.dim() == 2 else layer_input
            head_in = head_in.contiguous()
            hier = self._hierarchical()
            if hier:                                                            # :414-433, CLS row of view 0
                head_in = self._attn_forward(head_in, 0, self._draw_dropout_rng()).unsqueeze(1)

            h = ops.head_forward(head_in, self._packed_head(), self.cell_layer.bias.detach().float().contiguous(),
                                 self.lla_geocells.data, self.num_candidates)   # :447-459
            output, logits = h["pooled"], h["logits"]
            self._head_in = output
            # extension: view-averaged embedding, reused by evaluation.predict_batch as the refiner's input; the hierarchical
            # head's CLS row is not what the refiner reads (proto_refiner.py:138-139 averages the raw views)
            self.last_pooled = None if hier else output
            pred_LLH, geocell_preds = h["pred_lnglat"], h["pred_cell"]
            geocell_topk = TopK(h["topk_val"], h["topk_idx"])

            preds_mt = preds_climate = preds_month = None
            loss_reg = loss_climate = loss_month = 0
            self._saved_mt = None
            self._saved_mt_dx = None
            if self.multi_task:                                                 # :315-348
                (preds_mt, preds_climate, preds_month, loss_reg, loss_climate, loss_month, mt_dx, mt_grads) = self._multi_task(
                    output, labels_multi_task, labels_climate, labels_month, dev, want_grad)
                self._saved_mt = mt_grads
                self._saved_mt_dx = mt_dx

            if not self.training and self.serving:                              # :462-466
                if self.multi_task:
                    return pred_LLH, geocell_topk, preds_mt, embedding
                return pred_LLH, geocell_topk, embedding

            if labels_clf is None:
                # the reference dereferences labels_clf unconditionally here (:456 -> _to_one_hot -> .dim())
                raise AttributeError("'NoneType' object has no attribute 'dim' (labels_clf is required unless serving=True)")
            loss_clf = self._classification_loss(logits, labels, labels_clf, want_grad=want_grad)
            loss = loss_clf
            if self.multi_task:
                loss = loss_clf + loss_reg + loss_climate + loss_month
            return ModelOutput(loss, loss_clf, loss_reg, loss_climate, loss_month, pred_LLH, geocell_preds, preds_mt,
                               preds_climate, preds_month, geocell_topk, embedding)

    def __str__(self):
        """Same text as the reference prints at start-up (:486-501): one tab-aligned `name = value` line per switch."""
        fields = (('base_model\t', self.base_model is not None), ('panorama\t', self.panorama),
                  ('hierarchical\t', self.hierarchical), ('multi-task\t', self.multi_task), ('yfcc\t\t', self.yfcc),
                  ('embedding_size\t', self.hidden_size), ('input_dim\t', self.input_dim),
                  ('num_geocells\t', self.num_cells), ('label_smoothing\t', self.should_smooth_labels),
                  ('uses_headings\t', self.heading), ('freeze_base\t', self.freeze_base), ('serving\t\t', self.serving))
        return 'SuperGuessr(\n' + ''.join(f'\t{name}= {value}\n' for name, value in fields) + ')'
