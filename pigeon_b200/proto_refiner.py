"""ProtoRefiner — prototype-retrieval guess refinement, H100 execution behind the reference's interface.

Mirror of reference models/proto_refiner.py: same constructor arguments and `forward(...)` keyword names and
return value `(loss, preds_LLH, preds_geocell)`.  The per-query / per-candidate Python loops of the reference
(:154-222) run as three kernels over a CSR bank resident in HBM (csrc/refiner.cu); no CPU fallback.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch
from torch import Tensor, nn
from torch.nn.parameter import Parameter

from . import bank as bank_mod
from . import dist as dist_mod
from . import ops
from ._lib import PigeonB200Error
from .config import DATASET_PATH, PROTO_PATH


class ProtoRefiner(nn.Module):
    """Proto-Net refinement model (reference models/proto_refiner.py:17)."""

    def __init__(self, topk: int = 5, hedge: bool = False, max_refinement: int = 1000, temperature: float = 1.6,
                 proto_path: str = PROTO_PATH, dataset_path: str = DATASET_PATH, protos: Optional[object] = None,
                 verbose: bool = False, device: str | torch.device = 'cuda', shard_cells: bool = False):
        """Arguments as in the reference (:20-44).  `protos` may be

          * a dict of CSR arrays (layout of `pg_refiner_bank`; what `self.protos` of this class holds, so the
            reference's pickle-and-reload flow at evaluation/evaluate.py:67-80 round-trips), or
          * the reference's own list (one entry per geocell: None or a per-cell dataset with lng / lat / count /
            indices / embedding rows) — then `dataset_path` must still point at the training embeddings;
          * None: the bank is built from `proto_path` + `dataset_path` like the reference constructor does.

        `shard_cells` (extension, multi-GPU): under torch.distributed with world size W each rank keeps only the geocells
        with cell % W == rank in HBM, scans every query against its own cells, and the per-candidate partials are
        merged by owner through one small all-gather before the final stage — same outputs as the replicated bank.
        """
        super().__init__()
        if hedge:
            raise NotImplementedError("hedge=True (HedgeLayer, unused in the final model: models/README.md:11, "
                                      "evaluate.py:73,79) is outside the H100 hot path")
        self.topk = topk
        self.hedge = hedge
        self.max_refinement = max_refinement
        self.verbose = verbose
        self.shard_cells = bool(shard_cells)
        self._device = torch.device(device)

        if isinstance(protos, dict):
            arrays = protos
        elif protos is not None:
            from datasets import DatasetDict
            train = DatasetDict.load_from_disk(dataset_path)['train'].with_format('numpy')
            cells = [None if d is None else [d[i] for i in range(len(d))] for d in protos]
            arrays = bank_mod.bank_from_proto_rows(cells, np.asarray(train['embedding'], np.float32),
                                                   np.asarray(train['labels'], np.float32))
        else:
            print('Initializing ProtoRefiner. This might take a while ...')          # :263
            arrays = bank_mod.bank_from_reference_files(proto_path, dataset_path, device=self._device)
            print('Initialization of ProtoRefiner complete.')                        # :286
        self.protos: Dict[str, np.ndarray] = arrays
        self.num_geocells = int(arrays['cell_off'].shape[0]) - 1
        self._bank: Optional[ops.DeviceBank] = None

        # "Learnable" parameters, frozen in the reference (:89-90)
        self.temperature = Parameter(torch.tensor(temperature), requires_grad=False)
        self.geo_scaling = Parameter(torch.tensor(20.), requires_grad=False)

    def __getstate__(self):  # device handles are rebuilt after unpickling (torch.save(refiner), evaluate.py:71)
        d = self.__dict__.copy()
        d['_bank'] = None
        d.pop('_bank_world', None)
        return d

    def __str__(self):
        rep = 'ProtoRefiner(\n'
        rep += f'\ttopk\t\t= {self.topk}\n'
        rep += f'\thedge\t\t= {self.hedge}\n'
        rep += f'\tmax_refinement\t= {self.max_refinement}\n'
        rep += f'\ttemperature\t= {self.temperature.data.item()}\n'
        rep += f'\tgeo_scaling\t= {self.geo_scaling.data.item()}\n'
        rep += ')'
        return rep

    def device_bank(self) -> ops.DeviceBank:
        if self._bank is None:
            if self._device.type != 'cuda':
                raise PigeonB200Error("ProtoRefiner needs a CUDA device (no CPU path)")
            arrays = self.protos
            self._bank_world = 1
            if self.shard_cells and dist_mod.is_distributed():
                import torch.distributed as dist
                self._bank_world = dist.get_world_size()
                arrays = bank_mod.shard_bank(arrays, dist.get_rank(), self._bank_world)
            self._bank = ops.DeviceBank(self._device, **arrays)
        return self._bank

    @torch.no_grad()
    def forward(self, embedding: Tensor = None, geo_tensor: Tensor = None, initial_preds: Tensor = None,
                candidate_cells: Tensor = None, candidate_probs: Tensor = None, cluster: Tensor = None,
                return_debug: bool = False):
        """reference :121-231.  Returns (loss, preds_LLH float32 [B,2], preds_geocell int64 [B])."""
        assert self.topk <= candidate_cells.size(1), \
            '"topk" parameter must be smaller or equal to the number of geocell candidates \
             passed into the forward function.'
        bank = self.device_bank()
        dev = bank.device
        embedding = embedding.to(dev, torch.float32)
        candidate_cells = candidate_cells.to(dev)
        if candidate_probs is None:                                               # :143-145
            candidate_probs = torch.zeros(candidate_cells.shape, dtype=torch.float32, device=dev)
            candidate_probs[:, 0] = 1
        loss = 0 if self.training else None                                       # :151
        if getattr(self, "_bank_world", 1) > 1:
            return self._forward_sharded(bank, embedding, initial_preds.to(dev), candidate_cells, candidate_probs.to(dev),
                                         loss, return_debug)
        res = ops.refiner_forward(bank, embedding, initial_preds.to(dev), candidate_cells, candidate_probs.to(dev),
                                  self.topk, float(self.temperature.item()), float(self.max_refinement),
                                  debug=return_debug or self.verbose)
        if self.verbose:                                                          # :224-227 (costs a device sync)
            perc_changed = (res[2]["choice"] != 0).sum() / res[2]["choice"].size(0)
            print(f'Changed geocell predictions of {perc_changed * 100:.1f} % of guesses.')
        if return_debug:
            return loss, res[0], res[1], res[2]
        return loss, res[0], res[1]

    def _forward_sharded(self, bank, embedding, initial_preds, candidate_cells, candidate_probs, loss, return_debug):
        """Cell-sharded bank: every rank holds the SAME queries (the gathered batch), scans them against its own geocells,
        then one packed all-gather of the (B, topk, 3) partials, merge by owner, final stage on every rank."""
        world = self._bank_world
        cand = candidate_cells[:, : self.topk].to(torch.int64)
        bl, bll, bp = ops.refiner_scan(bank, embedding, candidate_cells, self.topk)
        gathered = dist_mod.all_gather_rows(dict(best_logit=bl, best_lnglat=bll))
        merged = dist_mod.merge_partials_by_owner(gathered, cand, world)
        ll, cell, choice = ops.refiner_finalize(merged["best_logit"], merged["best_lnglat"], initial_preds,
                                                candidate_cells, candidate_probs, self.topk,
                                                float(self.temperature.item()), float(self.max_refinement))
        if self.verbose:
            perc_changed = (choice != 0).sum() / choice.size(0)
            print(f'Changed geocell predictions of {perc_changed * 100:.1f} % of guesses.')
        if return_debug:
            return loss, ll, cell, dict(best_logit=merged["best_logit"], best_lnglat=merged["best_lnglat"], choice=choice)
        return loss, ll, cell
