"""Two-GPU check of the pretraining loop's data parallelism (torchrun --nproc-per-node 2): 2 ranks x acc 1 must give the same
parameters as 1 rank x acc 2 over the same micro-batches.  Each rank's contrastive batch is its own (HF CLIPModel does not
gather features across ranks), so rank r takes micro-batch r of each pair; the single-rank reference runs on rank 0 with
the two micro-batches of a pair accumulated.  Exit code 0 on success.

    python -m torch.distributed.run --nproc-per-node 2 tools/ddp_pretrain_check.py
"""
import os
import sys
from types import SimpleNamespace

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


class _Pairs(torch.utils.data.Dataset):
    def __init__(self, rows):
        self.rows = rows

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, i):
        return self.rows[i]


def _run(rows, acc, collate, out_dir):
    import make_clip_pretrain_golden as G
    from pigeon_b200 import CLIPModel
    from pigeon_b200.pretrain import CLIPPretrainer
    td, vd, P, sd, _, _, _ = G.setup()
    m = CLIPModel(td, vd, projection_dim=P)
    m.load_state_dict(sd)
    m = m.cuda()
    s = G.SETTINGS
    args = SimpleNamespace(output_dir=out_dir, per_device_train_batch_size=s["batch"], gradient_accumulation_steps=acc,
                           num_train_epochs=1, max_steps=3, learning_rate=s["lr"], adam_beta1=0.9, adam_beta2=0.98,
                           adam_epsilon=1e-6, weight_decay=0.1, max_grad_norm=s["max_grad_norm"], warmup_ratio=0.0,
                           lr_scheduler_type="linear", logging_steps=1, evaluation_strategy="no", save_strategy="no", seed=1)
    tr = CLIPPretrainer(m, args, rows, None, data_collator=collate)
    tr.train()
    return {n: p.detach().clone() for n, p in m.named_parameters()}


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    assert world == 2
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl")
    import make_clip_pretrain_golden as G
    _, _, _, _, rows, _, collate = G.setup()
    rows = rows[:24]
    # DistributedSampler(shuffle) with num_replicas=2 deals permutation[rank::2]; the single-rank run must see, per update,
    # the batch of rank 0 then that of rank 1: build its dataset in exactly that order and keep it unshuffled.
    g = torch.Generator().manual_seed(1)
    perm = torch.randperm(len(rows), generator=g).tolist()
    per_rank = [perm[r::2] for r in range(2)]
    b = G.SETTINGS["batch"]
    ordered = []
    for k in range(len(per_rank[0]) // b):
        for r in range(2):
            ordered += per_rank[r][k * b:(k + 1) * b]
    two = _run(_Pairs(rows), 1, collate, "/nonexistent")
    ok = True
    if rank == 0:
        dist.destroy_process_group()
        import pigeon_b200.pretrain as P
        orig = P.DistributedSampler

        class Ordered(torch.utils.data.Sampler):                     # the order above, for one rank
            def __init__(self, ds, **kw):
                self.n = len(ds)

            def set_epoch(self, e):
                pass

            def __iter__(self):
                return iter(ordered)

            def __len__(self):
                return self.n
        P.DistributedSampler = Ordered
        one = _run(_Pairs(rows), 2, collate, "/nonexistent")
        P.DistributedSampler = orig
        worst = max(((two[n].double() - one[n].double()).norm() / one[n].double().norm().clamp_min(1e-30)).item()
                    for n in one)
        print(f"ddp pretrain: 2 ranks x acc 1 vs 1 rank x acc 2, worst per-tensor relative difference {worst:.3e}",
              flush=True)
        ok = worst < 1e-3             # float-atomic LayerNorm / bias column sums differ in the last bits
    else:
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
