"""N-GPU check of SOLVER.GRAD_NORM_CLIP in the captured multi-GPU Trainer step: after the NCCL all-reduce of the gradient
arena, FusedAdamW.step(grad_scale=1/world, max_grad_norm=c) clips the RANK MEAN (DDP + clip_grad_norm_ in the reference),
on every rank alike.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/grad_clip_two_rank_check.py
c is half the mean gradient's norm of a first, unclipped step. Checked on the graph replays (steps 2 and 3): the norm the
kernel reports is above c and the same on every rank, world^-1 x the norm of the (summed) arena after the step is c, and the
parameter replicas are bit-identical. Prints one JSON line on rank 0; exit code != 0 on any mismatch."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monoflex_b200 import parallel                                    # noqa: E402
from monoflex_b200 import synthetic as syn                            # noqa: E402
from monoflex_b200.config import default_cfg                          # noqa: E402
from monoflex_b200.model.detector import KeypointDetector             # noqa: E402
from monoflex_b200.train import Trainer                               # noqa: E402


def same_on_all_ranks(x, world):
    x = x.reshape(-1)
    got = [torch.zeros_like(x) for _ in range(world)]
    dist.all_gather(got, x)
    return all(torch.equal(got[0], g) for g in got)


def main():
    rank, world, local = parallel.env_rank()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    parallel.init("nccl", dev)
    assert world > 1, "run under torchrun with >= 2 ranks"
    B = 2
    images = syn.make_images(B, 384, 1280, seed=100 + rank).to(dev)
    targets = [t.to(dev) for t in syn.make_train_param_lists(syn.make_train_targets(B, seed=5 + rank, empty_image=B))]

    def model():
        m = KeypointDetector(default_cfg()).to(dev)
        m.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        return m

    t0 = Trainer(model(), default_cfg(), loss_scale=128.0)
    t0.step(images, targets)                                           # arena = all-reduced SUM after the step
    c = 0.5 * float(t0.optimizer.arena.grads.double().norm()) / world
    del t0
    cfg = default_cfg()
    cfg.SOLVER.GRAD_NORM_CLIP = c
    tr = Trainer(model(), cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)
    res, ok = {"world": world, "clip": c}, True
    for i in range(4):
        tr.step(images, targets)
        if i < 2:
            continue
        torch.cuda.synchronize()
        norm = float(tr.optimizer.last_grad_norm)
        mean_after = float(tr.optimizer.arena.grads.double().norm()) / world
        want = c * norm / (norm + 1e-6)
        good = (tr._graph is not None and norm > c and abs(mean_after - want) <= 1e-5 * c
                and same_on_all_ranks(tr.optimizer.last_grad_norm, world)
                and same_on_all_ranks(tr.optimizer.arena.params, world))
        res["step%d" % i] = {"grad_norm": norm, "mean_norm_after_clip": mean_after, "ok": bool(good)}
        ok &= good
    ok &= tr.optimizer.skipped_steps() == 0
    ok = bool(parallel.max_over_ranks([0.0 if ok else 1.0], device=dev)[0] == 0.0)
    res["ok"] = ok
    if rank == 0:
        print(json.dumps(res), flush=True)
    tr._graph = None
    torch.cuda.synchronize()
    parallel.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
