"""N-rank check of monoflex_b200.train.do_train on the path the reference's main() takes with more than one GPU
(tools/plain_train_net.py:127-140): the model wrapped in DistributedDataParallel(device_ids=[local rank],
broadcast_buffers=False, find_unused_parameters=True) before train() builds the optimiser from the wrapped model.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/do_train_two_rank_check.py

Each rank loads different synthetic weights, so the replicas agree only through DDP's start-up broadcast. do_train runs 12
iterations of B = 2 per rank on a generated KITTI-layout directory (KittiTrainLoader shards the sampler by rank), with a
checkpoint and an evaluation at 5 and 10 and model_final at 12; SyncBatchNorm is off (cfg.MODEL.USE_SYNC_BN False, so
main() does not convert). Checked: the parameters are bit-identical on every rank after the run; only rank 0 called the
checkpointer, and it saved model_checkpoint at 5 and 10, model_final at 12 and a best model at each evaluation whose AP
is not below the best so far; every TensorBoard event file was written by rank 0's process; every rank finished with
arguments['iteration'] == 12 and evaluated at 5 and 10. Prints one JSON line on rank 0; exit code != 0 on any mismatch.

--backend gloo runs the same check with every rank on the visible GPUs round-robin (several ranks on one GPU), which
NCCL does not allow; the NCCL run needs one GPU per rank."""
import argparse
import json
import os
import shutil
import sys
import tempfile

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from monoflex_b200 import loader as L                                 # noqa: E402
from monoflex_b200 import parallel                                    # noqa: E402
from monoflex_b200 import solver                                      # noqa: E402
from monoflex_b200 import synthetic as syn                            # noqa: E402
from monoflex_b200 import train as TR                                 # noqa: E402
from monoflex_b200.config import default_cfg                          # noqa: E402
from monoflex_b200.model.detector import KeypointDetector             # noqa: E402

MAX_ITER, INTERVAL, B = 12, 5, 2
VAL_IDS = ["000004", "000001", "000010"]


class Checkpointer(object):
    """utils/check_point.py's save(name, **kwargs) interface; records the calls, writes the reference's dict"""

    def __init__(self, model, optimizer, scheduler, save_dir):
        self.model, self.optimizer, self.scheduler, self.save_dir = model, optimizer, scheduler, save_dir
        self.calls = []

    def save(self, name, **kwargs):
        data = {"model": self.model.state_dict(), "optimizer": self.optimizer.state_dict(),
                "scheduler": self.scheduler.state_dict()}
        data.update(kwargs)
        torch.save(data, os.path.join(self.save_dir, "{}.pth".format(name)))
        self.calls.append((name, int(kwargs["iteration"])))


def gather(obj, world):
    out = [None] * world
    dist.all_gather_object(out, obj)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl", choices=("nccl", "gloo"))
    a = ap.parse_args()
    rank, world, local = parallel.env_rank()
    dev_index = local % torch.cuda.device_count()
    torch.cuda.set_device(dev_index)
    dev = torch.device("cuda", dev_index)
    parallel.init(a.backend, dev)
    assert world > 1, "run under torchrun with >= 2 ranks"
    tmp = gather(tempfile.mkdtemp(prefix="do_train_ranks_") if rank == 0 else None, world)[0]
    root, out = os.path.join(tmp, "kitti"), os.path.join(tmp, "out")
    if rank == 0:
        from test_gpu_train_loader import make_kitti
        make_kitti(root)
        with open(os.path.join(root, "ImageSets", "val.txt"), "w") as f:
            f.write("".join(i + "\n" for i in VAL_IDS))
        os.makedirs(out)
    dist.barrier()

    cfg = default_cfg()
    cfg.DATASETS.TRAIN_SPLIT, cfg.DATASETS.TEST_SPLIT, cfg.DATASETS.TEST = "train", "val", ("kitti_val",)
    cfg.DATASETS.USE_RIGHT_IMAGE = False
    cfg.SOLVER.IMS_PER_BATCH, cfg.TEST.IMS_PER_BATCH = B * world, B
    cfg.SOLVER.MAX_ITERATION, cfg.SOLVER.STEPS = MAX_ITER, (8,)
    cfg.SOLVER.EVAL_INTERVAL = cfg.SOLVER.SAVE_CHECKPOINT_INTERVAL = INTERVAL
    cfg.SOLVER.EVAL_AND_SAVE_EPOCH = False
    cfg.OUTPUT_DIR, cfg.START_TIME = out, "ranks"

    model = KeypointDetector(cfg).to(dev)
    model.load_state_dict(syn.make_state_dict(seed=rank), strict=False)      # replicas differ until DDP broadcasts
    if cfg.MODEL.USE_SYNC_BN:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[dev_index], broadcast_buffers=False,
                                                      find_unused_parameters=True)
    data_loader = L.KittiTrainLoader(cfg, root)
    data_loaders_val = L.KittiEvalLoader(cfg, root)
    optimizer = solver.build_optimizer(model, cfg)
    scheduler, warmup_scheduler = solver.build_scheduler(optimizer, total_iters_each_epoch=3, optim_cfg=cfg.SOLVER)
    arguments = {"iteration": 0, "iter_per_epoch": 3}
    checkpointer = Checkpointer(model, optimizer, scheduler, out)
    evals = []
    real_eval = TR.do_eval

    def do_eval(cfg_, net, loaders, iteration):
        evals.append(iteration)
        return real_eval(cfg_, net, loaders, iteration)
    TR.do_eval = do_eval
    p0 = optimizer.arena.params.clone()
    TR.do_train(cfg, True, model, data_loader, data_loaders_val, optimizer, scheduler, warmup_scheduler, checkpointer,
                dev, arguments)
    torch.cuda.synchronize()

    params = optimizer.arena.params
    replicas = [torch.zeros_like(params) for _ in range(world)]
    dist.all_gather(replicas, params)
    same = all(torch.equal(replicas[0], r) for r in replicas[1:])
    moved = not torch.equal(params, p0)
    info = gather({"rank": rank, "pid": os.getpid(), "iteration": arguments["iteration"], "saves": checkpointer.calls,
                   "evals": evals, "skipped": optimizer.skipped_steps()}, world)
    ok = True
    if rank == 0:
        writer_dir = os.path.join(out, "writer", cfg.START_TIME)
        event_files = [os.path.join(d, f) for d, _, fs in os.walk(writer_dir) for f in fs if f.startswith("events.")]
        pids = {int(os.path.basename(f).split(".")[-2]) for f in event_files}       # events.out.tfevents.<t>.<host>.<pid>.<n>
        saves0 = [n for n, _ in info[0]["saves"] if n != "model_moderate_best_soft"]
        bests = [it for n, it in info[0]["saves"] if n == "model_moderate_best_soft"]
        checks = {
            "params_identical": same,
            "params_trained": moved,
            "iteration_on_every_rank": all(i["iteration"] == MAX_ITER for i in info),
            "evaluated_on_every_rank": all(i["evals"] == [INTERVAL, 2 * INTERVAL] for i in info),
            "saves_on_rank0_only": all(not i["saves"] for i in info[1:]),
            "rank0_saves": saves0 == ["model_checkpoint", "model_checkpoint", "model_final"] and
            [it for n, it in info[0]["saves"] if n != "model_moderate_best_soft"] == [5, 10, 12] and
            bests[:1] == [5] and set(bests) <= {5, 10},
            "events_from_rank0_only": bool(event_files) and pids == {info[0]["pid"]},
            "files_on_disk": all(os.path.isfile(os.path.join(out, n + ".pth"))
                                 for n in ("model_checkpoint", "model_final", "model_moderate_best_soft")),
        }
        ok = all(checks.values())
        print(json.dumps({"world": world, "backend": a.backend, "ok": ok, "checks": checks, "ranks": info,
                          "event_files": [os.path.relpath(f, out) for f in event_files]}), flush=True)
    ok = gather(ok, world)[0]
    dist.barrier()
    if rank == 0:
        shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
