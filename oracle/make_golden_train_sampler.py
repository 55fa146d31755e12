"""TEST INFRASTRUCTURE. Records tests/golden/train_sampler.npz from the UNMODIFIED reference's TrainingSampler
(data/samplers/distributed_sampler.py:12-54), torch's BatchSampler(drop_last=True) as data/build.py:104-107 wraps it, and
utils.comm.shared_random_seed after utils.envs.seed_all_rng, imported through oracle/ref_shims.py. utils.comm's rank and
world size are stubbed (no process group):

  * idx_s{size}_w{world}_r{rank}_seed{seed}: the first three epochs' part of the stream a rank iterates,
    `list(islice(iter(TrainingSampler(size, seed=seed)), n))` with n = ceil((3 * size - rank) / world), for SIZES x WORLDS
    (every rank of world 2, two ranks of world 8) x SEEDS;
  * batch_s{size}_w{world}_r{rank}_seed{seed}: the first BATCH_COUNT batches of BatchSampler(..., BATCH, drop_last=True)
    over size 7, which cross the epoch boundaries;
  * shared_seed: comm.shared_random_seed() at world 1 after seed_all_rng(s), for s in CFG_SEEDS - the sampler seed of a
    run with cfg.SEED = s (default_setup calls seed_all_rng(cfg.SEED + rank); nothing draws from numpy's global RNG before
    make_data_loader in tools/plain_train_net.py).

    python oracle/make_golden_train_sampler.py        (needs the reference tree; writes tests/golden/train_sampler.npz)
"""
import itertools
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "train_sampler.npz")

# read by tests/test_train_loader_host.py
SIZES = (7, 3712, 7424)
WORLDS = {1: (0,), 2: (0, 1), 8: (0, 5)}
SEEDS = (0, 1234567)
BATCH, BATCH_COUNT = 3, 6
BATCH_RANKS = ((1, 0), (2, 1))
CFG_SEEDS = (0, 7, 12345)


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_shims
    ref_shims.install()
    import torch
    from utils import comm
    from utils.envs import seed_all_rng
    from data.samplers.distributed_sampler import TrainingSampler

    out = {}
    for size in SIZES:
        for world, ranks in WORLDS.items():
            for rank in ranks:
                for seed in SEEDS:
                    with mock.patch.object(comm, "get_rank", lambda: rank), \
                            mock.patch.object(comm, "get_world_size", lambda: world):
                        s = TrainingSampler(size, seed=seed)
                    n = -(-(3 * size - rank) // world)
                    out["idx_s%d_w%d_r%d_seed%d" % (size, world, rank, seed)] = np.array(
                        [int(i) for i in itertools.islice(iter(s), n)], dtype=np.int16)          # every size < 2 ** 15
    for world, rank in BATCH_RANKS:
        for seed in SEEDS:
            with mock.patch.object(comm, "get_rank", lambda: rank), mock.patch.object(comm, "get_world_size", lambda: world):
                s = TrainingSampler(7, seed=seed)
            bs = torch.utils.data.sampler.BatchSampler(s, BATCH, drop_last=True)
            out["batch_s7_w%d_r%d_seed%d" % (world, rank, seed)] = np.array(
                [[int(i) for i in b] for b in itertools.islice(iter(bs), BATCH_COUNT)], dtype=np.int64)
    seeds = []
    for s in CFG_SEEDS:
        seed_all_rng(s)
        seeds.append(comm.shared_random_seed())
    out["shared_seed"] = np.array(seeds, dtype=np.int64)
    out["cfg_seeds"] = np.array(CFG_SEEDS, dtype=np.int64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "shared seeds", dict(zip(CFG_SEEDS, seeds)))


if __name__ == "__main__":
    main()
