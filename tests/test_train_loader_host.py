"""CPU: the training loader's sampler (monoflex_b200/loader.py TrainSampler, sampler_seed) against the unmodified
reference's TrainingSampler, BatchSampler(drop_last=True) and shared_random_seed (tests/golden/train_sampler.npz, written
by oracle/make_golden_train_sampler.py); the flip stream's properties; KittiTrainLoader's refusals, each before anything
is decoded; and the host-side flip of the camera matrix."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import GOLDEN
from monoflex_b200 import loader as L
from monoflex_b200 import targets as T
from monoflex_b200.config import default_cfg
from oracle import make_golden_train_sampler as mgs
from png_util import ihdr


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "train_sampler.npz")) as z:
        return {k: z[k] for k in z.files}


def rank_rows(size, seed, rank, world, n):
    s = L.TrainSampler(size, world, seed, rank, world)
    out, parts = [], s.rows()
    while sum(len(p) for p in out) < n:
        out.append(next(parts))
    return np.concatenate(out)[:n]


@pytest.mark.parametrize("size", mgs.SIZES)
@pytest.mark.parametrize("seed", mgs.SEEDS)
def test_indices_match_the_reference_sampler(gold, size, seed):
    for world, ranks in mgs.WORLDS.items():
        for rank in ranks:
            want = gold["idx_s%d_w%d_r%d_seed%d" % (size, world, rank, seed)].astype(np.int64)
            got = rank_rows(size, seed, rank, world, len(want))
            assert np.array_equal(got[:, 0], want), (world, rank)


@pytest.mark.parametrize("seed", mgs.SEEDS)
def test_batches_match_the_reference_batch_sampler_across_epochs(gold, seed):
    for world, rank in mgs.BATCH_RANKS:
        want = gold["batch_s7_w%d_r%d_seed%d" % (world, rank, seed)]
        it = iter(L.TrainSampler(7, mgs.BATCH * world, seed, rank, world))
        got = np.stack([next(it) for _ in range(len(want))])
        assert got.shape == (len(want), mgs.BATCH, 2)
        assert np.array_equal(got[:, :, 0], want), (world, rank)
        assert mgs.BATCH * mgs.BATCH_COUNT // world > 7           # the batches cross at least one epoch boundary


def test_seed_from_cfg_seed_is_the_reference_shared_seed(gold):
    state = np.random.get_state()
    for s, want in zip(gold["cfg_seeds"], gold["shared_seed"]):
        assert L.sampler_seed(NS(SEED=int(s))) == int(want)
    assert L.sampler_seed(NS(SEED=3), seed=99) == 99
    after = np.random.get_state()
    assert after[0] == state[0] and np.array_equal(after[1], state[1]) and after[2:] == state[2:]   # global RNG untouched


def test_default_seed_is_a_draw_from_the_global_rng_without_reseeding():
    for cfg in (NS(SEED=-1), NS()):                            # a cfg without SEED counts as -1 (config/defaults.py:338)
        np.random.seed(4321)
        want = np.random.RandomState(4321).randint(2 ** 31)
        assert L.sampler_seed(cfg) == want
        r = np.random.RandomState(4321)
        r.randint(2 ** 31)
        assert np.random.randint(1 << 30) == r.randint(1 << 30)    # one draw taken, nothing reseeded


@pytest.mark.parametrize("size,world", [(7, 2), (7, 8), (3712, 8), (13, 2)])
def test_rows_do_not_depend_on_the_world_size(size, world):
    n = 3 * size
    ref = rank_rows(size, 17, 0, 1, n)
    parts = [rank_rows(size, 17, r, world, -(-(n - r) // world)) for r in range(world)]
    inter = np.zeros((n, 2), dtype=np.int64)
    for r in range(world):
        inter[r::world] = parts[r]
    assert np.array_equal(inter, ref)


@pytest.mark.parametrize("size,world", [(3712, 2), (3712, 8), (7424, 8)])
def test_each_epoch_is_split_disjointly_across_ranks(size, world):
    for epoch in range(2):
        seen = []
        for r in range(world):
            rows = rank_rows(size, 5, r, world, 2 * size // world)
            seen.append(rows[epoch * (size // world):(epoch + 1) * (size // world), 0])
        allidx = np.concatenate(seen)
        assert len(np.unique(allidx)) == len(allidx) == size
        assert set(allidx.tolist()) == set(range(size))


def test_flips_are_deterministic_per_seed_and_differ_between_seeds():
    a = rank_rows(1000, 3, 0, 1, 3000)[:, 1]
    b = rank_rows(1000, 3, 0, 1, 3000)[:, 1]
    c = rank_rows(1000, 4, 0, 1, 3000)[:, 1]
    assert np.array_equal(a, b)
    assert not np.array_equal(a, c)
    assert set(np.unique(a).tolist()) == {0, 1}


def test_flip_frequency_is_p():
    n, p = 10 ** 5, 0.5
    flips = rank_rows(n, 11, 0, 1, n)[:, 1]
    assert abs(flips.mean() - p) <= 5 * np.sqrt(p * (1 - p) / n)


def test_flip_draws_leave_the_index_stream_untouched(gold, monkeypatch):
    want = gold["idx_s3712_w2_r1_seed0"].astype(np.int64)
    base = rank_rows(3712, 0, 1, 2, len(want))
    monkeypatch.setattr(L, "FLIP_SEED_OFFSET", 12345)
    moved = rank_rows(3712, 0, 1, 2, len(want))
    assert not np.array_equal(base[:, 1], moved[:, 1])
    assert np.array_equal(base[:, 0], want) and np.array_equal(moved[:, 0], want)
    s = L.TrainSampler(3712, 2, 0, 1, 2, flip_prob=0.0)
    assert np.array_equal(next(s.rows()), base[:1856] * [1, 0])             # p = 0: indices only


def test_ims_per_batch_not_divisible_by_the_world_raises():
    with pytest.raises(ValueError, match="IMS_PER_BATCH \\(6\\) must be divisible by the number of GPUs \\(4\\)"):
        L.TrainSampler(10, 6, 0, 0, 4)


def test_flip_calib_is_the_reference_formula():
    g = np.random.default_rng(2)
    P = g.normal(size=(6, 3, 4)) * 300
    widths = np.array([1242, 1224, 1238, 1241, 1226, 1234])
    flips = np.array([1, 0, 1, 1, 0, 1], dtype=bool)
    got = T.flip_calib(P, widths, flips)
    for b in range(6):
        want = P[b].copy()
        if flips[b]:
            want[0, 2] = widths[b] - want[0, 2] - 1
            want[0, 3] = -want[0, 3]
        assert np.array_equal(got[b], want)
    assert np.array_equal(T.flip_calib(P, widths, np.zeros(6, bool)), P)


# ----------------------------------------------------------------------------------------- refusals before any decode
IDS = ["000000", "000001", "000002"]


def train_cfg(right=False, split="train"):
    cfg = default_cfg()
    cfg.DATASETS.TRAIN_SPLIT = split
    cfg.DATASETS.USE_RIGHT_IMAGE = right
    cfg.SOLVER.IMS_PER_BATCH = 2
    return cfg


def make_dir(root, sizes=((64, 32), (48, 40), (80, 24)), right=True):
    from oracle import make_golden_targets as mg
    for d in ("image_2", "image_3", "label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    g = np.random.default_rng(0)
    for i, (w, h) in zip(IDS, sizes):
        for cam in ("image_2",) + (("image_3",) if right else ()):
            Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(os.path.join(root, cam, i + ".png"))
        with open(os.path.join(root, "calib", i + ".txt"), "w") as f:
            f.write(mg.calib_text(mg.make_P2(g, 1242, 375)))
        open(os.path.join(root, "label_2", i + ".txt"), "w").close()
    with open(os.path.join(root, "ImageSets", "train.txt"), "w") as f:
        f.write("".join(i + "\n" for i in IDS))


@pytest.fixture
def no_decode(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("decoded before the refusal")
    monkeypatch.setattr(L, "decode_windows", refuse)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (1 << 40, 1 << 40))


def test_refusals_without_a_split(tmp_path, no_decode):
    make_dir(str(tmp_path))
    with pytest.raises(ValueError, match="no split"):
        L.KittiTrainLoader(train_cfg(split=""), str(tmp_path))
    cfg = train_cfg()
    del cfg.DATASETS.TRAIN_SPLIT
    with pytest.raises(ValueError, match="no split"):
        L.KittiTrainLoader(cfg, str(tmp_path))
    with pytest.raises(FileNotFoundError, match="ImageSets file not exist.*trainval.txt"):
        L.KittiTrainLoader(train_cfg(), str(tmp_path), split="trainval")


def test_world_not_dividing_the_batch_raises(tmp_path, no_decode):
    make_dir(str(tmp_path))
    with pytest.raises(ValueError, match="must be divisible"):
        L.KittiTrainLoader(train_cfg(), str(tmp_path), rank=0, world=4)


def test_missing_right_image_raises(tmp_path, no_decode):
    make_dir(str(tmp_path))
    os.remove(os.path.join(str(tmp_path), "image_3", IDS[1] + ".png"))
    with pytest.raises(FileNotFoundError, match="image_3/%s.png" % IDS[1]):
        L.KittiTrainLoader(train_cfg(right=True), str(tmp_path))
    with pytest.raises(AssertionError, match="decoded before the refusal"):      # without USE_RIGHT_IMAGE it is not read
        L.KittiTrainLoader(train_cfg(right=False), str(tmp_path))


def test_oversize_image_raises(tmp_path, no_decode):
    make_dir(str(tmp_path))
    path = os.path.join(str(tmp_path), "image_3", IDS[2] + ".png")
    with open(path, "wb") as f:                                 # the IHDR alone is read before the decode
        f.write(b"\x89PNG\r\n\x1a\n" + ihdr(1281, 300))
    with pytest.raises(ValueError, match="image_3/%s.png: image 1281x300 larger than the input 1280x384" % IDS[2]):
        L.KittiTrainLoader(train_cfg(right=True), str(tmp_path))


def test_store_larger_than_free_memory_raises(tmp_path, no_decode, monkeypatch):
    make_dir(str(tmp_path))
    sizes = [(64, 32), (48, 40), (80, 24)] * 2
    store, filtered = L.window_bytes(sizes)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (store - 1, 1 << 40))
    with pytest.raises(MemoryError, match="take %d bytes on the device \\(%d with .*more than the %d bytes free"
                       % (store, store + 2 * filtered, store - 1)):
        L.KittiTrainLoader(train_cfg(right=True), str(tmp_path))
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (store + 2 * filtered, 1 << 40))
    with pytest.raises(AssertionError, match="decoded before the refusal"):        # fits: the decode comes next
        L.KittiTrainLoader(train_cfg(right=True), str(tmp_path))


def test_dataset_length_is_the_reference_len(tmp_path, no_decode):
    make_dir(str(tmp_path))
    for right in (False, True):
        ds = L.KittiTrainSplit(train_cfg(right=right), str(tmp_path), "train")
        assert len(ds) == T.dataset_len(3, train_cfg(right=right)) == (6 if right else 3)
