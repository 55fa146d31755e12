"""The evaluation loader: `make_data_loader(cfg, is_train=False)` of the reference (data/build.py, KITTIDataset +
BatchCollator, data/collate_batch.py) with the PNG decode, the padding / normalisation and the target encoding on the GPU.

    loader = KittiEvalLoader(cfg, "kitti/training")                # split: cfg.DATASETS.TEST_SPLIT, e.g. "val"
    for batch in loader:                                           # dict(images=ImageList, targets=(ParamsList, ...),
        output, eval_utils, _ = model(batch["images"], batch["targets"])   #      img_ids=("000001", ...))

It reads ImageSets/<split>.txt in order, TEST.IMS_PER_BATCH images per batch. Images are image_2/<id>.png through
decode_png (csrc/mf_png.cu) and GpuInputPipeline.images; a labelled split's targets are GpuTargetEncoder.encode(labels,
P2, sizes, flips=None).param_lists() from label_2 and calib, the test split's are encode_inference(P2, sizes). The
targets carry no `ori_img`: only the reference's visualiser reads it, and the visualiser is not part of this package.

The files are decoded DECODE_WINDOW images at a time (rounded up to whole batches). While the consumer runs the model on
one window, the next one decodes on a side stream ordered by events. The one after it has its host half (reading the
files, their CRCs, staging them in pinned memory: about 2.3-2.4 ms per 800 KB file) done on a worker thread. Each
window's status is checked before its first batch is yielded, so a malformed file raises ValueError before any
detection of its window is written; a file the host rejects raises one window earlier still. When the decoded split fits
in free device memory, the first complete pass keeps it and later passes read it back (KittiEvalLoader).

The training loader: `make_data_loader(cfg, is_train=True)` (data/build.py: TrainingSampler, BatchSampler(drop_last=True),
KITTIDataset with its horizontal flip and right-camera items) from images decoded once into device memory.

    loader = KittiTrainLoader(cfg, "kitti/training")               # split: cfg.DATASETS.TRAIN_SPLIT, e.g. "train"
    for batch in loader:                                           # infinite, as the reference's
        loss_dict, log = model(batch["images"], batch["targets"])  # or Trainer.step(batch["images"].tensors,
                                                                   #                 batch["encoded"], sync_log=False)

At construction it reads every label and calibration file and every image's IHDR, refuses what the reference would
refuse (before any decode), decodes every view (image_2, and image_3 with DATASETS.USE_RIGHT_IMAGE) into a store of
uint8 HWC images in device memory and encodes every view in both flip states once to find the items the reference
cannot encode. A batch is then GpuInputPipeline.images over store views and GpuTargetEncoder.encode over rows of host
tables: no file, no decode and no host synchronisation per batch.
"""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import targets as T
from .data import GpuInputPipeline
from .png import DecodedImages, PngBatch, read_ihdr, read_png, window_bytes
from .structures import to_image_list

# Images decoded per launch, chosen with tools/bench_png.py (README, "PNG decode and evaluation loader"). A launch takes
# about 215 ms for 8 to 256 images, because one warp inflates one image serially, so the window sets the kernels'
# throughput: 0.84 ms per image at 256. That is above the strict model's rate at B = 1 and B = 8. The whole loop still
# runs below the same loop fed from pinned memory. At 1024 the kernels take 0.26 ms per image, but the loop at B = 8
# ran slower than at 256.
DECODE_WINDOW = 256


def decode_windows(windows, device="cuda"):
    """Decode windows (lists of PNG paths) in order and yield each window's DecodedImages, checked and ordered before the
    current stream's later work. While the consumer works on window k, window k + 1 decodes on a side stream and window
    k + 2 is read, checked and staged in pinned memory on a worker thread. A malformed file raises ValueError when its
    window comes up, before that window is yielded; a file the host rejects raises one window earlier."""
    device = torch.device(device)
    main = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device)
    pool = ThreadPoolExecutor(max_workers=1)
    staged = []

    def launch(batch):
        with torch.cuda.stream(side):
            return DecodedImages(batch, device)

    try:
        staged = [pool.submit(_stage, w) for w in windows[:2]]
        pending = launch(staged.pop(0).result()) if windows else None
        for k in range(len(windows)):
            dec = pending
            if k + 2 < len(windows):
                staged.append(pool.submit(_stage, windows[k + 2]))
            pending = launch(staged.pop(0).result()) if staged else None
            dec.check()
            main.wait_event(dec.event)
            dec.buffer.record_stream(main)              # read on the main stream after the side stream lets it go
            yield dec
    finally:
        for f in staged:
            f.cancel()
        pool.shutdown(wait=True)


def _stage(paths):
    """the host half of a window's decode: read, check and stage its files (runs in the worker thread)"""
    return PngBatch([read_png(p) for p in paths])


def store_budget(sizes, window, device="cuda"):
    """(store bytes, bytes needed, bytes free) of decoding images of `sizes` ((w, h) each) `window` at a time and keeping
    them in device memory: the store is every window's images buffer (window_bytes), the need adds the transient filtered
    buffers of the two windows decode_windows has in flight, the free bytes are torch.cuda.mem_get_info's. Both loaders
    keep their images only when need <= free."""
    per_window = [window_bytes(sizes[i:i + window]) for i in range(0, len(sizes), window)]
    store = int(sum(b for b, _ in per_window))
    need = store + 2 * max([f for _, f in per_window] + [0])
    return store, need, torch.cuda.mem_get_info(device)[0]


class KittiSplit(object):
    """What the reference's KITTIDataset exposes to the evaluation (engine/inference.py, inference_all_depths): the split
    file, the label directory, the classes and the ids in the split's order."""

    def __init__(self, cfg, root, split):
        self.root, self.split = root, split
        self.image_dir = os.path.join(root, "image_2")
        self.label_dir = os.path.join(root, "label_2")
        self.calib_dir = os.path.join(root, "calib")
        self.imageset_txt = os.path.join(root, "ImageSets", "{}.txt".format(split))
        if not os.path.exists(self.imageset_txt):
            raise FileNotFoundError("ImageSets file not exist, dir = {}".format(self.imageset_txt))
        with open(self.imageset_txt) as f:
            self.ids = [line.replace("\n", "") for line in f]
        self.classes = cfg.DATASETS.DETECT_CLASSES
        self.labelled = split != "test"

    def __len__(self):
        return len(self.ids)


class KittiEvalLoader(object):
    """The reference's evaluation loader on the GPU (module docstring), TEST.IMS_PER_BATCH images per batch.

    The first complete pass also keeps what it decoded and encoded: each window's images buffer and every batch's
    targets. Later passes read them back - no file, no PNG decode, no label or calibration parsing and no host
    synchronisation per batch, only GpuInputPipeline.images over the kept views - and yield the same batches, bit for
    bit. Keeping is decided from free device memory, by KittiTrainLoader's rule (store_budget: the images plus the
    decode's transient buffers against torch.cuda.mem_get_info), before the first window and again before each later
    one. It is all or nothing: when a window does not fit, what was kept is dropped and every pass streams. KITTI val
    (3,769 images of about 1242x375) holds about 5.2 GB (`store_bytes`); dropping the loader releases it. The kept
    passes see the split as it was read: files changed after the first complete pass are not read again. A pass the
    consumer leaves early keeps nothing."""

    def __init__(self, cfg, root, split=None, device="cuda"):
        self.dataset = KittiSplit(cfg, root, cfg.DATASETS.TEST_SPLIT if split is None else split)
        self.batch_size = int(getattr(cfg.TEST, "IMS_PER_BATCH", 1))
        if self.batch_size < 1:
            raise ValueError("TEST.IMS_PER_BATCH = %d" % self.batch_size)
        self.window = -(-DECODE_WINDOW // self.batch_size) * self.batch_size
        self.device = torch.device(device)
        self.pipe = GpuInputPipeline(cfg, device)
        self.encoder = T.GpuTargetEncoder(cfg, device)
        self.max_objs = int(cfg.DATASETS.MAX_OBJECTS)
        self.store_bytes = None           # the images' device bytes, once a pass has read the headers
        self._kept = None                 # [(image views, targets, ids)] per batch, after a complete kept pass

    @property
    def kept(self):
        """True when the passes read the images and targets kept by the first complete pass"""
        return self._kept is not None

    def __len__(self):
        return -(-len(self.dataset) // self.batch_size)

    def batches(self):
        """the split's ids grouped as the loader yields them"""
        ids, B = self.dataset.ids, self.batch_size
        return [ids[i:i + B] for i in range(0, len(ids), B)]

    def _targets(self, ids, sizes):
        ds = self.dataset
        P2 = np.stack([T.read_kitti_calib(os.path.join(ds.calib_dir, i + ".txt")) for i in ids])
        sizes = np.asarray(sizes, dtype=np.int64).reshape(-1, 2)
        if not ds.labelled:
            return tuple(self.encoder.encode_inference(P2, sizes))
        labels = T.pack_labels([T.read_kitti_label(os.path.join(ds.label_dir, i + ".txt"), tuple(ds.classes))
                                for i in ids], self.max_objs)
        enc = self.encoder.encode(labels, P2, sizes, flips=None)
        out = tuple(enc.param_lists())
        enc.check()
        return out

    def _image_sizes(self, paths):
        """(w, h) of every image from its IHDR, or None when a header cannot be read: that file then raises where the
        streamed pass reaches it, as it does without keeping"""
        try:
            return [read_ihdr(p) for w in paths for p in w]
        except (OSError, ValueError, NotImplementedError):
            return None

    def _fits(self, sizes):
        store, need, free = store_budget(sizes, self.window, self.device)
        return need <= free

    def __iter__(self):
        if self._kept is not None:
            for views, targets, ids in self._kept:
                images, _ = self.pipe.images(views)
                yield dict(images=to_image_list(images), targets=targets, img_ids=ids)
            return
        batches = self.batches()
        per = self.window // self.batch_size
        windows = [sum(batches[i:i + per], []) for i in range(0, len(batches), per)]
        paths = [[os.path.join(self.dataset.image_dir, i + ".png") for i in w] for w in windows]
        sizes = self._image_sizes(paths)
        kept = None
        if sizes is not None:
            self.store_bytes = store_budget(sizes, self.window, self.device)[0]
            kept = [] if self._fits(sizes) else None
        for k, (ids, dec) in enumerate(zip(windows, decode_windows(paths, self.device))):
            if kept is not None and k and not self._fits(sizes[k * self.window:]):
                kept = None                                       # all or nothing: stream this pass and the next ones
            for j in range(0, len(ids), self.batch_size):
                b_ids = ids[j:j + self.batch_size]
                views = dec.images[j:j + len(b_ids)]
                images, _ = self.pipe.images(views)
                batch = dict(images=to_image_list(images), targets=self._targets(b_ids, dec.sizes[j:j + len(b_ids)]),
                             img_ids=tuple(b_ids))
                if kept is not None:
                    kept.append((views, batch["targets"], batch["img_ids"]))
                yield batch
        self._kept = kept


# Images decoded per launch while the training store is built. The build is bound by the host half of the decode (2.5-2.6
# ms per file on the worker thread), so the window only has to keep the kernels fed: tools/bench_train_loader.py built
# 1,024 views in 4.56-4.61 s at 256 and 4.59-5.40 s at 512 (README). The transient filtered buffer is about as large as
# a window's images, and two windows are in flight.
TRAIN_DECODE_WINDOW = 256
VALIDATE_CHUNK = 256                  # views per GpuTargetEncoder.encode call of the start-up validation
# The flip generator's seed is (sampler seed + FLIP_SEED_OFFSET) mod 2**64: a fixed rule, so that a run's flips follow
# from its seed, and a different stream from the index generator's, which keeps the reference's seed.
FLIP_SEED_OFFSET = 0x9E3779B97F4A7C15


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


def _dist_rank_world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def sampler_seed(cfg, seed=None):
    """The TrainingSampler seed of a run: `seed` if given; for cfg.SEED >= 0 the value comm.shared_random_seed() returns
    after default_setup's seed_all_rng(cfg.SEED + rank), rank 0's: np.random.RandomState(cfg.SEED).randint(2 ** 31);
    otherwise (SEED = -1, the default, also when cfg has no SEED) a draw from numpy's global RNG on rank 0, broadcast to
    every rank when torch.distributed is initialised. numpy's global RNG is never reseeded here."""
    if seed is not None:
        return int(seed)
    cfg_seed = int(getattr(cfg, "SEED", -1))
    if cfg_seed >= 0:
        return int(np.random.RandomState(cfg_seed).randint(2 ** 31))
    value = [int(np.random.randint(2 ** 31))]
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast_object_list(value, src=0)
    return value[0]


class TrainSampler(object):
    """TrainingSampler (data/samplers/distributed_sampler.py:12-54) followed by BatchSampler(drop_last=True), with the
    horizontal flip drawn alongside. Iterating yields int64 [images_per_batch // world, 2] arrays of (dataset index, flip)
    rows, forever, starting at position 0 of the stream.

    Indices: torch.randperm(size, generator=g) epoch after epoch, g = torch.Generator() seeded with `seed`; this rank's
    rows are positions rank, rank + world, ... of that stream, and batches run across epoch boundaries, as the
    reference's do. Flips: a second torch.Generator seeded with (seed + FLIP_SEED_OFFSET) mod 2**64 draws torch.rand(size)
    per epoch; position j of epoch e is flipped when u_e[j] < flip_prob. The index generator never sees these draws, and
    the (index, flip) at a global position depends on the seed alone, not on the world size, the rank or the batch size.
    The reference's flips come from random.random() in its DataLoader workers (worker_init_reset_seed), which depends on
    NUM_WORKERS and on torch's RNG after the model is built, so they are not reproduced."""

    def __init__(self, size, images_per_batch, seed, rank=0, world=1, flip_prob=0.5):
        if size < 1:
            raise ValueError("TrainSampler: dataset size %d" % size)
        if world < 1 or not 0 <= rank < world:
            raise ValueError("TrainSampler: rank %d of world %d" % (rank, world))
        if images_per_batch % world:
            raise ValueError("SOLVER.IMS_PER_BATCH (%d) must be divisible by the number of GPUs (%d) used"
                             % (images_per_batch, world))
        self.size, self.rank, self.world, self.seed = int(size), int(rank), int(world), int(seed)
        self.batch_size = images_per_batch // world
        if self.batch_size < 1:
            raise ValueError("SOLVER.IMS_PER_BATCH = %d" % images_per_batch)
        self.flip_prob = float(flip_prob)

    def epochs(self):
        """(indices int64 [size], flips bool [size]) of epoch 0, 1, ... of the global stream"""
        g, gf = torch.Generator(), torch.Generator()
        g.manual_seed(self.seed)
        gf.manual_seed((self.seed + FLIP_SEED_OFFSET) % 2 ** 64)
        while True:
            idx = torch.randperm(self.size, generator=g).numpy()
            flips = torch.rand(self.size, generator=gf).numpy() < self.flip_prob
            yield idx, flips

    def rows(self):
        """this rank's (index, flip) rows, one epoch's part at a time: int64 [n, 2] arrays"""
        for e, (idx, flips) in enumerate(self.epochs()):
            first = (self.rank - e * self.size) % self.world          # the first position j with e*size + j = rank (mod world)
            yield np.stack([idx[first::self.world], flips[first::self.world].astype(np.int64)], axis=1)

    def __iter__(self):
        B, pending = self.batch_size, np.zeros((0, 2), dtype=np.int64)
        for part in self.rows():
            pending = np.concatenate([pending, part])
            n = len(pending) // B * B
            for i in range(0, n, B):
                yield pending[i:i + B]
            pending = pending[n:]


class KittiTrainSplit(KittiSplit):
    """KittiSplit with the right camera's images: len() is len(KITTIDataset), twice the frames with
    DATASETS.USE_RIGHT_IMAGE (targets.dataset_len), as tools/plain_train_net.py reads it."""

    def __init__(self, cfg, root, split):
        super(KittiTrainSplit, self).__init__(cfg, root, split)
        self.image_right_dir = os.path.join(root, "image_3")
        self.use_right = T.dataset_len(1, cfg) == 2
        self._len = T.dataset_len(len(self.ids), cfg)

    def __len__(self):
        return self._len


class KittiTrainLoader(object):
    """The reference's training loader on the GPU (module docstring). rank / world default to torch.distributed's, or
    (0, 1); seed to sampler_seed(cfg), kept as `.seed` so a run can be repeated. Yields, per batch of
    SOLVER.IMS_PER_BATCH // world rows of TrainSampler:

        images   ImageList of GpuInputPipeline.images(store views, flips)
        targets  tuple of ParamsList (kitti.py:496-521 without ori_img), what do_train moves to the device
        encoded  EncodedTargets of GpuTargetEncoder.encode, for Trainer.step(images, encoded, sync_log=False)
        img_ids  the frames' 6-character ids, left and right items alike (kitti.py:261)

    Differences from the reference, besides the flip stream (TrainSampler): whatever the reference raises on when it
    draws an item - a missing image_3, an image larger than the input, an object it cannot encode in either flip state -
    raises here at construction, naming the file or the frame, camera and flip. Over the reference's 100 epochs every
    item is drawn in both flip states with near certainty, so it would raise too. The store has to fit in free device
    memory (KITTI train, left: about 5.2 GB; trainval, both cameras: about 20.9 GB); a larger one raises with both byte
    counts. A new iterator starts the stream at position 0, as the reference's do_train does on resume."""

    def __init__(self, cfg, root, split=None, rank=None, world=None, seed=None, device="cuda"):
        split = split if split is not None else getattr(cfg.DATASETS, "TRAIN_SPLIT", None)
        if not split:
            raise ValueError("KittiTrainLoader: no split (neither `split` nor cfg.DATASETS.TRAIN_SPLIT is set)")
        if rank is None or world is None:
            r, w = _dist_rank_world()
            rank, world = r if rank is None else rank, w if world is None else world
        self.device = torch.device(device)
        self.encoder = T.GpuTargetEncoder(cfg, device)          # refuses every INPUT / DATASETS option not built
        self.pipe = GpuInputPipeline(cfg, device)
        self.dataset = ds = KittiTrainSplit(cfg, root, split)
        if not ds.labelled:
            raise ValueError("KittiTrainLoader: split %r has no labels" % split)
        F = len(ds.ids)
        self.seed = sampler_seed(cfg, seed)
        self.sampler = TrainSampler(len(ds), int(cfg.SOLVER.IMS_PER_BATCH), self.seed, rank, world,
                                    flip_prob=float(getattr(cfg.INPUT, "AUG_PARAMS", [[0.5]])[0][0]))
        self.build_seconds = {}
        t0 = time.perf_counter()
        self.labels = self._read_labels(cfg)
        self.P = np.stack([T.read_kitti_calib(os.path.join(ds.calib_dir, i + ".txt")) for i in ds.ids]
                          + ([T.read_kitti_calib(os.path.join(ds.calib_dir, i + ".txt"), use_right_cam=True)
                              for i in ds.ids] if ds.use_right else [])).reshape(-1, 3, 4)
        # per dataset index (targets.dataset_view): frame, right flag, file, (w, h), camera matrix
        views = [T.dataset_view(i, F, cfg) for i in range(len(ds))]
        self.frames = np.array([f for f, _ in views], dtype=np.int64)
        self.right = np.array([r for _, r in views], dtype=bool)
        self.files = [os.path.join(ds.image_right_dir if r else ds.image_dir, ds.ids[f] + ".png")
                      for f, r in zip(self.frames, self.right)]
        t1 = time.perf_counter()
        self.sizes = np.array([self._ihdr(p) for p in self.files], dtype=np.int64).reshape(-1, 2)
        windows = [self.files[i:i + TRAIN_DECODE_WINDOW] for i in range(0, len(self.files), TRAIN_DECODE_WINDOW)]
        self.store_bytes, need, free = store_budget([tuple(s) for s in self.sizes], TRAIN_DECODE_WINDOW, self.device)
        if need > free:
            raise MemoryError("KittiTrainLoader: the decoded images of split %r take %d bytes on the device (%d with the "
                              "decode's transient buffers), more than the %d bytes free; streaming is not built"
                              % (split, self.store_bytes, need, free))
        t2 = time.perf_counter()
        self.store, self.images = [], []
        for dec in decode_windows(windows, self.device):
            self.store.append(dec.buffer)
            self.images += dec.images
        t3 = time.perf_counter()
        self._validate()
        torch.cuda.current_stream(self.device).synchronize()
        self.build_seconds = dict(labels_calib=t1 - t0, headers=t2 - t1, decode=t3 - t2, validate=time.perf_counter() - t3)

    def _read_labels(self, cfg):
        ds, M = self.dataset, int(cfg.DATASETS.MAX_OBJECTS)
        rows = []
        for i in ds.ids:
            path = os.path.join(ds.label_dir, i + ".txt")
            try:
                r = T.read_kitti_label(path, tuple(ds.classes))
            except ValueError as e:
                raise ValueError("%s: %s" % (path, e))
            if len(r) > M:
                raise ValueError("%s: %d objects of the detected classes, more than MAX_OBJECTS = %d" % (path, len(r), M))
            rows.append(r)
        return T.pack_labels(rows, M)

    def _ihdr(self, path):
        if not os.path.exists(path):
            raise FileNotFoundError("KittiTrainLoader: image file not found: %s" % path)
        w, h = read_ihdr(path)
        if w > self.encoder.W or h > self.encoder.H:
            raise ValueError("%s: image %dx%d larger than the input %dx%d (INPUT.WIDTH_TRAIN x HEIGHT_TRAIN)"
                             % (path, w, h, self.encoder.W, self.encoder.H))
        return w, h

    def _encode(self, idx, flips):
        """GpuTargetEncoder.encode of the dataset indices `idx` with `flips`, from rows of the host tables staged in pinned
        memory, so that their copies to the device do not wait for the stream"""
        right = _pinned(self.right[idx].astype(np.int32)) if self.dataset.use_right else None
        return self.encoder.encode(_pinned(self.labels[self.frames[idx]]), _pinned(self.P[idx]), _pinned(self.sizes[idx]),
                                   _pinned(np.asarray(flips, dtype=np.int32)), right=right)

    def _validate(self):
        """every item in both flip states through the encoder, one status read in all; a chunk that reports objects the
        reference cannot encode is encoded item by item to name the item"""
        n = len(self.dataset)
        chunks = [(np.arange(i, min(i + VALIDATE_CHUNK, n)), f) for i in range(0, n, VALIDATE_CHUNK) for f in (0, 1)]
        status = torch.cat([self._encode(idx, np.full(len(idx), f)).status for idx, f in chunks]).cpu().numpy()
        for (idx, f), s in zip(chunks, status):
            if not s:
                continue
            for i in idx:
                if int(self._encode(np.array([i]), np.array([f])).status.item()):
                    raise RuntimeError("KittiTrainLoader: frame %s, %s, %s: an object the reference cannot encode (an edge "
                                       "object with two non-zero heat-map radii, or an outside object whose 2D box centre "
                                       "lies outside the image)" % (self.dataset.ids[self.frames[i]],
                                                                    "image_3" if self.right[i] else "image_2",
                                                                    "flipped" if f else "not flipped"))

    def __iter__(self):
        ids = self.dataset.ids
        for rows in self.sampler:
            idx, flips = rows[:, 0], rows[:, 1].astype(bool)
            images, _ = self.pipe.images([self.images[i] for i in idx], flips=flips)
            enc = self._encode(idx, flips)
            P = T.flip_calib(self.P[idx], self.sizes[idx, 0], flips)
            yield dict(images=to_image_list(images), targets=tuple(enc.param_lists(P)), encoded=enc,
                       img_ids=tuple(ids[f] for f in self.frames[idx]))
