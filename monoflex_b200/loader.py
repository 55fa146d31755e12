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
detection of its window is written; a file the host rejects raises one window earlier still."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import targets as T
from .data import GpuInputPipeline
from .png import DecodedImages, PngBatch, read_png
from .structures import to_image_list

# Images decoded per launch, chosen with tools/bench_png.py (README, "PNG decode and evaluation loader"). A launch takes
# about 215 ms for 8 to 256 images, because one warp inflates one image serially, so the window sets the kernels'
# throughput: 0.84 ms per image at 256. That is above the strict model's rate at B = 1 and B = 8. The whole loop still
# runs below the same loop fed from pinned memory. At 1024 the kernels take 0.26 ms per image, but the loop at B = 8
# ran slower than at 256.
DECODE_WINDOW = 256


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

    def __iter__(self):
        batches = self.batches()
        per = self.window // self.batch_size
        windows = [sum(batches[i:i + per], []) for i in range(0, len(batches), per)]
        main = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(self.device)
        pool = ThreadPoolExecutor(max_workers=1)
        staged = []
        try:
            # window k + 2 is read and staged on the worker thread and window k + 1 decodes on the side stream while the
            # consumer runs the model on window k
            staged = [pool.submit(self._stage, w) for w in windows[:2]]
            pending = self._launch(staged.pop(0).result(), side) if windows else None
            for k in range(len(windows)):
                dec = pending
                if k + 2 < len(windows):
                    staged.append(pool.submit(self._stage, windows[k + 2]))
                pending = self._launch(staged.pop(0).result(), side) if staged else None
                dec.check()
                main.wait_event(dec.event)
                dec.buffer.record_stream(main)              # read on the main stream after the side stream lets it go
                for j in range(0, len(windows[k]), self.batch_size):
                    b_ids = windows[k][j:j + self.batch_size]
                    images, _ = self.pipe.images(dec.images[j:j + len(b_ids)])
                    yield dict(images=to_image_list(images),
                               targets=self._targets(b_ids, dec.sizes[j:j + len(b_ids)]), img_ids=tuple(b_ids))
        finally:
            for f in staged:
                f.cancel()
            pool.shutdown(wait=True)

    def _stage(self, ids):
        """the host half of a window's decode: read, check and stage its files (runs in the loader's worker thread)"""
        return PngBatch([read_png(os.path.join(self.dataset.image_dir, i + ".png")) for i in ids])

    def _launch(self, batch, side):
        with torch.cuda.stream(side):
            return DecodedImages(batch, self.device)
