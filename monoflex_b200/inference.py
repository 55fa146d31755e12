"""Drop-in for the reference's `inference_all_depths` (engine/inference.py:130-197, tools/plain_train_net.py
--eval_all_depths through engine/test_net.py:run_test): the KITTI AP of every depth estimator of the PostProcessor.

The reference runs the whole split through the model once per estimator. Here the loader, the host-to-device copy, the
backbone, the predictor, the NMS and the top-k run once per batch: KeypointDetector.forward_depths decodes all eight
estimators from one pass. Per estimator the same text files are written (`<output_folder>/eval_all_depths/<method>/`,
byte-identical to generate_kitti_3d_detection), the same R40 metric is computed (on the GPU, from the decode's rows
rather than by parsing the files back) and the same lines are logged to `monoflex.inference`.

Drop-in for the reference's `inference` (engine/inference.py:65-128: do_eval's evaluation during training and run_test
without --eval_all_depths): the model runs over the loader through KeypointDetector.forward_async, each batch's padded
rows and counts are copied on the stream into buffers that last the pass, and they are read to the host once, at its end.
The same files are written (`<output_folder>/data/<id>.txt`, on a worker thread while the metric runs), the same lines
logged and the same (ret_dicts, result, dis_ious) returned; the metric scores the decode's rows on the GPU against the
split's labels, parsed once per dataset. When the folder holds result files this call did not write (stale files, or
another rank's), the folder is scored as text by evaluate_python, as the reference scores it. With a KittiEvalLoader whose
split fits in device memory, later evaluations neither decode nor parse anything."""
import logging
import os
import re
import datetime
import threading
import time

import numpy as np
import torch

from . import evaluation as E
from . import parallel
from .model.detector import KeypointDetector

# engine/inference.py:146, in the reference's order (which also orders the log lines)
EVAL_DEPTH_METHODS = ('oracle', 'hard', 'soft', 'mean', 'direct', 'keypoints_center', 'keypoints_02', 'keypoints_13')
_RESULT_FILE = re.compile(r'^\d{6}$')       # the result files kitti_common.get_label_annos lists


def scored_rows(image_ids, counts, starts):
    """evaluate_python pairs the result files, sorted by id, with the split's ids in the split's order. Of the images of a
    pass - their ids, detection counts and the first row of each image's rows - the ones that name a result file
    (\\d{6}; of a repeated id the last, whose file is the last written) sorted by id -> (int64 row indices, counts)"""
    starts = np.asarray(starts, np.int64)
    last = {img_id: i for i, img_id in enumerate(image_ids) if _RESULT_FILE.match(img_id)}
    order = [last[k] for k in sorted(last, key=int)]
    pick = torch.from_numpy(np.concatenate([np.arange(starts[i], starts[i] + counts[i]) for i in order]
                                           + [np.zeros(0, np.int64)]))
    return pick, [counts[i] for i in order]


def inference_all_depths(model, data_loader, dataset_name, eval_types=("detections",), device="cuda", output_folder=None,
                         vis=False, eval_score_iou=False, metrics=('R40', 'R11')):
    """engine/inference.py:130-197 with its signature and return value (None, None, None). `metrics` is ignored and
    R40 used, `eval_score_iou` is unused, as in the reference. The loader yields the reference's batches (images,
    targets, img_ids) of any size; dataset.label_dir / imageset_txt / classes give the ground truth."""
    if vis:
        raise NotImplementedError("inference_all_depths(vis=True): the visualiser is out of scope")
    if not isinstance(model, KeypointDetector):
        raise TypeError("inference_all_depths needs a monoflex_b200 KeypointDetector (it decodes every estimator from "
                        "one forward_depths pass), got %s" % type(model).__name__)
    logger = logging.getLogger("monoflex.inference")
    dataset = data_loader.dataset
    folders = {}
    for method in EVAL_DEPTH_METHODS:
        folders[method] = os.path.join(output_folder, 'eval_all_depths', method)
        os.makedirs(folders[method], exist_ok=True)
        for name in os.listdir(folders[method]):            # remove all previous predictions
            os.remove(os.path.join(folders[method], name))

    model.eval()
    device = torch.device(device)
    results, counts, image_ids = [], [], []
    with torch.no_grad():
        for batch in data_loader:
            images, targets = batch["images"].to(device), [t.to(device) for t in batch["targets"]]
            out = model.forward_depths(images, targets, EVAL_DEPTH_METHODS)
            n = out[EVAL_DEPTH_METHODS[0]][1]['counts']
            rows = torch.stack([out[m][0] for m in EVAL_DEPTH_METHODS])          # [methods, rows, 14], one copy out
            host = rows.cpu()
            for i, method in enumerate(EVAL_DEPTH_METHODS):
                for img_id, r in zip(batch["img_ids"], host[i].split(n)):
                    E.write_kitti_detections(r, os.path.join(folders[method], img_id + '.txt'))
            results.append(rows)
            counts += n
            image_ids += list(batch["img_ids"])

    rows = torch.cat(results, 1) if results else torch.zeros(len(EVAL_DEPTH_METHODS), 0, 14, device=device)
    pick, dt_counts = scored_rows(image_ids, counts, np.concatenate([[0], np.cumsum(counts)]))
    with open(dataset.imageset_txt, 'r') as f:
        split_ids = [int(line) for line in f.readlines()]
    gt = E.KittiAnnos.from_label_dir(dataset.label_dir, split_ids)

    ret_dicts = []
    for i, method in enumerate(EVAL_DEPTH_METHODS):
        logger.info("evaluation with depth method: {}".format(method))
        dt = E.KittiAnnos.from_results(rows[i].index_select(0, pick.to(rows.device)), dt_counts)
        ret_dicts.append(E.get_official_eval_result(gt, dt, dataset.classes, metric='R40')[1])

    # engine/inference.py:171-195: bev / 3d AP of every method for Car at IoU 0.7, then the methods sorted by 3d moderate
    for cls, thresh in (('Car', 0.7),):
        logger.info('{} AP@{:.2f}, {:.2f}:'.format(cls, thresh, thresh))
        sort_metric = []
        for method, ret in zip(EVAL_DEPTH_METHODS, ret_dicts):
            key = lambda kind, level: ret['{}_{}_{:.2f}/{}'.format(cls, kind, thresh, level)]
            logger.info('bev/3d AP, method {}:'.format(method))
            logger.info('{:.4f}/{:.4f}, {:.4f}/{:.4f}, {:.4f}/{:.4f}'.format(
                key('bev', 'easy'), key('3d', 'easy'), key('bev', 'moderate'), key('3d', 'moderate'), key('bev', 'hard'),
                key('3d', 'hard')))
            sort_metric.append(key('3d', 'moderate'))
        order = np.argsort(-np.array(sort_metric))
        logger.info('Cls {}, Thresh {}, Sort: '.format(cls, thresh) + ' > '.join(EVAL_DEPTH_METHODS[j] for j in order))
    return None, None, None


def get_time_str(seconds):
    """utils/timer.py:get_time_str"""
    return str(datetime.timedelta(seconds=seconds))


def _world_size():
    import torch.distributed as dist
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _is_main_process():
    import torch.distributed as dist
    return not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0


class DetectionPass(object):
    """The decode's padded rows of every image of one pass, gathered on the device: `result` float32 [n, K, 14] and
    `count` int32 [n] in the loader's order, `img_ids` the n ids. append() copies a decode workspace in on the current
    stream (no host synchronisation); read() copies both to the host once."""

    def __init__(self, capacity, device):
        self.capacity, self.device = max(int(capacity), 1), torch.device(device)
        self.result = self.count = None
        self.n, self.img_ids = 0, []

    def append(self, ws, img_ids):
        B, K = ws.result.shape[0], ws.result.shape[1]
        if self.result is None:
            self.result = torch.empty(self.capacity, K, 14, device=self.device)
            self.count = torch.empty(self.capacity, dtype=torch.int32, device=self.device)
        if self.n + B > self.result.shape[0]:         # a loader longer than its dataset's len(): grow, on the device
            cap = max(2 * self.result.shape[0], self.n + B)
            result, count = torch.empty(cap, K, 14, device=self.device), torch.empty(cap, dtype=torch.int32, device=self.device)
            result[:self.n].copy_(self.result[:self.n])
            count[:self.n].copy_(self.count[:self.n])
            self.result, self.count = result, count
        self.result[self.n:self.n + B].copy_(ws.result)
        self.count[self.n:self.n + B].copy_(ws.count)
        self.n += B
        self.img_ids += list(img_ids)

    def rows(self):
        """the device rows [n * K, 14], image i's valid rows starting at i * K"""
        return self.result[:self.n].reshape(-1, 14) if self.n else torch.zeros(0, 14, device=self.device)

    def read(self):
        """-> (result float32 [n, K, 14], counts int list) on the host: one copy of each into pinned memory, one wait"""
        if not self.n:
            return np.zeros((0, 1, 14), np.float32), []
        res = torch.empty(self.result[:self.n].shape, pin_memory=True)
        cnt = torch.empty(self.n, dtype=torch.int32, pin_memory=True)
        res.copy_(self.result[:self.n], non_blocking=True)
        cnt.copy_(self.count[:self.n], non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        return res.numpy(), cnt.tolist()


def detect_pass(model, data_loader, device="cuda"):
    """compute_on_dataset's model loop (engine/inference.py:17-63) without its host reads: every batch moved to the
    device as the reference moves it, enqueued with forward_async, its rows copied into a DetectionPass. Nothing here
    waits for the device unless the loader's batches or a graph capture do."""
    model.eval()
    try:
        capacity = len(data_loader.dataset)
    except TypeError:
        capacity = 1
    rows = DetectionPass(capacity, device)
    with torch.no_grad():
        for batch in data_loader:
            images = batch["images"].to(device)
            targets = [t.to(device) for t in batch["targets"]]
            rows.append(model.forward_async(images, targets).ws, batch["img_ids"])
    return rows


def write_result_files(folder, img_ids, result, counts):
    """generate_kitti_3d_detection of every image of a pass, in the pass's order: `result` the host padded rows [n, K, 14],
    `counts` the valid rows of each"""
    for img_id, res, n in zip(img_ids, result, counts):
        E.write_kitti_detections(res[:n], os.path.join(folder, img_id + '.txt'))


def split_ground_truth(dataset):
    """KittiAnnos of the split's labels (evaluate_python's ground truth), parsed on the first call and kept on the
    dataset for the later ones; a dataset that cannot hold an attribute is parsed on every call"""
    with open(dataset.imageset_txt, 'r') as f:
        split_ids = [int(line) for line in f.readlines()]
    key = (dataset.label_dir, tuple(split_ids), torch.cuda.current_device())
    cached = getattr(dataset, '_kitti_ground_truth', None)
    if cached is not None and cached[0] == key:
        return cached[1]
    gt = E.KittiAnnos.from_label_dir(dataset.label_dir, split_ids)
    try:
        dataset._kitti_ground_truth = (key, gt)
    except (AttributeError, TypeError):
        pass
    return gt


def inference(model, data_loader, dataset_name, eval_types=("detections",), device="cuda", output_folder=None,
              metrics=['R40'], vis=False, eval_score_iou=False):
    """engine/inference.py:65-128 with its signature and return value: (ret_dicts, result, dis_ious) - one ret_dict per
    metric, the last metric's text and {} - on the main rank, (None, None, None) on the others, after parallel.barrier()
    where the reference calls comm.synchronize(). The loader yields the reference's batches (images, targets, img_ids) of
    any size (the reference's test loader has batch 1; each image gets its own file at every batch size);
    dataset.label_dir / imageset_txt / classes give the ground truth, which is kept on the dataset between calls.
    `eval_score_iou` is unused, as in the reference; TEST.EVAL_DIS_IOUS raises (out of scope)."""
    if vis:
        raise NotImplementedError("inference(vis=True): the visualiser is out of scope")
    if not isinstance(model, KeypointDetector):
        raise TypeError("inference needs a monoflex_b200 KeypointDetector (it reads the decode's rows on the device "
                        "through forward_async), got %s" % type(model).__name__)
    model.heads.post_processor.check_config()          # TEST.EVAL_DIS_IOUS (--eval_iou) raises
    device = torch.device(device)
    num_devices = _world_size()
    logger = logging.getLogger("monoflex.inference")
    dataset = data_loader.dataset
    logger.info("Start evaluation on {} dataset({} images).".format(dataset_name, len(dataset)))
    predict_folder = os.path.join(output_folder, 'data')
    os.makedirs(predict_folder, exist_ok=True)

    start = time.time()
    rows = detect_pass(model, data_loader, device)
    result, counts = rows.read()
    inference_time = time.time() - start
    failed = []

    def write():
        try:
            write_result_files(predict_folder, rows.img_ids, result, counts)
        except BaseException as e:                      # re-raised on the calling thread
            failed.append(e)
    writer = threading.Thread(target=write, name="kitti-result-files")
    writer.start()

    def written():
        writer.join()
        if failed:
            raise failed.pop()

    try:
        if not _is_main_process():
            written()                                   # the main rank lists the folder after the barrier
        parallel.barrier()
        total_time = time.time() - start
        logger.info("Total run time: {} ({} s / img per device, on {} devices)".format(
            get_time_str(total_time), total_time * num_devices / len(dataset), num_devices))
        logger.info("Model inference time: {} ({} s / img per device, on {} devices)".format(
            get_time_str(inference_time), inference_time * num_devices / len(dataset), num_devices))
        if not _is_main_process():
            return None, None, None

        logger.info('Finishing generating predictions, start evaluating ...')
        mine = {i + '.txt' for i in rows.img_ids if _RESULT_FILE.match(i)}
        others = {n for n in os.listdir(predict_folder) if _RESULT_FILE.match(n[:-4]) and n.endswith('.txt')} - mine
        if others:                                      # files this call did not write: score the folder as text
            written()
            dt = None
        else:
            pick, dt_counts = scored_rows(rows.img_ids, counts, np.arange(rows.n) * max(result.shape[1], 1))
            dt = E.KittiAnnos.from_results(rows.rows().index_select(0, pick.to(rows.device)), dt_counts)
            gt = split_ground_truth(dataset)
        ret_dicts = []
        for metric in metrics:
            if dt is None:
                result_text, ret_dict = E.evaluate_python(label_path=dataset.label_dir, result_path=predict_folder,
                                                          label_split_file=dataset.imageset_txt,
                                                          current_class=dataset.classes, metric=metric)
            else:
                result_text, ret_dict = E.get_official_eval_result(gt, dt, dataset.classes, metric=metric)
            logger.info('metric = {}'.format(metric))
            logger.info('\n' + result_text)
            ret_dicts.append(ret_dict)
        return ret_dicts, result_text, {}
    finally:
        written()
