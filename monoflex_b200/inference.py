"""Drop-in for the reference's `inference_all_depths` (engine/inference.py:130-197, tools/plain_train_net.py
--eval_all_depths through engine/test_net.py:run_test): the KITTI AP of every depth estimator of the PostProcessor.

The reference runs the whole split through the model once per estimator. Here the loader, the host-to-device copy, the
backbone, the predictor, the NMS and the top-k run once per batch: KeypointDetector.forward_depths decodes all eight
estimators from one pass. Per estimator the same text files are written (`<output_folder>/eval_all_depths/<method>/`,
byte-identical to generate_kitti_3d_detection), the same R40 metric is computed (on the GPU, from the decode's rows
rather than by parsing the files back) and the same lines are logged to `monoflex.inference`."""
import logging
import os
import re

import numpy as np
import torch

from . import evaluation as E
from .model.detector import KeypointDetector

# engine/inference.py:146, in the reference's order (which also orders the log lines)
EVAL_DEPTH_METHODS = ('oracle', 'hard', 'soft', 'mean', 'direct', 'keypoints_center', 'keypoints_02', 'keypoints_13')
_RESULT_FILE = re.compile(r'^\d{6}$')       # the result files kitti_common.get_label_annos lists


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

    # evaluate_python pairs the result files, sorted by id, with the split's ids in the split's order
    rows = torch.cat(results, 1) if results else torch.zeros(len(EVAL_DEPTH_METHODS), 0, 14, device=device)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    last = {img_id: i for i, img_id in enumerate(image_ids) if _RESULT_FILE.match(img_id)}   # a re-written file: the last
    order = [last[k] for k in sorted(last, key=int)]
    pick = torch.from_numpy(np.concatenate([np.arange(offsets[i], offsets[i + 1]) for i in order] + [np.zeros(0, np.int64)]))
    dt_counts = [counts[i] for i in order]
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
