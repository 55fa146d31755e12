"""KITTI official 3D-detection metric on the GPU: 2D / BEV / 3D / AOS AP at R40 and R11, and the COCO-style AP over a
sweep of overlap thresholds.

A drop-in for the reference's `evaluate_python` (data/datasets/evaluation/__init__.py:33), which every `inference()`
ends in, for `get_official_eval_result` (kitti_object_eval_python/eval.py:644-726) and `get_coco_eval_result`
(eval.py:729-788): the same `result` text and the same `ret_dict`; and for kitti_object_eval_python's `evaluate()`
entry (evaluate.py:14-32), also as a command line:

    python -m monoflex_b200.evaluation --label_path L --result_path R --label_split_file S [--current_class 0,1,2]
        [--coco] [--score_thresh T] [--metric R40|R11]

Overlaps, flags, matching, thresholds and AP run in monoflex_b200/csrc/mf_kitti_eval.cu; the host parses label files,
packs the objects and formats the text. There is no CPU fallback: without the library or a GPU, calls raise.
"""
import argparse
import ctypes
import io
import os
import pathlib
import re
import sys

import numpy as np
import torch

from . import _lib

CLASS_NAMES = ('car', 'pedestrian', 'cyclist', 'van', 'person_sitting', 'truck')
CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting', 5: 'Truck'}
NAME_TO_CLASS = {v: k for k, v in CLASS_TO_NAME.items()}
ID_TYPE_CONVERSION = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist'}     # the decode's class ids
DONTCARE = 6          # MF_KITTI_DONTCARE
OBJ = 16              # MF_KITTI_OBJ
MAX_DT = 128          # MF_KITTI_MAX_DT
N_SAMPLE_PTS = 41
# min_overlaps[k, metric, class] of get_official_eval_result
MIN_OVERLAPS = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3),
                         np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5],
                                   [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]])], axis=0)
# get_coco_eval_result's classes and their (start, stop, count) of overlap thresholds; Truck has none
COCO_CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting'}
COCO_CLASS_TO_RANGE = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10], 3: [0.5, 0.95, 10],
                       4: [0.25, 0.7, 10]}


def class_code(name):
    """clean_data compares lower-cased names with the class list and 'DontCare' case-sensitively"""
    if name == 'DontCare':
        return DONTCARE
    low = name.lower()
    return CLASS_NAMES.index(low) if low in CLASS_NAMES else -1


def get_label_anno(label_path):
    """One label or result file as kitti_common.get_label_anno returns it: a dict of per-object arrays, dimensions in
    (l, h, w) order. An empty file, or one whose first line is shorter than 15 characters, has no objects (the reference's
    writer leaves a lone newline for an image without detections); a file whose first line has no 16th column gets
    score 0."""
    with open(label_path, 'r') as f:
        lines = f.readlines()
    rows = [line.strip().split(' ') for line in lines] if lines and len(lines[0]) >= 15 else []
    # columns 1..14: truncated, occluded, alpha, x1, y1, x2, y2, h, w, l, x, y, z, rotation_y
    v = np.array([[float(t) for t in r[1:15]] for r in rows], np.float64).reshape(-1, 14)
    scored = bool(rows) and len(rows[0]) == 16
    return {'name': np.array([r[0] for r in rows]), 'truncated': v[:, 0], 'occluded': np.array([int(r[2]) for r in rows]),
            'alpha': v[:, 2], 'bbox': v[:, 3:7], 'dimensions': v[:, [9, 7, 8]], 'location': v[:, 10:13],
            'rotation_y': v[:, 13], 'score': np.array([float(r[15]) for r in rows]) if scored else np.zeros(len(rows))}


class KittiAnnos:
    """Ground truth or detections of a set of images, packed for the device: `objects` is a float64 [N, 16] tensor
    (class code, truncated, occluded, alpha, x1, y1, x2, y2, l, h, w, x, y, z, rotation_y, score), image i owning rows
    offsets[i]:offsets[i + 1]; `counts` stays on the host. The metric takes CUDA tensors only; device='cpu' packs for
    inspection."""

    def __init__(self, objects, counts):
        if not isinstance(objects, torch.Tensor) or objects.dtype != torch.float64 or objects.dim() != 2 \
                or objects.shape[1] != OBJ:
            raise ValueError("KittiAnnos: objects must be a float64 [N, %d] tensor, got %s" % (
                OBJ, "%s %s" % (objects.dtype, tuple(objects.shape)) if isinstance(objects, torch.Tensor) else type(objects)))
        self.objects = objects.contiguous()
        self.counts = np.asarray(counts, np.int64).reshape(-1)
        off = np.zeros(len(self.counts) + 1, np.int32)
        np.cumsum(self.counts, out=off[1:])
        if off[-1] != objects.shape[0]:
            raise ValueError("counts sum to %d, objects has %d rows" % (off[-1], objects.shape[0]))
        self.offsets = torch.from_numpy(off).to(objects.device)

    def __len__(self):
        return len(self.counts)

    @classmethod
    def from_annos(cls, annos, device='cuda'):
        """the reference's get_label_anno dicts, one per image"""
        rows = []
        for a in annos:
            n = len(a['name'])
            score = a['score'] if 'score' in a else np.zeros(n)
            r = np.zeros((n, OBJ), np.float64)
            r[:, 0] = [class_code(s) for s in a['name']]
            r[:, 1], r[:, 2], r[:, 3] = a['truncated'], a['occluded'], a['alpha']
            r[:, 4:8] = np.asarray(a['bbox']).reshape(n, 4)
            r[:, 8:11] = np.asarray(a['dimensions']).reshape(n, 3)
            r[:, 11:14] = np.asarray(a['location']).reshape(n, 3)
            r[:, 14], r[:, 15] = a['rotation_y'], score
            rows.append(r)
        obj = np.concatenate(rows, 0) if rows else np.zeros((0, OBJ))
        return cls(torch.from_numpy(obj).to(device), [len(a['name']) for a in annos])

    @classmethod
    def from_label_dir(cls, path, image_ids=None, device='cuda'):
        """kitti_common.get_label_annos: without ids, every ^\\d{6}.txt$ file of the folder, sorted by id"""
        if image_ids is None:
            prog = re.compile(r'^\d{6}.txt$')
            image_ids = sorted(int(p.stem) for p in pathlib.Path(path).glob('*.txt') if prog.match(p.name))
        if not isinstance(image_ids, list):
            image_ids = list(range(image_ids))
        return cls.from_annos([get_label_anno(os.path.join(path, '%06d.txt' % i)) for i in image_ids], device)

    @classmethod
    def from_results(cls, result, counts):
        """the decode's rows (result [N, 14] fp32 on the GPU, counts per image) exactly as generate_kitti_3d_detection
        writes them and get_label_anno parses them back, without the text files"""
        result = result.detach().float().contiguous()
        if not result.is_cuda or result.dim() != 2 or result.shape[1] != 14:
            raise ValueError("from_results: result must be a CUDA [N, 14] tensor, got %s" % (tuple(result.shape),))
        out = torch.empty(result.shape[0], OBJ, dtype=torch.float64, device=result.device)
        _lib.call("mf_kitti_pack_results", _lib.ptr(result), result.shape[0], _lib.ptr(out), _lib.stream())
        return cls(out, counts)


def _as_annos(a):
    return a if isinstance(a, KittiAnnos) else KittiAnnos.from_annos(a)


def eval_tables(gt, dt, classes, events=None, min_overlaps=None):
    """every configuration at once on the GPU. Returns (tables, overlaps): tables has recall / precision / aos
    [3 metric][ncls][3 difficulty][n_sets overlap set][41] (eval_class's arrays per metric), ap [2 (R40, R11)][4 (bbox,
    bev, 3d, aos)][ncls][3][n_sets] and compute_aos; overlaps is the device tensor [3, n_pair] of the per-image blocks.
    min_overlaps: eval_class's float64 table [n_sets][3 metric][ncls], its values compared as given; None is
    get_official_eval_result's two sets. `events`, if given, receives CUDA events recorded before and after each stage."""
    if min_overlaps is not None:
        min_overlaps = np.ascontiguousarray(min_overlaps, dtype=np.float64)
        if min_overlaps.ndim != 3 or min_overlaps.shape[1:] != (3, len(classes)) or min_overlaps.shape[0] < 1:
            raise ValueError("eval_tables: min_overlaps must be [n_sets >= 1, 3, %d], got %s"
                             % (len(classes), min_overlaps.shape))
    gt, dt = _as_annos(gt), _as_annos(dt)
    for name, a in (("ground truth", gt), ("detections", dt)):
        if not a.objects.is_cuda:
            raise ValueError("eval_tables: the %s are on %s; the metric runs on CUDA tensors only (there is no CPU "
                             "fallback): build KittiAnnos with device='cuda'" % (name, a.objects.device))
    dev = torch.device("cuda", torch.cuda.current_device())
    if gt.objects.device != dev or dt.objects.device != dev:
        raise ValueError("eval_tables: ground truth on %s and detections on %s, the current stream on %s"
                         % (gt.objects.device, dt.objects.device, dev))
    if len(gt) != len(dt):
        raise ValueError("%d ground-truth images but %d detection images" % (len(gt), len(dt)))
    if len(gt) == 0:
        raise ValueError("no images to evaluate")
    ncls = len(classes)
    pairs = gt.counts * dt.counts
    pair_off = np.zeros(len(pairs), np.int64)
    np.cumsum(pairs[:-1], out=pair_off[1:])
    n_pair = int(pairs.sum())
    pair_off = torch.from_numpy(pair_off).to(dev)
    n_gt, n_dt = gt.objects.shape[0], dt.objects.shape[0]
    overlaps = torch.empty(3, max(n_pair, 1), dtype=torch.float64, device=dev)
    n_sets = 2 if min_overlaps is None else min_overlaps.shape[0]
    if min_overlaps is None:
        ws_bytes = _lib.load().mf_kitti_eval_workspace(n_gt, n_dt, ncls)
    else:
        size = ctypes.c_size_t(0)
        if _lib.load().mf_kitti_eval_sets_workspace_size(n_gt, n_dt, ncls, n_sets, ctypes.byref(size)) != 0:
            raise ValueError(_lib.load().mf_last_error().decode())
        ws_bytes = size.value
    if ws_bytes == 0:
        raise ValueError("%d classes: between 1 and 8 are supported" % ncls)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    C = 9 * n_sets * ncls
    out = torch.empty(3 * C * N_SAMPLE_PTS + 8 * C // 3 + 2, dtype=torch.float64, device=dev)
    st = _lib.stream()
    cls_arr = (ctypes.c_int * ncls)(*classes)
    common = (_lib.ptr(gt.objects), _lib.ptr(gt.offsets), _lib.ptr(dt.objects), _lib.ptr(dt.offsets), _lib.ptr(pair_off))

    def mark():
        if events is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            events.append(e)
    mark()
    _lib.call("mf_kitti_eval_overlaps", *common, len(gt), n_pair, _lib.ptr(overlaps), st)
    mark()
    max_dt = int(dt.counts.max())
    if min_overlaps is None:
        _lib.call("mf_kitti_eval_statistics", *common, len(gt), n_gt, n_dt, max_dt, _lib.ptr(overlaps), n_pair,
                  cls_arr, ncls, _lib.ptr(ws), ws_bytes, st)
    else:
        _lib.call("mf_kitti_eval_sets_statistics", *common, len(gt), n_gt, n_dt, max_dt, _lib.ptr(overlaps), n_pair,
                  cls_arr, ncls, min_overlaps.ctypes.data, n_sets, _lib.ptr(ws), ws_bytes, st)
    mark()
    if min_overlaps is None:
        _lib.call("mf_kitti_eval_ap", _lib.ptr(ws), n_gt, n_dt, ncls, _lib.ptr(out), st)
    else:
        _lib.call("mf_kitti_eval_sets_ap", _lib.ptr(ws), n_gt, n_dt, ncls, n_sets, _lib.ptr(out), st)
    mark()
    h = out.cpu().numpy()
    if h[-1] > 0:
        raise RuntimeError("eval_tables: an image has %d detections, more than the %d per image the matching kernels take"
                           % (int(h[-1]), MAX_DT))
    shape = (3, ncls, 3, n_sets, N_SAMPLE_PTS)
    n = int(np.prod(shape))
    n_ap = 8 * ncls * 3 * n_sets
    tables = {'recall': h[:n].reshape(shape), 'precision': h[n:2 * n].reshape(shape),
              'orientation': h[2 * n:3 * n].reshape(shape),
              'ap': h[3 * n:3 * n + n_ap].reshape(2, 4, ncls, 3, n_sets), 'compute_aos': bool(h[-2])}
    return tables, overlaps[:, :n_pair]


def print_str(value):
    s = io.StringIO()
    print(value, file=s)
    return s.getvalue()


def get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None, metric='R40'):
    """eval.py:644-726 on the GPU: the same `result` text and `ret_dict`. gt_annos / dt_annos: KittiAnnos or the
    reference's lists of get_label_anno dicts. AOS is computed when the first non-empty detection set's first alpha is
    not -10."""
    if metric not in ('R40', 'R11'):
        raise ValueError("unknown metric %r: 'R40' or 'R11'" % (metric,))
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    current_classes = [NAME_TO_CLASS[c] if isinstance(c, str) else c for c in current_classes]
    min_overlaps = MIN_OVERLAPS[:, :, current_classes]
    tables, _ = eval_tables(gt_annos, dt_annos, current_classes)
    compute_aos = tables['compute_aos']
    ap = tables['ap'][0 if metric == 'R40' else 1]
    mAPbbox, mAPbev, mAP3d = ap[0], ap[1], ap[2]
    mAPaos = ap[3] if compute_aos else None
    if PR_detail_dict is not None:
        PR_detail_dict['bbox'] = tables['precision'][0]
        if compute_aos:
            PR_detail_dict['aos'] = tables['orientation'][0]
        PR_detail_dict['bev'] = tables['precision'][1]
        PR_detail_dict['3d'] = tables['precision'][2]

    result = ''
    ret_dict = {}
    for j, curcls in enumerate(current_classes):
        name = CLASS_TO_NAME[curcls]
        for i in range(min_overlaps.shape[0]):
            result += print_str((f"{name} " "AP@{:.2f}, {:.2f}, {:.2f}:".format(*min_overlaps[i, :, j])))
            result += print_str(f"bbox AP:{mAPbbox[j, 0, i]:.4f}, {mAPbbox[j, 1, i]:.4f}, {mAPbbox[j, 2, i]:.4f}")
            result += print_str(f"bev  AP:{mAPbev[j, 0, i]:.4f}, {mAPbev[j, 1, i]:.4f}, {mAPbev[j, 2, i]:.4f}")
            result += print_str(f"3d   AP:{mAP3d[j, 0, i]:.4f}, {mAP3d[j, 1, i]:.4f}, {mAP3d[j, 2, i]:.4f}")
            if compute_aos:
                result += print_str(f"aos  AP:{mAPaos[j, 0, i]:.2f}, {mAPaos[j, 1, i]:.2f}, {mAPaos[j, 2, i]:.2f}")
                if i == 0:
                    ret_dict['%s_aos/easy' % name] = mAPaos[j, 0, 0]
                    ret_dict['%s_aos/moderate' % name] = mAPaos[j, 1, 0]
                    ret_dict['%s_aos/hard' % name] = mAPaos[j, 2, 0]
            for key, m, col in (('3d', mAP3d, 1), ('bev', mAPbev, 2)):
                thr = min_overlaps[i, col, j]
                ret_dict['{}_{}_{:.2f}/easy'.format(name, key, thr)] = m[j, 0, i]
                ret_dict['{}_{}_{:.2f}/moderate'.format(name, key, thr)] = m[j, 1, i]
                ret_dict['{}_{}_{:.2f}/hard'.format(name, key, thr)] = m[j, 2, i]
            ret_dict['{}_image/easy'.format(name)] = mAPbbox[j, 0, 0]
            ret_dict['{}_image/moderate'.format(name)] = mAPbbox[j, 1, 0]
            ret_dict['{}_image/hard'.format(name)] = mAPbbox[j, 2, 0]
    return result, ret_dict


def coco_min_overlaps(current_classes):
    """do_coco_style_eval's [10 set][3 metric][ncls] table: each class's (start, stop, count) through np.linspace with an
    integer count, the same thresholds for 2D, BEV and 3D. A class without a range (Truck) raises KeyError."""
    overlap_ranges = np.zeros([3, 3, len(current_classes)])
    for i, curcls in enumerate(current_classes):
        overlap_ranges[:, :, i] = np.array(COCO_CLASS_TO_RANGE[curcls])[:, np.newaxis]
    min_overlaps = np.zeros([10, *overlap_ranges.shape[1:]])
    for i in range(overlap_ranges.shape[1]):
        for j in range(overlap_ranges.shape[2]):
            start, stop, num = overlap_ranges[:, i, j]
            min_overlaps[:, i, j] = np.linspace(start, stop, int(num))
    return min_overlaps


def get_coco_eval_result(gt_annos, dt_annos, current_classes):
    """eval.py:729-788 on the GPU: the same text. 2D / BEV / 3D / AOS AP at R40 per overlap set, averaged over the ten
    sets of coco_min_overlaps by numpy's mean. gt_annos / dt_annos: KittiAnnos or the reference's lists of get_label_anno
    dicts; classes by id or name, Truck excluded (KeyError, as in the reference)."""
    name_to_class = {v: n for n, v in COCO_CLASS_TO_NAME.items()}
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    current_classes = [name_to_class[c] if isinstance(c, str) else c for c in current_classes]
    min_overlaps = coco_min_overlaps(current_classes)
    tables, _ = eval_tables(gt_annos, dt_annos, current_classes, min_overlaps=min_overlaps)
    return coco_result_text(current_classes, tables['ap'][0], tables['compute_aos'])


def coco_result_text(current_classes, ap, compute_aos):
    """get_coco_eval_result's text from the AP at R40 (do_eval's default metric) per overlap set, ap [4 (bbox, bev, 3d,
    aos)][ncls][3][10], of the class ids current_classes"""
    mAPbbox, mAPbev, mAP3d = (np.ascontiguousarray(ap[i]).mean(-1) for i in range(3))
    mAPaos = np.ascontiguousarray(ap[3]).mean(-1) if compute_aos else None
    result = ''
    for j, curcls in enumerate(current_classes):
        o_range = np.array(COCO_CLASS_TO_RANGE[curcls])[[0, 2, 1]]
        o_range[1] = (o_range[2] - o_range[0]) / (o_range[1] - 1)
        result += print_str((f"{COCO_CLASS_TO_NAME[curcls]} " "coco AP@{:.2f}:{:.2f}:{:.2f}:".format(*o_range)))
        result += print_str(f"bbox AP:{mAPbbox[j, 0]:.2f}, {mAPbbox[j, 1]:.2f}, {mAPbbox[j, 2]:.2f}")
        result += print_str(f"bev  AP:{mAPbev[j, 0]:.2f}, {mAPbev[j, 1]:.2f}, {mAPbev[j, 2]:.2f}")
        result += print_str(f"3d   AP:{mAP3d[j, 0]:.2f}, {mAP3d[j, 1]:.2f}, {mAP3d[j, 2]:.2f}")
        if compute_aos:
            result += print_str(f"aos  AP:{mAPaos[j, 0]:.2f}, {mAPaos[j, 1]:.2f}, {mAPaos[j, 2]:.2f}")
    return result


def filter_low_score(annos, thresh):
    """kitti_common.filter_annos_low_score on the device: the detections whose score is >= thresh, in order, each image
    recounted"""
    annos = _as_annos(annos)
    obj = annos.objects
    keep = obj[:, 15] >= thresh
    image = torch.repeat_interleave(torch.arange(len(annos), device=obj.device),
                                    torch.from_numpy(annos.counts).to(obj.device))
    counts = torch.bincount(image[keep], minlength=len(annos))
    return KittiAnnos(obj[keep], counts.cpu().numpy())


def write_kitti_detections(rows, path):
    """generate_kitti_3d_detection (kitti_object_eval_python/evaluate.py:34-53), byte for byte: one line per row of the
    decode's result [n, 14] (class, alpha, x1, y1, x2, y2, h, w, l, x, y, z, ry, score) - the class name, 0, 0, then the
    row after np.round(4) in float32, each value printed as the Python float it widens to - and a lone newline for an
    image without detections. The reference's check_last_line_break leaves the file as written: its `os.SEEK_END` raises
    NameError (evaluate.py does not import os), which its bare `except` swallows."""
    rows = np.asarray(rows, dtype=np.float32).reshape(-1, 14).round(4)
    lines = ["%s 0 0 %s\n" % (ID_TYPE_CONVERSION[int(r[0])], " ".join(repr(v) for v in r[1:])) for r in rows.tolist()]
    with open(path, 'w', newline='') as f:
        f.write("".join(lines) if lines else "\n")


def evaluate_python(label_path, result_path, label_split_file, current_class, metric):
    """data/datasets/evaluation/__init__.py:33: the detection files (sorted ids) are paired by position with the ground
    truth of the split file's ids, in the split file's order."""
    dt = KittiAnnos.from_label_dir(result_path)
    with open(label_split_file, 'r') as f:
        ids = [int(line) for line in f.readlines()]
    gt = KittiAnnos.from_label_dir(label_path, ids)
    return get_official_eval_result(gt, dt, current_class, metric=metric)


def evaluate(label_path, result_path, label_split_file, current_class=0, coco=False, score_thresh=-1, metric='R40'):
    """kitti_object_eval_python/evaluate.py:14-32: the result folder's detection files (sorted ids) against the ground
    truth of the split file's ids, paired by position. score_thresh > 0 first drops the detections scored below it.
    Returns get_coco_eval_result's text when coco, else get_official_eval_result's (result, ret_dict) at `metric`."""
    dt = KittiAnnos.from_label_dir(result_path)
    if score_thresh > 0:
        dt = filter_low_score(dt, score_thresh)
    with open(label_split_file, 'r') as f:
        ids = [int(line) for line in f.readlines()]
    gt = KittiAnnos.from_label_dir(label_path, ids)
    if coco:
        return get_coco_eval_result(gt, dt, current_class)
    return get_official_eval_result(gt, dt, current_class, metric=metric)


def parse_classes(text):
    """'0,1,2' or 'Car,Pedestrian': class ids and names as evaluate() takes them"""
    return [int(c) if re.fullmatch(r'-?\d+', c) else c for c in (t.strip() for t in text.split(','))]


def main(argv=None):
    p = argparse.ArgumentParser(prog="python -m monoflex_b200.evaluation",
                                description="Score a folder of KITTI result files against the labels of a split: the "
                                            "official AP table, or the COCO-style AP over overlap thresholds.")
    p.add_argument("--label_path", required=True, help="folder of ground-truth label files (000123.txt)")
    p.add_argument("--result_path", required=True, help="folder of detection files, one per image of the split")
    p.add_argument("--label_split_file", required=True, help="image ids of the split, one per line")
    p.add_argument("--current_class", default="0", help="comma-separated class ids or names (default: 0)")
    p.add_argument("--coco", action="store_true", help="AP averaged over ten overlap thresholds per class")
    p.add_argument("--score_thresh", type=float, default=-1, help="drop detections scored below it when > 0")
    p.add_argument("--metric", choices=("R40", "R11"), default="R40", help="recall positions of the official AP")
    args = p.parse_args(argv)
    out = evaluate(args.label_path, args.result_path, args.label_split_file, parse_classes(args.current_class),
                   coco=args.coco, score_thresh=args.score_thresh, metric=args.metric)
    sys.stdout.write(out if args.coco else out[0])


if __name__ == "__main__":
    main()
