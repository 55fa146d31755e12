"""Training-target encoding of KITTIDataset.__getitem__ (data/datasets/kitti.py:126-179, 202-216, 335-521) with its horizontal
flip (data/augmentations/augmentations.py:28-77) on the GPU, for a whole batch, from raw KITTI labels (csrc/mf_targets.cu).

    labels = pack_labels([read_kitti_label(path) for path in label_files], max_objs=40)    # float64 [B, 40, 16], host
    P2 = np.stack([read_kitti_calib(path) for path in calib_files])                          # float64 [B, 3, 4]
    enc = GpuTargetEncoder(cfg).encode(labels, P2, image_sizes, flips)                       # no host synchronisation
    loss_dict, log = model._forward_train(images, enc.edge_targets(), prepared=enc.prepared)
    enc.check()                                                                              # outside a captured step

`flips` are the flags the caller also passes to `GpuInputPipeline.images(flips=...)`. What stays on the host is parsing the
label text and the class filter, O(objects). Only the runs/monoflex.yaml configuration is built, with DATASETS.USE_RIGHT_IMAGE
either way (runs/monoflex_right.yaml); anything else raises NotImplementedError. A right-camera item (dataset index >=
num_samples, see dataset_view) is encoded with `right` set for its image, its calibration's P3
(read_kitti_calib(..., use_right_cam=True)) in place of P2 and the image_3 size; its label boxes are rebuilt from the
projected 3D boxes on the device (kitti.py:232-252). The reference raises on two label geometries (an edge object with two non-zero heat-map radii,
kitti.py:457; an outside object whose 2D box centre is outside the image, where approx_proj_center returns None); the kernel
cannot raise, so it counts them in a device status word, leaves them out of every output, and `EncodedTargets.check()` raises.
"""
import numpy as np
import torch

from ._lib import call, ptr, stream
from .structures import Calibration, ParamsList

LABEL_COLS = 16          # MF_TARGET_LABEL_COLS: valid + the 14 values of read_kitti_label + one zero column
ROW_COLS = 14            # type id, truncation, occlusion, xmin, ymin, xmax, ymax, h, w, l, tx, ty, tz, ry
CLASSES = ("Car", "Pedestrian", "Cyclist")
DOWN_RATIO = 4
_OBJ_SLICES = [("cls_ids", 0, 1), ("target_centers", 1, 3), ("2d_bboxes", 3, 7), ("reg_mask", 7, 8), ("trunc_mask", 8, 9),
               ("dimensions", 9, 12), ("locations", 12, 15), ("rotys", 15, 16), ("offset_3D", 16, 18),
               ("orientations", 18, 26), ("keypoints_depth_mask", 26, 29), ("keypoints", 29, 59)]   # OBJ_FIELDS columns
_INT_FIELDS = {"cls_ids": torch.int32, "target_centers": torch.int32, "reg_mask": torch.uint8, "trunc_mask": torch.uint8}


def _lines(path_or_lines):
    if isinstance(path_or_lines, str):
        with open(path_or_lines) as f:
            return [line.rstrip() for line in f]
    return [line.rstrip() for line in path_or_lines]


def read_kitti_label(path_or_lines, classes=CLASSES):
    """Object3d + filtrate_objects (kitti_utils.py:61-93, kitti.py:202-216): one float64 row per kept object, in file order:
    type id, truncation, occlusion, xmin, ymin, xmax, ymax, h, w, l, tx, ty, tz, ry. The location is rounded to float32 like
    Object3d.t; the box stays in doubles (the flip works on them, the kernel rounds Object3d.box2d to float32 itself). The
    file's alpha column is not used: alpha is recomputed from ry and the location."""
    rows = []
    for line in _lines(path_or_lines):
        data = line.split(" ")
        vals = [float(x) for x in data[1:]]
        if len(vals) < 14:
            raise ValueError("KITTI label line with %d values, 15 expected: %r" % (len(data), line))
        if data[0] not in classes:
            continue
        t = np.array(vals[10:13], dtype=np.float32).astype(np.float64)
        rows.append([float(classes.index(data[0])), vals[0], float(int(vals[1]))] + vals[3:10] + list(t) + [vals[13]])
    return np.array(rows, dtype=np.float64).reshape(-1, ROW_COLS)


def read_kitti_calib(path, use_right_cam=False):
    """P2 (or P3 with use_right_cam, Calibration(..., use_right_cam=True)) of a KITTI calibration file
    (Calibration.read_calib_file, kitti_utils.py:193-238) as float64 [3, 4]."""
    data = {}
    with open(path) as f:
        for line in f.readlines():
            line = line.rstrip()
            if len(line) == 0:
                continue
            key, value = line.split(":", 1)
            try:
                data[key] = np.array([float(x) for x in value.split()])
            except ValueError:
                pass
    return np.reshape(data["P3" if use_right_cam else "P2"], [3, 4]).astype(np.float64)


def dataset_len(num_samples, cfg, is_train=True):
    """len(KITTIDataset) (kitti.py:100-104): 2 * num_samples when DATASETS.USE_RIGHT_IMAGE and is_train, else num_samples."""
    return 2 * num_samples if _use_right(cfg, is_train) else num_samples


def dataset_view(idx, num_samples, cfg, is_train=True):
    """The view a KITTIDataset index stands for (kitti.py:232-259), for a sampler feeding GpuTargetEncoder: (frame index,
    right flag). Indices >= num_samples (present only with DATASETS.USE_RIGHT_IMAGE and is_train) are frame
    idx - num_samples seen by the right camera: image_3, P3 and the right flag of encode()."""
    idx = int(idx)
    if not 0 <= idx < dataset_len(num_samples, cfg, is_train):
        raise IndexError("dataset index %d outside 0..%d" % (idx, dataset_len(num_samples, cfg, is_train) - 1))
    return (idx - num_samples, True) if idx >= num_samples else (idx, False)


def flip_calib(P, widths, flips):
    """The camera matrices encode() writes to EncodedTargets.P2, on the host: float64 P [B, 3, 4] with the horizontal flip's
    calibration change (augmentations.py:71-74, P[0, 2] = w - P[0, 2] - 1, P[0, 3] = -P[0, 3]) where flips[b] is set,
    w = widths[b] the width of the view's own image."""
    P = np.array(P, dtype=np.float64).reshape(-1, 3, 4)
    f = np.asarray(flips, dtype=bool).reshape(-1)
    w = np.asarray(widths, dtype=np.float64).reshape(-1)
    P[f, 0, 2] = w[f] - P[f, 0, 2] - 1
    P[f, 0, 3] = -P[f, 0, 3]
    return P


def _use_right(cfg, is_train):
    return bool(_get(cfg.DATASETS, "USE_RIGHT_IMAGE", False)) and bool(is_train)


def pack_labels(list_of_rows, max_objs):
    """Per-image rows of read_kitti_label -> float64 [B, max_objs, 16]: slot = index in the filtered list (kitti.py:335),
    column 0 = 1 for a present object. More than max_objs kept objects raise ValueError (the reference: IndexError)."""
    out = np.zeros((len(list_of_rows), max_objs, LABEL_COLS), dtype=np.float64)
    for b, rows in enumerate(list_of_rows):
        rows = np.asarray(rows, dtype=np.float64).reshape(-1, ROW_COLS)
        if rows.shape[0] > max_objs:
            raise ValueError("image %d has %d objects of the detected classes, more than MAX_OBJECTS = %d"
                             % (b, rows.shape[0], max_objs))
        out[b, :rows.shape[0], 0] = 1.0
        out[b, :rows.shape[0], 1:1 + ROW_COLS] = rows
    return out


def _get(node, name, default):
    return getattr(node, name, default)


class GpuTargetEncoder(object):
    """KITTIDataset's training targets for a batch, on the device (see the module docstring)."""

    def __init__(self, cfg, device="cuda"):
        self._check_config(cfg, right_views=True)
        self.H, self.W = int(cfg.INPUT.HEIGHT_TRAIN), int(cfg.INPUT.WIDTH_TRAIN)
        if self.H % DOWN_RATIO or self.W % DOWN_RATIO:
            raise ValueError("input size %dx%d is not a multiple of the down ratio %d" % (self.W, self.H, DOWN_RATIO))
        self.max_objs = int(cfg.DATASETS.MAX_OBJECTS)
        self.ncls = len(CLASSES)
        self.K = 2 * (self.W // DOWN_RATIO + self.H // DOWN_RATIO)
        self.device = torch.device(device)

    @staticmethod
    def _check_config(cfg, right_views=False):
        """Only runs/monoflex.yaml's INPUT / DATASETS options are built; an option the cfg does not carry takes that value.
        right_views=False checks them for a caller that encodes left views only, which cannot serve DATASETS.USE_RIGHT_IMAGE
        (half of that training set is right-camera items); right_views=True, what the encoder itself checks, also accepts
        USE_RIGHT_IMAGE = True (runs/monoflex_right.yaml), whose right items encode() takes with its `right` flags."""
        inp, ds = cfg.INPUT, cfg.DATASETS
        right = _get(ds, "USE_RIGHT_IMAGE", False)
        if right not in ((True, False) if right_views else (False,)):
            raise NotImplementedError("GpuTargetEncoder: DATASETS.USE_RIGHT_IMAGE = %r; %s" % (
                right, "True or False expected" if right_views else
                "only False (runs/monoflex.yaml) is served by left views alone; right_views=True accepts True"))
        want = [(inp, "INPUT", "HEATMAP_CENTER", '3D'), (inp, "INPUT", "APPROX_3D_CENTER", 'intersect'),
                (inp, "INPUT", "ADJUST_BOUNDARY_HEATMAP", True), (inp, "INPUT", "KEYPOINT_VISIBLE_MODIFY", True),
                (inp, "INPUT", "HEATMAP_RATIO", 0.5), (inp, "INPUT", "ORIENTATION", 'multi-bin'),
                (inp, "INPUT", "ORIENTATION_BIN_SIZE", 4), (inp, "INPUT", "AUG_PARAMS", [[0.5]]),
                (ds, "DATASETS", "CONSIDER_OUTSIDE_OBJS", True), (ds, "DATASETS", "FILTER_ANNO_ENABLE", True),
                (ds, "DATASETS", "FILTER_ANNOS", [0.9, 20]), (ds, "DATASETS", "DETECT_CLASSES", list(CLASSES)),
                (cfg.MODEL.BACKBONE, "MODEL.BACKBONE", "DOWN_RATIO", DOWN_RATIO),
                (cfg.MODEL.HEAD, "MODEL.HEAD", "ENABLE_EDGE_FUSION", True)]
        for node, path, key, v in want:
            got = _get(node, key, v)
            got = [list(g) if isinstance(g, (list, tuple)) else g for g in got] if isinstance(got, (list, tuple)) else got
            if got != v:
                raise NotImplementedError("GpuTargetEncoder: %s.%s = %r; only %r (runs/monoflex.yaml) is built" % (path, key, got, v))

    def _dev(self, x, dtype):
        t = torch.as_tensor(x)
        if t.device != self.device:
            t = t.to(self.device, non_blocking=True)
        return t.to(dtype).contiguous()

    def encode(self, labels, P2, image_sizes, flips=None, out=None, edge_out=None, right=None):
        """labels float64 [B, max_objs, 16] (pack_labels), P2 float64 [B, 3, 4], image_sizes [B, 2] original (w, h), flips [B]
        (or None). Host arrays are copied up; for a CUDA-graph capture pass device tensors and refill them between replays.
        out: (hm, obj, img) tensors to write instead of allocating (a captured step's static buffers); edge_out:
        (edge_indices int64 [B, K, 2], edge_len int64 [B]) likewise. right [B] (or None: all left) marks right-camera items,
        host or device like flips: for such an image P2[b] is its P3, image_sizes[b] the right image's size, and the label
        rows' box columns are not read. Returns EncodedTargets; nothing here reads the device."""
        B, M = int(labels.shape[0]), self.max_objs
        if tuple(labels.shape) != (B, M, LABEL_COLS):
            raise ValueError("labels: [B, %d, %d] expected, got %s" % (M, LABEL_COLS, tuple(labels.shape)))
        if tuple(P2.shape) != (B, 3, 4) or tuple(image_sizes.shape) != (B, 2):
            raise ValueError("P2 [B, 3, 4] and image_sizes [B, 2] expected, got %s, %s" % (tuple(P2.shape), tuple(image_sizes.shape)))
        for name, flags in (("flips", flips), ("right", right)):
            if flags is not None and tuple(flags.shape if hasattr(flags, "shape") else (len(flags),)) != (B,):
                raise ValueError("%s: one flag per image expected" % name)
        if not (torch.is_tensor(image_sizes) and image_sizes.is_cuda):
            s = np.asarray(image_sizes.cpu() if torch.is_tensor(image_sizes) else image_sizes)
            if (s < 1).any() or (s[:, 0] > self.W).any() or (s[:, 1] > self.H).any():
                raise ValueError("image sizes %s outside 1..%dx%d" % (s.tolist(), self.W, self.H))
        inputs = (self._dev(labels, torch.float64), self._dev(P2, torch.float64), self._dev(image_sizes, torch.int32),
                  None if flips is None else self._dev(flips, torch.int32),
                  None if right is None else self._dev(right, torch.int32))
        dev, f32 = self.device, torch.float32
        h, w = self.H // DOWN_RATIO, self.W // DOWN_RATIO
        shapes = ((B, self.ncls, h, w), (B * M, _obj_cols()), (B, 8))
        if out is None:
            out = tuple(torch.empty(s, dtype=f32, device=dev) for s in shapes)
        for t, s in zip(out, shapes):
            if tuple(t.shape) != s or t.dtype != f32 or not t.is_cuda or not t.is_contiguous():
                raise ValueError("out: contiguous fp32 CUDA tensors of shapes %s expected" % (shapes,))
        if edge_out is None:
            edge_out = (torch.empty(B, self.K, 2, dtype=torch.int64, device=dev), torch.empty(B, dtype=torch.int64, device=dev))
        if tuple(edge_out[0].shape) != (B, self.K, 2) or tuple(edge_out[1].shape) != (B,) or \
                any(t.dtype != torch.int64 or not t.is_contiguous() for t in edge_out):
            raise ValueError("edge_out: int64 [B, %d, 2] and [B] expected" % self.K)
        e = EncodedTargets(self, inputs, out, edge_out)
        lab, p2, sz, fl, rt = inputs
        hm, obj, img = out
        call("mf_encode_targets_views", lab.data_ptr(), p2.data_ptr(), sz.data_ptr(), ptr(fl), ptr(rt), B, M,
             self.H, self.W, hm.data_ptr(), obj.data_ptr(), img.data_ptr(), e.alphas.data_ptr(), e.gt_bboxes.data_ptr(),
             e.reg_weight.data_ptr(), e.occlusions.data_ptr(), e.truncations.data_ptr(), e.obj6.data_ptr(), e.P2.data_ptr(),
             edge_out[0].data_ptr(), edge_out[1].data_ptr(), e.status.data_ptr(), stream())
        return e

    def encode_inference(self, P2, image_sizes):
        """The test split's fields (kitti.py:287-299): per image a ParamsList with pad_size, calib, edge_len, edge_indices
        (the edge fields on the device). P2 and image_sizes are host values here: pad_size and calib are host fields."""
        s = np.asarray(image_sizes.cpu() if torch.is_tensor(image_sizes) else image_sizes).astype(np.int64).reshape(-1, 2)
        P2 = np.asarray(P2.cpu() if torch.is_tensor(P2) else P2, dtype=np.float64).reshape(-1, 3, 4)
        B = s.shape[0]
        if (s < 1).any() or (s[:, 0] > self.W).any() or (s[:, 1] > self.H).any():
            raise ValueError("image sizes %s outside 1..%dx%d" % (s.tolist(), self.W, self.H))
        sz = self._dev(torch.from_numpy(s), torch.int32)
        edge = torch.empty(B, self.K, 2, dtype=torch.int64, device=self.device)
        edge_len = torch.empty(B, dtype=torch.int64, device=self.device)
        call("mf_encode_edges", sz.data_ptr(), B, self.H, self.W, edge.data_ptr(), edge_len.data_ptr(), stream())
        out = []
        for b in range(B):
            t = ParamsList(image_size=(self.W, self.H), is_train=False)
            t.add_field("pad_size", torch.tensor([(self.W - s[b, 0]) // 2, (self.H - s[b, 1]) // 2], dtype=torch.int64))
            t.add_field("calib", Calibration(P2[b]))
            t.add_field("edge_len", edge_len[b])
            t.add_field("edge_indices", edge[b])
            out.append(t)
        self._keep = sz                            # alive until the kernel has run (stream ordered)
        return out


def _obj_cols():
    from ._lib import load
    return load().mf_loss_obj_cols()


class EncodedTargets(object):
    """Device outputs of one GpuTargetEncoder.encode call.

    prepared      (hm, obj, img): what Loss_Computation.prepare_targets returns, for `_forward_train(..., prepared=)`
    edge_indices  int64 [B, K, 2], edge_len int64 [B]
    alphas, gt_bboxes, reg_weight, occlusions, truncations: the remaining per-slot fields of kitti.py:497-521
    obj6          int32 [B, M, 6] heat-map table (valid, class, cx, cy, rx, ry)
    P2            float64 [B, 3, 4]: the (flipped) camera matrix each image was encoded with (P3 for a right-camera item)
    status        int32 [1]: objects left out where the reference raises (read by check())
    inputs        (labels, P2, image_sizes, flips, right) on the device, as encode_into encodes them again"""

    def __init__(self, encoder, inputs, out, edge_out):
        B, M, dev = out[2].shape[0], encoder.max_objs, encoder.device
        self.encoder, self.inputs = encoder, inputs
        self.prepared = tuple(out)
        self.edge_indices, self.edge_len = edge_out
        self.alphas = torch.empty(B, M, dtype=torch.float32, device=dev)
        self.gt_bboxes = torch.empty(B, M, 4, dtype=torch.float32, device=dev)
        self.reg_weight = torch.empty(B, M, dtype=torch.float32, device=dev)
        self.occlusions = torch.empty(B, M, dtype=torch.float64, device=dev)
        self.truncations = torch.empty(B, M, dtype=torch.float64, device=dev)
        self.obj6 = torch.empty(B, M, 6, dtype=torch.int32, device=dev)
        self.P2 = torch.empty(B, 3, 4, dtype=torch.float64, device=dev)
        self.status = torch.empty(1, dtype=torch.int32, device=dev)

    def __len__(self):
        return self.P2.shape[0]

    def check(self):
        """Raise where the reference's __getitem__ raises. Reads the status word: a host synchronisation, so call it outside a
        captured step (e.g. on the previous batch's targets)."""
        n = int(self.status.item())
        if n:
            raise RuntimeError("GpuTargetEncoder: %d object(s) or image(s) the reference cannot encode (an edge object with two "
                               "non-zero heat-map radii, an outside object whose 2D box centre lies outside the image, an image "
                               "larger than the input); they were left out of the targets" % n)

    def encode_into(self, out, edge_out):
        """Encode the same inputs again into other buffers (a captured training step's static targets)."""
        lab, p2, sz, fl, rt = self.inputs
        return self.encoder.encode(lab, p2, sz, fl, out=out, edge_out=edge_out, right=rt)

    def edge_targets(self):
        """Per-image ParamsLists with only the edge-fusion fields (device views): what the predictor reads when the loss
        gets `prepared`."""
        enc = self.encoder
        out = []
        for b in range(len(self)):
            t = ParamsList(image_size=(enc.W, enc.H), is_train=True)
            t.add_field("edge_len", self.edge_len[b])
            t.add_field("edge_indices", self.edge_indices[b])
            out.append(t)
        return out

    def param_lists(self, P2=None):
        """Reference-shaped ParamsLists (kitti.py:496-521 without ori_img): device tensor views of the encoded tables and a
        host Calibration of the (flipped) P2 or P3 (one device-to-host copy). prepare_targets(param_lists()) == prepared.
        P2: host float64 [B, 3, 4] equal to self.P2 (flip_calib of the encoded matrices) for the Calibrations, so that
        nothing here waits for the device."""
        enc = self
        hm, obj, img = self.prepared
        B, M = len(self), self.encoder.max_objs
        o = obj.view(B, M, obj.shape[1])
        if P2 is None:
            P2 = self.P2.cpu().numpy()
        elif np.shape(P2) != (B, 3, 4):
            raise ValueError("P2: [%d, 3, 4] host matrices expected, got %s" % (B, np.shape(P2)))
        pad = img[:, 6:8].to(torch.int64)
        out = []
        for b in range(B):
            t = ParamsList(image_size=(self.encoder.W, self.encoder.H), is_train=True)
            for name, c0, c1 in _OBJ_SLICES:
                v = o[b, :, c0:c1]
                if c1 - c0 == 1:
                    v = v.reshape(M)
                elif name == "keypoints":
                    v = v.reshape(M, 10, 3)
                if name in _INT_FIELDS:
                    v = v.to(_INT_FIELDS[name])
                t.add_field(name, v)
            t.add_field("calib", Calibration(P2[b]))
            t.add_field("pad_size", pad[b])
            t.add_field("reg_weight", enc.reg_weight[b])
            t.add_field("alphas", enc.alphas[b])
            t.add_field("hm", hm[b])
            t.add_field("gt_bboxes", enc.gt_bboxes[b])
            t.add_field("occlusions", enc.occlusions[b])
            t.add_field("truncations", enc.truncations[b])
            t.add_field("edge_len", enc.edge_len[b])
            t.add_field("edge_indices", enc.edge_indices[b])
            out.append(t)
        return out
