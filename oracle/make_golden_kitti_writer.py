"""Golden fixture of the KITTI detection text writer from the UNMODIFIED reference: tests/golden/kitti_writer.npz.

    python -m oracle.make_golden_kitti_writer

Runs the reference's generate_kitti_3d_detection (kitti_object_eval_python/evaluate.py:34-53, which ends in
check_last_line_break) on decode-shaped float32 rows [n, 14] (class, alpha, x1, y1, x2, y2, h, w, l, x, y, z, ry, score)
and stores each file's bytes. The images: none, one and many detections; every class; negative zeros, values that round
to -0.0, values half a unit from the fourth decimal (which np.round's float32 arithmetic may send either way), values
that float32 cannot hold to four decimals, large pixel coordinates, tiny magnitudes and random decode-like rows."""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden_kitti_eval import reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "kitti_writer.npz")


def awkward_images(rng):
    row = lambda cls, *v: [float(cls)] + list(v)
    edge = [
        row(0, -0.0, 0.0, -0.0, 1279.99995, 383.00005, 1.23445, 1.23455, -2.50005, -0.00004, 0.00005, 99.99995, -3.14159265, 0.99995),
        row(1, 3.14159265, 1241.5, 374.49995, 1242.0, 375.0, 1.76, 0.66, 0.84, -12.345649, 1.7, 45.67895, 3.1416, 0.2),
        row(2, -1e-5, 1e-7, 5e-5, 15e-5, 0.123456789, 1.74, 0.6, 1.76, 1e-9, -5e-5, 0.1, -1e-4, 0.0),
        row(0, 0.30000001, 0.1 + 0.2, 2.675, 1.005, 2.5e-4, 7.77775, 0.33335, 8.88885, -0.44445, 0.55555, 66.66665, 1.11115, 0.5),
    ]
    images = [np.zeros((0, 14)), np.array(edge[:1]), np.array(edge)]
    for n in (1, 7, 50):                    # decode-like rows
        r = np.zeros((n, 14))
        r[:, 0] = rng.integers(0, 3, n)
        r[:, 1] = rng.uniform(-np.pi, np.pi, n)
        x1, y1 = rng.uniform(0, 1200, n), rng.uniform(0, 350, n)
        r[:, 2:6] = np.stack([x1, y1, x1 + rng.uniform(0, 80, n), y1 + rng.uniform(0, 25, n)], 1)
        r[:, 6:9] = rng.uniform(0.5, 4, (n, 3))
        r[:, 9:12] = np.stack([rng.uniform(-20, 20, n), rng.uniform(0.5, 2.5, n), rng.uniform(0.1, 100, n)], 1)
        r[:, 12] = rng.uniform(-np.pi, np.pi, n)
        r[:, 13] = rng.uniform(0, 1, n)
        images.append(r)
    return [np.asarray(i, np.float32).reshape(-1, 14) for i in images]


def main(seed=20261018):
    _, evl, _ = reference()
    images = awkward_images(np.random.default_rng(seed))
    texts = []
    with tempfile.TemporaryDirectory() as d:
        for i, rows in enumerate(images):
            path = os.path.join(d, "%06d.txt" % i)
            evl.generate_kitti_3d_detection(torch.from_numpy(rows), path)
            with open(path, "rb") as f:
                texts.append(f.read())
    z = {"rows": np.concatenate(images, 0), "counts": np.array([len(r) for r in images], np.int64),
         "text": np.array(texts, dtype=object).astype(np.bytes_)}
    np.savez_compressed(OUT, **z)
    print("wrote %s: %d files, %d rows" % (OUT, len(images), len(z["rows"])))


if __name__ == "__main__":
    main()
