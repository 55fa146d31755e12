"""CPU: evaluation.write_kitti_detections against the unmodified reference's generate_kitti_3d_detection
(oracle/make_golden_kitti_writer.py -> tests/golden/kitti_writer.npz), byte for byte."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import evaluation as E


@pytest.fixture(scope="module")
def z():
    with np.load(os.path.join(GOLDEN, "kitti_writer.npz")) as f:
        return {k: f[k] for k in f.files}


def images(z):
    off = np.concatenate([[0], np.cumsum(z["counts"])])
    return [z["rows"][a:b] for a, b in zip(off[:-1], off[1:])]


def test_writer_matches_the_reference_byte_for_byte(z, tmp_path):
    for i, (rows, text) in enumerate(zip(images(z), z["text"])):
        for arg in (rows, torch.from_numpy(rows)):              # the host rows as numpy or as the decode's tensor
            path = tmp_path / ("%06d.txt" % i)
            E.write_kitti_detections(arg, str(path))
            assert path.read_bytes() == bytes(text), i


def test_fixture_covers_the_awkward_rows(z):
    rows = z["rows"]
    assert 0 in z["counts"] and z["counts"].max() >= 50
    assert set(rows[:, 0].tolist()) == {0.0, 1.0, 2.0}
    texts = [bytes(t).decode() for t in z["text"]]
    assert texts[0] == "\n" and all(t.endswith("\n") for t in texts)
    assert any(" -0.0 " in t for t in texts)
    scaled = rows.astype(np.float64) * 1e4
    assert (np.abs(np.abs(scaled - np.floor(scaled)) - 0.5) < 1e-2).any()     # half a unit from the fourth decimal
