"""TEST INFRASTRUCTURE. Records tests/golden/pretrain_dla34.npz from the UNMODIFIED reference's KeypointDetector built
with MODEL.PRETRAIN = True (DLASeg -> dla34(pretrained=True) -> DLA.load_pretrained_model, model/backbone/dla_dcn.py:
333-352), imported through oracle/ref_shims.py.

The ImageNet file is a seeded stand-in (synthetic.dla34_imagenet_weights: the reference DLA-34 base's keys and shapes plus
`fc`) written to <TORCH_HOME>/hub/checkpoints/dla34-ba72cf86.pth in a temporary TORCH_HOME, where model_zoo.load_url
finds it. torch.hub.download_url_to_file and urllib.request.urlopen are patched to raise before anything runs, so a
missing file fails instead of reaching the network. Recorded:

  * file_keys / file_shapes: the stand-in file's entries in order (checked against the reference DLA's own state_dict);
  * model_keys / model_shapes: the reference detector's state_dict after the load, `backbone.base.fc.*` included;
  * file_equal: 1 where the reference's loaded backbone.base tensor equals the file's bit for bit.

    python oracle/make_golden_pretrain.py        (needs the reference tree; writes tests/golden/pretrain_dla34.npz)
"""
import os
import sys
import tempfile
import urllib.request
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "pretrain_dla34.npz")
SEED = 3


def _no_network(*a, **k):
    raise RuntimeError("make_golden_pretrain: a network call was attempted")


def _shape_str(t):
    return ",".join(str(int(s)) for s in t.shape)


def main():
    sys.path.insert(0, ROOT)
    with mock.patch("torch.hub.download_url_to_file", _no_network), mock.patch.object(urllib.request, "urlopen",
                                                                                     _no_network):
        import torch
        from oracle import ref_shims as rs
        from monoflex_b200 import synthetic as syn
        with tempfile.TemporaryDirectory() as home:
            os.environ["TORCH_HOME"] = home
            torch.hub.set_dir(os.path.join(home, "hub"))
            fake = syn.dla34_imagenet_weights(SEED)
            path = os.path.join(torch.hub.get_dir(), "checkpoints", "dla34-ba72cf86.pth")
            os.makedirs(os.path.dirname(path))
            torch.save(fake, path)
            cfg = rs.reference_cfg()
            rs.install()
            from model.backbone.dla_dcn import DLA, BasicBlock
            ref_base = DLA([1, 1, 1, 2, 2, 1], [16, 32, 64, 128, 256, 512], block=BasicBlock)
            ref_keys = [k for k in ref_base.state_dict() if not k.endswith("num_batches_tracked")]
            if ref_keys != list(fake)[:-2] or list(fake)[-2:] != ["fc.weight", "fc.bias"]:
                raise RuntimeError("the stand-in file's keys are not the reference DLA-34 base's plus fc")
            cfg.MODEL.PRETRAIN = True
            model = rs.build_reference_model(cfg)
            sd = model.state_dict()
            equal = [int(torch.equal(sd["backbone.base." + k], v)) for k, v in fake.items()]
    np.savez_compressed(OUT, file_keys=np.array(list(fake)), file_shapes=np.array([_shape_str(v) for v in fake.values()]),
                        model_keys=np.array(list(sd)), model_shapes=np.array([_shape_str(v) for v in sd.values()]),
                        file_equal=np.array(equal, dtype=np.int8), seed=np.array(SEED))
    print("wrote", OUT, len(fake), "file entries,", len(sd), "model entries, all equal:", all(equal))


if __name__ == "__main__":
    main()
