"""MODEL.PRETRAIN = True (monoflex_b200/model/backbone/dla_dcn.py: load_pretrained) on the CPU, and do_train's refusals
that need no GPU. The network functions raise for the whole module: a test that reached them fails.

The fixture tests/golden/pretrain_dla34.npz (oracle/make_golden_pretrain.py) holds the keys and shapes of the reference's
KeypointDetector built with PRETRAIN = True from the same stand-in file, and that file's entries."""
import os
import urllib.request

import numpy as np
import pytest
import torch

from monoflex_b200 import synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.model.backbone import dla_dcn

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "pretrain_dla34.npz"))


def _no_network(*a, **k):
    raise AssertionError("a network call was attempted")


@pytest.fixture(autouse=True)
def no_network(monkeypatch):
    monkeypatch.setattr(torch.hub, "download_url_to_file", _no_network)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", _no_network)
    monkeypatch.setattr(urllib.request, "urlopen", _no_network)


@pytest.fixture
def hub(tmp_path, monkeypatch):
    """a temporary torch.hub directory holding the stand-in file -> (path, its entries)"""
    old = torch.hub.get_dir()
    torch.hub.set_dir(str(tmp_path / "hub"))
    try:
        path = os.path.join(torch.hub.get_dir(), "checkpoints", "dla34-ba72cf86.pth")
        os.makedirs(os.path.dirname(path))
        fake = syn.dla34_imagenet_weights(int(GOLDEN["seed"]))
        torch.save(fake, path)
        yield path, fake
    finally:
        torch.hub.set_dir(old)


def shapes(sd):
    return [",".join(str(s) for s in v.shape) for v in sd.values()]


def pretrain_cfg():
    cfg = default_cfg(device="cpu")
    cfg.MODEL.PRETRAIN = True
    return cfg


def test_stand_in_file_has_the_recorded_entries():
    fake = syn.dla34_imagenet_weights(int(GOLDEN["seed"]))
    assert list(fake) == GOLDEN["file_keys"].tolist() and shapes(fake) == GOLDEN["file_shapes"].tolist()
    assert list(fake)[-2:] == ["fc.weight", "fc.bias"] and fake["fc.bias"].shape == (1000,)
    assert GOLDEN["file_equal"].all()


def test_pretrained_detector_has_the_reference_layout_and_the_file_bit_for_bit(hub):
    from monoflex_b200.model.detector import KeypointDetector
    path, fake = hub
    sd = KeypointDetector(pretrain_cfg()).state_dict()
    assert list(sd) == GOLDEN["model_keys"].tolist()
    assert shapes(sd) == GOLDEN["model_shapes"].tolist()
    for k, v in fake.items():
        got = sd["backbone.base." + k]
        assert got.dtype == v.dtype and torch.equal(got, v), k
    assert isinstance(dla_dcn.dla34(pretrained=True).fc, torch.nn.Conv2d)


def test_num_classes_is_the_length_of_the_last_entry(hub):
    path, fake = hub
    fake = dict(fake)
    fake["fc.weight"], fake["fc.bias"] = torch.zeros(7, 512, 1, 1), torch.arange(7, dtype=torch.float32)
    torch.save(fake, path)
    base = dla_dcn.dla34(pretrained=True)
    assert base.fc.out_channels == 7 and torch.equal(base.fc.bias.detach(), fake["fc.bias"])


def test_missing_file_raises_with_the_path_and_url(tmp_path):
    old = torch.hub.get_dir()
    torch.hub.set_dir(str(tmp_path / "empty"))
    try:
        path = os.path.join(torch.hub.get_dir(), "checkpoints", "dla34-ba72cf86.pth")
        with pytest.raises(RuntimeError) as e:
            dla_dcn.dla34(pretrained=True)
        assert path in str(e.value) and dla_dcn.DLA34_URL in str(e.value)
        assert not os.path.exists(path)
    finally:
        torch.hub.set_dir(old)


def test_wrong_key_raises_as_a_strict_load(hub):
    path, fake = hub
    fake = dict(fake)
    fake["level9.weight"] = fake.pop("level0.0.weight")
    fake["fc.bias"] = fake.pop("fc.bias")                       # keep the classifier last
    torch.save(fake, path)
    with pytest.raises(RuntimeError, match=r"Missing key\(s\).*level0\.0\.weight"):
        dla_dcn.dla34(pretrained=True)


def test_pretrain_false_builds_no_classifier():
    assert not hasattr(dla_dcn.dla34(pretrained=False), "fc")


def test_do_train_refuses_a_torch_optimiser_before_anything_runs():
    from monoflex_b200.train import do_train
    model = torch.nn.Linear(2, 2)
    opt = torch.optim.AdamW(model.parameters())
    with pytest.raises(TypeError, match="monoflex_b200.solver import build_optimizer"):
        do_train(default_cfg(), False, model, [], None, opt, None, None, None, "cuda", {"iteration": 0})


def test_trainer_refuses_a_torch_optimiser():
    from monoflex_b200.train import Trainer
    model = torch.nn.Linear(2, 2)
    with pytest.raises(TypeError, match="build_optimizer"):
        Trainer(model, default_cfg(), optimizer=torch.optim.SGD(model.parameters(), lr=0.1))


def test_metric_logger_means_are_float32_and_global_means_float64():
    from monoflex_b200.train import MetricLogger
    m = MetricLogger()
    vals = [0.1 * i + 1e-9 for i in range(13)]
    for v in vals:
        m.update(loss=v)
    meter = m.meters["loss"]
    assert meter.avg == torch.tensor(vals[-10:]).mean().item()
    assert meter.value == torch.tensor(vals[-1:]).item() and meter.global_avg == sum(vals) / 13
    assert str(m) == "loss: {:.4f}".format(meter.avg)
