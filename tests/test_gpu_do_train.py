"""-m gpu: monoflex_b200.train.do_train, the drop-in for engine/trainer.py:do_train, on a generated KITTI-layout directory
(the training loader's seven frames, a three-frame `val` split of the same directory), B = 2, synthetic weights.

One 25-iteration run with EVAL_INTERVAL = SAVE_CHECKPOINT_INTERVAL = 10 and LambdaLR decays at 13 and 22 is checked for:
its log records against a restatement of the reference's MetricLogger fed the per-step log_loss_dicts the drop-in
resolved (wall-clock fields masked); its TensorBoard tags, steps and values; the lr at each step against the reference's
scheduler.step(iteration); its per-step losses against the eager reference-shaped loop; its checkpoints (names,
iterations, reference keys, an optimiser state that loads into torch.optim.AdamW); no host synchronisation between
boundaries; and an evaluation that leaves the training state bit-identical. Separate runs cover the warm-up schedule, a
resume from iteration 10 with a dynamic loss scale, and tools/plain_train_net.py:train()'s call sequence with
runs/monoflex.yaml's settings and MODEL.PRETRAIN from a stand-in cached ImageNet file."""
import collections
import io
import itertools
import logging
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from monoflex_b200 import loader as L
from monoflex_b200 import solver
from monoflex_b200 import synthetic as syn
from monoflex_b200 import train as TR
from monoflex_b200.config import default_cfg
from monoflex_b200.model.detector import KeypointDetector

pytestmark = pytest.mark.gpu
VAL_IDS = ["000004", "000001", "000010"]
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "pretrain_dla34.npz"))


@pytest.fixture(scope="module")
def kitti(tmp_path_factory):
    from test_gpu_train_loader import make_kitti
    root = str(tmp_path_factory.mktemp("kitti"))
    make_kitti(root)
    with open(os.path.join(root, "ImageSets", "val.txt"), "w") as f:
        f.write("".join(i + "\n" for i in VAL_IDS))
    return root


def run_cfg(out, max_iter=25, steps=(13, 22), warmup=False):
    cfg = default_cfg()
    cfg.DATASETS.TRAIN_SPLIT, cfg.DATASETS.TEST_SPLIT, cfg.DATASETS.TEST = "train", "val", ("kitti_val",)
    cfg.DATASETS.USE_RIGHT_IMAGE = False
    cfg.SOLVER.IMS_PER_BATCH, cfg.TEST.IMS_PER_BATCH = 2, 2
    cfg.SOLVER.MAX_ITERATION, cfg.SOLVER.STEPS = max_iter, steps
    cfg.SOLVER.EVAL_INTERVAL = cfg.SOLVER.SAVE_CHECKPOINT_INTERVAL = 10
    cfg.SOLVER.EVAL_AND_SAVE_EPOCH = False
    cfg.SOLVER.LR_WARMUP, cfg.SOLVER.WARMUP_STEPS = warmup, 5
    cfg.OUTPUT_DIR, cfg.START_TIME = str(out), "10-19 00:00:00"
    return cfg


def make_model(cfg, seed=0):
    m = KeypointDetector(cfg).cuda()
    m.load_state_dict(syn.make_state_dict(seed=seed), strict=False)
    return m


class Checkpointer(object):
    """utils/check_point.py's save(name, **kwargs) / load(f) interface: torch.save of the model, optimiser and scheduler
    states plus the kwargs. Every save is also kept in memory as (name, bytes)."""

    def __init__(self, model, optimizer, scheduler, save_dir):
        self.model, self.optimizer, self.scheduler, self.save_dir = model, optimizer, scheduler, save_dir
        self.saved = []
        self.logger = logging.getLogger("monoflex.checkpointer")

    def save(self, name, **kwargs):
        data = {"model": self.model.state_dict(), "optimizer": self.optimizer.state_dict(),
                "scheduler": self.scheduler.state_dict()}
        data.update(kwargs)
        f = os.path.join(self.save_dir, "{}.pth".format(name))
        self.logger.info("Saving checkpoint to {}".format(f))
        torch.save(data, f)
        buf = io.BytesIO()
        torch.save(data, buf)
        self.saved.append((name, buf.getvalue()))

    def load(self, f):
        ck = torch.load(io.BytesIO(f) if isinstance(f, bytes) else f, map_location="cpu", weights_only=False)
        self.model.load_state_dict(ck.pop("model"))
        self.optimizer.load_state_dict(ck.pop("optimizer"))
        self.scheduler.load_state_dict(ck.pop("scheduler"))
        return ck


class Recorder(object):
    """what the drop-in fed its meters (the resolved log_loss_dicts, in order), and whether the host synchronised"""

    def __init__(self, monkeypatch):
        self.logs = []
        orig = TR.MetricLogger.update

        def update(meters, **kw):
            if "loss" in kw:
                self.logs.append({k: v for k, v in kw.items() if k != "loss"})
            return orig(meters, **kw)
        monkeypatch.setattr(TR.MetricLogger, "update", update)


def guarded(loader, start, warm, boundaries):
    """the loader's batches; the steps between boundaries after the graph was captured run with the sync debug mode at
    "error", the first step after a checkpoint or an evaluation included. The step that ends on a boundary runs at
    "default": the boundary's reads (flush, optimiser state_dict, evaluation) follow it before the next batch is drawn."""
    for it, batch in zip(range(start, 10 ** 9), loader):
        quiet = it >= start + warm + 1 and (it + 1) not in boundaries
        torch.cuda.set_sync_debug_mode("error" if quiet else "default")
        yield batch
    torch.cuda.set_sync_debug_mode("default")


class Skipped(object):
    """the loader's stream from batch `skip` on: the batches an uninterrupted run trains on after `skip` iterations"""

    def __init__(self, loader, skip):
        self.loader, self.skip, self.dataset = loader, skip, loader.dataset

    def __iter__(self):
        return itertools.islice(iter(self.loader), self.skip, None)


class ParamsListBatches(object):
    """the loader's batches without `encoded`: images and the reference-shaped ParamsList targets, what any loader other
    than KittiTrainLoader yields"""

    def __init__(self, loader):
        self.loader, self.dataset = loader, loader.dataset

    def __iter__(self):
        for batch in self.loader:
            yield {"images": batch["images"], "targets": batch["targets"], "img_ids": batch["img_ids"]}


class Guarded(object):
    def __init__(self, loader, start, boundaries, warm=2):
        self.loader, self.start, self.boundaries, self.warm = loader, start, boundaries, warm
        self.dataset = loader.dataset

    def __iter__(self):
        return guarded(self.loader, self.start, self.warm, self.boundaries)


def run(cfg, model, arguments, skip=0, optimizer=None, scheduler=None, warmup=None, ckpt=None, guard=None,
        params_lists=False):
    if optimizer is None:
        optimizer = solver.build_optimizer(model, cfg)
        scheduler, warmup = solver.build_scheduler(optimizer, total_iters_each_epoch=3, optim_cfg=cfg.SOLVER)
    ckpt = ckpt or Checkpointer(model, optimizer, scheduler, cfg.OUTPUT_DIR)
    train_loader = L.KittiTrainLoader(cfg, arguments["root"], seed=5)
    val = L.KittiEvalLoader(cfg, arguments["root"])
    args = {k: v for k, v in arguments.items() if k != "root"}
    if skip:
        train_loader = Skipped(train_loader, skip)
    if params_lists:
        train_loader = ParamsListBatches(train_loader)
    if guard is not None:
        train_loader = Guarded(train_loader, args["iteration"], guard)
    try:
        trainer = TR.do_train(cfg, False, model, train_loader, val, optimizer, scheduler, warmup, ckpt,
                              torch.device("cuda"), args)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    return trainer, ckpt, args


class RefMeter(object):
    """utils/metric_logger.py, restated: SmoothedValue(window 10) and MetricLogger.__str__"""

    def __init__(self):
        self.deque, self.total, self.count = collections.deque(maxlen=10), 0.0, 0

    def update(self, v):
        self.deque.append(v)
        self.total += v
        self.count += 1


def reference_records(logs, lrs, max_iter, start=0):
    """the reference loop's log lines and non-timing TensorBoard scalars {tag: {step: value}} from the same log_loss_dicts"""
    meters = collections.OrderedDict()
    lines, scalars = [], collections.defaultdict(dict)

    def update(**kw):
        for k, v in kw.items():
            meters.setdefault(k, RefMeter()).update(v)
    for i, (log, lr) in enumerate(zip(logs, lrs)):
        it = start + i + 1
        update(loss=sum(v for k, v in log.items() if k.find('loss') >= 0), **log)
        update(time=0.0, data=0.0)
        scalars["stat/lr"][it] = lr
        for name, m in meters.items():
            if name.find('MAE') >= 0:
                scalars["train_metric_depth_errors_" + name][it] = torch.tensor(list(m.deque))[-1].item()
            elif name not in ('time', 'data'):
                scalars["train_metric/" + name][it] = torch.tensor(list(m.deque))[-1].item()
        if it % 10 == 0 or it == max_iter:
            body = " ".join("{}: {:.4f}".format(n, torch.tensor(list(m.deque)).mean().item()) for n, m in meters.items())
            lines.append(mask(" ".join(["eta: {}".format("0:00:00"), "iter: {}".format(it), body,
                                        "lr: {:.8f} \n".format(lr)])))
    return lines, scalars


def mask(line):
    return re.sub(r"(eta|time|data): \S+", r"\1: *", line)


def trainer_lines(caplog):
    return [mask(r.getMessage()) for r in caplog.records if r.name == "monoflex.trainer" and r.getMessage().startswith("eta")]


def events(folder):
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    out = {}
    for d, _, fs in os.walk(folder):
        if not any(f.startswith("events.") for f in fs):
            continue
        acc = EventAccumulator(d, size_guidance={"scalars": 0})
        acc.Reload()
        sub = os.path.relpath(d, folder)
        for tag in acc.Tags()["scalars"]:
            name = tag if sub == "." else os.path.basename(sub)
            out[name] = {e.step: e.value for e in acc.Scalars(tag)}
    return out


def reference_lrs(cfg, n, start=0):
    """optimizer.param_groups[0]["lr"] after each step of the reference's loop (warmup.step(i) / scheduler.step(i))"""
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=cfg.SOLVER.BASE_LR)
    sched, warm = solver.build_scheduler(opt, cfg.SOLVER)
    warm_iters = cfg.SOLVER.WARMUP_STEPS if cfg.SOLVER.LR_WARMUP else -1
    out = []
    for i in range(n):
        if i < warm_iters:
            warm.step(i)
        else:
            sched.step(i)
        if i >= start:
            out.append(opt.param_groups[0]["lr"])
    return out


def state_of(model, optimizer):
    opt = getattr(optimizer, "opt", optimizer)
    return ([p.detach().clone() for p in model.parameters()] + [b.detach().clone() for b in model.buffers()]
            + [opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt._state4.clone()], opt.step_count)


@pytest.fixture(scope="module")
def main_run(kitti, tmp_path_factory):
    """the 25-iteration run, with its log records, resolved logs, evaluation-state checks and checkpoints"""
    mp = pytest.MonkeyPatch()
    out = tmp_path_factory.mktemp("run")
    cfg = run_cfg(out)
    model = make_model(cfg)
    rec = Recorder(mp)
    handler = _ListHandler()
    logging.getLogger("monoflex").addHandler(handler)
    logging.getLogger("monoflex").setLevel(logging.INFO)
    states = []
    orig_eval = TR.do_eval

    def do_eval(cfg_, net, loaders, iteration):
        torch.cuda.synchronize()
        before = state_of(net, optimizer)
        ret = orig_eval(cfg_, net, loaders, iteration)
        torch.cuda.synchronize()
        states.append((iteration, before, state_of(net, optimizer)))
        return ret
    mp.setattr(TR, "do_eval", do_eval)
    optimizer = solver.build_optimizer(model, cfg)
    scheduler, warmup = solver.build_scheduler(optimizer, cfg.SOLVER)
    try:
        trainer, ckpt, args = run(cfg, model, {"iteration": 0, "iter_per_epoch": 3, "root": kitti}, optimizer=optimizer,
                                  scheduler=scheduler, warmup=warmup, guard={10, 20, 25})
    finally:
        mp.undo()
        logging.getLogger("monoflex").removeHandler(handler)
    return dict(cfg=cfg, model=model, trainer=trainer, ckpt=ckpt, args=args, logs=rec.logs, records=handler.records,
                states=states, out=str(out))


class _ListHandler(logging.Handler):
    def __init__(self):
        super().__init__()
        self.records = []

    def emit(self, record):
        self.records.append(record)


def test_log_lines_and_tensorboard_follow_the_reference_loop(main_run):
    cfg, logs = main_run["cfg"], main_run["logs"]
    assert len(logs) == 25 and all(np.isfinite(sum(l.values())) for l in logs)
    lrs = reference_lrs(cfg, 25)
    want_lines, want_scalars = reference_records(logs, lrs, 25)
    recs = main_run["records"]
    msgs = [r.getMessage() for r in recs]
    got_lines = [mask(m) for r, m in zip(recs, msgs) if r.name == "monoflex.trainer" and m.startswith("eta")]
    assert got_lines == want_lines
    # the reference's order of records around the boundaries
    order = [m.split(" ")[0] if not m.startswith("eta") else "eta%s" % m.split("iter: ")[1].split(" ")[0]
             for r, m in zip(recs, msgs) if r.name in ("monoflex.trainer", "monoflex.checkpointer")]
    assert order[:7] == ["Start", "eta10", "iteration", "Saving", "iteration", "Saving", "iteration"], order
    assert msgs[-3].startswith("Total training time: ") and msgs[-2] == "The best performance is as follows"
    assert msgs[-1].startswith("\n") and len(msgs[-1]) > 1
    ev = events(os.path.join(cfg.OUTPUT_DIR, "writer", cfg.START_TIME))
    for tag in ("stat/lr", "stat/time", "stat/data", "train_metric/loss", "train_metric/hm_loss"):
        assert sorted(ev[tag]) == list(range(1, 26)), tag
    for tag, want in want_scalars.items():
        assert tag in ev, tag
        for step, v in want.items():
            assert ev[tag][step] == np.float32(v), (tag, step)
    evals = [t for t in ev if t.startswith("eval_soft_0.70/")]
    assert "eval_soft_0.70/Car_3d_0.70/moderate" in evals and all(sorted(ev[t]) == [1, 2] for t in evals)


def test_lr_changes_at_the_reference_iterations(main_run):
    cfg = main_run["cfg"]
    ev = events(os.path.join(cfg.OUTPUT_DIR, "writer", cfg.START_TIME))
    got = [ev["stat/lr"][i] for i in range(1, 26)]
    want = reference_lrs(cfg, 25)
    assert got == [np.float32(v) for v in want]
    # the lr logged at iteration i + 1 is the one after step i: the decays at 13 and 22 show at 14 and 23 (a plain
    # scheduler.step() would show them at 13 and 22)
    assert [i + 2 for i in range(24) if want[i + 1] != want[i]] == [14, 23]


def test_losses_match_the_eager_reference_loop(main_run, kitti):
    """model(images, targets), FusedAdamW, scheduler.step(i) on the same batches; the captured-against-eager tolerances"""
    cfg = main_run["cfg"]
    model = make_model(cfg)
    model.train()
    opt = solver.build_optimizer(model, cfg)
    sched, _ = solver.build_scheduler(opt, cfg.SOLVER)
    for i, batch in zip(range(6), L.KittiTrainLoader(cfg, kitti, seed=5)):
        loss_dict, log = model(batch["images"].tensors, list(batch["targets"]))
        losses = sum(loss_dict.values())
        opt.zero_grad()
        losses.backward()
        if i == 0:
            opt.mark_unused({n for n, _ in model.named_parameters()} - set(model.last_grad_names), model)
        opt.step()
        sched.step(i)
        a = sum(v for k, v in log.items() if k.endswith("_loss"))
        b = sum(v for k, v in main_run["logs"][i].items() if k.endswith("_loss"))
        assert np.isfinite(b) and abs(a - b) <= (0.03 if i <= 2 else 0.25) * abs(a), (i, a, b)


def test_checkpoints_at_the_reference_iterations(main_run):
    saved = [(n, torch.load(io.BytesIO(b), map_location="cpu", weights_only=False)) for n, b in main_run["ckpt"].saved]
    names = [(n, c["iteration"]) for n, c in saved]
    assert names == [("model_checkpoint", 10), ("model_moderate_best_soft", 10), ("model_checkpoint", 20),
                     ("model_moderate_best_soft", 20), ("model_final", 25)]          # synthetic weights: AP 0 >= best 0
    want_keys = [k for k in GOLDEN["model_keys"].tolist() if not k.startswith("backbone.base.fc.")]
    cpu = KeypointDetector(default_cfg(device="cpu"))
    for n, c in saved:
        assert list(c["model"]) == want_keys and c["iter_per_epoch"] == 3 and "mf_loss_scale" not in c
        ref = torch.optim.AdamW(solver.get_model_params(cpu, main_run["cfg"]), lr=3e-4, betas=(0.9, 0.99))
        ref.load_state_dict(c["optimizer"])
        assert int(float(next(iter(c["optimizer"]["state"].values()))["step"])) == c["iteration"]
    for name in ("model_checkpoint", "model_final", "model_moderate_best_soft"):
        assert os.path.isfile(os.path.join(main_run["out"], name + ".pth"))


def test_evaluation_between_captured_steps_leaves_training_state_unchanged(main_run):
    assert [it for it, _, _ in main_run["states"]] == [10, 20]
    for it, (a, na), (b, nb) in main_run["states"]:
        assert na == nb == it
        assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b)), it
    assert main_run["trainer"]._graph is not None and main_run["trainer"].optimizer.skipped_steps() == 0
    assert main_run["trainer"].optimizer.step_count == 25


def test_warmup_lr_follows_the_reference(kitti, tmp_path):
    cfg = run_cfg(tmp_path, max_iter=9, steps=(7,), warmup=True)
    cfg.SOLVER.EVAL_INTERVAL = cfg.SOLVER.SAVE_CHECKPOINT_INTERVAL = 100
    trainer, _, _ = run(cfg, make_model(cfg), {"iteration": 0, "iter_per_epoch": 3, "root": kitti})
    ev = events(os.path.join(cfg.OUTPUT_DIR, "writer", cfg.START_TIME))
    assert [ev["stat/lr"][i] for i in range(1, 10)] == [np.float32(v) for v in reference_lrs(cfg, 9)]


def test_resume_from_iteration_10_equals_an_uninterrupted_run(kitti, tmp_path, monkeypatch):
    monkeypatch.setenv("MF_LOSS_SCALE", "dynamic")
    cfg = run_cfg(tmp_path / "a", max_iter=20)
    os.makedirs(cfg.OUTPUT_DIR)
    _, ck_a, _ = run(cfg, make_model(cfg), {"iteration": 0, "iter_per_epoch": 3, "root": kitti})
    at10 = [b for n, b in ck_a.saved if n == "model_checkpoint"][0]
    cfg_b = run_cfg(tmp_path / "b", max_iter=20)
    os.makedirs(cfg_b.OUTPUT_DIR)
    model = make_model(cfg_b, seed=1)
    opt = solver.build_optimizer(model, cfg_b)
    sched, _ = solver.build_scheduler(opt, cfg_b.SOLVER)
    ck_b = Checkpointer(model, opt, sched, cfg_b.OUTPUT_DIR)
    arguments = {"iteration": 0, "iter_per_epoch": 3}
    arguments.update(ck_b.load(at10))                     # tools/plain_train_net.py:train()
    assert arguments["iteration"] == 10 and "mf_loss_scale" in arguments
    # the drop-in restarts the data stream at position 0, as the reference does; fed the stream the uninterrupted run
    # trained on, it must reach the same state
    run(cfg_b, model, dict(arguments, root=kitti), skip=10, optimizer=opt, scheduler=sched, ckpt=ck_b, guard={20})
    a20 = torch.load(io.BytesIO([b for n, b in ck_a.saved if n == "model_checkpoint"][1]), weights_only=False)
    b20 = torch.load(io.BytesIO([b for n, b in ck_b.saved if n == "model_checkpoint"][0]), weights_only=False)
    assert a20["iteration"] == b20["iteration"] == 20
    steps = lambda c: {int(float(s["step"])) for s in c["optimizer"]["state"].values()}
    assert steps(a20) == steps(b20) and len(steps(a20)) == 1         # updates applied: skipped steps left out
    assert a20["optimizer"]["param_groups"][0]["lr"] == b20["optimizer"]["param_groups"][0]["lr"]
    assert a20["scheduler"] == b20["scheduler"]
    assert a20["mf_loss_scale"] == b20["mf_loss_scale"]


def test_plain_train_net_sequence_with_pretrained_weights(kitti, tmp_path):
    """tools/plain_train_net.py:train() restated: EVAL_AND_SAVE_EPOCH's interval rule over runs/monoflex.yaml's SOLVER
    settings (MAX_EPOCHS and DECAY_EPOCH_STEPS shortened), build_optimizer, build_scheduler(total_iters_each_epoch=...),
    arguments = {iteration: 0, iter_per_epoch}, MODEL.PRETRAIN from a stand-in cached ImageNet file.

    `fc` is outside the forward, so the reference's autograd leaves its gradient None and AdamW skips it. Here every
    parameter's .grad is a view of the fused optimiser's gradient arena (solver.ParamArena), so it cannot be None: the
    equivalent is that the backward never writes it (not in last_grad_names, the view stays all zero) and the optimiser
    marks it unused, so the update skips it and fc stays bit-identical."""
    old = torch.hub.get_dir()
    torch.hub.set_dir(str(tmp_path / "hub"))
    try:
        path = os.path.join(torch.hub.get_dir(), "checkpoints", "dla34-ba72cf86.pth")
        os.makedirs(os.path.dirname(path))
        fake = syn.dla34_imagenet_weights(int(GOLDEN["seed"]))
        torch.save(fake, path)
        cfg = run_cfg(tmp_path)
        cfg.MODEL.PRETRAIN = True
        s = cfg.SOLVER                                            # runs/monoflex.yaml
        s.OPTIMIZER, s.BASE_LR, s.WEIGHT_DECAY, s.LR_WARMUP, s.WARMUP_STEPS, s.LR_DECAY = "adamw", 3e-4, 1e-5, False, 2000, 0.1
        s.EVAL_AND_SAVE_EPOCH, s.EVAL_EPOCH_INTERVAL, s.SAVE_CHECKPOINT_EPOCH_INTERVAL = True, 1, 2
        s.MAX_EPOCHS, s.DECAY_EPOCH_STEPS, s.WARMUP_EPOCH = 4, [2, 3], 1
        model = KeypointDetector(cfg)
        heads = {k: v for k, v in syn.make_state_dict(seed=0).items() if not k.startswith("backbone.base.")}
        model.load_state_dict(heads, strict=False)
        model = model.cuda()
        fc0 = (model.backbone.base.fc.weight.detach().clone(), model.backbone.base.fc.bias.detach().clone())
        base0 = model.backbone.base.level5.tree1.conv1.weight.detach().clone()
        data_loader = L.KittiTrainLoader(cfg, kitti)
        data_loaders_val = L.KittiEvalLoader(cfg, kitti)
        total_iters_each_epoch = len(data_loader.dataset) // cfg.SOLVER.IMS_PER_BATCH
        assert total_iters_each_epoch == 3
        s.MAX_ITERATION = s.MAX_EPOCHS * total_iters_each_epoch
        s.SAVE_CHECKPOINT_INTERVAL = total_iters_each_epoch * s.SAVE_CHECKPOINT_EPOCH_INTERVAL
        s.EVAL_INTERVAL = total_iters_each_epoch * s.EVAL_EPOCH_INTERVAL
        s.STEPS = [total_iters_each_epoch * x for x in s.DECAY_EPOCH_STEPS]
        s.WARMUP_STEPS = s.WARMUP_EPOCH * total_iters_each_epoch
        optimizer = solver.build_optimizer(model, cfg)
        scheduler, warmup_scheduler = solver.build_scheduler(optimizer, total_iters_each_epoch=total_iters_each_epoch,
                                                             optim_cfg=cfg.SOLVER)
        arguments = {"iteration": 0, "iter_per_epoch": total_iters_each_epoch}
        checkpointer = Checkpointer(model, optimizer, scheduler, cfg.OUTPUT_DIR)
        handler = _ListHandler()
        logging.getLogger("monoflex").addHandler(handler)
        logging.getLogger("monoflex").setLevel(logging.INFO)
        try:
            TR.do_train(cfg, False, model, data_loader, data_loaders_val, optimizer, scheduler, warmup_scheduler,
                        checkpointer, torch.device("cuda"), arguments)
        finally:
            logging.getLogger("monoflex").removeHandler(handler)
    finally:
        torch.hub.set_dir(old)
    msgs = [r.getMessage() for r in handler.records if r.name == "monoflex.trainer"]
    print("\n".join(msgs))
    assert arguments["iteration"] == 12
    assert [m for m in msgs if m.startswith("epoch = ") and "evaluate" in m] == [
        "epoch = %d, evaluate model on validation set with depth soft" % e for e in (1, 2, 3, 4)]
    assert [m.split("iter: ")[1].split(" ")[0] for m in msgs if m.startswith("eta")] == ["10", "12"]
    names = [n for n, _ in checkpointer.saved]
    # checkpoints at 6 and 12, model_final at 12 before that iteration's evaluation, a best model at every evaluation
    # whose AP is not below the best so far
    assert [n for n in names if n != "model_moderate_best_soft"] == ["model_checkpoint"] * 2 + ["model_final"], names
    assert names[0] == "model_moderate_best_soft" and names.count("model_moderate_best_soft") >= 1
    ev = events(os.path.join(cfg.OUTPUT_DIR, "writer", cfg.START_TIME))
    assert sorted(ev["stat/lr"]) == list(range(1, 13)) and sorted(ev["eval_soft_0.70/Car_3d_0.70/moderate"]) == [1, 2, 3, 4]
    last = torch.load(io.BytesIO(checkpointer.saved[-1][1]), weights_only=False)["model"]
    assert list(last) == GOLDEN["model_keys"].tolist()
    fc = model.backbone.base.fc
    assert "backbone.base.fc.weight" not in model.last_grad_names and "backbone.base.fc.bias" not in model.last_grad_names
    assert torch.equal(fc.weight.detach(), fc0[0]) and torch.equal(fc.bias.detach(), fc0[1])
    assert not fc.weight.grad.any() and not fc.bias.grad.any()
    arena = optimizer.arena
    skipped = {id(p) for p, skip in zip(arena.tensors, optimizer._skip) if skip}
    assert id(fc.weight) in skipped and id(fc.bias) in skipped
    assert not torch.equal(model.backbone.base.level5.tree1.conv1.weight.detach(), base0)     # the pretrained base trains


def test_params_list_batches_train_without_host_synchronisation(main_run, kitti, tmp_path, monkeypatch):
    """a batch without `encoded`: the ParamsList targets are prepared and loaded into the captured step on every replay,
    still without a host synchronisation between boundaries, and the losses follow the encoded run's on the same batches"""
    cfg = run_cfg(tmp_path, max_iter=14)
    rec = Recorder(monkeypatch)
    trainer, ckpt, args = run(cfg, make_model(cfg), {"iteration": 0, "iter_per_epoch": 3, "root": kitti}, guard={10, 14},
                              params_lists=True)
    assert args["iteration"] == 14 and trainer._graph is not None and len(rec.logs) == 14
    assert [n for n, _ in ckpt.saved if n != "model_moderate_best_soft"] == ["model_checkpoint", "model_final"]
    for i, (a, b) in enumerate(zip(main_run["logs"][:6], rec.logs)):
        ta, tb = (sum(v for k, v in l.items() if k.endswith("_loss")) for l in (a, b))
        assert np.isfinite(tb) and abs(ta - tb) <= (0.03 if i <= 2 else 0.25) * abs(ta), (i, ta, tb)


def test_two_ranks_under_distributed_data_parallel():
    """world >= 2 only (skipped on a 1-GPU box): the reference's main() path - DistributedDataParallel around the model,
    the optimiser built from the wrapped model - through do_train with a checkpoint and an evaluation inside: identical
    replicas, checkpoints and event files from rank 0 only, every rank at max_iter (tools/do_train_two_rank_check.py)"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29553", os.path.join(root, "tools", "do_train_two_rank_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert '"ok": true' in r.stdout
