"""CPU: the checkpoint file round-trips; a checkpoint of another spec, setup or config is refused before anything reaches
the device; fit's schedule (train.lua:221-361) with a recording trainer against a table worked by hand: the decay
epochs, the switch to phase 2 with its step / decay overrides, the snapshots and `final`, and a resume from a snapshot."""
import os
import types

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200._lib import CTrainConfig
from multipathnet_b200.train import Trainer


class _Recorder:
    """a Trainer and its BatchProviderROI as fit sees them: the calls are recorded, a step's losses are its sample index"""

    def __init__(self, phase2=True):
        self.model = types.SimpleNamespace(spec=models.vgg16_fast_rcnn(21, seed=None, width_div=16, fc_dim=64))
        self.cfg = CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 555)
        self.phase2, self.steps, self.calls, self.bbox_regr = phase2, 0, [], None

    # the provider
    def setup_data(self):
        self.calls.append(("setup_data",))
        self.bbox_regr = (np.arange(4, dtype=np.float32), np.ones(4, np.float32))

    def sample(self, k):
        return k

    def sample_integral(self, k):
        return 1000 + k

    # the trainer
    def step_batch(self, k):
        self.calls.append(("step", k))
        self.steps += 1
        return float(k), float(k) / 2, float(k) / 4

    def decay(self, f):
        self.calls.append(("decay", f))
        self.cfg.lr = float(np.float32(self.cfg.lr) * np.float32(f))

    def set_phase2(self, lr):
        self.calls.append(("phase2", lr))
        if lr is not None:
            self.cfg.lr = lr

    def set_lr(self, lr):
        self.calls.append(("set_lr", lr))
        self.cfg.lr = lr

    def _zero_buffers(self):
        self.calls.append(("zero_buffers",))

    def state_dict(self):
        self.calls.append(("save", self.steps))
        return {"fingerprint": {"name": "rec"}, "config": {}, "state": {"steps": self.steps, "lr": self.cfg.lr},
                "tensors": {3: (np.full((2, 2), self.steps, np.float32), np.zeros((2, 2), np.float32))}}

    def load_state_dict(self, d):
        self.calls.append(("load", d["state"]["steps"]))
        self.steps, self.cfg.lr = d["state"]["steps"], d["state"]["lr"]

    def weights(self):
        return self.model.spec.weights


OPT = dict(nEpochs=6, epochSize=2, step=2, decay=0.1, snapshot=3, phase2_epoch=4, phase2_learningRate=0.01, phase2_step=1,
           phase2_decay=0.5)
f32 = lambda x: float(np.float32(x))
LR = [f32(1e-3), f32(np.float32(1e-3) * np.float32(0.1))]
LR += [LR[1], f32(np.float32(0.01) * np.float32(0.5))]
LR += [f32(np.float32(LR[3]) * np.float32(0.5))]
LR += [f32(np.float32(LR[4]) * np.float32(0.5))]
# train.lua's hooks for OPT by hand: (epoch, the calls of the epoch, learningRate and decay logged at its end, snapshot)
TABLE = [(1, [("step", 0), ("step", 1)], LR[0], 0.1, False),
         (2, [("step", 2), ("step", 3), ("decay", 0.1)], LR[1], 0.1, False),                    # 2 % step == 0
         (3, [("step", 4), ("step", 5), ("save", 6)], LR[2], 0.1, True),                          # snapshot
         (4, [("phase2", 0.01), ("step", 6), ("step", 7), ("decay", 0.5)], LR[3], 0.5, False),  # the switch: step 1, decay 0.5
         (5, [("step", 8), ("step", 9), ("decay", 0.5)], LR[4], 0.5, False),
         (6, [("step", 10), ("step", 11), ("decay", 0.5), ("save", 12)], LR[5], 0.5, True)]


def _flat(rows):
    return [c for _, cs, _, _, _ in rows for c in cs]


def test_schedule_follows_train_lua(tmp_path):
    rec, lines = _Recorder(), []
    stats = np.arange(12, dtype=np.float64) / 100
    r = mpn.fit(rec, rec, dict(OPT, save_folder=str(tmp_path)), validate_fn=lambda m: stats, log=lines.append)
    assert rec.calls == [("setup_data",)] + _flat(TABLE) + [("save", 12)]
    want = []
    for epoch, _, lr, decay, snap in TABLE:
        want.append((epoch, lr, decay, 0.0, 0.0))
        if snap:
            want.append((epoch, lr, decay, 0.01, 0.0))            # voc_metric = res[2], coco_metric = res[1]
    want.append((7, LR[5], 0.5, 0.01, 0.0))                       # onEnd logs state.epoch + 1
    assert [(x["epoch"], x["learningRate"], x["decay"], x["voc_metric"], x["coco_metric"]) for x in r] == want
    assert r[0]["train_loss"] == 0.5 and r[0]["primary_loss"] == 0.25 and r[0]["bboxregr_loss"] == 0.125
    assert len(lines) == len(r) and all(s.startswith("json_stats: {") for s in lines)
    assert set(r[0]) == {"epoch", "learningRate", "decay", "train_loss", "primary_loss", "bboxregr_loss", "voc_metric", "coco_metric",
                         "train_time"}
    assert sorted(os.listdir(tmp_path)) == ["checkpoint_3.npz", "checkpoint_6.npz", "checkpoint_final.npz", "model_3.t7", "model_6.t7",
                                            "model_final.t7"]
    ck = mpn.load_checkpoint(str(tmp_path / "checkpoint_3.npz"))
    assert ck["extra"] == {"epoch": 3, "step": 2, "decay": 0.1, "bbox_mean": [0.0, 1.0, 2.0, 3.0], "bbox_std": [1.0] * 4}
    assert mpn.load_checkpoint(str(tmp_path / "checkpoint_6.npz"))["extra"]["step"] == 1           # phase2_step in force
    # resuming from epoch 3's snapshot runs epochs 4 .. 6 as the uninterrupted run did
    res = _Recorder()
    r2 = mpn.fit(res, res, dict(OPT, resume=str(tmp_path / "checkpoint_3.npz")), log=lambda s: None)
    assert res.calls == [("load", 6)] + [c for c in _flat(TABLE[3:]) if c[0] != "save"]
    assert [x["learningRate"] for x in r2] == LR[3:] and res.bbox_regr[0].tolist() == [0.0, 1.0, 2.0, 3.0]
    # integral: the threshold set is drawn per step; no save_folder: nothing written; a model without phase 2 still takes
    # the phase-2 rate and zeroed buffers (train.lua:244-259)
    plain = _Recorder(phase2=False)
    mpn.fit(plain, plain, dict(OPT, nEpochs=4, integral=True), log=lambda s: None)
    assert plain.calls[1:3] == [("step", 1000), ("step", 1001)]
    assert ("set_lr", 0.01) in plain.calls and ("zero_buffers",) in plain.calls and not any(c[0] == "save" for c in plain.calls)


def test_bad_options_are_refused():
    rec = _Recorder()
    with pytest.raises(mpn.MpnError, match="unknown options"):
        mpn.fit(rec, rec, {"nEpoch": 3})
    with pytest.raises(mpn.MpnError, match="epochSize"):
        mpn.fit(rec, rec, {"epochSize": 0})


def test_checkpoint_file_round_trips(tmp_path):
    rec = _Recorder()
    rec.steps = 5
    path = str(tmp_path / "c.npz")
    mpn.save_checkpoint(path, rec, epoch=2, step=3, decay=0.1, bbox_mean=np.array([0.5, 0, 0, 0], np.float32))
    d = mpn.load_checkpoint(path)
    want = rec.state_dict()
    assert d["fingerprint"] == want["fingerprint"] and d["state"] == want["state"] and d["config"] == want["config"]
    assert d["extra"] == {"epoch": 2, "step": 3, "decay": 0.1, "bbox_mean": [0.5, 0.0, 0.0, 0.0]}
    assert list(d["tensors"]) == [3]
    for a, b in zip(d["tensors"][3], want["tensors"][3]):
        assert a.dtype == np.float32 and np.array_equal(a, b)


def _offline_trainer(spec, **cfg):
    """a Trainer as its constructor leaves it for load_state_dict's checks, without a device (they refuse before any call)"""
    t = Trainer.__new__(Trainer)
    t.model = types.SimpleNamespace(spec=spec)
    c = dict(lr=1e-3, momentum=0.9, dampening=0.0, weight_decay=5e-4, dropout=0.5, bbox_regression=1.0, seed=555)
    c.update(cfg)
    t.cfg = CTrainConfig(*c.values())
    t.trunk_from, t.phase2, t.phase = 0, False, 1
    t.trained = sorted(t._trained_indices())
    t._fingerprint = {"name": spec.name, "shapes": [list(np.shape(w)) for w in spec.weights], "trained": list(t.trained), "trunk_from": 0,
                      "phase2_from": 0, "integral_k": len(spec.cls_heads), "fixed_bn": sorted(spec.fixed_bn)}
    return t


def test_a_mismatched_checkpoint_is_refused_without_a_gpu():
    spec = models.vgg16_fast_rcnn(21, seed=None, width_div=16, fc_dim=64)
    a = _offline_trainer(spec)
    d = {"fingerprint": dict(a._fingerprint), "config": {k: getattr(a.cfg, k) for k, _ in CTrainConfig._fields_},
         "state": {"step": 0, "lr": 1e-3, "head": 0, "last_head": 0, "phase2": 0, "steps": 0}, "tensors": {}}
    for other, what in ((models.vgg16_fast_rcnn(21, seed=None, width_div=8, fc_dim=64), "name"),
                        (models.vgg16_fast_rcnn(21, seed=None, width_div=16, fc_dim=64, integral_k=3), "shapes"),
                        (models.vgg16_multipathnet(21, seed=None, width_div=16, fc_dim=64), "name")):
        with pytest.raises(mpn.MpnError, match=what):
            _offline_trainer(other).load_state_dict(d)
    with pytest.raises(mpn.MpnError, match="config seed"):
        _offline_trainer(spec, seed=7).load_state_dict(d)
    with pytest.raises(mpn.MpnError, match="config dropout"):
        _offline_trainer(spec, dropout=0.0).load_state_dict(d)
    with pytest.raises(mpn.MpnError, match="phase2=True"):
        a.load_state_dict(dict(d, state=dict(d["state"], phase2=1)))
    with pytest.raises(mpn.MpnError, match="holds tensors"):
        a.load_state_dict(d)
    wrong = {i: (np.zeros(3, np.float32), np.zeros(3, np.float32)) for i in a.trained}
    with pytest.raises(mpn.MpnError, match="tensor"):
        a.load_state_dict(dict(d, tensors=wrong))
