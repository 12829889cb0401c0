"""train.lua's loop around the step (train.lua:188-361): epochs of `epochSize` steps, the learning-rate schedule, the
switch to MultiPathNet's phase 2, snapshots, validation and resuming from a snapshot.

`fit` drives a `Trainer` with a `BatchProviderROI` through train.lua's hooks: onStartEpoch (the phase-2 switch at
`phase2_epoch`), one sampled minibatch per step, onEndEpoch (lr and momentum buffers x `decay` every `step` epochs, a
`json_stats:` line, and every `snapshot` epochs a checkpoint and a validation) and onEnd (the `final` checkpoint and
validation). The minibatch of a step is drawn for its global index ((epoch - 1) * epochSize + n), and a checkpoint holds
the whole device state of the trainer, so a run resumed from a snapshot trains exactly as the uninterrupted run.

`validate` is Tester_FRCNN:test (Tester_FRCNN.lua:141-187) over a test set held in memory, scored by the device COCO
evaluator; it runs on the training model's own handle.
"""
from __future__ import annotations

import dataclasses
import json
import os
import time
from typing import Callable, Dict, Optional, Sequence, Union

import numpy as np

from . import coco_eval, t7, utils
from ._lib import MpnError
from .modules import ImageTransformer
from .tester import Tester
from .train import load_checkpoint, save_checkpoint

# train.lua's defaults of the options fit reads (train.lua:23-81)
DEFAULTS = dict(nEpochs=400, epochSize=100, step=300, decay=0.1, snapshot=100, phase2_epoch=-1, phase2_learningRate=-1,
                phase2_step=-1, phase2_decay=-1, integral=False, save_folder="", resume="")


def validate(model, transformer: Union[str, ImageTransformer], images: Union[Sequence[np.ndarray], Callable[[int], np.ndarray]], proposals: Sequence[np.ndarray],
             image_ids: Sequence[int], gt: Union[Dict, coco_eval.CocoGroundTruth], scale: float = 600, max_size: float = 1000,
             test_num_per_image: int = 100, category_ids: Optional[Sequence[int]] = None, images_per_batch: int = 1,
             **tester_opts) -> np.ndarray:
    """Tester_FRCNN:test on n test images: per image Tester.testOne (images[i] or images(i): the raw 3 x H x W image,
    proposals[i]: its N_i x 4 boxes), then keepTopKPerImage(test_num_per_image), transposeBoxes, utils.coco_results and
    coco_eval.coco_evaluate -> the 12 COCO stats (stats[0] = train.lua's coco_metric, stats[1] its voc_metric).
    transformer: "ross" | "imagenet" (ModelSpec.transformer) or an ImageTransformer.
    category_ids: the category of each foreground class (default: gt's categories in ascending id order). An image
    without proposals has no detections. images_per_batch > 1: Tester.testMany over that many consecutive images at a
    time (the same bits as image by image). tester_opts go to Tester (nms_thresh, bbox_voting, ...)."""
    if int(images_per_batch) < 1:
        raise MpnError(f"validate: images_per_batch must be >= 1, got {images_per_batch}")
    g = gt if isinstance(gt, coco_eval.CocoGroundTruth) else coco_eval.CocoGroundTruth.from_dict(gt)
    tf = ImageTransformer(transformer) if isinstance(transformer, str) else transformer
    tester = Tester(model, tf, [scale], max_size, **tester_opts)
    nfg = model.spec.num_classes - 1
    aboxes_t = []
    step = int(images_per_batch)

    def get(i):
        return images(i) if callable(images) else images[i]
    for i0 in range(0, len(proposals), step):
        idx = range(i0, min(i0 + step, len(proposals)))
        boxes = {i: np.asarray(proposals[i], np.float32).reshape(-1, 4) for i in idx}
        live = [i for i in idx if boxes[i].shape[0]]
        if step == 1:
            found = {i: tester.testOne(get(i), boxes[i]) for i in live}
        else:
            found = dict(zip(live, tester.testMany([get(i) for i in live], [boxes[i] for i in live]))) if live else {}
        for i in idx:
            aboxes_t.append(found[i] if i in found else [np.zeros((0, 5), np.float32) for _ in range(nfg)])
    aboxes = tester.transposeBoxes(tester.keepTopKPerImage(aboxes_t, test_num_per_image))
    cats = list(g.cat_ids) if category_ids is None else list(category_ids)
    if len(cats) != nfg:
        raise MpnError(f"validate: {len(cats)} categories for the model's {nfg} foreground classes")
    return coco_eval.coco_evaluate(model.ctx, g, utils.coco_results(aboxes, list(image_ids), cats))["stats"]


def _save(trainer, folder: str, tag, extra: dict) -> None:
    """train.lua's save: the checkpoint (model + optim state) and, where t7.model_to_t7 exports the graph, model_<tag>.t7"""
    save_checkpoint(os.path.join(folder, f"checkpoint_{tag}.npz"), trainer, **extra)
    try:
        graph = t7.model_to_t7(dataclasses.replace(trainer.model.spec, weights=trainer.weights()))
    except NotImplementedError:
        return
    t7.save(os.path.join(folder, f"model_{tag}.t7"), graph)


def fit(trainer, provider, opt: Optional[Dict] = None, validate_fn: Optional[Callable] = None, log: Callable[[str], None] = print):
    """Run train.lua's schedule. opt: train.lua's options (DEFAULTS for those not given): nEpochs, epochSize, step,
    decay, snapshot, phase2_epoch, phase2_learningRate, phase2_step, phase2_decay (< 0: unset), integral (sample the
    threshold set per step), save_folder (snapshots are written there; '' writes none), resume (a checkpoint file to
    continue from). validate_fn(model) -> the 12 COCO stats (e.g. a `validate` bound to a test set); None skips
    validation. Returns the json_stats records logged, in order."""
    o = dict(DEFAULTS)
    unknown = set(opt or {}) - set(DEFAULTS)
    if unknown:
        raise MpnError(f"fit: unknown options {sorted(unknown)}")
    o.update(opt or {})
    n_epochs, epoch_size, snapshot = int(o["nEpochs"]), int(o["epochSize"]), int(o["snapshot"])
    if n_epochs < 0 or epoch_size < 1 or snapshot < 1 or int(o["step"]) < 1:
        raise MpnError("fit: nEpochs >= 0, epochSize >= 1, snapshot >= 1 and step >= 1")
    folder = str(o["save_folder"])
    if folder:
        os.makedirs(folder, exist_ok=True)
    state = {"step": int(o["step"]), "decay": float(o["decay"])}
    start = 0
    if o["resume"]:                                              # train.lua:226-234
        d = load_checkpoint(str(o["resume"]))
        trainer.load_state_dict(d)
        ex = d["extra"]
        start, state["step"], state["decay"] = int(ex["epoch"]), int(ex["step"]), float(ex["decay"])
        provider.bbox_regr = (np.asarray(ex["bbox_mean"], np.float32), np.asarray(ex["bbox_std"], np.float32))
    elif provider.bbox_regr is None:
        provider.setup_data()
    records = []
    meters = {}

    def emit(epoch, voc=0.0, coco=0.0):
        n = max(meters["n"], 1)
        r = {"epoch": epoch, "learningRate": float(trainer.cfg.lr), "decay": state["decay"], "train_loss": meters["loss"] / n,
             "primary_loss": meters["cls"] / n, "bboxregr_loss": meters["bbox"] / n, "voc_metric": float(voc),
             "coco_metric": float(coco), "train_time": meters["time"]}
        records.append(r)
        log("json_stats: " + json.dumps(r))

    def snapshot_and_validate(epoch, tag):
        if folder:
            mean, std = provider.bbox_regr
            _save(trainer, folder, tag, {"epoch": epoch, "step": state["step"], "decay": state["decay"],
                                         "bbox_mean": np.asarray(mean).tolist(), "bbox_std": np.asarray(std).tolist()})
        if validate_fn is not None:
            res = validate_fn(trainer.model)
            emit(epoch if tag != "final" else epoch + 1, voc=res[1], coco=res[0])

    for epoch in range(start + 1, n_epochs + 1):
        if epoch == int(o["phase2_epoch"]):                      # onStartEpoch, train.lua:237-269
            lr2 = float(o["phase2_learningRate"])
            if trainer.phase2:
                trainer.set_phase2(lr2 if lr2 >= 0 else None)
            elif lr2 >= 0:
                trainer.set_lr(lr2)
                trainer._zero_buffers()
            if int(o["phase2_step"]) >= 0:
                state["step"] = int(o["phase2_step"])
            if float(o["phase2_decay"]) >= 0:
                state["decay"] = float(o["phase2_decay"])
            if state["step"] < 1:
                raise MpnError("fit: phase2_step must be >= 1")
        meters = {"n": 0, "loss": 0.0, "cls": 0.0, "bbox": 0.0}
        t0 = time.perf_counter()
        for n in range(epoch_size):
            k = (epoch - 1) * epoch_size + n
            batch = provider.sample_integral(k) if o["integral"] else provider.sample(k)
            loss, cls, bbox = trainer.step_batch(batch)
            meters["n"] += 1; meters["loss"] += loss; meters["cls"] += cls; meters["bbox"] += bbox
        meters["time"] = time.perf_counter() - t0
        if epoch % state["step"] == 0:                           # onEndEpoch, train.lua:319-346
            trainer.decay(state["decay"])
        emit(epoch)
        if epoch % snapshot == 0:
            snapshot_and_validate(epoch, epoch)
    if meters:                                                   # onEnd, train.lua:348-360 (logged as epoch nEpochs + 1)
        snapshot_and_validate(n_epochs, "final")
    return records
