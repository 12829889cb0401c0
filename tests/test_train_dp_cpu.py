"""CPU: the host side of data-parallel training (Trainer(replicas=...)): the sharding rule of train.lua's train_nGPU, the
refusals that need no device, and that a checkpoint carries no replica count, so it loads into a trainer with any."""
import dataclasses
import types

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200._lib import CTrainConfig
from multipathnet_b200.train import Trainer, check_replicas, shard_plan


def test_shards_are_contiguous_image_ranges_in_batch_order():
    assert shard_plan([3, 5, 2, 7], 1) == [(0, 4, 0, 17)]
    assert shard_plan([3, 5, 2, 7], 2) == [(0, 2, 0, 8), (2, 4, 8, 17)]
    assert shard_plan([3, 5, 2, 7], 4) == [(0, 1, 0, 3), (1, 2, 3, 8), (2, 3, 8, 10), (3, 4, 10, 17)]
    assert shard_plan([4, 0, 1, 6, 0, 2], 3) == [(0, 2, 0, 4), (2, 4, 4, 11), (4, 6, 11, 13)]   # an image without rows is fine


@pytest.mark.parametrize("counts,k,match", [
    ([3, 5, 2], 2, "images_per_batch must be a multiple of train_nGPU: 3 images over 2 replicas"),
    ([3, 5], 4, "images_per_batch must be a multiple of train_nGPU"),
    ([], 1, "images_per_batch must be a multiple of train_nGPU"),
    ([3, 5, 0, 0], 2, r"replica 1's images 2..3 have no ROIs"),
    ([0, 5], 2, r"replica 0's images 0..0 have no ROIs"),
    ([1, 2], 0, "at least one"),
])
def test_the_sharding_refusals(counts, k, match):
    with pytest.raises(mpn.MpnError, match=match):
        shard_plan(counts, k)


def _spec(seed=None, **kw):
    return models.vgg16_fast_rcnn(21, seed=seed, width_div=16, fc_dim=64, **kw)


def test_replicas_of_another_spec_or_the_same_model_twice_are_refused():
    spec = _spec(3)
    m0 = types.SimpleNamespace(spec=spec)
    check_replicas(m0, [types.SimpleNamespace(spec=spec), types.SimpleNamespace(spec=dataclasses.replace(spec))])
    copy = dataclasses.replace(spec, weights=[np.array(w, copy=True) for w in spec.weights])
    check_replicas(m0, [types.SimpleNamespace(spec=copy)])                     # equal weights in other arrays
    with pytest.raises(mpn.MpnError, match="replica 1 is the same Model as replica 0"):
        check_replicas(m0, [m0])
    r1 = types.SimpleNamespace(spec=spec)
    with pytest.raises(mpn.MpnError, match="replica 2 is the same Model as replica 1"):
        check_replicas(m0, [r1, r1])
    bumped = [np.array(w, copy=True) for w in spec.weights]
    bumped[-1].flat[0] += 1
    for other in (_spec(4), _spec(3, integral_k=2), dataclasses.replace(spec, weights=bumped),
                  dataclasses.replace(spec, bbox_mean=(0.1, 0.0, 0.0, 0.0)), models.vgg16_multipathnet(21, seed=3, width_div=16, fc_dim=64)):
        with pytest.raises(mpn.MpnError, match="replica 1 has another spec"):
            check_replicas(m0, [types.SimpleNamespace(spec=other)])


def _offline(spec, n_models):
    """a Trainer as its constructor leaves it, over n_models replicas, with the library calls recorded instead of made"""
    t = Trainer.__new__(Trainer)
    t.model = types.SimpleNamespace(spec=spec, name="replica 0")
    t.models = [t.model] + [types.SimpleNamespace(spec=spec, name=f"replica {j}") for j in range(1, n_models)]
    t.cfg = CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 555)
    t.trunk_from, t.phase2, t.phase = 0, False, 1
    t.trained = sorted(t._trained_indices())
    t._fingerprint = {"name": spec.name, "shapes": [list(np.shape(w)) for w in spec.weights], "trained": list(t.trained), "trunk_from": 0,
                      "phase2_from": 0, "integral_k": len(spec.cls_heads), "fixed_bn": sorted(spec.fixed_bn)}
    t.calls = []

    def each(fn, *args):
        for m in t.models:
            t.calls.append((m.name, fn))
    t._each = each
    return t


def test_a_checkpoint_loads_into_any_number_of_replicas():
    spec = _spec()
    one, two, four = _offline(spec, 1), _offline(spec, 2), _offline(spec, 4)
    assert one._fingerprint == two._fingerprint == four._fingerprint
    d = {"fingerprint": dict(one._fingerprint), "config": {k: getattr(one.cfg, k) for k, _ in CTrainConfig._fields_},
         "state": {"step": 3, "lr": 1e-3, "head": 0, "last_head": 0, "phase2": 0, "steps": 3},
         "tensors": {i: (np.zeros(spec.weights[i].shape, np.float32),) * 2 for i in one.trained}}
    for t, n in ((one, 1), (two, 2), (four, 4)):
        t.load_state_dict(d)
        assert t.steps == 3
        # every replica takes the state and every tensor's master and buffer
        for j in range(n):
            mine = [fn for who, fn in t.calls if who == f"replica {j}"]
            assert mine.count("mpn_model_train_set_state") == 1
            assert mine.count("mpn_model_train_set") == 2 * len(t.trained)
    # a mismatched checkpoint is refused the same way whatever the replica count, before any call
    bad = dict(d, config=dict(d["config"], seed=7))
    for t in (_offline(spec, 1), _offline(spec, 2)):
        with pytest.raises(mpn.MpnError, match="config seed"):
            t.load_state_dict(bad)
        assert t.calls == []
