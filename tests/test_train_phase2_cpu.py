"""CPU: MultiPathNet's phase 2. Which trunk layer the builders and the t7 reader start it from (spec.phase2_from), the
library's acceptances and refusals (mpn_train_check, phase2 = 1), and the numpy rules the kernel-level GPU test restates:
the foveal region of a ROI, the normalisation's (a, b) and the in-order gather, on hand-made inputs with known answers."""
import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, t7
from multipathnet_b200.train import check_spec
from _train_phase2_ref import bin_windows, gather, norm_ab, region_box, roi_argmax
from test_t7_cpu import _roundtrip
from test_t7_graphs_cpu import O, _conv, _ident, _pool, _relu, _seq, _tiny_multipathnet


def test_builders_phase2_from():
    s = models.vgg16_multipathnet(81, seed=None)
    assert s.phase2_from == 6 and s.trunk_train_from == 0
    L = s.trunk_layers[6]
    assert L.kind == mpn._lib.MPN_LAYER_CONV and L.cin == 128 and L.cout == 256          # conv3_1
    assert models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256, integral_k=3).phase2_from == 6
    for other in (models.vgg16_fast_rcnn(21, seed=None), models.resnet50_fast_rcnn(81, seed=None),
                  models.resnet18_fast_rcnn(81, seed=None, fixed_bn=True)):
        assert other.phase2_from == 0
    check_spec(s, phase2=True)
    check_spec(models.vgg16_multipathnet(21, seed=None, integral_k=6), integral=True, phase2=True)


def test_check_phase2_refusals():
    with pytest.raises(mpn.MpnError, match="phase2_from is 0"):
        check_spec(models.vgg16_fast_rcnn(21, seed=None), phase2=True)
    with pytest.raises(mpn.MpnError, match="fixed batch norm"):
        r = models.resnet18_fast_rcnn(81, seed=None, fixed_bn=True)
        r.phase2_from = r.trunk_train_from
        check_spec(r, phase2=True)
    with pytest.raises(mpn.MpnError, match="integral loss"):
        check_spec(models.vgg16_multipathnet(21, seed=None, integral_k=3), phase2=True)
    s = models.vgg16_multipathnet(81, seed=None)
    s.phase2_from = len(s.trunk_layers)
    with pytest.raises(mpn.MpnError, match="out of range"):
        check_spec(s, phase2=True)
    s = models.vgg16_multipathnet(81, seed=None)
    s.trunk_layers[8].stride = 2                                        # conv3_3, inside the range
    with pytest.raises(mpn.MpnError, match="3x3 / stride 1"):
        check_spec(s, phase2=True)
    s = models.vgg16_multipathnet(81, seed=None)
    s.phase2_from = 10                                                  # conv3_3's slot, pooled by two towers, stays frozen
    with pytest.raises(mpn.MpnError, match="every tower level must pool"):
        check_spec(s, phase2=True)
    s = models.vgg16_multipathnet(81, seed=None)
    s.towers[2].layers[0].kind = mpn._lib.MPN_LAYER_MAXPOOL
    with pytest.raises(mpn.MpnError, match="must start with a convolution of the pooled map"):
        check_spec(s, phase2=True)
    s = models.vgg16_multipathnet(81, seed=None)
    s.towers[1].layers[2].relu = 0
    s.towers[1].layers[2].kh = 3                                        # fc6 as a 3x3: not a per-ROI chain layer
    with pytest.raises(mpn.MpnError, match="every per-ROI layer"):
        check_spec(s, phase2=True)
    # trunk training without phase 2 keeps its refusal of MultiPathNet's trunk
    with pytest.raises(mpn.MpnError, match="exactly one tower"):
        check_spec(models.vgg16_multipathnet(81, seed=None), 6)


def _ten_plain(rng):
    """conv1_1 .. pool2 of a tiny VGG: the 10 plain modules disableFeatureBackprop(skip, 10) wraps"""
    return [_conv(rng, 3, 8, gain=1 / 8.0), _relu(), _conv(rng, 8, 8), _relu(), _pool(),
            _conv(rng, 8, 8), _relu(), _conv(rng, 8, 8), _relu(), _pool()]


def _deep_multipathnet(rng, phase):
    """_tiny_multipathnet with a skip trunk of 10 plain modules, then conv3 (conv, ReLU) before its conv4 branch.
    phase 1: the whole skip trunk under nn.NoBackprop (multipathnet.lua:60-62); phase 2: as vggSetPhase2_outer leaves it,
    nn.NoBackprop around the first 10 modules only (model_utils.lua:197-207)"""
    model = _tiny_multipathnet(rng)
    nb = model.modules[0].modules[0]
    dpt = nb.modules[0]
    skip = dpt.modules[0]
    tail = [_conv(rng, 8, 8), _relu()] + list(skip.modules[5:])
    if phase == 1:
        skip.fields["modules"] = _ten_plain(rng) + tail
    else:
        skip.fields["modules"] = [O("nn.NoBackprop", modules=[_seq(*_ten_plain(rng))])] + tail
        model.modules[0].fields["modules"][0] = dpt
    return model


def test_t7_reader_phase2_from():
    rng = np.random.default_rng(7)
    one = t7.model_from_t7(_roundtrip(_deep_multipathnet(rng, 1)))
    two = t7.model_from_t7(_roundtrip(_deep_multipathnet(rng, 2)))
    kinds = [L.kind for L in one.trunk_layers[:7]]
    assert kinds == [1, 1, 2, 1, 1, 2, 1] and [L.kind for L in two.trunk_layers] == [L.kind for L in one.trunk_layers]
    assert one.phase2_from == 6 and one.trunk_train_from == 0                        # conv1_1 .. pool2: 6 layers, ReLUs fused
    assert two.phase2_from == 6 and two.trunk_train_from == 6
    check_spec(one, phase2=True)
    check_spec(two, phase2=True)
    # five plain modules before the conv4 branch: the switch would wrap a branch, so there is no phase 2
    assert t7.model_from_t7(_roundtrip(_tiny_multipathnet(np.random.default_rng(1)))).phase2_from == 0
    # a non-plain module among the first 10 (a Dropout)
    m = _deep_multipathnet(np.random.default_rng(3), 1)
    skip = m.modules[0].modules[0].modules[0].modules[0]
    skip.modules[3] = O("nn.Dropout", p=0.5, v2=True, inplace=True)
    assert t7.model_from_t7(_roundtrip(m)).phase2_from == 0
    # single-tower graphs and the builders' exports
    assert t7.model_from_t7(_roundtrip(t7.model_to_t7(models.vgg16_fast_rcnn(21, seed=1, width_div=8, fc_dim=64)))).phase2_from == 0


def test_region_box_and_clipped_bins():
    box = (10.0, 20.0, 30.0, 60.0)                                      # w 20, h 40
    assert region_box(box, 0) == tuple(np.float32(v) for v in box)
    assert region_box(box, 1) == (np.float32(5.0), np.float32(10.0), np.float32(35.0), np.float32(70.0))
    assert region_box(box, 2) == (np.float32(0.0), np.float32(0.0), np.float32(40.0), np.float32(80.0))
    assert region_box(box, 3) == (np.float32(-20.0), np.float32(-40.0), np.float32(60.0), np.float32(120.0))
    wins = bin_windows(box, 3, 1.0 / 8, 2, 2, 2, 8, 6)                  # x4 leaves the 8 x 6 map at the top and left
    assert wins[0][0] == 0 and wins[0][2] == 0                          # clipped at 0
    assert all(he <= 8 and we <= 6 for _, he, _, we in wins)
    # an empty bin: a region entirely outside the map
    wins = bin_windows((200.0, 200.0, 210.0, 210.0), 0, 1.0 / 8, 2, 2, 2, 8, 6)
    assert all(he <= hs or we <= ws for hs, he, ws, we in wins)
    fm = np.zeros((1, 8, 6), np.float32)
    assert (roi_argmax(fm, [(200.0, 200.0, 210.0, 210.0)], 0, 1.0 / 8, 2, 2, 2) == -1).all()


def test_roi_argmax_ties_take_the_first_cell():
    fm = np.array([[[1, 3, 3], [3, 2, 0]]], np.float32)                 # 1 x 2 x 3
    am = roi_argmax(fm, [(1.0, 1.0, 3.0, 2.0)], 0, 1.0, 2, 1, 1)        # one bin over the whole map
    assert am.shape == (1, 1, 1) and am[0, 0, 0] == 1                   # the first 3 in (h, w) order


def test_norm_ab_known_answer():
    a, b = norm_ab([3.0, 4.0], [1.0, 0.0])
    n = np.sqrt(25.0 + float(np.float32(1e-10)))
    assert a == 1000.0 / n and b == 1000.0 * 3.0 / n ** 3
    assert abs(a - 200.0) < 1e-9 and abs(b - 24.0) < 1e-9
    assert norm_ab(np.zeros(4), np.ones(4)) == (1000.0 / np.sqrt(float(np.float32(1e-10))), 0.0)


def test_gather_known_answer_in_job_order():
    """two jobs on a 1 x 2 x 1 map (x = 1, 2): an unnormalised one names cells 0 and 1; a normalised one (a, b) =
    (2, 0.5) names cell 1 once and has an empty bin. cell 1 = 0.25 + fl(fl(2 * 1) - fl(0.5 * 2)) = 1.25"""
    x = np.array([[[1.0], [2.0]]], np.float32)
    jobs = [dict(argmax=np.array([[[0], [1]]]), g=np.array([[[0.5], [0.25]]], np.float32), ab=None),
            dict(argmax=np.array([[[1], [-1]]]), g=np.array([[[1.0], [7.0]]], np.float32), ab=np.array([[2.0, 0.5]]))]
    out = gather(x, jobs)
    assert out.shape == (1, 2, 1) and out[0, 0, 0] == 0.5 and out[0, 1, 0] == 1.25
    # the order is job, then r, then bin, from +0: a sum that rounds differently when reordered
    big, tiny = np.float32(1.0), np.float32(2.0 ** -24)
    jobs = [dict(argmax=np.array([[[0], [0]]]), g=np.array([[[big], [tiny]]], np.float32), ab=None),
            dict(argmax=np.array([[[0]]]), g=np.array([[[tiny]]], np.float32), ab=None)]
    out = gather(np.zeros((1, 1, 1), np.float32), jobs)
    assert out[0, 0, 0] == np.float32(big + tiny + tiny)                # (1 + 2^-24) + 2^-24 = 1 in fp32
