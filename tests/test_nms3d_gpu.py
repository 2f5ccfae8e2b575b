"""GPU: the 3D-IoU box filter (csrc/nms3d.cu) against the float64 oracle, exact equality of the kept lists, and the
posed RGB-D inference entry point end to end.

The one place where fp32 and float64 clipping may legitimately decide `iou > iou_thr` differently is an IoU within 1e-4
of the threshold. The scene generator (`nms3d_ref.clustered_scene`) computes the oracle matrix in float64 and draws the
jitter of any box of such a pair again (seeded, so the set of boxes is fixed); outside that band no tolerance applies."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nms3d_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
IOU_THR = 0.15
INF = 10 ** 9
# n -> (copies per cuboid, cuboids per 6 m x 6 m): the large scenes are spread out so that the Python oracle clips
# thousands of pairs, not millions; tile edges (64) and multi-word masks are crossed all the same
SCENES = {1: (5, 24), 63: (5, 24), 64: (5, 24), 65: (5, 24), 500: (5, 6), 3000: (4, 3)}


@functools.lru_cache(maxsize=None)
def scene(n, seed=0):
    copies, per_room = SCENES[n]
    return R.clustered_scene(n, seed + n, copies=copies, per_room=per_room, iou_thr=IOU_THR)


def gpu_keep(boxes, scores, labels, **kw):
    from embodiedscan_b200.geometry import nms3d_9dof
    out = nms3d_9dof(torch.from_numpy(boxes).to(DEV), torch.from_numpy(scores).to(DEV), torch.from_numpy(labels).to(DEV),
                     **kw)
    return [o.tolist() for o in out] if isinstance(out, list) else out.tolist()


@pytest.mark.parametrize('n', sorted(SCENES))
def test_kept_list_equals_oracle(n):
    boxes, scores, labels, iou = scene(n)
    dup = (np.round(scores * 8) / 8).astype(np.float32)                     # many exact ties: input order decides
    cases = [dict(score_thr=-np.inf, topk=None, scores=scores), dict(score_thr=-np.inf, topk=2, scores=scores),
             dict(score_thr=0.3, topk=None, scores=scores), dict(score_thr=0.3, topk=3, scores=dup),
             dict(score_thr=-np.inf, topk=None, scores=dup)]
    for c in cases:
        ref = R.nms_filter(boxes, c['scores'], labels, IOU_THR, c['score_thr'], INF if c['topk'] is None else c['topk'],
                           iou=iou)
        got = gpu_keep(boxes, c['scores'], labels, iou_thr=IOU_THR, score_thr=c['score_thr'], topk_per_class=c['topk'])
        assert got == ref, (n, c['score_thr'], c['topk'])
        if c['topk'] is not None and n >= 500:
            assert max(np.bincount(labels[ref])) == c['topk'], 'the cap must bind'
    assert n < 500 or len(R.nms_filter(boxes, scores, labels, IOU_THR, -np.inf, INF, iou=iou)) < 0.8 * n, \
        'the scene must exercise suppression'


def test_segments_equal_single_calls():
    parts = [scene(65), scene(1), None, scene(500)]
    boxes = np.concatenate([p[0] for p in parts if p is not None])
    scores = np.concatenate([p[1] for p in parts if p is not None])
    labels = np.concatenate([p[2] for p in parts if p is not None])
    seg_off = np.cumsum([0] + [0 if p is None else len(p[1]) for p in parts]).tolist()
    got = gpu_keep(boxes, scores, labels, iou_thr=IOU_THR, score_thr=0.1, topk_per_class=4, seg_off=seg_off)
    assert len(got) == 4 and got[2] == []
    for s, p in enumerate(parts):
        if p is None:
            continue
        single = gpu_keep(p[0], p[1], p[2], iou_thr=IOU_THR, score_thr=0.1, topk_per_class=4)
        assert got[s] == [seg_off[s] + i for i in single]
        assert single == R.nms_filter(p[0], p[1], p[2], IOU_THR, 0.1, 4, iou=p[3])


def test_empty_input_and_argument_checks():
    from embodiedscan_b200.geometry import nms3d_9dof
    e = nms3d_9dof(torch.zeros((0, 9), device=DEV), torch.zeros(0, device=DEV), torch.zeros(0, dtype=torch.long, device=DEV),
                   iou_thr=0.15)
    assert e.dtype == torch.long and e.numel() == 0
    with pytest.raises(AssertionError, match='no CPU fallback'):
        nms3d_9dof(torch.zeros((1, 9)), torch.zeros(1), torch.zeros(1, dtype=torch.long), iou_thr=0.15)
    from embodiedscan_b200 import _ffi
    z = torch.zeros(16, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match='iou_thr must be >= 0'):
        _ffi.call('esb_nms3d_9dof', z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 1, 1, -0.5, 0.0, 1, 1,
                  z.data_ptr(), z.data_ptr(), z.data_ptr(), 64, _ffi.stream())


def test_degenerate_boxes_overlap_nothing():
    """A zero size or a NaN makes a box overlap nothing: it is kept, suppresses nothing and is never suppressed."""
    unit = [0, 0, 0, 1, 1, 1, 0, 0, 0]
    boxes = np.array([unit, [0, 0, 0, 0, 1, 1, 0, 0, 0], [np.nan, 0, 0, 1, 1, 1, 0, 0, 0], unit, unit], dtype=np.float32)
    boxes[4, 0] = 0.02
    scores = np.array([.6, .9, .8, .7, .5], dtype=np.float32)
    labels = np.zeros(5, dtype=np.int64)
    ref = R.nms_filter(boxes, scores, labels, IOU_THR, -np.inf, INF)
    assert ref == [1, 2, 3]
    assert gpu_keep(boxes, scores, labels, iou_thr=IOU_THR) == ref


def test_mask_phase_agrees_with_box3d_overlap():
    """Thresholding the full matrix of esb_box3d_overlap and walking it on the host gives the kept list of the NMS kernel:
    both run the clipping of csrc/iou3d.cuh."""
    from embodiedscan_b200.geometry import box3d_overlap, box_corners_container
    boxes, scores, labels, _ = scene(500)
    k = box_corners_container(torch.from_numpy(boxes).to(DEV))
    iou32 = box3d_overlap(k, k)[1].cpu().numpy()
    for topk in (None, 2):
        ref = R.nms_filter(boxes, scores, labels, np.float32(IOU_THR), 0.2, INF if topk is None else topk, iou=iou32)
        assert gpu_keep(boxes, scores, labels, iou_thr=IOU_THR, score_thr=0.2, topk_per_class=topk) == ref


def _scan(n_views=2):
    from embodiedscan_b200.synth import synth_scan
    s = synth_scan(3, n_views=n_views, H=240, W=320, n_points=2000, device=DEV)
    pm = s['data_sample'].metainfo['depth2img']
    imgs = s['img'].permute(0, 2, 3, 1).contiguous()
    return imgs, s['depth'], pm['intrinsic'][0], pm['extrinsic']


def _model(kind):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_det3d_config
    torch.manual_seed(0)
    cfg = mv_det3d_config('C1')
    cfg['test_cfg'] = dict(nms_pre=50, iou_thr=.5, score_thr=.01)
    if kind == 'Embodied3DDetector':
        cfg['type'] = kind
        cfg['data_preprocessor'] = dict(cfg['data_preprocessor'], batchwise_inputs=True)
    model = MODELS.build(cfg).to(DEV).eval()
    with torch.no_grad():                          # three classes clear the thresholds, with spread-out scores
        bias = torch.full((284, ), -9.0)
        bias[[3, 77, 200]] = -1.5
        model.bbox_head.conv_cls.bias.copy_(bias.view(1, -1))
        model.bbox_head.conv_cls.kernel.mul_(20.)
        model.bbox_head.conv_center.kernel.mul_(20.)
    return model


@pytest.mark.parametrize('kind', ['SparseFeatureFusionSingleStage3DDetector', 'Embodied3DDetector'])
def test_inference_scan_end_to_end(kind):
    from embodiedscan_b200.inference import inference_scan, nms_filter
    from embodiedscan_b200.structures import Det3DDataSample
    model = _model(kind)
    imgs, depth, K, extr = _scan()
    kw = dict(num_points=2000, points_per_view=1500, seed=5)
    results, _ = inference_scan(model, imgs, depth, K, extr, **kw)
    assert len(results) == (2 if kind == 'Embodied3DDetector' else 1)
    assert all(isinstance(r, Det3DDataSample) for r in results)
    preds = [r.pred_instances_3d for r in results]
    # The oracle clips pairs in Python, so the score threshold is set where about 60 boxes of each result pass it. A box
    # under the threshold is skipped before any IoU is read, so the oracle matrix is needed among the passing boxes only.
    score_thr = max(float(np.sort(p.scores_3d.cpu().numpy())[::-1][:60][-1]) for p in preds)
    mats = []
    for p in preds:
        b, s = p.bboxes_3d.tensor.cpu().numpy(), p.scores_3d.cpu().numpy()
        live = np.nonzero(s >= score_thr)[0]
        m = np.zeros((len(s), len(s)))
        m[np.ix_(live, live)] = R.iou_matrix(b[live])
        mats.append(m)
    # a threshold no oracle IoU of these predictions comes within 1e-4 of (see the module docstring)
    thr = next(t for t in (0.15, 0.2, 0.25, 0.3, 0.35, 0.4, 0.45, 0.5)
               if all((np.abs(m - t) >= 1e-4).all() for m in mats))
    flt = dict(iou_thr=thr, score_thr=score_thr, topk_per_class=10)
    results, filtered = inference_scan(model, imgs, depth, K, extr, filter=flt, **kw)
    again, filtered2 = inference_scan(model, imgs, depth, K, extr, filter=flt, **kw)
    assert len(filtered) == len(results)
    suppressed = 0
    for r, r2, (fb, fl), (fb2, fl2), m in zip(results, again, filtered, filtered2, mats):
        p = r.pred_instances_3d
        assert len(p.scores_3d) > 60, 'the scan must produce candidates on both sides of the score threshold'
        assert torch.equal(p.bboxes_3d.tensor, r2.pred_instances_3d.bboxes_3d.tensor)
        assert torch.equal(fb, fb2) and torch.equal(fl, fl2)
        b, s, l = p.bboxes_3d.tensor.cpu().numpy(), p.scores_3d.cpu().numpy(), p.labels_3d.cpu().numpy()
        ref = R.nms_filter(b, s, l, thr, score_thr, 10, iou=m)
        assert fb.is_cuda and fb.shape == (len(ref), 9)
        assert np.array_equal(fb.cpu().numpy(), b[ref]) and np.array_equal(fl.cpu().numpy(), l[ref])
        assert len(ref) == 0 or np.bincount(l[ref]).max() <= 10
        suppressed += len(s) - len(ref)
        one_b, one_l = nms_filter(p, **flt)                                  # a single InstanceData, no list
        assert torch.equal(one_b, fb) and torch.equal(one_l, fl)
    assert suppressed > 0, 'the filter must have something to remove'


def test_inference_scan_rejects_models_without_boxes():
    from embodiedscan_b200.inference import inference_scan
    with pytest.raises(TypeError, match='predicts no boxes'):
        inference_scan(torch.nn.Linear(1, 1), None, None, None, None, num_points=1, points_per_view=1)
