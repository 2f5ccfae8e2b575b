"""GPU: esb_img_resize_linear_u8 equals cv2.resize(INTER_LINEAR) on every byte (tests/golden/resize.npz), for 1, 20 and
50 views in one launch; and inference_scan(img_scale=(480, 480)) equals the configs' pipeline route, cv2-resized frames
with mmcv's Resize meta, bit for bit, for both box detectors."""
import os
import sys

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

from resize_cases import CASES, N_VIEWS, digest, frames  # noqa: E402

from oracle import resize_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLD, 'resize.npz')))


@pytest.mark.parametrize('name', list(CASES))
def test_kernel_equals_cv2(gold, name):
    from embodiedscan_b200.transforms import resize_multiview
    (W, H), (w, h) = CASES[name]
    src_np = frames(name)
    src = torch.from_numpy(src_np).to(DEV)
    for V in (1, 20, N_VIEWS):
        out = resize_multiview(src[:V], (w, h))
        assert out.shape == (V, 3, h, w) and out.dtype == torch.uint8
        hwc = out.permute(0, 2, 3, 1).cpu().numpy()
        for v in range(V):
            if not np.array_equal(digest(hwc[v]), gold[f'{name}/sha256'][v]):
                ref = R.resize_linear_u8(src_np[v], (w, h))       # the oracle equals cv2 (test_resize_cpu.py)
                bad = np.argwhere(hwc[v] != ref)
                pytest.fail(f'{name} V={V} view {v}: {len(bad)} bytes differ from cv2, '
                            f'first (y, x, c) {bad[:4].tolist()}')
    assert torch.equal(src, torch.from_numpy(src_np).to(DEV)), 'the source frames must be left unchanged'


def _model(kind):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_det3d_config
    torch.manual_seed(0)
    cfg = mv_det3d_config('C1')
    cfg['test_cfg'] = dict(nms_pre=200, iou_thr=.5, score_thr=.01)
    if kind == 'Embodied3DDetector':
        cfg['type'] = kind
        cfg['data_preprocessor'] = dict(cfg['data_preprocessor'], batchwise_inputs=True)
    model = MODELS.build(cfg).to(DEV).eval()
    with torch.no_grad():                          # three classes clear the demo's score threshold
        bias = torch.full((284, ), -9.0)
        bias[[3, 77, 200]] = -1.5
        model.bbox_head.conv_cls.bias.copy_(bias.view(1, -1))
        model.bbox_head.conv_cls.kernel.mul_(20.)
        model.bbox_head.conv_center.kernel.mul_(20.)
    return model


def _pipeline_route(model, imgs_chw, depth, K, extr, *, num_points, points_per_view, seed, filter):
    """What the configs' test pipeline hands the model for a 640x480 scan: frames already resized to 480x480 (cv2's
    bytes) and mmcv Resize's meta, then data_preprocessor, predict and nms_filter."""
    from embodiedscan_b200.detectors import Embodied3DDetector
    from embodiedscan_b200.inference import nms_filter
    from embodiedscan_b200.structures import Det3DDataSample, EulerDepthInstance3DBoxes, InstanceData
    from embodiedscan_b200.transforms import MultiViewDepthToPoints
    V, H, W = depth.shape
    K = np.asarray(K, dtype=np.float32)
    K4 = np.eye(4, dtype=np.float32)
    K4[:K.shape[0], :K.shape[1]] = K
    extr = [np.asarray(e, dtype=np.float32) for e in extr]
    meta = dict(img_shape=(480, 480), ori_shape=(H, W), scale_factor=(0.75, 1.0), flip=False, transformation_3d_flow=[],
                depth2img=dict(extrinsic=extr, intrinsic=[K4] * V, origin=np.array([.0, .0, .5], dtype=np.float32)),
                box_type_3d=EulerDepthInstance3DBoxes)
    sample = Det3DDataSample(metainfo=meta)
    if isinstance(model, Embodied3DDetector):
        per_frame = [MultiViewDepthToPoints(points_per_view, points_per_view, seed=seed + v)(
            dict(depth_imgs=depth[v:v + 1], depth2img=dict(intrinsic=[K4], extrinsic=[extr[v]])))['points']
            for v in range(V)]
        allp = torch.cat(per_frame)
        points = [[allp[:e]] for e in np.cumsum([p.shape[0] for p in per_frame]).tolist()]
        gt = InstanceData()
        gt.bboxes_3d = [EulerDepthInstance3DBoxes(torch.zeros((0, 9)), box_dim=9) for _ in range(V)]
        gt.labels_3d = [torch.zeros((0, ), dtype=torch.long) for _ in range(V)]
        sample.gt_instances_3d = gt
    else:
        points = [MultiViewDepthToPoints(num_points, points_per_view, seed=seed)(
            dict(depth_imgs=depth, depth2img=meta['depth2img']))['points']]
    with torch.no_grad():
        data = model.data_preprocessor(dict(inputs=dict(points=points, img=[imgs_chw]), data_samples=[sample]), False)
        results = model(**data, mode='predict')
    filtered = nms_filter([r.pred_instances_3d for r in results], num_classes=model.bbox_head.num_classes, **filter)
    return results, filtered


def _same(a, b):
    pa, pb = a.pred_instances_3d, b.pred_instances_3d
    return torch.equal(pa.bboxes_3d.tensor, pb.bboxes_3d.tensor) and torch.equal(pa.scores_3d, pb.scores_3d) and \
        torch.equal(pa.labels_3d, pb.labels_3d)


@pytest.mark.parametrize('kind', ['SparseFeatureFusionSingleStage3DDetector', 'Embodied3DDetector'])
def test_inference_scan_resize_equals_pipeline_route(gold, kind):
    from embodiedscan_b200.inference import inference_scan
    from embodiedscan_b200.synth import synth_scan
    V = 3
    s = synth_scan(3, n_views=V, H=480, W=640, n_points=2000, device=DEV)
    depth = s['depth']
    pm = s['data_sample'].metainfo['depth2img']
    K, extr = pm['intrinsic'][0], pm['extrinsic']
    # colour frames: the fixture's ScanNet-sized frames, whose cv2 480x480 bytes the fixture pins
    imgs = frames('scannet_640x480', V)
    resized = R.resize_linear_u8(imgs, (480, 480))
    for v in range(V):
        assert np.array_equal(digest(resized[v]), gold['scannet_640x480/sha256'][v])
    imgs_chw = torch.from_numpy(resized).permute(0, 3, 1, 2).contiguous().to(DEV)
    model = _model(kind)
    # the demo's IoU threshold and per-class cap; no score floor, so the filter has boxes to keep and to suppress
    kw = dict(num_points=2000, points_per_view=1500, seed=5, filter=dict(iou_thr=.15, score_thr=0., topk_per_class=10))
    ref, ref_filtered = _pipeline_route(model, imgs_chw, depth, K, extr, **kw)
    imgs_dev = torch.from_numpy(imgs).to(DEV)
    results, filtered = inference_scan(model, imgs_dev, depth, K, extr, img_scale=(480, 480), **kw)
    assert len(results) == len(ref) == (V if kind == 'Embodied3DDetector' else 1)
    for r, q in zip(results, ref):
        assert r.metainfo['img_shape'] == (480, 480) and r.metainfo['scale_factor'] == (0.75, 1.0)
        assert len(r.pred_instances_3d.scores_3d) > 0
        assert _same(r, q)
    assert len(filtered) == len(ref_filtered)
    assert all(len(b) > 0 for b, _ in filtered)
    for (b, l), (rb, rl) in zip(filtered, ref_filtered):
        assert torch.equal(b, rb) and torch.equal(l, rl)
    # the frames reach the prediction: the native-size route (no Resize) predicts other boxes
    native, _ = inference_scan(model, imgs_dev, depth, K, extr, **kw)
    assert not all(_same(a, b) for a, b in zip(native, results))
