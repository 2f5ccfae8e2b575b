"""Inference on one posed RGB-D sequence, the job of the reference's ``demo/demo.py``: camera poses -> extrinsics
(:174-197), colour + depth frames -> model input -> ``predict`` (:199-206), then the final box filter ``nms_filter``
(:84-130) as one launch of the 3D-IoU NMS (csrc/nms3d.cu). Reading the image, depth and pose files is the caller's job.

``nms_filter`` is opt-in post-processing: the ``pred_instances_3d`` the detectors return are what ``predict`` returns
in the reference (per-class BEV NMS of the head) and are left untouched.

The grounder takes the same scan inputs plus K free-text prompts. None of its visual work reads the text, so the visual
branch runs once and only the text encoder, the decoder and the head see the K prompts, in one batch.
"""
import contextlib
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .detectors import Embodied3DDetector, SparseFeatureFusionSingleStage3DDetector
from .geometry import nms3d_9dof
from .grounding import SparseFeatureFusion3DGrounder
from .precision import fp32_exact
from .structures import Det3DDataSample, EulerDepthInstance3DBoxes, InstanceData
from .transforms import MultiViewDepthToPoints, MultiViewResize

# camera axes (x right, y down, z forward) -> the pose file's body axes (demo.py:180-181)
_CAM_AXES = np.array([[0., 0., 1.], [-1., 0., 0.], [0., -1., 0.]])


def nms_filter(pred_instances_3d: Union[InstanceData, Sequence[InstanceData]], iou_thr: float = 0.15,
               score_thr: float = 0.075, topk_per_class: int = 10, num_classes=None):
    """The reference's ``nms_filter`` (same name, defaults and return order): greedy class-agnostic suppression on the
    exact 9-DoF 3D IoU by descending score, boxes under `score_thr` dropped, at most `topk_per_class` kept per label.
    Returns ``(boxes (K,9), labels (K,))`` in selection order. The reference returns numpy arrays; here the tensors stay
    on the device. A list of results is filtered in one launch and a list of pairs comes back."""
    single = isinstance(pred_instances_3d, InstanceData)
    preds = [pred_instances_3d] if single else list(pred_instances_3d)
    if not preds:
        return []
    boxes = torch.cat([p.bboxes_3d.tensor for p in preds])
    scores = torch.cat([p.scores_3d for p in preds])
    labels = torch.cat([p.labels_3d for p in preds])
    seg_off = np.cumsum([0] + [len(p.scores_3d) for p in preds]).tolist()
    keeps = nms3d_9dof(boxes, scores, labels, iou_thr, score_thr, topk_per_class, seg_off=seg_off,
                       num_classes=num_classes)
    out = [(boxes[k], labels[k]) for k in keeps]
    return out[0] if single else out


def scan_from_poses(poses, intrinsic, axis_align_matrix) -> Tuple[np.ndarray, List[np.ndarray]]:
    """Camera poses of a sequence -> what ``depth2img`` needs (demo.py:174-197).

    poses: (V,7) rows ``x y z qx qy qz qw`` (camera in the unaligned global frame; the timestamp column of
    ``poses.txt`` removed). The demo's own loop starts at the second line of ``poses.txt``; a caller that wants the
    demo's frames drops the first line before calling. intrinsic: (4,4) or (3,3). axis_align_matrix: (4,4).
    Returns ``(intrinsic fp32, [extrinsic_v (4,4) fp32])`` with
    ``extrinsic_v = inv(axis_align_matrix @ cam2global_v)`` computed in fp64: aligned world -> camera."""
    poses = np.asarray(poses, dtype=np.float64).reshape(-1, 7)
    align = np.asarray(axis_align_matrix, dtype=np.float64).reshape(4, 4)
    extrinsics = []
    for x, y, z, qx, qy, qz, qw in poses:
        n = qx * qx + qy * qy + qz * qz + qw * qw
        assert n > 0, 'zero quaternion in poses'
        s = 2.0 / n
        rot = np.array([[1 - s * (qy * qy + qz * qz), s * (qx * qy - qz * qw), s * (qx * qz + qy * qw)],
                        [s * (qx * qy + qz * qw), 1 - s * (qx * qx + qz * qz), s * (qy * qz - qx * qw)],
                        [s * (qx * qz - qy * qw), s * (qy * qz + qx * qw), 1 - s * (qx * qx + qy * qy)]])
        cam2global = np.eye(4)
        cam2global[:3, :3] = rot @ _CAM_AXES
        cam2global[:3, 3] = (x, y, z)
        extrinsics.append(np.linalg.inv(align @ cam2global).astype(np.float32))
    return np.asarray(intrinsic, dtype=np.float32), extrinsics


def _intrinsic44(intrinsic) -> np.ndarray:
    k = np.eye(4, dtype=np.float32)
    a = np.asarray(intrinsic, dtype=np.float32)
    k[:a.shape[0], :a.shape[1]] = a
    return k


def _scan_inputs(model, imgs_u8: torch.Tensor, depth_u16: torch.Tensor, intrinsic, extrinsics, *, num_points: int,
                 points_per_view: int, depth_shift: float, seed: int, img_scale):
    """A posed RGB-D scan -> what the configs' test pipeline hands a model: ``(points, img, meta)`` with `points` the
    per-sample list of ``data_preprocessor``'s inputs, `img` (V,3,h,w) uint8 on the model's device and `meta` the scan's
    metainfo. The one copy of this step for every model ``inference_scan`` runs."""
    dev = next(model.parameters()).device
    assert dev.type == 'cuda', 'inference_scan runs on the GPU'
    V, H, W = depth_u16.shape
    assert imgs_u8.dtype == torch.uint8 and tuple(imgs_u8.shape) == (V, H, W, 3) and len(extrinsics) == V
    depth = depth_u16.to(dev)
    if img_scale is None:
        img = imgs_u8.to(dev).permute(0, 3, 1, 2).contiguous()               # (V,3,H,W) uint8, as Pack3DDetInputs
        img_shape, scale_factor = (H, W), (1.0, 1.0)
    else:
        resized = MultiViewResize(img_scale)(dict(img=imgs_u8.to(dev)))
        img, img_shape, scale_factor = resized['img'], resized['img_shape'], resized['scale_factor']
    K = _intrinsic44(intrinsic)
    extr = [np.asarray(e, dtype=np.float32).reshape(4, 4) for e in extrinsics]
    meta = dict(img_shape=img_shape, ori_shape=(H, W), scale_factor=scale_factor, flip=False, transformation_3d_flow=[],
                depth2img=dict(extrinsic=extr, intrinsic=[K] * V, origin=np.array([.0, .0, .5], dtype=np.float32)),
                box_type_3d=EulerDepthInstance3DBoxes)
    if isinstance(model, Embodied3DDetector):
        # frame-ordered per-view samples; prefix i = frames 0..i, views into one buffer (ConstructMultiSweeps)
        frames = []
        for v in range(V):
            to_points = MultiViewDepthToPoints(points_per_view, points_per_view, depth_shift, seed=seed + v)
            frames.append(to_points(dict(depth_imgs=depth[v:v + 1],
                                         depth2img=dict(intrinsic=[K], extrinsic=[extr[v]])))['points'])
        allp = torch.cat(frames)
        ends = np.cumsum([f.shape[0] for f in frames]).tolist()
        points = [[allp[:e]] for e in ends]
    else:
        to_points = MultiViewDepthToPoints(num_points, points_per_view, depth_shift, seed=seed)
        points = [to_points(dict(depth_imgs=depth, depth2img=meta['depth2img']))['points']]
    return points, img, meta


def _check_prompts(model: SparseFeatureFusion3DGrounder, prompts) -> List[str]:
    """The prompts of one ``inference_scan`` call as a list, or ``ValueError``: a non-empty sequence of strings, none
    longer than the contrastive head's ``max_text_len`` tokens (the head has no column for the tokens past it)."""
    if prompts is None:
        raise ValueError(f'inference_scan on a {type(model).__name__} needs prompts=[...], the sentences to ground')
    if isinstance(prompts, str):
        raise ValueError('prompts is a sequence of sentences, not one string: pass [prompt]')
    prompts = list(prompts)
    if not prompts:
        raise ValueError('prompts is empty: pass at least one sentence')
    for k, p in enumerate(prompts):
        if not isinstance(p, str):
            raise ValueError(f'prompts[{k}] is a {type(p).__name__}, not a str')
    max_len = model.bbox_head.max_text_len
    lengths = model.tokenizer.batch_encode_plus(prompts, padding='longest', return_tensors='pt')['attention_mask'].sum(1)
    for p, n in zip(prompts, lengths.tolist()):
        if n > max_len:
            raise ValueError(f'prompt {p!r} is {n} tokens long; the grounding head takes at most max_text_len = '
                             f'{max_len}')
    return prompts


def _rank_queries(scores: torch.Tensor, topk: int) -> torch.Tensor:
    """Indices of the `topk` best queries: descending score, equal scores in ascending query order (a stable sort; the
    reference's ``argsort`` leaves the order of ties open)."""
    return torch.sort(scores, descending=True, stable=True).indices[:topk]


def _ground_scan(model: SparseFeatureFusion3DGrounder, points, img, meta, prompts: List[str], topk: int):
    """K prompts on one scan: the visual branch (2D backbone, sparse backbone, painting, ``MinkNeck``) runs once at
    batch size 1, and its per-scan outputs are repeated K times into one text-encoder and decoder batch, which is what
    ``predict`` computes for K samples holding the same scan. Each sample names its whole prompt as its one phrase
    (``tokens_positive``): ``encode_text`` writes the positive maps from it, which the prediction does not read. Returns
    ``(results, ranked)``."""
    with torch.no_grad(), (fp32_exact() if model.compute_dtype == torch.float32 else contextlib.nullcontext()):
        data = model.data_preprocessor(dict(inputs=dict(points=points, img=[img]),
                                            data_samples=[Det3DDataSample(metainfo=meta)]), False)
        scan = data['data_samples'][0]
        feats, scores, xyz = model.extract_feat(data['inputs'], [scan])
        K = len(prompts)
        samples = []
        for p in prompts:
            ds = Det3DDataSample(metainfo=scan.metainfo)
            ds.text = p
            ds.tokens_positive = [[[0, len(p)]]]                            # one phrase: the whole prompt
            ds.gt_instances_3d = InstanceData()                             # encode_text writes the positive maps here
            samples.append(ds)
        text_dict = model.encode_text(samples, feats[0].device)
        head_in = model.forward_transformer(feats * K, scores * K, xyz * K, text_dict, samples)
        preds = model.bbox_head.predict(**head_in, batch_data_samples=samples)
    ranked = []
    for ds, r in zip(samples, preds):
        ds.pred_instances_3d = r
        order = _rank_queries(r.scores_3d, topk)
        ranked.append((r.bboxes_3d.tensor[order], r.scores_3d[order]))
    return samples, ranked


def inference_scan(model, imgs_u8: torch.Tensor, depth_u16: torch.Tensor, intrinsic, extrinsics, *, num_points: int,
                   points_per_view: int, depth_shift: float = 1000., seed: int = 0, filter=None, img_scale=None,
                   prompts: Optional[Sequence[str]] = None, topk: Optional[int] = None):
    """One posed RGB-D scan through a detector and the final box filter, or through the grounder with free-text prompts.

    imgs_u8 (V,H,W,3) uint8 colour frames in the channel order the model's preprocessor expects, depth_u16 (V,H,W)
    integer depth in 1/`depth_shift` metres (0 = no return), intrinsic (3,3)/(4,4), extrinsics V x (4,4) world ->
    camera (``scan_from_poses``). Points are sampled as ``MultiViewDepthToPoints`` samples them, seeded by `seed`.

    `img_scale` ``(w, h)`` resizes the colour frames as the config's ``Resize(scale=(w, h), keep_ratio=False)`` does
    (``MultiViewResize``, cv2 bilinear bit for bit) and records its ``img_shape`` and ``scale_factor``, so point
    painting maps the intrinsics of the original frames onto the resized ones. The config's ``Resize`` scale (480x480 in
    every published config) is what reproduces ``demo.py``, which runs the config's test pipeline. ``None`` passes the
    frames at their own size, as a pipeline without ``Resize`` would.

    Detectors (``SparseFeatureFusionSingleStage3DDetector``, ``Embodied3DDetector``): `filter` holds the ``nms_filter``
    arguments (default: the demo's 0.15 / 0.075 / 10). Returns ``(results, filtered)``: `results` is the list of
    ``Det3DDataSample`` of ``model.forward(mode='predict')`` with ``pred_instances_3d`` set, one for
    ``SparseFeatureFusionSingleStage3DDetector`` and one per frame prefix 1..V for ``Embodied3DDetector``;
    `filtered[i]` is ``nms_filter(results[i].pred_instances_3d)``, all results filtered in one launch.

    ``SparseFeatureFusion3DGrounder``: `prompts` (required) are the K sentences to ground in the scan, each a ``str`` of
    at most the head's ``max_text_len`` tokens (``ValueError`` otherwise). The visual branch runs once and the K prompts
    share one text-encoder and decoder batch. Returns ``(results, ranked)``, K of each in prompt order: `results[k]` is
    the ``Det3DDataSample`` ``predict`` produces for the scan with ``text = prompts[k]`` (``pred_instances_3d`` with
    ``bboxes_3d``, ``scores_3d`` and ``target_scores_3d`` of every query), and `ranked[k]` is ``(boxes (n,9), scores
    (n,))`` of its `topk` best queries (default 10, the number ``GroundingMetric`` scores) by descending score, equal
    scores in ascending query order. No box filter is applied, as in the reference. Everything stays on the device. A
    prompt's text features depend on the other prompts of the call: the tokens are padded to the longest prompt, as in
    the reference's batched test."""
    grounder = isinstance(model, SparseFeatureFusion3DGrounder)
    if not grounder and not isinstance(model, SparseFeatureFusionSingleStage3DDetector):
        raise TypeError(f'inference_scan runs the box detectors (SparseFeatureFusionSingleStage3DDetector, '
                        f'Embodied3DDetector) and the grounder (SparseFeatureFusion3DGrounder); {type(model).__name__} '
                        f'predicts no boxes (occupancy models are not supported)')
    kw = dict(num_points=num_points, points_per_view=points_per_view, depth_shift=depth_shift, seed=seed,
              img_scale=img_scale)
    if grounder:
        prompts = _check_prompts(model, prompts)
        if filter is not None:
            raise ValueError('filter is the box detectors\' nms_filter; grounding outputs are not filtered')
        topk = 10 if topk is None else int(topk)
        if topk < 1:
            raise ValueError(f'topk must be >= 1, got {topk}')
        points, img, meta = _scan_inputs(model, imgs_u8, depth_u16, intrinsic, extrinsics, **kw)
        return _ground_scan(model, points, img, meta, prompts, topk)
    if prompts is not None or topk is not None:
        raise ValueError(f'prompts and topk are for the grounder; {type(model).__name__} is a box detector')
    filter = dict(iou_thr=.15, score_thr=.075, topk_per_class=10) if filter is None else dict(filter)
    points, img, meta = _scan_inputs(model, imgs_u8, depth_u16, intrinsic, extrinsics, **kw)
    sample = Det3DDataSample(metainfo=meta)
    if isinstance(model, Embodied3DDetector):
        V = len(points)
        gt = InstanceData()                                                  # empty annotation per prefix (demo.py:166-171)
        gt.bboxes_3d = [EulerDepthInstance3DBoxes(torch.zeros((0, 9)), box_dim=9) for _ in range(V)]
        gt.labels_3d = [torch.zeros((0, ), dtype=torch.long) for _ in range(V)]
        sample.gt_instances_3d = gt
    with torch.no_grad():
        data = model.data_preprocessor(dict(inputs=dict(points=points, img=[img]), data_samples=[sample]), False)
        results = model(**data, mode='predict')
    num_classes = getattr(model.bbox_head, 'num_classes', None)
    filtered = nms_filter([r.pred_instances_3d for r in results], num_classes=num_classes, **filter)
    return results, filtered
