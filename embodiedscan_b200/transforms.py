"""Device-side data front-end (SURVEY §8 rows a2 / f1): depth maps -> world points for all views of a scan in one
launch, replacing LoadDepthFromFile's `/ depth_shift`, ConvertRGBDToPoints + points_img2cam and AggregateMultiViewPoints
(embodiedscan/datasets/transforms/loading.py:70-73, points.py:30-81, structures/bbox_3d/utils.py:335-368,
multiview.py:139-169), followed by the reference's two PointSample stages (points.py:119-153) as seeded permutations.
The colour frames' `Resize` of the same pipeline (cv2 bilinear, bit for bit) is `MultiViewResize`, all views in one
launch.

The 3D augmentations of the training pipeline (configs/detection/mv-det3d_*.py:147-158) follow as torch operations on
the device-resident points and the (tiny) box tensor: `RandomFlip3D` (datasets/transforms/augmentation.py:11-250, the
`flip_2d=False` configuration) and `GlobalRotScaleTrans` (:253-420). They draw from `numpy.random` in the reference's
order, so a seeded run makes the same decisions as the reference pipeline, and they record the same `img_meta` keys
(`pcd_horizontal_flip`, `pcd_vertical_flip`, `pcd_rotation`, `pcd_scale_factor`, `pcd_trans`,
`transformation_3d_flow`) that point painting reverses (fusion.py).
"""
from typing import Optional, Sequence

import numpy as np
import torch

from ._ffi import call, ptr, query, stream
from .registry import TRANSFORMS


def unproject_multiview(depth_u16: torch.Tensor, intrinsics: Sequence, extrinsics: Sequence, depth_shift: float = 1000.0,
                        return_view: bool = False):
    """depth (V,H,W) integer millimetres on the GPU -> (n_valid, 3) fp32 world points, zero-depth pixels dropped, views
    concatenated in order and pixels row-major (the reference's `nonzero` order). The per-view matrix
    ``E^-1 @ K^-1`` is composed on the host in fp64 and applied as one fp32 4x4 per pixel."""
    assert depth_u16.is_cuda and depth_u16.dim() == 3
    V, H, W = depth_u16.shape
    dev = depth_u16.device
    d16 = depth_u16.to(torch.int32).clamp_(0, 65535).to(torch.int16).contiguous()       # uint16 bit pattern
    mats = []
    for v in range(V):
        K = np.eye(4, dtype=np.float64)
        Kin = np.asarray(intrinsics[v], dtype=np.float64)
        K[:Kin.shape[0], :Kin.shape[1]] = Kin
        E = np.asarray(extrinsics[v], dtype=np.float64).reshape(4, 4)
        mats.append((np.linalg.inv(E) @ np.linalg.inv(K)).astype(np.float32))
    md = torch.from_numpy(np.stack(mats)).to(dev).contiguous()
    out = torch.empty((V * H * W, 3), dtype=torch.float32, device=dev)
    view_of = torch.empty(V * H * W, dtype=torch.int32, device=dev) if return_view else None
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    wsb = query('esb_unproject_depth_workspace_bytes', V, H, W)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    call('esb_unproject_depth', ptr(d16), V, H, W, float(depth_shift), ptr(md), ptr(out), ptr(view_of), ptr(cnt), ptr(ws), wsb,
         stream())
    n = int(cnt.item())
    return (out[:n], view_of[:n]) if return_view else out[:n]


@TRANSFORMS.register_module()
class MultiViewDepthToPoints:
    """results['depth_imgs'] (V,H,W) + results['depth2img'] {'intrinsic': [...], 'extrinsic': [...]} -> results['points']
    (n_points, 3): per-view sample of `points_per_view`, then a global sample of `num_points` (seeded permutations; the
    reference draws with np.random.choice)."""

    def __init__(self, num_points: int = 100000, points_per_view: int = 10000, depth_shift: float = 1000.0,
                 seed: Optional[int] = None):
        self.num_points, self.points_per_view, self.depth_shift, self.seed = num_points, points_per_view, depth_shift, seed

    def __call__(self, results: dict) -> dict:
        depth = results['depth_imgs']
        pm = results['depth2img']
        pts, view = unproject_multiview(depth, pm['intrinsic'], pm['extrinsic'], self.depth_shift, return_view=True)
        gen = torch.Generator(device=pts.device)
        if self.seed is not None:
            gen.manual_seed(self.seed)
        keep = []
        for v in range(depth.shape[0]):
            idx = torch.nonzero(view == v).squeeze(1)
            perm = torch.randperm(idx.numel(), generator=gen, device=pts.device)[:self.points_per_view]
            keep.append(idx[perm])
        keep = torch.cat(keep)
        keep = keep[torch.randperm(keep.numel(), generator=gen, device=pts.device)[:self.num_points]]
        results['points'] = pts[keep].contiguous()
        return results


def resize_multiview(img_u8: torch.Tensor, size) -> torch.Tensor:
    """(V,H,W,3) uint8 frames on the GPU -> (V,3,h,w) uint8 for ``size = (w, h)``: ``cv2.resize(frame, size,
    interpolation=cv2.INTER_LINEAR)`` of every view, bit for bit, in one launch (csrc/resize.cu). Channels keep their
    order; the output is the layout ``Pack3DDetInputs`` stacks."""
    assert isinstance(img_u8, torch.Tensor) and img_u8.is_cuda and img_u8.dtype == torch.uint8 and \
        img_u8.dim() == 4 and img_u8.shape[-1] == 3, 'frames are one (V,H,W,3) uint8 GPU tensor (one source size)'
    w, h = (int(s) for s in size)
    V, H, W, _ = img_u8.shape
    src = img_u8.contiguous()
    out = torch.empty((V, 3, h, w), dtype=torch.uint8, device=src.device)
    call('esb_img_resize_linear_u8', ptr(src), V, H, W, h, w, ptr(out), stream())
    return out


@TRANSFORMS.register_module()
class MultiViewResize:
    """mmcv's ``Resize(scale=(w, h), keep_ratio=False)`` as the configs run it inside ``MultiViewPipeline``
    (configs/detection/mv-det3d_*.py:143,171), for all views of a scan at once: results['img'] (V,H,W,3) uint8 on the
    GPU -> (V,3,h,w). It leaves the keys mmcv's ``Resize._resize_img`` writes for the last view, which
    ``MultiViewPipeline`` keeps (multiview.py:90-92): ``img_shape = (h, w)``, ``scale = (w, h)``,
    ``scale_factor = (w / W, h / H)`` and ``keep_ratio``. Point painting reads ``scale_factor`` to map the original
    intrinsics onto the resized pixels (fusion.py). Only the configured mode is implemented: a fixed size, bilinear
    (mmcv's default cv2 backend)."""

    def __init__(self, scale, keep_ratio: bool = False, interpolation: str = 'bilinear'):
        if keep_ratio:
            raise ValueError('MultiViewResize: keep_ratio=True is not on the configured path (the configs resize to a '
                             'fixed size)')
        if interpolation != 'bilinear':
            raise ValueError(f'MultiViewResize: only bilinear interpolation is implemented, got {interpolation!r}')
        self.scale = (scale, scale) if isinstance(scale, int) else tuple(scale)
        self.keep_ratio = keep_ratio

    def __call__(self, results: dict) -> dict:
        img = results['img']
        results['img'] = resize_multiview(img, self.scale)
        H, W = img.shape[1:3]
        w, h = self.scale
        results['img_shape'] = (h, w)
        results['scale'] = self.scale
        results['scale_factor'] = (w / W, h / H)
        results['keep_ratio'] = self.keep_ratio
        return results

    transform = __call__


@TRANSFORMS.register_module()
class RandomFlip3D:
    """BEV flips of points + 9-DoF boxes. Only the configured mode is implemented: 3D flips decided independently of the
    images (``sync_2d=False, flip_2d=False``)."""

    def __init__(self, sync_2d: bool = True, flip_2d: bool = True, flip_3d: bool = True,
                 flip_ratio_bev_horizontal: float = 0.0, flip_ratio_bev_vertical: float = 0.0, flip_box3d: bool = True,
                 **kwargs):
        assert not flip_2d and not sync_2d, 'image flips are not on the configured path (cfg :147-152)'
        self.flip_3d, self.flip_box3d = flip_3d, flip_box3d
        self.flip_ratio_bev_horizontal, self.flip_ratio_bev_vertical = flip_ratio_bev_horizontal, flip_ratio_bev_vertical

    def _flip(self, results, direction):
        if 'gt_bboxes_3d' in results and self.flip_box3d:
            if 'points' in results:
                results['points'] = results['gt_bboxes_3d'].flip(direction, points=results['points'])
            else:
                results['gt_bboxes_3d'].flip(direction)
        elif 'points' in results:
            results['points'][:, 0 if direction == 'horizontal' else 1] *= -1

    def __call__(self, results: dict) -> dict:
        if not self.flip_3d:
            return results
        if 'pcd_horizontal_flip' not in results:
            results['pcd_horizontal_flip'] = bool(np.random.rand() < self.flip_ratio_bev_horizontal)
        if 'pcd_vertical_flip' not in results:
            results['pcd_vertical_flip'] = bool(np.random.rand() < self.flip_ratio_bev_vertical)
        flow = results.setdefault('transformation_3d_flow', [])
        if results['pcd_horizontal_flip']:
            self._flip(results, 'horizontal')
            flow.extend(['HF'])
        if results['pcd_vertical_flip']:
            self._flip(results, 'vertical')
            flow.extend(['VF'])
        return results

    transform = __call__


@TRANSFORMS.register_module()
class GlobalRotScaleTrans:
    """Random yaw (or 3-DoF) rotation, isotropic scale and Gaussian translation of points + boxes."""

    def __init__(self, rot_range=(-0.78539816, 0.78539816), rot_dof: int = 1, scale_ratio_range=(0.95, 1.05),
                 translation_std=(0, 0, 0), shift_height: bool = False, **kwargs):
        if not isinstance(rot_range, (list, tuple, np.ndarray)):
            rot_range = [-rot_range, rot_range]
        if not isinstance(translation_std, (list, tuple, np.ndarray)):
            translation_std = [translation_std] * 3
        assert not shift_height
        self.rot_range, self.rot_dof = rot_range, rot_dof
        self.scale_ratio_range, self.translation_std = scale_ratio_range, translation_std

    def __call__(self, results: dict) -> dict:
        flow = results.setdefault('transformation_3d_flow', [])
        pts, boxes = results.get('points'), results.get('gt_bboxes_3d')
        # rotation (augmentation.py:330-362)
        if self.rot_dof == 1:
            noise = -np.random.uniform(self.rot_range[0], self.rot_range[1])
        else:
            noise = np.array([-np.random.uniform(self.rot_range[0], self.rot_range[1]) for _ in range(3)])
        if boxes is not None and len(boxes.tensor) != 0:
            if pts is not None:
                pts, rot_mat_T = boxes.rotate(noise, pts)
                results['points'] = pts
            else:
                rot_mat_T = boxes.rotate(noise)
        elif pts is not None:
            from .geometry import euler_angles_to_matrix
            ang = torch.as_tensor(noise, dtype=pts.dtype, device=pts.device).reshape(-1)
            if ang.numel() == 1:
                ang = torch.cat([ang, ang.new_zeros(2)])
            rot_mat_T = euler_angles_to_matrix(ang, 'ZXY').T
            pts[:, :3] = pts[:, :3] @ rot_mat_T
        results['pcd_rotation'] = rot_mat_T
        results['pcd_rotation_angle'] = noise
        # scale (:364-395)
        if 'pcd_scale_factor' not in results:
            results['pcd_scale_factor'] = np.random.uniform(self.scale_ratio_range[0], self.scale_ratio_range[1])
        scale = results['pcd_scale_factor']
        if pts is not None:
            pts[:, :3] *= scale
        if boxes is not None:
            boxes.scale(scale)
        # translation (:309-328)
        trans = np.random.normal(scale=np.array(self.translation_std, dtype=np.float32), size=3).T
        if pts is not None:
            pts[:, :3] += torch.as_tensor(trans, dtype=pts.dtype, device=pts.device)
        results['pcd_trans'] = trans
        if boxes is not None:
            boxes.translate(trans)
        flow.extend(['R', 'S', 'T'])
        return results

    transform = __call__


@TRANSFORMS.register_module()
class ConstructMultiSweeps:
    """N aggregated frames -> the 1..N growing prefixes of the continuous setting (multiview.py:172-246):
    ``points`` (tensor of all frames, frame order) + ``points_slice_indices`` -> list of N prefix clouds;
    ``gt_bboxes_3d`` / ``gt_labels_3d`` -> per-prefix lists of the instances visible in any frame so far
    (``visible_instance_masks``), ``visible_occupancy_masks`` -> cumulative ``gt_occupancy_masks``.
    Prefix clouds are views into ONE buffer ordered by frame, so no point is copied N times."""

    def __call__(self, results: dict) -> dict:
        pts = results['points']
        pts = pts.tensor if hasattr(pts, 'tensor') else pts
        sl = results['points_slice_indices']
        n = len(sl) - 1
        results['points'] = [pts[sl[0]:sl[i + 1]] for i in range(n)]
        if 'visible_instance_masks' in results:
            boxes, labels = results['gt_bboxes_3d'], results['gt_labels_3d']
            seen = set()
            out_b, out_l = [], []
            for i in range(n):
                seen |= set(np.argwhere(np.array(results['visible_instance_masks'][i])).flatten().tolist())
                idx = np.array(list(seen), dtype=np.int32)       # the reference's set -> list order, kept on purpose
                out_b.append(boxes[torch.as_tensor(idx, dtype=torch.long)])
                out_l.append(labels[idx])
            results['gt_bboxes_3d'], results['gt_labels_3d'] = out_b, out_l
            if 'eval_ann_info' in results:
                results['eval_ann_info']['gt_bboxes_3d'] = out_b
                results['eval_ann_info']['gt_labels_3d'] = out_l
        if 'visible_occupancy_masks' in results:
            cum, out_m = None, []
            for i in range(n):
                m = np.asarray(results['visible_occupancy_masks'][i])
                cum = m if cum is None else np.logical_or(cum, m)
                out_m.append(cum)
            results['gt_occupancy_masks'] = out_m
            if 'eval_ann_info' in results:
                results['eval_ann_info']['gt_occupancy_masks'] = out_m
        return results

    transform = __call__
