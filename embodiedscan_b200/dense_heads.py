"""The FCAF3D heads — sparse FPN + anchor-free head — registered under the reference's names
(embodiedscan/models/dense_heads/fcaf3d_head.py): ``FCAF3DHeadRotMat`` (:827-1725, 9-DoF boxes from a 6D rotation, corner
chamfer box loss) and ``FCAF3DHead`` (:29-826, raw yaw or Euler angles, rotated 3D IoU box loss), with their losses
(``BBoxCDLoss``, ``ChamferDistance``, ``RotatedIoU3DLoss``). Same constructor arguments, ``forward`` / ``loss`` /
``predict`` contract and parameter names (``up_block_i.{0,3}.kernel``, ``out_block_i.0.kernel``, ``conv_cls.bias``,
``scales.i.scale``). Host-side differences that do not change results:
  * target assignment is one fused kernel pipeline per scan (csrc/head.cu) instead of dense (Np,Ng,*) temporaries;
  * the per-scan scalar ``reduce_mean`` calls are fused into ONE device-side vector all-reduce (no host sync);
  * the 284-iteration per-class NMS loop is one segmented kernel launch (csrc/nms.cu).
"""
import ctypes
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _ffi
from . import sparse as SP
from ._ffi import call, ptr, query, stream
from .geometry import (CD_GROUPS, CD_MODES, CD_REDUCTIONS, bbox_cd_loss, bbox_to_corners, chamfer_src,
                       euler_angles_to_matrix, matrix_to_euler_angles_zxy, ortho_6d_2_mat, rotation_3d_in_axis,
                       rotation_3d_in_euler)
from .registry import MODELS
from .structures import EulerDepthInstance3DBoxes, InstanceData


class Scale(nn.Module):
    """mmcv.cnn.Scale: a learnable scalar."""

    def __init__(self, scale: float = 1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(scale, dtype=torch.float))

    def forward(self, x):
        return x * self.scale.to(x.dtype)


def _check_cd_options(mode=None, group=None, reduction=None):
    for value, valid, what in ((mode, CD_MODES, 'mode'), (group, CD_GROUPS, 'group'), (reduction, CD_REDUCTIONS, 'reduction')):
        if value is not None and value not in valid:
            raise ValueError(f'chamfer {what} must be one of {valid}, got {value!r}')


def check_head_box_loss(loss):
    """A head averages its box loss itself, so the loss module must keep reduction='mean' (the reference's heads stack
    per-scan 'sum' / 'none' results into values that are not a loss)."""
    reduction = getattr(loss, 'reduction', 'mean')
    if reduction != 'mean':
        raise ValueError(f"the box loss of a head supports reduction='mean' only, got reduction={reduction!r}")


@MODELS.register_module()
class BBoxCDLoss(nn.Module):
    """embodiedscan/models/losses/chamfer_distance.py:206-285: chamfer distance from the 8 corners of each source box
    to the corners of its target box (src->dst only), criterion 'l1' / 'l2' / 'smooth_l1', corner groups 'g8' / 'g4'."""

    def __init__(self, mode='l2', group='g8', reduction='mean', loss_weight=1.0):
        super().__init__()
        _check_cd_options(mode, group, reduction)
        self.mode, self.group, self.reduction, self.loss_weight = mode, group, reduction, loss_weight

    def forward(self, source, target, loss_weight=1.0, reduction_override=None, **kwargs):
        _check_cd_options(reduction=reduction_override)
        reduction = reduction_override if reduction_override else self.reduction
        return bbox_cd_loss(source, target, self.loss_weight, self.mode, self.group, reduction, loss_weight)


_REDUCTIONS = ('none', 'mean', 'sum')


def weight_reduce_loss(loss, weight=None, reduction='mean', avg_factor=None):
    """embodiedscan/models/losses/reduce_loss.py:30-65: element-wise weight, then 'none' / 'mean' / 'sum'; with an
    avg_factor, 'mean' is sum / (avg_factor + eps_fp32) and 'sum' is an error."""
    if weight is not None:
        loss = loss * weight
    if avg_factor is None:
        return loss.mean() if reduction == 'mean' else loss.sum() if reduction == 'sum' else loss
    if reduction == 'mean':
        return loss.sum() / (avg_factor + torch.finfo(torch.float32).eps)
    if reduction != 'none':
        raise ValueError('avg_factor can not be used with reduction="sum"')
    return loss


def _box_rows(t: torch.Tensor) -> torch.Tensor:
    """fp32 rows whose first 7 columns the IoU kernel reads in place (unit column stride, row stride >= 7)."""
    t = t.detach().float()
    if t.stride(1) != 1 or t.stride(0) < 7:
        t = t.contiguous()
    return t


class _RotatedIoU3D(torch.autograd.Function):
    """csrc/rotiou3d.cu: the IoU of one-to-one rotated box pairs and, in backward, its analytic gradient for both
    arguments (the target's only when it requires one)."""

    @staticmethod
    def forward(ctx, pred, target):
        a, b = _box_rows(pred), _box_rows(target)
        n = a.shape[0]
        iou = torch.empty(n, dtype=torch.float32, device=a.device)
        call('esb_rotated_iou3d_fwd', ptr(a), a.stride(0), ptr(b), b.stride(0), n, ptr(iou), stream())
        ctx.save_for_backward(a, b)
        ctx.like = (pred.shape, pred.dtype, target.shape, target.dtype)
        return iou

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        n = a.shape[0]
        need_b = ctx.needs_input_grad[1]
        grad_a = torch.empty((n, 7), dtype=torch.float32, device=a.device)
        grad_b = torch.empty((n, 7), dtype=torch.float32, device=a.device) if need_b else None
        call('esb_rotated_iou3d_bwd', ptr(a), a.stride(0), ptr(b), b.stride(0), n, ptr(g.float().contiguous()),
             ptr(grad_a), ptr(grad_b), stream())

        def widen(grad, shape, dtype):          # columns past 7 do not enter the IoU
            if shape[1] == 7:
                return grad.to(dtype)
            return torch.cat((grad, grad.new_zeros(n, shape[1] - 7)), 1).to(dtype)

        pshape, pdtype, tshape, tdtype = ctx.like
        return (widen(grad_a, pshape, pdtype) if ctx.needs_input_grad[0] else None,
                widen(grad_b, tshape, tdtype) if need_b else None)


def rotated_iou_3d(pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """mmcv.ops.diff_iou_rotated_3d for one-to-one pairs on csrc/rotiou3d.cu: pred, target (N, >=7) CUDA rows
    (x, y, z, w, l, h, alpha, ...), z the box centre; columns past 7 are ignored. Returns iou (N,) fp32,
    differentiable in both arguments."""
    if pred.dim() != 2 or target.dim() != 2 or pred.shape[0] != target.shape[0] or pred.shape[1] < 7 or \
            target.shape[1] < 7:
        raise ValueError(f'rotated_iou_3d takes one-to-one boxes (N, >=7), got {tuple(pred.shape)} and '
                         f'{tuple(target.shape)}')
    if not (pred.is_cuda and target.is_cuda):
        raise ValueError('rotated_iou_3d runs on CUDA tensors only (there is no CPU implementation)')
    return _RotatedIoU3D.apply(pred, target)


@MODELS.register_module()
class RotatedIoU3DLoss(nn.Module):
    """embodiedscan/models/losses/rotated_iou_loss.py:37-91: loss_weight * weight_reduce_loss(1 - IoU) of one-to-one
    rotated boxes (N, >=7) on csrc/rotiou3d.cu. A weight (N, k > 1) is averaged over its last dimension; a weight with
    no element > 0 returns pred.sum() * weight.sum()."""

    def __init__(self, reduction='mean', loss_weight=1.0):
        super().__init__()
        if reduction not in _REDUCTIONS:
            raise ValueError(f'reduction must be one of {_REDUCTIONS}, got {reduction!r}')
        self.reduction, self.loss_weight = reduction, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None, **kwargs):
        if weight is not None and not torch.any(weight > 0):
            return pred.sum() * weight.sum()
        if reduction_override not in (None, ) + _REDUCTIONS:
            raise ValueError(f'reduction_override must be None or one of {_REDUCTIONS}, got {reduction_override!r}')
        reduction = reduction_override if reduction_override else self.reduction
        if weight is not None and weight.dim() > 1:
            weight = weight.mean(-1)
        return self.loss_weight * weight_reduce_loss(1 - rotated_iou_3d(pred, target), weight, reduction, avg_factor)


_CD_MODE_CODE = {'l1': 0, 'l2': 1, 'smooth_l1': 2}     # ESB_CD_L1 / ESB_CD_L2 / ESB_CD_SMOOTH_L1


class _ChamferNN(torch.autograd.Function):
    """csrc/chamfer.cu: nearest-neighbour distances in both directions (dist1 (B,N), dist2 (B,M)) and their int64
    arg-minima; backward maps d/d dist1 and d/d dist2 to the points, deterministically."""

    @staticmethod
    def forward(ctx, src, dst, mode):
        s, d = src.float().contiguous(), dst.float().contiguous()
        B, N, C = s.shape
        M = d.shape[1]
        dev = s.device
        dist1 = torch.empty((B, N), dtype=torch.float32, device=dev)
        dist2 = torch.empty((B, M), dtype=torch.float32, device=dev)
        idx1 = torch.empty((B, N), dtype=torch.int64, device=dev)
        idx2 = torch.empty((B, M), dtype=torch.int64, device=dev)
        call('esb_chamfer_fwd', ptr(s), ptr(d), B, N, M, C, _CD_MODE_CODE[mode], ptr(dist1), ptr(dist2), ptr(idx1),
             ptr(idx2), stream())
        ctx.save_for_backward(s, d, idx1, idx2)
        ctx.mode, ctx.dtypes = mode, (src.dtype, dst.dtype)
        ctx.mark_non_differentiable(idx1, idx2)
        return dist1, dist2, idx1, idx2

    @staticmethod
    def backward(ctx, g1, g2, _g_idx1, _g_idx2):
        s, d, idx1, idx2 = ctx.saved_tensors
        B, N, C = s.shape
        M = d.shape[1]
        g1 = None if g1 is None else g1.float().contiguous()
        g2 = None if g2 is None else g2.float().contiguous()
        grad_src, grad_dst = torch.empty_like(s), torch.empty_like(d)
        call('esb_chamfer_bwd', ptr(s), ptr(d), ptr(idx1), ptr(idx2), ptr(g1), ptr(g2), B, N, M, C,
             _CD_MODE_CODE[ctx.mode], ptr(grad_src), ptr(grad_dst), stream())
        return grad_src.to(ctx.dtypes[0]), grad_dst.to(ctx.dtypes[1]), None


def chamfer_distance(src, dst, src_weight=1.0, dst_weight=1.0, criterion_mode='l2', reduction='mean'):
    """chamfer_distance.py:13-79 on csrc/chamfer.cu. src (B,N,C), dst (B,M,C) CUDA tensors, 1 <= C <= 8, computed in fp32.
    Returns (loss_src, loss_dst, indices1 (B,N), indices2 (B,M)); on ties the lowest index wins. The weights (float or
    tensors broadcasting to (B,N) / (B,M)) and the reduction are applied in ATen, so tensor weights get gradients."""
    if criterion_mode not in CD_MODES:
        raise NotImplementedError(f'criterion_mode must be one of {CD_MODES}, got {criterion_mode!r}')
    if reduction not in CD_REDUCTIONS:
        raise NotImplementedError(f'reduction must be one of {CD_REDUCTIONS}, got {reduction!r}')
    if src.dim() != 3 or dst.dim() != 3 or src.shape[0] != dst.shape[0] or src.shape[2] != dst.shape[2]:
        raise ValueError(f'chamfer_distance takes src (B, N, C) and dst (B, M, C), got {tuple(src.shape)} and '
                         f'{tuple(dst.shape)}')
    if not (src.is_cuda and dst.is_cuda):
        raise ValueError('chamfer_distance runs on CUDA tensors only (there is no CPU implementation)')
    if not (src.is_floating_point() and dst.is_floating_point()):
        raise ValueError('chamfer_distance takes floating-point points')
    if src.shape[2] < 1 or src.shape[2] > 8:
        raise ValueError(f'chamfer_distance supports 1 to 8 coordinates per point, got C={src.shape[2]}')
    if src.numel() == 0 or dst.numel() == 0:
        raise ValueError(f'chamfer_distance of an empty point set: src {tuple(src.shape)}, dst {tuple(dst.shape)}')
    dist1, dist2, indices1, indices2 = _ChamferNN.apply(src, dst, criterion_mode)
    loss_src = dist1 * src_weight
    loss_dst = dist2 * dst_weight
    if reduction == 'sum':
        loss_src, loss_dst = loss_src.sum(), loss_dst.sum()
    elif reduction == 'mean':
        loss_src, loss_dst = loss_src.mean(), loss_dst.mean()
    return loss_src, loss_dst, indices1, indices2


@MODELS.register_module()
class ChamferDistance(nn.Module):
    """embodiedscan/models/losses/chamfer_distance.py:82-157 on the chamfer_distance kernel above."""

    def __init__(self, mode='l2', reduction='mean', loss_src_weight=1.0, loss_dst_weight=1.0):
        super().__init__()
        _check_cd_options(mode=mode, reduction=reduction)
        self.mode, self.reduction = mode, reduction
        self.loss_src_weight, self.loss_dst_weight = loss_src_weight, loss_dst_weight

    def forward(self, source, target, src_weight=1.0, dst_weight=1.0, reduction_override=None, return_indices=False,
                **kwargs):
        _check_cd_options(reduction=reduction_override)
        reduction = reduction_override if reduction_override else self.reduction
        loss_source, loss_target, indices1, indices2 = chamfer_distance(source, target, src_weight, dst_weight, self.mode,
                                                                        reduction)
        loss_source = loss_source * self.loss_src_weight
        loss_target = loss_target * self.loss_dst_weight
        if return_indices:
            return loss_source, loss_target, indices1, indices2
        return loss_source, loss_target


@MODELS.register_module(name=['mmdet.FocalLoss', 'FocalLoss'])
class FocalLoss(nn.Module):
    """mmdet.FocalLoss(use_sigmoid=True, gamma=2, alpha=.25, reduction='mean') on mmcv's CUDA sigmoid_focal_loss:
    label -1 (or any label outside [0, C)) means "no positive class" (SURVEY H6)."""

    def __init__(self, use_sigmoid=True, gamma=2.0, alpha=0.25, reduction='mean', loss_weight=1.0, **kwargs):
        super().__init__()
        assert use_sigmoid and reduction == 'mean'
        self.gamma, self.alpha, self.loss_weight = gamma, alpha, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, row_weight=None):
        """Integer targets (N,) on (N,C) logits: mmcv's CUDA op semantics, sum(focal) / avg_factor, or
        sum(row_weight[r] * focal[r, :]) when per-row weights are given. Float targets of pred's shape: mmdet's
        ``py_sigmoid_focal_loss`` (soft / token-level targets, the grounding head's call, grounding_head.py:760-763)."""
        if target.is_floating_point() and target.shape == pred.shape:
            return sigmoid_focal_loss_soft(pred, target, weight, self.gamma, self.alpha, avg_factor) * self.loss_weight
        if row_weight is None:
            if not torch.is_tensor(avg_factor):
                avg_factor = torch.tensor(float(avg_factor), device=pred.device)
            row_weight = (1.0 / avg_factor.to(torch.float32).reshape(1)).expand(pred.shape[0]).contiguous()
        return _Focal.apply(pred, target, row_weight, self.gamma, self.alpha) * self.loss_weight


def sigmoid_focal_loss_soft(pred, target, weight=None, gamma=2.0, alpha=0.25, avg_factor=None):
    """mmdet ``py_sigmoid_focal_loss`` + ``weight_reduce_loss(reduction='mean')`` (†upstream): with an avg_factor the
    result is sum / (avg_factor + eps_fp32), else the plain mean."""
    pred = pred.float()
    p = pred.sigmoid()
    target = target.type_as(pred)
    pt = (1 - p) * target + p * (1 - target)
    focal_weight = (alpha * target + (1 - alpha) * (1 - target)) * pt.pow(gamma)
    loss = F.binary_cross_entropy_with_logits(pred, target, reduction='none') * focal_weight
    if weight is not None:
        loss = loss * weight
    if avg_factor is None:
        return loss.mean()
    return loss.sum() / (avg_factor + torch.finfo(torch.float32).eps)


class _Focal(torch.autograd.Function):

    @staticmethod
    def forward(ctx, logits, target, row_w, gamma, alpha):
        logits = logits.contiguous()
        row_w = row_w.to(torch.float32).contiguous()
        n, C = logits.shape
        total = torch.zeros(1, dtype=torch.float32, device=logits.device)
        call('esb_focal_loss_fwd', ptr(logits), ptr(target), n, C, gamma, alpha, ptr(row_w), ptr(total),
             _ffi.dtype_code(logits.dtype), stream())
        ctx.save_for_backward(logits, target, row_w)
        ctx.hp = (gamma, alpha)
        return total.squeeze(0)

    @staticmethod
    def backward(ctx, g):
        logits, target, row_w = ctx.saved_tensors
        gamma, alpha = ctx.hp
        scale = g.to(torch.float32).reshape(1).contiguous()
        grad = torch.empty_like(logits)
        n, C = logits.shape
        call('esb_focal_loss_bwd', ptr(logits), ptr(target), n, C, gamma, alpha, ptr(row_w), ptr(scale), ptr(grad),
             _ffi.dtype_code(logits.dtype), stream())
        return grad, None, None, None, None


@MODELS.register_module(name=['mmdet.CrossEntropyLoss', 'CrossEntropyLoss'])
class CrossEntropyLoss(nn.Module):
    """mmdet.CrossEntropyLoss(use_sigmoid=True): BCE-with-logits, 'mean' over avg_factor."""

    def __init__(self, use_sigmoid=False, reduction='mean', loss_weight=1.0, **kwargs):
        super().__init__()
        assert use_sigmoid and reduction == 'mean'
        self.loss_weight = loss_weight

    def forward(self, pred, target, avg_factor):
        loss = F.binary_cross_entropy_with_logits(pred.float(), target.float(), reduction='none')
        return loss.sum() / avg_factor * self.loss_weight


class _BBoxCD(torch.autograd.Function):
    """Fused decode + decoupled corner-chamfer loss over the positives (csrc/head.cu::bbox_cd_loss_kernel): value and
    the gradient w.r.t. the 12 regression channels in one launch; backward only scales the stored gradient.
    mode 'l1' / 'l2' / 'smooth_l1', group 'g8' / 'g4'; norm_decouple divides the three decoupled terms of a row by
    clamp(|target size|, 0.1)."""

    @staticmethod
    def forward(ctx, points, bbox_pred, targets, row_w, weights, mode='l1', group='g8', norm_decouple=False):
        P = bbox_pred.shape[0]
        dev = bbox_pred.device
        loss = torch.zeros(1, dtype=torch.float32, device=dev)
        grad = torch.empty((P, 12), dtype=torch.float32, device=dev)
        w4 = (ctypes.c_float * 4)(*[float(w) for w in weights])
        call('esb_bbox_cd_loss', ptr(points.float().contiguous()), ptr(bbox_pred.float().contiguous()),
             ptr(targets.float().contiguous()), ptr(row_w.float().contiguous()), ctypes.cast(w4, ctypes.c_void_p), P,
             _CD_MODE_CODE[mode], 8 if group == 'g8' else 4, 1 if norm_decouple else 0, ptr(loss), ptr(grad), stream())
        ctx.save_for_backward(grad)
        ctx.dtype = bbox_pred.dtype
        return loss.squeeze(0)

    @staticmethod
    def backward(ctx, g):
        (grad, ) = ctx.saved_tensors
        return None, (grad * g).to(ctx.dtype), None, None, None, None, None, None


def fcaf3d_targets_batched(points: torch.Tensor, level_sizes: List[int], pt_batch: Optional[torch.Tensor],
                            boxes9_list: List[torch.Tensor], labels_list: List[torch.Tensor], assign_thr: int,
                            center_thr: int):
    """Fused get_targets (fcaf3d_head.py:1578-1664) for ALL scans of the batch in one kernel pipeline.
    points (Np,3) level by level (natural row order, scans interleaved), pt_batch (Np) int32 scan ids,
    boxes9_list[b] (Ng_b, 9) gravity-centred. Returns center_t (Np), bbox_t (Np,9), cls_t (Np) int64."""
    dev = points.device
    pts = points.float().contiguous()
    Np, L, B = pts.shape[0], len(level_sizes), len(boxes9_list)
    offs = [0]
    for n in level_sizes:
        offs.append(offs[-1] + n)
    box_offs = [0]
    for bx in boxes9_list:
        box_offs.append(box_offs[-1] + bx.shape[0])
    NgT, max_ng = box_offs[-1], max([bx.shape[0] for bx in boxes9_list] + [0])
    meta = torch.tensor(offs + box_offs, dtype=torch.int32).to(dev, non_blocking=True)
    level_off, box_off = meta[:L + 1], meta[L + 1:]
    boxes = torch.cat([bx.float() for bx in boxes9_list]).to(dev).contiguous() if NgT else pts.new_zeros((0, 9))
    labels = torch.cat([lb.to(torch.int64) for lb in labels_list]).to(dev).contiguous() if NgT else \
        torch.zeros((0, ), dtype=torch.int64, device=dev)
    rneg = euler_angles_to_matrix(-boxes[:, 6:9], 'ZXY').contiguous().view(-1, 9)
    center_t = torch.empty(Np, dtype=torch.float32, device=dev)
    bbox_t = torch.empty((Np, 9), dtype=torch.float32, device=dev)
    cls_t = torch.empty(Np, dtype=torch.int64, device=dev)
    wsb = query('esb_fcaf3d_targets_workspace_bytes', L, max(NgT, 1), B)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    call('esb_fcaf3d_targets', ptr(pts), ptr(level_off), L, Np, ptr(pt_batch), ptr(boxes), ptr(rneg), ptr(labels),
         ptr(box_off), B, NgT, max_ng, assign_thr, center_thr, ptr(center_t), ptr(bbox_t), ptr(cls_t), None, ptr(ws), wsb,
         stream())
    return center_t, bbox_t, cls_t


def fcaf3d_targets(points_lvls: List[torch.Tensor], gt_boxes9: torch.Tensor, gt_labels: torch.Tensor,
                   assign_thr: int, center_thr: int):
    """Single-scan form of the reference's get_targets(points, gt_bboxes, gt_labels)."""
    return fcaf3d_targets_batched(torch.cat(points_lvls), [p.shape[0] for p in points_lvls], None,
                                  [gt_boxes9.to(points_lvls[0].device)], [gt_labels.to(points_lvls[0].device)],
                                  assign_thr, center_thr)


def multiclass_nms_bev(bboxes: torch.Tensor, scores: torch.Tensor, score_thr: float, iou_thr: float,
                       with_yaw: bool = True):
    """_single_scene_multiclass_nms (fcaf3d_head.py:1666-1725) as one segmented launch.
    Returns (boxes (M, 7 or 6), scores (M,), labels (M,) int64) ordered class-major, score-descending (stable)."""
    dev = bboxes.device
    if bboxes.shape[-1] == 9:
        bboxes = bboxes[..., :7]
    if not with_yaw:
        bboxes = torch.cat((bboxes[:, :6], torch.zeros_like(bboxes[:, :1])), 1)
    C = scores.shape[1]
    cls_idx, box_idx = torch.nonzero((scores > score_thr).t(), as_tuple=True)
    if cls_idx.numel() == 0:
        return bboxes.new_zeros((0, 7 if with_yaw else 6)), bboxes.new_zeros((0, )), \
            torch.zeros((0, ), dtype=torch.long, device=dev)
    s = scores[box_idx, cls_idx]
    o1 = torch.sort(s, descending=True, stable=True).indices
    o2 = torch.sort(cls_idx[o1], stable=True).indices
    order = o1[o2]
    cls_s, box_s, s_s = cls_idx[order], box_idx[order], s[order]
    boxes_s = bboxes[box_s].float().contiguous()
    seg_off = torch.searchsorted(cls_s, torch.arange(C + 1, device=dev)).to(torch.int32)
    max_seg = int((seg_off[1:] - seg_off[:-1]).max().item())
    keep = torch.empty(boxes_s.shape[0], dtype=torch.uint8, device=dev)
    call('esb_nms_bev_segmented', ptr(boxes_s), ptr(seg_off), C, max_seg, float(iou_thr), 1 if with_yaw else 0, ptr(keep),
         stream())
    sel = keep.bool()
    out_boxes = boxes_s[sel]
    if not with_yaw:
        out_boxes = out_boxes[:, :6]
    return out_boxes, s_s[sel], cls_s[sel]


class SparseFPN(nn.Module):
    """The pruned sparse FPN of FCAF3D (fcaf3d_head.py:993-1114, mink_neck.py:133-244), shared by ``FCAF3DHeadRotMat``
    and ``MinkNeck``. Subclasses set ``pts_prune_threshold`` and call ``_init_fpn`` where the reference builds the
    blocks, so parameters register in the reference's order."""

    def _init_fpn(self, in_channels, out_channels):
        self.pruning = SP.MinkowskiPruning()
        for i in range(len(in_channels)):
            if i > 0:
                setattr(self, f'up_block_{i}', self._make_up_block(in_channels[i], in_channels[i - 1]))
            setattr(self, f'out_block_{i}', self._make_block(in_channels[i], out_channels))

    @staticmethod
    def _make_block(in_channels, out_channels):
        return nn.Sequential(SP.MinkowskiConvolution(in_channels, out_channels, kernel_size=3, dimension=3),
                             SP.MinkowskiBatchNorm(out_channels), SP.MinkowskiELU())

    @staticmethod
    def _make_up_block(in_channels, out_channels):
        return nn.Sequential(
            SP.MinkowskiGenerativeConvolutionTranspose(in_channels, out_channels, kernel_size=2, stride=2, dimension=3),
            SP.MinkowskiBatchNorm(out_channels), SP.MinkowskiELU(),
            SP.MinkowskiConvolution(out_channels, out_channels, kernel_size=3, dimension=3),
            SP.MinkowskiBatchNorm(out_channels), SP.MinkowskiELU())

    def _run_block(self, seq: nn.Sequential, x: SP.SparseTensor) -> SP.SparseTensor:
        """(conv|deconv) -> BN -> ELU triples with BN+ELU fused into one kernel."""
        mods = list(seq)
        assert len(mods) % 3 == 0
        for i in range(0, len(mods), 3):
            x = SP.conv_norm_act(mods[i], mods[i + 1], SP.ACT_ELU, x, training=self.training)
        return x

    def _top_down(self, inputs: List[SP.SparseTensor], level_fn) -> list:
        """Top-down pass (fcaf3d_head.py:993-1020): from the coarsest level, up block, union add with the finer input and
        prune by the coarser level's score, then the level's out block. ``level_fn(i, out)`` returns (result, prune score
        for the next finer level); the results come back coarse -> fine."""
        results = []
        x = inputs[-1]
        prune_score = None
        for i in range(len(inputs) - 1, -1, -1):
            if i < len(inputs) - 1:
                x = self._run_block(getattr(self, f'up_block_{i + 1}'), x)
                x = inputs[i] + x
                x = self._prune(x, prune_score)
            res, prune_score = level_fn(i, self._run_block(getattr(self, f'out_block_{i}'), x))
            results.append(res)
        return results

    def _prune(self, x: SP.SparseTensor, scores: SP.SparseTensor) -> SP.SparseTensor:
        """Per-scan top-k by the multilinearly interpolated parent max-class score (fcaf3d_head.py:1091-1114).
        Identity whenever every scan holds <= pts_prune_threshold rows."""
        if len(x) <= self.pts_prune_threshold:      # no scan can exceed the threshold: skip without a host sync
            return x
        perms, _, counts = x.cmap.decomposition(x.coordinate_manager.batch_size)
        if max(counts) <= self.pts_prune_threshold:
            return x
        with torch.no_grad():
            interpolated = scores.features_at_coordinates(x.C)      # integer child coordinates: the fused kernel
            prune_mask = torch.zeros(len(interpolated), dtype=torch.bool, device=x.device)
            for perm in perms:
                score = interpolated[perm].squeeze(1)
                topk = min(len(score), self.pts_prune_threshold)
                # torch.topk leaves ties unspecified; frozen rule: descending score, lowest row first among ties
                ids = torch.sort(score, descending=True, stable=True).indices[:topk]
                prune_mask[perm[ids]] = True
        return self.pruning(x, prune_mask)


class FCAF3DHeadBase(SparseFPN):
    """What the reference's two FCAF3D heads share line for line (fcaf3d_head.py: ``forward`` / ``_prune``,
    ``_forward_single``, ``get_targets``, ``predict_by_feat`` and the NMS at :179-335, 461-540, 626-824 and
    :993-1149, 1352-1431, 1527-1725): the layers, the forward pass, target assignment, the focal and centre losses and
    predict. A subclass decodes boxes (``_bbox_pred_to_bbox``) and adds the box term of the loss (``_box_loss``)."""

    def _init_layers(self, in_channels, out_channels, num_reg_outs, num_classes):
        self._init_fpn(in_channels, out_channels)
        self.conv_center = SP.MinkowskiConvolution(out_channels, 1, kernel_size=1, dimension=3)
        self.conv_reg = SP.MinkowskiConvolution(out_channels, num_reg_outs, kernel_size=1, dimension=3)
        self.conv_cls = SP.MinkowskiConvolution(out_channels, num_classes, kernel_size=1, bias=True, dimension=3)
        self.scales = nn.ModuleList([Scale(1.) for _ in range(len(in_channels))])

    def init_weights(self):
        nn.init.normal_(self.conv_center.kernel, std=.01)
        nn.init.normal_(self.conv_reg.kernel, std=.01)
        nn.init.normal_(self.conv_cls.kernel, std=.01)
        nn.init.constant_(self.conv_cls.bias, -4.59511985013459)  # bias_init_with_prob(.01)

    # ---- forward ------------------------------------------------------------------------------------------
    def _forward_levels(self, x: List[SP.SparseTensor]):
        """Top-down pass (fcaf3d_head.py:993-1020). Returns, per level (fine -> coarse), a dict of whole-batch tensors
        center (N,1), bbox (N,num_reg_outs), cls (N,C), points (N,3), batch (N,) int32, perms (per-scan row indices)."""
        f0 = x[-1].F
        w_all = self._head_weights(f0) if f0.is_cuda and f0.dtype == torch.bfloat16 else None
        return self._top_down(x, lambda i, out: self._forward_single_level(out, self.scales[i], need_prune_score=i > 0,
                                                                           w_all=w_all))[::-1]

    def forward(self, x: List[SP.SparseTensor]):
        """Reference return format: four lists (level-major) of per-scan tensor lists."""
        center_preds, bbox_preds, cls_preds, points = [], [], [], []
        for lv in self._forward_levels(x):
            perms = lv['tensor'].decomposition_permutations
            center_preds.append([lv['center'][p] for p in perms])
            bbox_preds.append([lv['bbox'][p] for p in perms])
            cls_preds.append([lv['cls'][p] for p in perms])
            points.append([lv['points'][p] for p in perms])
        return center_preds, bbox_preds, cls_preds, points

    def _head_weights(self, f: torch.Tensor):
        """[cls | centre | reg | zero pad] (C_in, width) fp32, width a multiple of 64: the operand of the ONE tensor-core GEMM
        behind the three 1x1 heads. The heads are shared by all levels, so it is concatenated once per pass; each level
        casts it to the feature dtype itself, which keeps the sum of the per-level weight gradients in fp32."""
        n_cls, n_reg = self.conv_cls.kernel.shape[1], self.conv_reg.kernel.shape[1]
        width = (n_cls + 1 + n_reg + 63) // 64 * 64
        return torch.cat([self.conv_cls.kernel, self.conv_center.kernel, self.conv_reg.kernel,
                          self.conv_cls.kernel.new_zeros(self.conv_cls.kernel.shape[0], width - n_cls - 1 - n_reg)], 1)

    def _forward_single_level(self, x: SP.SparseTensor, scale: Scale, need_prune_score: bool = True, w_all=None):
        """_forward_single (fcaf3d_head.py:1116-1149) on whole-batch rows: bf16 features with a multiple of 64 channels take
        one GEMM for the three 1x1 heads (rows_gemm), other rows one product for cls and one for centre + reg. Everything after
        the products (bias, Scale, exp, clamp, the column split and the pruning score) is ATen."""
        f = x.F
        coords = x.C
        n_cls, n_reg = self.conv_cls.kernel.shape[1], self.conv_reg.kernel.shape[1]
        if f.is_cuda and f.dtype == torch.bfloat16 and f.shape[1] % 64 == 0:
            out = SP.rows_gemm(f, (self._head_weights(f) if w_all is None else w_all).to(f.dtype))
            cls_pred = out[:, :n_cls] + self.conv_cls.bias.to(f.dtype)
            small = out[:, n_cls:n_cls + 1 + n_reg].float()
        else:
            w_small = torch.cat([self.conv_center.kernel, self.conv_reg.kernel], 1).to(f.dtype)
            small = (f @ w_small).float()
            cls_pred = torch.addmm(self.conv_cls.bias.to(f.dtype), f, self.conv_cls.kernel.to(f.dtype))
        center_pred = small[:, :1]
        reg_final = small[:, 1:]
        prune_scores = x.replace_feature(cls_pred.max(dim=1, keepdim=True).values.float()) if need_prune_score else None
        reg_distance = torch.exp(scale(reg_final[:, :6])).clamp(min=1e-3)
        bbox_pred = torch.cat((reg_distance, reg_final[:, 6:]), dim=1)
        lv = dict(center=center_pred, bbox=bbox_pred, cls=cls_pred, points=coords[:, 1:] * self.voxel_size,
                  batch=coords[:, 0].contiguous(), tensor=x)
        return lv, prune_scores

    # ---- loss ---------------------------------------------------------------------------------------------
    def loss(self, x, batch_data_samples, **kwargs) -> dict:
        levels = self._forward_levels(x)
        gts = [ds.gt_instances_3d for ds in batch_data_samples]
        return self.loss_by_levels(levels, gts)

    def _reduce_mean(self, t: torch.Tensor) -> torch.Tensor:
        """utils/dist_utils.py:4-10 for the whole batch at once, on the device."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return t
        t = t / dist.get_world_size(self.process_group)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.process_group)
        return t

    def loss_by_feat(self, center_preds, bbox_preds, cls_preds, points, batch_gt_instances_3d, batch_input_metas=None,
                     batch_gt_instances_ignore=None, **kwargs) -> dict:
        """Reference signature (lists of per-scan tensors); regrouped into whole-batch rows for the fused path."""
        dev = points[0][0].device
        levels = []
        for l in range(len(points)):
            B = len(points[l])
            levels.append(dict(center=torch.cat(center_preds[l]), bbox=torch.cat(bbox_preds[l]), cls=torch.cat(cls_preds[l]),
                               points=torch.cat(points[l]),
                               batch=torch.cat([torch.full((len(points[l][b]), ), b, dtype=torch.int32, device=dev)
                                                for b in range(B)])))
        return self.loss_by_levels(levels, batch_gt_instances_3d)

    def loss_by_levels(self, levels, batch_gt_instances_3d) -> dict:
        """_loss_by_feat_single + the batch mean (fcaf3d_head.py:337-459, 1151-1350), evaluated for all scans at once:
        per-scan normalisers become per-row weights, so there is no Python loop over scans and one host sync."""
        B = len(batch_gt_instances_3d)
        dev = levels[0]['points'].device
        pts = torch.cat([lv['points'] for lv in levels])
        pt_batch = torch.cat([lv['batch'] for lv in levels]).contiguous()
        sizes = [lv['points'].shape[0] for lv in levels]
        boxes9 = [torch.cat((g.bboxes_3d.gravity_center, g.bboxes_3d.tensor[:, 3:]), 1) for g in batch_gt_instances_3d]
        labels = [g.labels_3d for g in batch_gt_instances_3d]
        center_t, bbox_t, cls_t = fcaf3d_targets_batched(pts, sizes, pt_batch, boxes9, labels, self.pts_assign_threshold,
                                                         self.pts_center_threshold)
        pos_mask = cls_t >= 0
        pb_all = pt_batch.long()
        # positives per scan: a (B, N) one-hot reduction (index_add_ into B bins serialises ~100k atomics: 0.7 ms)
        scan_ids = torch.arange(B, device=dev, dtype=pb_all.dtype).unsqueeze(1)
        pos_in_scan = (pb_all.unsqueeze(0) == scan_ids) & pos_mask.unsqueeze(0)
        n_pos_local = pos_in_scan.sum(1).float()
        scan_sums = self._scan_box_sums(pos_in_scan, center_t)
        if scan_sums is None:
            n_pos = torch.clamp(self._reduce_mean(n_pos_local.clone()), min=1.)      # (B,) one fused all-reduce
        else:                                                                        # (2B,): still one all-reduce
            reduced = self._reduce_mean(torch.cat((n_pos_local, scan_sums)))
            n_pos, scan_sums = torch.clamp(reduced[:B], min=1.), reduced[B:]
        row_w = (1.0 / (n_pos * B))[pb_all]                                         # 1/(n_pos[scan] * B) per row
        # classification: sum_rows focal(row) / n_pos[scan(row)], mean over scans
        loss_cls, off = 0., 0
        for lv, n in zip(levels, sizes):
            loss_cls = loss_cls + self.cls_loss(lv['cls'], cls_t[off:off + n], row_weight=row_w[off:off + n])
            off += n
        center_preds = torch.cat([lv['center'] for lv in levels])
        bbox_preds = torch.cat([lv['bbox'] for lv in levels])
        pos_inds = torch.nonzero(pos_mask).squeeze(1)                                # the one host sync of the loss
        pos_center_preds = center_preds[pos_inds]
        pos_bbox_preds = bbox_preds[pos_inds]
        if pos_inds.numel() > 0:
            w_pos = row_w[pos_inds]
            pos_center_t = center_t[pos_inds]
            bce = F.binary_cross_entropy_with_logits(pos_center_preds.float(), pos_center_t.unsqueeze(1), reduction='none')
            loss_center = (bce.squeeze(1) * w_pos).sum() * self.center_loss.loss_weight
            loss_bbox = self._box_loss(pts[pos_inds], pos_bbox_preds, bbox_t[pos_inds], pos_center_t, pb_all[pos_inds],
                                       n_pos_local, scan_sums, B)
        else:
            loss_center = pos_center_preds.sum()
            loss_bbox = pos_bbox_preds.sum()
        return dict(loss_center=loss_center, loss_bbox=loss_bbox, loss_cls=loss_cls)

    def _scan_box_sums(self, pos_in_scan: torch.Tensor, center_t: torch.Tensor) -> Optional[torch.Tensor]:
        """(B,) per-scan sums the box term is normalised by, all-reduced (mean) together with the positive counts; None
        when the box term needs none."""
        return None

    def _box_loss(self, points, bbox_pred, bbox_t, center_t, batch, n_pos_local, scan_sums, B):
        """The box term over the P positives: their points (P,3), regression outputs, 9-DoF targets (P,9), centre targets
        (P,), scan ids (P,), the local positive counts per scan (B,) and the all-reduced ``_scan_box_sums`` (or None)."""
        raise NotImplementedError

    def get_targets(self, points, gt_bboxes, gt_labels):
        boxes9 = torch.cat((gt_bboxes.gravity_center, gt_bboxes.tensor[:, 3:]), 1).to(points[0].device)
        return fcaf3d_targets(points, boxes9, gt_labels.to(points[0].device), self.pts_assign_threshold,
                              self.pts_center_threshold)

    # ---- predict ------------------------------------------------------------------------------------------
    def predict(self, x, batch_data_samples, rescale: bool = False):
        metas = [ds.metainfo for ds in batch_data_samples]
        outs = self(x)
        return self.predict_by_feat(*outs, batch_input_metas=metas, rescale=rescale)

    def predict_by_feat(self, center_preds, bbox_preds, cls_preds, points, batch_input_metas, **kwargs):
        return [
            self._predict_by_feat_single([x[i] for x in center_preds], [x[i] for x in bbox_preds],
                                         [x[i] for x in cls_preds], [x[i] for x in points], batch_input_metas[i])
            for i in range(len(batch_input_metas))
        ]

    def _predict_by_feat_single(self, center_preds, bbox_preds, cls_preds, points, input_meta) -> InstanceData:
        nms_pre = self.test_cfg['nms_pre']
        mlvl_bboxes, mlvl_scores = [], []
        for center_pred, bbox_pred, cls_pred, point in zip(center_preds, bbox_preds, cls_preds, points):
            scores = cls_pred.sigmoid() * center_pred.sigmoid()
            max_scores, _ = scores.max(dim=1)
            if len(scores) > nms_pre > 0:
                _, ids = max_scores.topk(nms_pre)
                bbox_pred, scores, point = bbox_pred[ids], scores[ids], point[ids]
            mlvl_bboxes.append(self._bbox_pred_to_bbox(point, bbox_pred))
            mlvl_scores.append(scores)
        bboxes = torch.cat(mlvl_bboxes)
        scores = torch.cat(mlvl_scores)
        bboxes, scores, labels = multiclass_nms_bev(bboxes, scores, self.test_cfg['score_thr'], self.test_cfg['iou_thr'],
                                                    with_yaw=True)
        box_type = input_meta.get('box_type_3d', EulerDepthInstance3DBoxes)
        results = InstanceData()
        # 9-DoF boxes are truncated to 7 columns by the NMS stage and padded back with zero beta/gamma (SURVEY H4)
        results.bboxes_3d = box_type(bboxes, box_dim=bboxes.shape[1], with_yaw=bboxes.shape[1] == 7,
                                     origin=(.5, .5, .5))
        results.scores_3d = scores
        results.labels_3d = labels
        return results


@MODELS.register_module()
class FCAF3DHeadRotMat(FCAF3DHeadBase):

    def __init__(self, num_classes: int, in_channels: Tuple[int], out_channels: int, num_reg_outs: int,
                 voxel_size: float, pts_prune_threshold: int, pts_assign_threshold: int, pts_center_threshold: int,
                 center_loss: dict = dict(type='mmdet.CrossEntropyLoss', use_sigmoid=True),
                 bbox_loss: dict = dict(type='BBoxCDLoss', mode='l1', loss_weight=1.0, group='g8'),
                 cls_loss: dict = dict(type='mmdet.FocalLoss'), decouple_bbox_loss: bool = False,
                 decouple_groups: int = 3, decouple_weights: Optional[list] = None, norm_decouple_loss: bool = False,
                 train_cfg: Optional[dict] = None, test_cfg: Optional[dict] = None, init_cfg: Optional[dict] = None):
        super().__init__()
        self.voxel_size = voxel_size
        self.pts_prune_threshold = pts_prune_threshold
        self.pts_assign_threshold = pts_assign_threshold
        self.pts_center_threshold = pts_center_threshold
        self.center_loss = MODELS.build(center_loss)
        self.bbox_loss = MODELS.build(bbox_loss)
        check_head_box_loss(self.bbox_loss)
        self.cls_loss = MODELS.build(cls_loss)
        self.decouple_bbox_loss = decouple_bbox_loss
        self.decouple_groups = decouple_groups
        self.norm_decouple_loss = norm_decouple_loss
        self.decouple_weights = decouple_weights or [1.0 / decouple_groups] * decouple_groups
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.num_classes = num_classes
        self._init_layers(in_channels, out_channels, num_reg_outs, num_classes)
        self.init_weights()
        self.process_group = None

    def _box_loss(self, points, bbox_pred, tgt, center_t, batch, n_pos_local, scan_sums, B):
        """BBoxCDLoss on the decoded positives (fcaf3d_head.py:1224-1281)."""
        # per-scan mean over (P_scan x K) corners, then mean over scans -> weight 1 / (K * P_scan * B) per corner; K = 8
        # for 'g8', and 4 for 'g4', whose mean is mean(corners 0-3) + mean(corners 4-7)
        mode, group = self.bbox_loss.mode, self.bbox_loss.group
        p_scan = n_pos_local[batch]
        w_box = (1.0 / ((8.0 if group == 'g8' else 4.0) * p_scan * B))[:, None]
        norm = self.decouple_bbox_loss and self.norm_decouple_loss
        fused = bbox_pred.is_cuda and bbox_pred.shape[1] == 12 and \
            (not self.decouple_bbox_loss or self.decouple_groups in (3, 4))
        if fused:
            if self.decouple_bbox_loss:
                wts = list(self.decouple_weights[:3]) + [self.decouple_weights[3] if self.decouple_groups == 4 else 0.]
            else:
                wts = [0., 0., 0., 1.]
            return _BBoxCD.apply(points, bbox_pred, tgt, w_box[:, 0] * self.bbox_loss.loss_weight, wts, mode, group, norm)
        decoded = self._bbox_pred_to_bbox(points, bbox_pred)
        tgt_corners = bbox_to_corners(tgt)

        def cd(src, w=w_box):
            return (chamfer_src(bbox_to_corners(src), tgt_corners, mode, group) * w).sum() * self.bbox_loss.loss_weight

        if self.decouple_bbox_loss:
            tc, ts, te = tgt[:, :3], tgt[:, 3:6], tgt[:, 6:]
            pc, ps, pe = decoded[:, :3], decoded[:, 3:6], decoded[:, 6:]
            assert self.decouple_groups in (3, 4)
            # norm_decouple_loss: the decoupled terms of a row are divided by clamp(|target size|, 0.1)
            w_dec = w_box / ts.norm(dim=-1)[:, None].clamp(min=0.1) if norm else w_box
            w = self.decouple_weights
            loss_bbox = w[0] * cd(torch.cat((pc, ts, te), -1), w_dec) + w[1] * cd(torch.cat((tc, ps, te), -1), w_dec) + \
                w[2] * cd(torch.cat((tc, ts, pe), -1), w_dec)
            if self.decouple_groups == 4:
                loss_bbox = loss_bbox + w[3] * cd(decoded)
            return loss_bbox
        return cd(decoded)

    @staticmethod
    def _bbox_pred_to_bbox(points: torch.Tensor, bbox_pred: torch.Tensor) -> torch.Tensor:
        """(N,3) + (N,12) [6 face distances, 6D rotation] -> (N,9) centre/size/euler (fcaf3d_head.py:1454-1525)."""
        if bbox_pred.shape[0] == 0:
            return bbox_pred
        assert bbox_pred.shape[-1] == 12, 'RotMat head decodes 12-channel predictions'
        shift = torch.stack(((bbox_pred[:, 1] - bbox_pred[:, 0]) / 2, (bbox_pred[:, 3] - bbox_pred[:, 2]) / 2,
                             (bbox_pred[:, 5] - bbox_pred[:, 4]) / 2), dim=-1).view(-1, 1, 3)
        rot_mat = ortho_6d_2_mat(bbox_pred[:, 6:9], bbox_pred[:, 9:])
        euler = matrix_to_euler_angles_zxy(rot_mat)
        shift = rotation_3d_in_euler(shift, euler)[:, 0, :]
        center = points + shift
        size = torch.stack((bbox_pred[:, 0] + bbox_pred[:, 1], bbox_pred[:, 2] + bbox_pred[:, 3],
                            bbox_pred[:, 4] + bbox_pred[:, 5]), dim=-1)
        return torch.cat((center, size, euler), dim=-1)


@MODELS.register_module()
class FCAF3DHead(FCAF3DHeadBase):
    """The FCAF3D head with raw-angle box regression and the rotated 3D IoU box loss (fcaf3d_head.py:29-826).
    ``num_reg_outs`` 7: 6 face distances + 1 yaw; 9: 6 face distances + 3 ZXY Euler angles. The box loss must be a
    ``RotatedIoU3DLoss``; the reference's default ``AxisAlignedIoULoss`` is registered nowhere, so building with the
    default raises ``KeyError`` as it does there."""

    def __init__(self, num_classes: int, in_channels: Tuple[int], out_channels: int, num_reg_outs: int,
                 voxel_size: float, pts_prune_threshold: int, pts_assign_threshold: int, pts_center_threshold: int,
                 center_loss: dict = dict(type='mmdet.CrossEntropyLoss', use_sigmoid=True),
                 bbox_loss: dict = dict(type='AxisAlignedIoULoss'), cls_loss: dict = dict(type='mmdet.FocalLoss'),
                 train_cfg: Optional[dict] = None, test_cfg: Optional[dict] = None, init_cfg: Optional[dict] = None):
        super().__init__()
        if num_reg_outs not in (7, 9):
            raise ValueError(f'FCAF3DHead supports num_reg_outs 7 (yaw) or 9 (ZXY Euler angles), got {num_reg_outs}')
        self.voxel_size = voxel_size
        self.pts_prune_threshold = pts_prune_threshold
        self.pts_assign_threshold = pts_assign_threshold
        self.pts_center_threshold = pts_center_threshold
        self.center_loss = MODELS.build(center_loss)
        self.bbox_loss = MODELS.build(bbox_loss)
        if not isinstance(self.bbox_loss, RotatedIoU3DLoss):
            raise ValueError(f'FCAF3DHead supports a RotatedIoU3DLoss box loss, got {type(self.bbox_loss).__name__}')
        check_head_box_loss(self.bbox_loss)
        self.cls_loss = MODELS.build(cls_loss)
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.num_classes = num_classes
        self._init_layers(in_channels, out_channels, num_reg_outs, num_classes)
        self.init_weights()
        self.process_group = None

    def _scan_box_sums(self, pos_in_scan, center_t):
        return torch.where(pos_in_scan, center_t.unsqueeze(0), 0.).sum(1)        # the positives' centre targets

    def _box_loss(self, points, bbox_pred, tgt, center_t, batch, n_pos_local, scan_sums, B):
        """fcaf3d_head.py:377-405 and the mean over scans (:444-459): per scan, RotatedIoU3DLoss(decoded[:, :7],
        target[:, :7], weight=centre targets, avg_factor=center_denorm) with center_denorm = max(reduce_mean(sum of the
        scan's centre targets), 1e-6), i.e. one sum over all positives with the weight ct / ((center_denorm + eps) B).
        Summed directly rather than through the module's forward, whose all-zero-weight test would sync the host."""
        denorm = torch.clamp(scan_sums, min=1e-6) + torch.finfo(torch.float32).eps
        w = center_t / (denorm * B)[batch]
        iou = rotated_iou_3d(self._bbox_pred_to_bbox(points, bbox_pred)[:, :7], tgt[:, :7])
        return ((1 - iou) * w).sum() * self.bbox_loss.loss_weight

    @staticmethod
    def _bbox_pred_to_bbox(points: torch.Tensor, bbox_pred: torch.Tensor) -> torch.Tensor:
        """(N,3) + (N,7|9) [6 face distances, yaw | ZXY Euler angles] -> (N,7|9) centre/size/angles
        (fcaf3d_head.py:563-624)."""
        if bbox_pred.shape[0] == 0:
            return bbox_pred
        if bbox_pred.shape[-1] not in (7, 9):
            raise ValueError(f'FCAF3DHead decodes 7- or 9-channel predictions, got {bbox_pred.shape[-1]}')
        shift = torch.stack(((bbox_pred[:, 1] - bbox_pred[:, 0]) / 2, (bbox_pred[:, 3] - bbox_pred[:, 2]) / 2,
                             (bbox_pred[:, 5] - bbox_pred[:, 4]) / 2), dim=-1).view(-1, 1, 3)
        if bbox_pred.shape[-1] == 7:
            shift = rotation_3d_in_axis(shift, bbox_pred[:, 6], axis=2)[:, 0, :]
        else:
            shift = rotation_3d_in_euler(shift, bbox_pred[:, 6:])[:, 0, :]
        center = points + shift
        size = torch.stack((bbox_pred[:, 0] + bbox_pred[:, 1], bbox_pred[:, 2] + bbox_pred[:, 3],
                            bbox_pred[:, 4] + bbox_pred[:, 5]), dim=-1)
        return torch.cat((center, size, bbox_pred[:, 6:]), dim=-1)
