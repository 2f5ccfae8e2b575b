"""Box / rotation geometry of the hot path (device-agnostic torch; tiny tensors).

Restates the pytorch3d transforms the reference imports (†upstream pytorch3d 0.7.x, convention 'ZXY':
``R = Rz(a) @ Rx(b) @ Ry(c)``) and the helpers of ``embodiedscan/models/dense_heads/fcaf3d_head.py:1728-1750``
(``ortho_6d_2_Mat``), ``embodiedscan/models/losses/chamfer_distance.py:160-203`` (``bbox_to_corners``) and
``embodiedscan/structures/bbox_3d/euler_box3d.py:137-184`` (corner order of the box container).
"""
import torch


def _axis_rot(axis: str, angle: torch.Tensor) -> torch.Tensor:
    c, s = torch.cos(angle), torch.sin(angle)
    one, zero = torch.ones_like(angle), torch.zeros_like(angle)
    if axis == 'X':
        flat = (one, zero, zero, zero, c, -s, zero, s, c)
    elif axis == 'Y':
        flat = (c, zero, s, zero, one, zero, -s, zero, c)
    else:
        flat = (c, -s, zero, s, c, zero, zero, zero, one)
    return torch.stack(flat, -1).reshape(angle.shape + (3, 3))


def euler_angles_to_matrix(euler: torch.Tensor, convention: str = 'ZXY') -> torch.Tensor:
    mats = [_axis_rot(c, e) for c, e in zip(convention, torch.unbind(euler, -1))]
    return torch.matmul(torch.matmul(mats[0], mats[1]), mats[2])


def matrix_to_euler_angles_zxy(m: torch.Tensor) -> torch.Tensor:
    """pytorch3d.matrix_to_euler_angles(M, 'ZXY'): (alpha, beta, gamma) with
    beta = asin(M[2,1]); alpha = atan2(-M[0,1], M[1,1]); gamma = atan2(-M[2,0], M[2,2])."""
    beta = torch.asin(m[..., 2, 1])
    alpha = torch.atan2(-m[..., 0, 1], m[..., 1, 1])
    gamma = torch.atan2(-m[..., 2, 0], m[..., 2, 2])
    return torch.stack((alpha, beta, gamma), -1)


def ortho_6d_2_mat(x_raw: torch.Tensor, y_raw: torch.Tensor) -> torch.Tensor:
    """Gram-Schmidt with y first (fcaf3d_head.py:1739-1750); columns (x, y, z)."""
    y = y_raw / (torch.norm(y_raw, dim=1, keepdim=True) + 1e-8)
    z = torch.cross(x_raw, y, dim=1)
    z = z / (torch.norm(z, dim=1, keepdim=True) + 1e-8)
    x = torch.cross(y, z, dim=1)
    return torch.stack((x, y, z), 2)


def rotation_3d_in_euler(points: torch.Tensor, angles: torch.Tensor) -> torch.Tensor:
    """points (N, M, 3) @ R(angles)^T  (embodiedscan/structures/bbox_3d/utils.py:32-86)."""
    rot_t = euler_angles_to_matrix(angles, 'ZXY').transpose(-2, -1)
    if points.shape[0] == 0:
        return points
    return torch.bmm(points, rot_t)


def rotation_3d_in_axis(points: torch.Tensor, angles: torch.Tensor, axis: int = 2) -> torch.Tensor:
    """points (N, M, 3) rotated counter-clockwise about z by angles (N,): x' = x cos - y sin, y' = x sin + y cos
    (embodiedscan/structures/bbox_3d/utils.py:90-171 with clockwise=False; the same einsum). Only axis 2 is needed."""
    if axis not in (2, -1):
        raise NotImplementedError(f'rotation_3d_in_axis implements axis 2 only, got axis={axis}')
    if points.shape[0] == 0:
        return points
    c, s = torch.cos(angles), torch.sin(angles)
    o, z = torch.ones_like(c), torch.zeros_like(c)
    rot_mat_t = torch.stack([torch.stack([c, s, z]), torch.stack([-s, c, z]), torch.stack([z, z, o])])
    return torch.einsum('aij,jka->aik', points, rot_mat_t)


_CORNER_SIGNS = None


def bbox_to_corners(bbox: torch.Tensor) -> torch.Tensor:
    """(N, 9) -> (N, 8, 3) with the sign pattern of chamfer_distance.py:184-196."""
    n = bbox.shape[0]
    if bbox.shape[-1] == 9:
        rot = euler_angles_to_matrix(bbox[:, 6:], 'ZXY')
    elif bbox.shape[-1] == 7:
        ang = torch.cat((bbox[:, 6:], torch.zeros_like(bbox[:, 6:]).repeat(1, 2)), 1)
        rot = euler_angles_to_matrix(ang, 'ZXY')
    else:
        rot = torch.eye(3, device=bbox.device, dtype=bbox.dtype).expand(n, 3, 3)
    sx = bbox.new_tensor([1, 1, 1, 1, -1, -1, -1, -1])
    sy = bbox.new_tensor([1, 1, -1, -1, 1, 1, -1, -1])
    sz = bbox.new_tensor([1, -1, 1, -1, 1, -1, 1, -1])
    signs = torch.stack((sx, sy, sz), -1)[None]                      # (1, 8, 3)
    corners = signs * (bbox[:, None, 3:6] / 2)
    return bbox[:, None, :3] + torch.matmul(corners, rot.transpose(1, 2))


def box_corners_container(boxes9: torch.Tensor) -> torch.Tensor:
    """EulerInstance3DBoxes.corners order (euler_box3d.py:137-184): unravel(2,2,2)[[0,1,3,2,4,5,7,6]] - 0.5."""
    if boxes9.numel() == 0:
        return boxes9.new_zeros((0, 8, 3))
    base = torch.tensor([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]],
                        dtype=boxes9.dtype, device=boxes9.device) - 0.5
    corners = boxes9[:, None, 3:6] * base[None]
    corners = rotation_3d_in_euler(corners, boxes9[:, 6:9])
    return corners + boxes9[:, None, :3]


CD_MODES = ('l1', 'l2', 'smooth_l1')
CD_GROUPS = ('g8', 'g4')
CD_REDUCTIONS = ('mean', 'sum', 'none')


def chamfer_src(src: torch.Tensor, dst: torch.Tensor, mode: str = 'l1', group: str = 'g8') -> torch.Tensor:
    """(N,8,3),(N,8,3) -> (N,8): per source corner, the minimum over target corners of the criterion summed over x, y, z
    (chamfer_distance.py:55-61, src->dst only). Criteria: l1_loss, mse_loss, smooth_l1_loss (beta 1), reduction 'none'.
    'g4' lets corners 0-3 and 4-7 search only their own half of the target corners (chamfer_distance.py:265-276)."""
    diff = src[:, :, None, :] - dst[:, None, :, :]
    if mode == 'l1':
        d = diff.abs().sum(-1)
    elif mode == 'l2':
        d = (diff * diff).sum(-1)
    elif mode == 'smooth_l1':
        a = diff.abs()
        d = torch.where(a < 1, 0.5 * a * a, a - 0.5).sum(-1)
    else:
        raise ValueError(f'chamfer mode must be one of {CD_MODES}, got {mode!r}')
    if group == 'g8':
        return d.min(dim=2).values
    if group != 'g4':
        raise ValueError(f'chamfer group must be one of {CD_GROUPS}, got {group!r}')
    return torch.cat((d[:, :4, :4].min(dim=2).values, d[:, 4:, 4:].min(dim=2).values), 1)


def bbox_cd_loss(source: torch.Tensor, target: torch.Tensor, loss_weight: float = 1.0, mode: str = 'l1',
                 group: str = 'g8', reduction: str = 'mean', src_weight=1.0) -> torch.Tensor:
    """BBoxCDLoss (chamfer_distance.py:240-285): boxes (N, 6/7/9); src_weight a float or a tensor broadcasting to
    (N, 8) ('g8') or (N, 4) ('g4', applied to each half). 'g4' reduces each half on its own and adds the results, so
    'mean' is mean(half 1) + mean(half 2) and 'none' is the (N, 4) sum of the halves."""
    if reduction not in CD_REDUCTIONS:
        raise ValueError(f'reduction must be one of {CD_REDUCTIONS}, got {reduction!r}')
    d = chamfer_src(bbox_to_corners(source), bbox_to_corners(target), mode, group)
    weighted = torch.is_tensor(src_weight) or src_weight != 1.0
    halves = (d, ) if group == 'g8' else (d[:, :4], d[:, 4:])
    if weighted:
        halves = tuple(h * src_weight for h in halves)
    if reduction == 'mean':
        parts = [h.mean() for h in halves]
    elif reduction == 'sum':
        parts = [h.sum() for h in halves]
    else:
        parts = list(halves)
    loss = parts[0] if len(parts) == 1 else parts[0] + parts[1]
    return loss * loss_weight


def box3d_overlap(corners1: torch.Tensor, corners2: torch.Tensor, eps: float = 1e-4):
    """pytorch3d.ops.box3d_overlap contract: corners (N,8,3), (M,8,3) in the container's corner order -> (vol, iou),
    both (N,M). Exact convex clipping on the GPU (csrc/iou3d.cu); `eps` is accepted for signature parity."""
    from ._ffi import call, ptr, stream
    assert corners1.is_cuda, 'box3d_overlap runs in libesb200.so (no CPU fallback)'
    c1, c2 = corners1.float().contiguous(), corners2.float().contiguous()
    n1, n2 = c1.shape[0], c2.shape[0]
    vol = torch.empty((n1, n2), dtype=torch.float32, device=c1.device)
    iou = torch.empty((n1, n2), dtype=torch.float32, device=c1.device)
    call('esb_box3d_overlap', ptr(c1), n1, ptr(c2), n2, ptr(vol), ptr(iou), stream())
    return vol, iou


def box3d_best_overlap(qcorners: torch.Tensor, tcorners: torch.Tensor, tidx: torch.Tensor, qbeg: torch.Tensor,
                       qend: torch.Tensor):
    """Per query box i, the best 9-DoF IoU against the targets ``tidx[qbeg[i]:qend[i]]`` and the target index that gives
    it: corners (M,8,3) and (G,8,3) as for :func:`box3d_overlap`, ``tidx`` / ``qbeg`` / ``qend`` integer CUDA tensors ->
    (best (M,) fp32, arg (M,) int32). An empty range gives (-inf, -1). Each IoU has the bits ``box3d_overlap`` gives the
    pair; the choice is ``torch.max``'s (a NaN wins, ties to the smallest target index). One launch (csrc/iou3d.cu)."""
    from ._ffi import call, ptr, stream
    assert qcorners.is_cuda, 'box3d_best_overlap runs in libesb200.so (no CPU fallback)'
    cq, ct = qcorners.float().contiguous(), tcorners.float().contiguous()
    tidx, qbeg, qend = (x.to(device=cq.device, dtype=torch.int32).contiguous() for x in (tidx, qbeg, qend))
    m = cq.shape[0]
    assert qbeg.shape == qend.shape == (m, ) and ct.shape[1:] == (8, 3) and cq.shape[1:] == (8, 3)
    assert ct.shape[0] < 2 ** 31 and tidx.numel() < 2 ** 31
    best = torch.empty(m, dtype=torch.float32, device=cq.device)
    arg = torch.empty(m, dtype=torch.int32, device=cq.device)
    call('esb_box3d_best_overlap', ptr(cq), m, ptr(ct), ptr(tidx), ptr(qbeg), ptr(qend), ptr(best), ptr(arg), stream())
    return best, arg


def nms3d_9dof(boxes9: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, iou_thr: float,
               score_thr: float = float('-inf'), topk_per_class=None, seg_off=None, num_classes=None):
    """Class-agnostic greedy NMS on the exact 9-DoF 3D IoU with a score threshold and a per-label cap, the semantics of
    the reference's ``nms_filter`` (demo/demo.py:107-130): walking the boxes by descending score (stable: ties keep
    input order), a box is skipped when its label already has `topk_per_class` kept boxes, when its score is below
    `score_thr`, or when its IoU with a kept box exceeds `iou_thr`; a skipped box suppresses nothing.

    boxes9 (M,9), scores (M), labels (M) CUDA tensors -> LongTensor of kept input indices in selection order. With
    `seg_off` (S+1 host integers, segment s = rows seg_off[s]:seg_off[s+1]) every segment is filtered on its own in
    the same launch and a list of S index tensors comes back. Runs in libesb200.so (csrc/nms3d.cu, no CPU fallback);
    the kept counts of all segments are read back once. `num_classes` bounds the labels when the cap is set; left
    None it is read from ``labels.max()`` (one more small read-back)."""
    from ._ffi import call, ptr, query, stream
    assert boxes9.is_cuda, 'nms3d_9dof runs in libesb200.so (no CPU fallback)'
    assert boxes9.dim() == 2 and boxes9.shape[1] == 9 and scores.shape == labels.shape == boxes9.shape[:1]
    assert iou_thr >= 0, 'iou_thr must be >= 0'
    dev, M = boxes9.device, boxes9.shape[0]
    offs = [0, M] if seg_off is None else [int(o) for o in seg_off]
    assert offs[0] == 0 and offs[-1] == M and all(a <= b for a, b in zip(offs, offs[1:])), 'seg_off must cover 0..M'
    S = len(offs) - 1
    lens = [b - a for a, b in zip(offs, offs[1:])]
    max_seg = max(lens) if lens else 0
    if M == 0:
        out = [torch.empty(0, dtype=torch.long, device=dev) for _ in range(S)]
        return out[0] if seg_off is None else out
    scores = scores.float()
    order = torch.sort(scores, stable=True, descending=True).indices
    if S > 1:                                     # segment-major, score-descending inside each segment, still stable
        seg_of = torch.repeat_interleave(torch.arange(S, device=dev), torch.tensor(lens, device=dev), output_size=M)
        order = order[torch.sort(seg_of[order], stable=True).indices]
    if topk_per_class is None:                    # no cap: one label, a limit no count reaches
        lab, topk, ncls = torch.zeros(M, dtype=torch.int32, device=dev), 2 ** 31 - 1, 1
    else:
        lab, topk = labels[order].to(torch.int32).contiguous(), int(topk_per_class)
        ncls = int(num_classes) if num_classes is not None else int(labels.max()) + 1
    b = boxes9.float()[order].contiguous()
    sc = scores[order].contiguous()
    so = torch.tensor(offs, dtype=torch.int32).to(dev)
    keep = torch.empty(M, dtype=torch.int32, device=dev)
    n_keep = torch.empty(S, dtype=torch.int32, device=dev)
    wsb = query('esb_nms3d_9dof_workspace_bytes', M, S, max_seg)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    call('esb_nms3d_9dof', ptr(b), ptr(sc), ptr(lab), ptr(so), S, max_seg, float(iou_thr), float(score_thr), topk,
         max(ncls, 1), ptr(keep), ptr(n_keep), ptr(ws), wsb, stream())
    counts = n_keep.tolist()
    out = [order[keep[o:o + k].long()] for o, k in zip(offs, counts)]
    return out[0] if seg_off is None else out
