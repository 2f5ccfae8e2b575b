"""Oracle of the 3D-IoU box filter and the pose front-end (test helper; pytest does not collect this file).

Restates, on top of ``oracle.geometry_ref.container_corners`` + ``box3d_overlap`` (float64 clipping):
  * demo/demo.py:102-130 (``nms_filter``: stable descending sort, per-label cap, score threshold, greedy 3D-IoU walk)
  * demo/demo.py:174-197 (pose rows -> ``inv(axis_align_matrix @ cam2global)``) with scipy's Rotation, as the demo does
and holds the seeded scene generator the CPU and GPU tests and the timing script share.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import geometry_ref as G  # noqa: E402


def corners64(boxes9: np.ndarray) -> np.ndarray:
    return G.container_corners(torch.as_tensor(np.asarray(boxes9), dtype=torch.float64)).numpy()


def valid_boxes(boxes9: np.ndarray) -> np.ndarray:
    """The rule of csrc/nms3d.cu: a size <= 0 or a non-finite value makes the box overlap nothing."""
    b = np.asarray(boxes9, dtype=np.float64).reshape(-1, 9)
    return np.isfinite(b).all(1) & (b[:, 3:6] > 0).all(1)


def iou_matrix(boxes9: np.ndarray, prev: np.ndarray = None, changed: np.ndarray = None) -> np.ndarray:
    """(N,N) float64 IoU. Each unordered pair is clipped once (the lower-index box as A) and mirrored; the float64 result
    differs between the two orders far below anything a threshold test here can see. Pairs whose axis-aligned bounds are
    disjoint are 0 without clipping (disjoint bounds = empty intersection), which keeps thousands of boxes affordable in
    Python. With `prev` and `changed`, only the rows and columns of the changed boxes are recomputed."""
    b = np.asarray(boxes9, dtype=np.float64).reshape(-1, 9)
    n = len(b)
    ok = valid_boxes(b)
    safe = np.where(ok[:, None], b, np.array([0, 0, 0, 1, 1, 1, 0, 0, 0.]))
    k = corners64(safe) if n else np.zeros((0, 8, 3))
    lo, hi = k.min(1), k.max(1)
    near = ((lo[:, None] <= hi[None]) & (lo[None] <= hi[:, None])).all(-1) & ok[:, None] & ok[None]
    near = np.triu(near, 1)
    if prev is None:
        iou = np.zeros((n, n))
    else:
        iou = prev.copy()
        touched = np.zeros(n, dtype=bool)
        touched[changed] = True
        iou[touched, :] = 0
        iou[:, touched] = 0
        near &= touched[:, None] | touched[None]
    for i, j in zip(*np.nonzero(near)):
        iou[i, j] = iou[j, i] = G.box3d_overlap(k[i:i + 1], k[j:j + 1])[1][0, 0]
    return iou


def nms_filter(boxes9, scores, labels, iou_thr, score_thr, topk_per_class, iou=None):
    """demo/demo.py:102-130: kept indices into the input, in selection order."""
    score, label = np.asarray(scores), np.asarray(labels)
    if iou is None:
        iou = iou_matrix(boxes9)
    selected_per_class = dict()
    idx = list(range(len(score)))
    idx.sort(key=lambda x: score[x], reverse=True)
    selected_idx = []
    for i in idx:
        if selected_per_class.get(label[i], 0) >= topk_per_class:
            continue
        if score[i] < score_thr:
            continue
        bo = False
        for j in selected_idx:
            if iou[i][j] > iou_thr:
                bo = True
                break
        if not bo:
            selected_idx.append(i)
            selected_per_class[label[i]] = selected_per_class.get(label[i], 0) + 1
    return selected_idx


def scan_from_poses(poses, axis_align_matrix):
    """demo/demo.py:174-197 for already-parsed rows (x y z qx qy qz qw): world -> camera extrinsics, fp32."""
    from scipy.spatial.transform import Rotation as R
    out = []
    for x, y, z, qx, qy, qz, qw in np.asarray(poses, dtype=np.float64).reshape(-1, 7):
        transform_matrix = np.identity(4)
        transform_matrix[:3, :3] = R.from_quat([qx, qy, qz, qw]).as_matrix() @ [[0, 0, 1], [-1, 0, 0], [0, -1, 0]]
        transform_matrix[:3, 3] = [x, y, z]
        out.append(np.linalg.inv(np.asarray(axis_align_matrix, dtype=np.float64) @ transform_matrix).astype(np.float32))
    return out


# ---- the reject rule of csrc/nms3d.cu (`separated`), restated in float64 without the rounding slack ---------------
def euler_zxy(e: np.ndarray) -> np.ndarray:
    return G.euler_to_matrix(torch.as_tensor(e, dtype=torch.float64)).numpy()


def sat_separated(a9: np.ndarray, b9: np.ndarray) -> np.ndarray:
    """(P,9),(P,9) -> (P,) bool: one of the 15 axes of the two oriented boxes separates them."""
    Ra, Rb = euler_zxy(a9[:, 6:9]), euler_zxy(b9[:, 6:9])
    ha, hb = a9[:, 3:6] / 2, b9[:, 3:6] / 2
    d = b9[:, :3] - a9[:, :3]
    t = np.einsum('pk,pka->pa', d, Ra)
    Rm = np.einsum('pka,pkb->pab', Ra, Rb)
    Ab = np.abs(Rm)
    sep = np.zeros(len(a9), dtype=bool)
    sep |= (np.abs(t) > ha + np.einsum('pab,pb->pa', Ab, hb)).any(1)
    sep |= (np.abs(np.einsum('pa,pab->pb', t, Rm)) > np.einsum('pa,pab->pb', ha, Ab) + hb).any(1)
    for a in range(3):
        a1, a2 = (a + 1) % 3, (a + 2) % 3
        for b in range(3):
            b1, b2 = (b + 1) % 3, (b + 2) % 3
            ra = ha[:, a1] * Ab[:, a2, b] + ha[:, a2] * Ab[:, a1, b]
            rb = hb[:, b1] * Ab[:, a, b2] + hb[:, b2] * Ab[:, a, b1]
            sep |= np.abs(t[:, a2] * Rm[:, a1, b] - t[:, a1] * Rm[:, a2, b]) > ra + rb + 1e-12
    return sep


# ---- seeded scenes --------------------------------------------------------------------------------------------
ROOM = (-3.0, 3.0, -3.0, 3.0, 0.0, 2.8)


def _gt_cuboids(rng, n):
    """Cuboids drawn like embodiedscan_b200.synth.synth_scan draws its ground truth."""
    ctr = np.stack([rng.uniform(ROOM[0] + .3, ROOM[1] - .3, n), rng.uniform(ROOM[2] + .3, ROOM[3] - .3, n),
                    rng.uniform(0.3, 2.2, n)], 1)
    size = rng.uniform(0.2, 1.5, (n, 3))
    euler = np.stack([rng.uniform(-np.pi, np.pi, n), rng.normal(0, 0.05, n), rng.normal(0, 0.05, n)], 1)
    return np.concatenate([ctr, size, euler], 1)


def _jitter(rng, gt):
    out = gt.copy()
    out[:, :3] += rng.normal(0, 0.08, (len(gt), 3))
    out[:, 3:6] *= np.exp(rng.normal(0, 0.12, (len(gt), 3)))
    out[:, 6:9] += rng.normal(0, 0.12, (len(gt), 3))
    return out


def cluster_boxes(n: int, seed: int, copies: int = 10, per_room: float = 24, num_classes: int = 20):
    """n candidate boxes as a detector emits them around objects: ceil(n / copies) ground-truth cuboids at `per_room`
    cuboids per 6 m x 6 m of floor (24 = one synth room; the floor grows with n), each with `copies` jittered copies
    (centre sigma 8 cm, log-size sigma 0.12, all three angles sigma 0.12 rad), the label of its cuboid with probability
    0.8 (else random) and a random score, in random order. Returns fp32 boxes, scores, int64 labels, the cuboid of each
    box, the cuboids and the generator."""
    rng = np.random.default_rng(seed)
    n_gt = -(-n // copies)
    gt = _gt_cuboids(rng, n_gt)
    gt[:, :2] *= max(1.0, np.sqrt(n_gt / per_room))
    src = np.repeat(np.arange(n_gt), copies)[:n]
    boxes = _jitter(rng, gt[src]).astype(np.float32)
    gt_label = rng.integers(0, num_classes, n_gt)
    labels = np.where(rng.random(n) < 0.8, gt_label[src], rng.integers(0, num_classes, n)).astype(np.int64)
    scores = rng.random(n).astype(np.float32)
    perm = rng.permutation(n)
    return boxes[perm], scores[perm], labels[perm], src[perm], gt, rng


def clustered_scene(n: int, seed: int, copies: int = 10, per_room: float = 24, num_classes: int = 20, iou_thr=None,
                    band: float = 1e-4):
    """`cluster_boxes` plus the float64 oracle IoU matrix of the fp32 boxes: (boxes, scores, labels, iou).

    With `iou_thr`, any pair whose oracle IoU lies within `band` of it has the jitter of its second box drawn again
    (seeded, so the set is fixed): inside that band the order of fp32 clipping operations may legitimately decide the
    comparison either way, everywhere else the kernel must agree exactly."""
    boxes, scores, labels, src, gt, rng = cluster_boxes(n, seed, copies, per_room, num_classes)
    iou = iou_matrix(boxes)
    if iou_thr is not None:
        for _ in range(20):
            bad = np.unique(np.nonzero(np.abs(iou - iou_thr) < band)[1])
            if len(bad) == 0:
                break
            boxes[bad] = _jitter(rng, gt[src[bad]]).astype(np.float32)
            iou = iou_matrix(boxes, iou, bad)
        else:
            raise AssertionError('could not clear the threshold band')
    return boxes, scores, labels, iou
