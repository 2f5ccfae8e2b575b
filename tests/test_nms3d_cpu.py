"""CPU: the oracle of the 3D-IoU box filter on cases with countable answers, the pose front-end against its scipy
restatement and closed forms, and the exactness argument of the kernel's separating-axis reject."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nms3d_ref as R  # noqa: E402
from oracle import geometry_ref as G  # noqa: E402

INF = 10 ** 9


def box(x=0., y=0., z=0., dx=1., dy=1., dz=1., a=0., b=0., c=0.):
    return [x, y, z, dx, dy, dz, a, b, c]


def keep(boxes, scores, labels=None, iou_thr=0.15, score_thr=-np.inf, topk=INF):
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 9)
    labels = np.zeros(len(boxes), dtype=np.int64) if labels is None else np.asarray(labels)
    return R.nms_filter(boxes, np.asarray(scores, dtype=np.float32), labels, iou_thr, score_thr, topk)


def test_identical_disjoint_empty_and_single():
    assert keep([box(), box()], [.9, .8]) == [0]
    assert keep([box(), box(x=5.)], [.8, .9]) == [1, 0]
    assert keep([], []) == []
    assert keep([box()], [.5]) == [0]


def test_known_overlap_fraction_on_both_sides_of_the_threshold():
    # unit cubes shifted by s along x: intersection 1 - s, IoU (1 - s) / (1 + s); s = 0.5 -> 1/3
    pair = [box(), box(x=0.5)]
    assert abs(R.iou_matrix(np.array(pair))[0, 1] - 1 / 3) < 1e-12
    assert keep(pair, [.9, .8], iou_thr=0.30) == [0]
    assert keep(pair, [.9, .8], iou_thr=0.35) == [0, 1]


def test_cap_drops_the_third_box_of_a_label():
    assert keep([box(), box(x=3.), box(x=6.)], [.9, .8, .7], labels=[4, 4, 4], topk=2) == [0, 1]


def test_a_box_skipped_by_the_cap_does_not_suppress():
    # label 1 is full after boxes 0 and 1; box 2 (label 1) is skipped, so box 3 (label 2) on the same spot survives
    boxes = [box(), box(x=3.), box(x=6.), box(x=6.)]
    assert keep(boxes, [.9, .8, .7, .6], labels=[1, 1, 1, 2], topk=2) == [0, 1, 3]
    assert keep(boxes, [.9, .8, .7, .6], labels=[1, 1, 1, 2]) == [0, 1, 2]


def test_a_box_under_the_score_threshold_does_not_suppress_and_is_not_kept():
    assert keep([box(), box()], [.05, .04], score_thr=0.075) == []
    assert keep([box(), box(x=3.)], [.5, .05], score_thr=0.075) == [0]


def test_equal_scores_keep_input_order():
    assert keep([box(x=0.), box(x=3.), box(x=6.)], [.5, .5, .5]) == [0, 1, 2]
    assert keep([box(), box()], [.5, .5]) == [0]


def test_degenerate_boxes_overlap_nothing():
    boxes = np.array([box(), box(dx=0.), box(x=np.nan), box()])
    assert R.valid_boxes(boxes).tolist() == [True, False, False, True]
    assert keep(boxes, [.6, .9, .8, .7]) == [1, 2, 3]


def test_pitched_box_survives_3d_filter_but_not_the_heads_bev_nms():
    """The head's NMS reads 7 columns: a box pitched and rolled is BEV-identical to its upright twin and is suppressed
    there. Their true 3D IoU is well under 1, so a 3D threshold between the two keeps both."""
    upright, tilted = box(dx=2., dy=.6, dz=.6), box(dx=2., dy=.6, dz=.6, b=0.5, c=0.5)
    b9 = np.array([upright, tilted])
    bev = G.iou_bev(b9[0, :7].astype(np.float32), b9[1, :7].astype(np.float32))
    iou3d = R.iou_matrix(b9)[0, 1]
    assert bev > 0.99 and 0.2 < iou3d < 0.8
    assert G.nms3d(b9[:, :7].astype(np.float32), np.array([.9, .8], dtype=np.float32), 0.9).tolist() == [0]
    assert keep(b9, [.9, .8], iou_thr=0.9) == [0, 1]
    assert keep(b9, [.9, .8], iou_thr=iou3d - 0.05) == [0]


def test_scan_from_poses_closed_forms_and_restatement():
    from embodiedscan_b200.inference import scan_from_poses
    P = np.array([[0., 0., 1.], [-1., 0., 0.], [0., -1., 0.]])
    K = np.eye(4)
    _, (e, ) = scan_from_poses([[0, 0, 0, 0, 0, 0, 1]], K, np.eye(4))
    assert e.dtype == np.float32 and np.allclose(e[:3, :3], P.T, atol=1e-7) and np.allclose(e[:3, 3], 0)
    # 90 degree yaw about z, camera at (1, 2, 3): cam2global = [Rz(90) P | t], extrinsic = its inverse
    s = np.sqrt(0.5)
    Rz = np.array([[0., -1., 0.], [1., 0., 0.], [0., 0., 1.]])
    _, (e, ) = scan_from_poses([[1, 2, 3, 0, 0, s, s]], K, np.eye(4))
    assert np.allclose(e[:3, :3], (Rz @ P).T, atol=1e-6)
    assert np.allclose(e[:3, 3], -(Rz @ P).T @ [1, 2, 3], atol=1e-6)
    # random poses and alignment: equal to the scipy restatement, and a true inverse
    rng = np.random.default_rng(3)
    q = rng.normal(size=(6, 4))
    poses = np.concatenate([rng.uniform(-3, 3, (6, 3)), q / np.linalg.norm(q, axis=1, keepdims=True)], 1)
    ang = 0.3
    align = np.eye(4)
    align[:2, :2] = [[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]]
    align[:3, 3] = [0.4, -1.2, 0.1]
    intr, ext = scan_from_poses(poses, np.eye(3), align)
    assert intr.dtype == np.float32 and len(ext) == 6
    for e, ref, (x, y, z, qx, qy, qz, qw) in zip(ext, R.scan_from_poses(poses, align), poses):
        assert np.abs(e - ref).max() <= 1e-6
        from scipy.spatial.transform import Rotation
        c2g = np.eye(4)
        c2g[:3, :3] = Rotation.from_quat([qx, qy, qz, qw]).as_matrix() @ P
        c2g[:3, 3] = [x, y, z]
        assert np.abs(e.astype(np.float64) @ (align @ c2g) - np.eye(4)).max() <= 1e-6


def test_separating_axis_reject_is_exact():
    """The kernel never clips a pair for which one of the 15 axes separates the boxes. On 20000 seeded random pairs at
    touching distance, "separated" implies the oracle's IoU is 0, so the reject cannot change a decision."""
    rng = np.random.default_rng(11)
    n = 20000
    a = np.concatenate([rng.uniform(-1, 1, (n, 3)), rng.uniform(0.2, 1.5, (n, 3)), rng.uniform(-np.pi, np.pi, (n, 3))], 1)
    b = np.concatenate([a[:, :3] + rng.normal(0, 0.7, (n, 3)), rng.uniform(0.2, 1.5, (n, 3)),
                        rng.uniform(-np.pi, np.pi, (n, 3))], 1)
    sep = R.sat_separated(a, b)
    assert 0.2 < sep.mean() < 0.9, 'the sample must hold both separated and overlapping pairs'
    idx = np.nonzero(sep)[0]
    ka, kb = R.corners64(a[idx]), R.corners64(b[idx])
    worst = max(G.box3d_overlap(ka[i:i + 1], kb[i:i + 1])[1][0, 0] for i in range(len(idx)))
    assert worst == 0.0
    # and the test is not vacuous the other way: overlapping pairs exist among the non-separated ones
    jdx = np.nonzero(~sep)[0][:200]
    kc, kd = R.corners64(a[jdx]), R.corners64(b[jdx])
    assert sum(G.box3d_overlap(kc[i:i + 1], kd[i:i + 1])[1][0, 0] > 0 for i in range(len(jdx))) >= 190
