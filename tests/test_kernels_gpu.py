"""GPU parity tests proper: every CUDA entry point (called through the C ABI via the host package) against the CPU
oracle on the same seeded inputs. Integer outputs bit-exact; floating point within the stated tolerance."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

RTOL = 1e-3   # BASELINE.json north_star: "within 1e-3 relative fp32"


def _dev():
    return torch.device('cuda:0')


def _rand_coords(n, extent, n_batch, seed):
    g = np.random.RandomState(seed)
    c = g.randint(-extent, extent, size=(n, 3))
    b = np.sort(g.randint(0, n_batch, size=(n, 1)), axis=0)
    return np.concatenate([b, c], 1).astype(np.int64)


def _close(a, b, rtol=RTOL, what=''):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    scale = max(float(b.abs().max()), 1e-6)
    err = float((a - b).abs().max())
    assert err <= rtol * scale, f'{what}: max abs err {err} vs scale {scale}'


# ------------------------------------------------------------------------------------------------ coordinates
@pytest.mark.parametrize('n,extent,div', [(1, 4, 1), (5000, 12, 1), (5000, 12, 2), (60000, 40, 4), (0, 4, 1)])
def test_coord_unique_bit_exact(n, extent, div):
    from embodiedscan_b200.sparse import CoordinateManager
    from oracle import sparse_ref as R
    c = _rand_coords(n, extent, 3, 1) if n else np.zeros((0, 4), dtype=np.int64)
    ref_out, ref_map = R.unique_first(c, div)
    mgr = CoordinateManager(_dev())
    cm, in2out = mgr._unique(torch.from_numpy(c).to(_dev(), torch.int32), div, div)
    assert np.array_equal(cm.coords.cpu().numpy().astype(np.int64), ref_out)
    assert np.array_equal(in2out.cpu().numpy().astype(np.int64), ref_map)


def test_voxelize_bit_exact():
    from embodiedscan_b200 import _ffi
    from oracle import sparse_ref as R
    g = torch.Generator().manual_seed(3)
    p = (torch.rand(20000, 3, generator=g) - 0.5) * 7
    p[:100] = torch.round(p[:100] * 100) / 100          # values sitting on voxel boundaries
    ref = R.voxelize(p, 0.01, 2)
    out = torch.empty((p.shape[0], 4), dtype=torch.int32, device=_dev())
    pd = p.to(_dev())
    inv = float(np.float32(1.) / np.float32(0.01))
    _ffi.call('esb_voxelize_points', pd.data_ptr(), p.shape[0], 3, 2, inv, out.data_ptr(), _ffi.stream())
    assert np.array_equal(out.cpu().numpy().astype(np.int64), ref)


@pytest.mark.parametrize('ksize,stride', [(3, 1), (3, 2), (2, 2), (1, 2)])
def test_kernel_map_bit_exact(ksize, stride):
    from embodiedscan_b200.sparse import CoordinateManager
    from oracle import sparse_ref as R
    c = R.unique_first(_rand_coords(8000, 10, 2, 5))[0]
    mgr = CoordinateManager(_dev())
    key = mgr.insert_unique(torch.from_numpy(c).to(_dev(), torch.int32), 1)
    mgr.batch_size = 2
    out_key = mgr.stride_key(key, stride) if stride > 1 else key
    km = mgr.kernel_map(key, out_key, ksize)
    ref_out = R.unique_first(c, stride)[0] if stride > 1 else c
    ref = R.kernel_map(c, ref_out, R.offsets(ksize, 1))
    assert np.array_equal(mgr.maps[out_key].coords.cpu().numpy().astype(np.int64), ref_out)
    assert np.array_equal(km.nbr_out.cpu().numpy().astype(np.int64), ref)
    # transposed map and pair lists are consistent with nbr_out
    nbr_in = km.nbr_in.cpu().numpy()
    for k in range(ref.shape[0]):
        o = np.nonzero(ref[k] >= 0)[0]
        assert np.array_equal(nbr_in[k][ref[k][o]], o)
    pin, pout, koff, _ = km.pairs
    koff = koff.cpu().numpy()
    assert koff[-1] == (ref >= 0).sum()
    for k in range(ref.shape[0]):
        o = np.nonzero(ref[k] >= 0)[0]
        assert np.array_equal(pout[koff[k]:koff[k + 1]].cpu().numpy(), o)
        assert np.array_equal(pin[koff[k]:koff[k + 1]].cpu().numpy(), ref[k][o])


def test_generative_and_union_bit_exact():
    from embodiedscan_b200.sparse import CoordinateManager
    from oracle import sparse_ref as R
    parents = R.unique_first(_rand_coords(500, 6, 2, 7) * np.array([1, 4, 4, 4]))[0]
    other = R.unique_first(_rand_coords(3000, 12, 2, 8) * np.array([1, 2, 2, 2]))[0]
    mgr = CoordinateManager(_dev())
    pk = mgr.insert_unique(torch.from_numpy(parents).to(_dev(), torch.int32), 4)
    ok = mgr.insert_unique(torch.from_numpy(other).to(_dev(), torch.int32), 2)
    ck = mgr.generative_key(pk)
    ref_child = R.generative_children(parents, 2)
    assert np.array_equal(mgr.maps[ck].coords.cpu().numpy().astype(np.int64), ref_child)
    uk, map_b = mgr.union_key(ok, ck)
    ref_u, ref_map = R.union(other, ref_child)
    assert np.array_equal(mgr.maps[uk].coords.cpu().numpy().astype(np.int64), ref_u)
    assert np.array_equal(map_b.cpu().numpy(), ref_map)


# ------------------------------------------------------------------------------------------------ sparse conv
@pytest.mark.parametrize('cin,cout,ksize,stride,dtype', [
    (3, 64, 3, 2, torch.float32), (64, 64, 3, 1, torch.float32), (64, 128, 3, 2, torch.float32),
    (128, 128, 3, 1, torch.float32), (64, 128, 1, 2, torch.float32), (96, 40, 3, 1, torch.float32),
    (64, 64, 3, 1, torch.bfloat16), (128, 256, 3, 2, torch.bfloat16), (128, 128, 3, 1, torch.bfloat16),
    (256, 512, 3, 2, torch.bfloat16), (512, 512, 3, 1, torch.bfloat16), (1024, 128, 3, 1, torch.bfloat16),
    (64, 128, 1, 2, torch.bfloat16), (192, 64, 3, 1, torch.bfloat16)])
def test_spconv_fwd_bwd(cin, cout, ksize, stride, dtype):
    from embodiedscan_b200 import sparse as SP
    from oracle import sparse_ref as R
    torch.manual_seed(0)
    c = R.unique_first(_rand_coords(6000, 9, 2, 11))[0]
    x = torch.randn(c.shape[0], cin)
    K = ksize ** 3
    w = torch.randn((K, cin, cout) if K > 1 else (cin, cout)) / math.sqrt(cin * K)
    if dtype == torch.bfloat16:
        x, w = x.bfloat16().float(), w.bfloat16().float()
    out_c = R.unique_first(c, stride)[0] if stride > 1 else c
    nbr = R.kernel_map(c, out_c, R.offsets(ksize, 1))
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    yr = R.conv(xr, wr, nbr)
    gy = torch.randn_like(yr)
    if dtype == torch.bfloat16:
        gy = gy.bfloat16().float()
    yr.backward(gy)

    mgr = SP.CoordinateManager(_dev())
    key = mgr.insert_unique(torch.from_numpy(c).to(_dev(), torch.int32), 1)
    conv = SP.MinkowskiConvolution(cin, cout, kernel_size=ksize, stride=stride).to(_dev())
    with torch.no_grad():
        conv.kernel.copy_(w.to(_dev()))
    xd = x.to(_dev(), dtype).requires_grad_(True)
    y = conv(SP.SparseTensor(xd, coordinate_map_key=key, coordinate_manager=mgr))
    assert np.array_equal(y.C.cpu().numpy().astype(np.int64), out_c)
    y.F.backward(gy.to(_dev(), dtype))
    # bf16 storage (8-bit mantissa outputs); the wgmma path (channels % 64 == 0) accumulates in fp32 registers
    tol = RTOL if dtype == torch.float32 else 2e-2
    _close(y.F, yr, tol, 'fwd')
    _close(xd.grad, xr.grad, tol, 'dgrad')
    _close(conv.kernel.grad, wr.grad.view_as(conv.kernel), tol, 'wgrad')


def test_spconv_dense_equivalence():
    """Closed form: on a fully occupied cube the sparse conv equals F.conv3d (zero padding)."""
    from embodiedscan_b200 import sparse as SP
    torch.manual_seed(1)
    D, cin, cout = 6, 8, 16
    zz, yy, xx = np.meshgrid(np.arange(D), np.arange(D), np.arange(D), indexing='ij')
    c = np.stack([np.zeros(D ** 3, dtype=np.int64), xx.ravel(), yy.ravel(), zz.ravel()], 1)
    x = torch.randn(D ** 3, cin)
    w = torch.randn(27, cin, cout) * 0.1
    dense = x.view(D, D, D, cin).permute(3, 0, 1, 2)[None]                       # (1,C,z,y,x)
    wd = w.view(3, 3, 3, cin, cout).permute(4, 3, 0, 1, 2)                        # k = x + 3y + 9z -> (z,y,x)
    ref = torch.nn.functional.conv3d(dense, wd, padding=1)[0].permute(1, 2, 3, 0).reshape(-1, cout)
    mgr = SP.CoordinateManager(_dev())
    key = mgr.insert_unique(torch.from_numpy(c).to(_dev(), torch.int32), 1)
    conv = SP.MinkowskiConvolution(cin, cout, kernel_size=3).to(_dev())
    with torch.no_grad():
        conv.kernel.copy_(w.to(_dev()))
    y = conv(SP.SparseTensor(x.to(_dev()), coordinate_map_key=key, coordinate_manager=mgr))
    _close(y.F, ref, 1e-4, 'dense equivalence')


def test_maxpool_and_norms():
    from embodiedscan_b200 import sparse as SP
    from oracle import sparse_ref as R
    torch.manual_seed(2)
    c = R.unique_first(_rand_coords(5000, 8, 3, 13))[0]
    C = 64
    x = torch.randn(c.shape[0], C) * 2 + 0.5
    pooled = R.unique_first(c, 2)[0]
    nbr = R.kernel_map(c, pooled, R.offsets(2, 1))
    xr = x.clone().requires_grad_(True)
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    h = torch.relu(R.instance_norm(xr, c[:, 0], 3, gr, br))
    yr = R.maxpool(h, nbr)
    g2, b2 = torch.rand(C) + 0.5, torch.randn(C)
    g2r, b2r = g2.clone().requires_grad_(True), b2.clone().requires_grad_(True)
    res = torch.randn(pooled.shape[0], C)
    resr = res.clone().requires_grad_(True)
    zr = torch.nn.functional.elu(R.batch_norm(yr, g2r, b2r) + resr)
    gz = torch.randn_like(zr)
    zr.backward(gz)

    mgr = SP.CoordinateManager(_dev())
    key = mgr.insert_unique(torch.from_numpy(c).to(_dev(), torch.int32), 1)
    mgr.batch_size = 3
    inorm = SP.MinkowskiInstanceNorm(C).to(_dev())
    bn = SP.MinkowskiBatchNorm(C).to(_dev())
    with torch.no_grad():
        inorm.weight.copy_(gamma.view(1, -1)); inorm.bias.copy_(beta.view(1, -1))
        bn.bn.weight.copy_(g2); bn.bn.bias.copy_(b2)
    xd = x.to(_dev()).requires_grad_(True)
    resd = res.to(_dev()).requires_grad_(True)
    t = inorm(SP.SparseTensor(xd, coordinate_map_key=key, coordinate_manager=mgr), act=SP.ACT_RELU)
    t = SP.MinkowskiMaxPooling()(t)
    z = bn(t, act=SP.ACT_ELU, res=resd)
    assert np.array_equal(z.C.cpu().numpy().astype(np.int64), pooled)
    z.F.backward(gz.to(_dev()))
    _close(z.F, zr, RTOL, 'norm/pool fwd')
    _close(xd.grad, xr.grad, RTOL, 'dx')
    _close(resd.grad, resr.grad, RTOL, 'dres')
    _close(bn.bn.weight.grad, g2r.grad, RTOL, 'dgamma_bn')
    _close(bn.bn.bias.grad, b2r.grad, RTOL, 'dbeta_bn')
    _close(inorm.weight.grad.view(-1), gr.grad, RTOL, 'dgamma_in')
    _close(inorm.bias.grad.view(-1), br.grad, RTOL, 'dbeta_in')
    # running statistics follow nn.BatchNorm1d (momentum .1, unbiased variance)
    ref_bn = torch.nn.BatchNorm1d(C)
    ref_bn.train()
    ref_bn(yr.detach())
    _close(bn.bn.running_mean, ref_bn.running_mean, RTOL, 'running_mean')
    _close(bn.bn.running_var, ref_bn.running_var, RTOL, 'running_var')


# ------------------------------------------------------------------------------------------------ point painting
@pytest.mark.parametrize('augment,C,dtype', [(False, 64, torch.float32), (True, 128, torch.float32),
                                             (True, 512, torch.float32), (False, 256, torch.bfloat16)])
def test_point_painting(augment, C, dtype):
    from embodiedscan_b200.fusion import pack_paint_metas, pack_projections, paint_points
    from embodiedscan_b200.synth import synth_scan
    from oracle import model_ref as M
    torch.manual_seed(4)
    V, H, W = 3, 96, 128
    scans = [synth_scan(i, n_views=V, H=H, W=W, n_points=1500, augment=augment) for i in range(2)]
    metas = [s['data_sample'].metainfo for s in scans]
    Hf, Wf = H // 8, W // 8
    feat = torch.randn(2 * V, C, Hf, Wf)
    if dtype == torch.bfloat16:
        feat = feat.bfloat16().float()
    coords, ref_rows, ref_cnt = [], [], []
    for b, s in enumerate(scans):
        q = torch.floor(s['points'] / 0.08).to(torch.int64) * 8                      # stride-8 lattice, 1 cm voxels
        q = torch.unique(q, dim=0)
        coords.append(torch.cat([torch.full((q.shape[0], 1), b), q], 1))
        pm = metas[b]['depth2img']
        proj = torch.from_numpy(np.stack([M.compose_projection(pm['intrinsic'][v], pm['extrinsic'][v]) for v in range(V)]))
        pts = q.to(torch.int32) * 0.01
        fr = feat[b * V:(b + 1) * V].clone().requires_grad_(True)
        out, cnt = M.batch_point_sample(metas[b], fr, pts, proj, (H, W))
        ref_rows.append((out, fr))
        ref_cnt.append(cnt)
    coords = torch.cat(coords).to(_dev(), torch.int32)
    fd = feat.to(_dev(), dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    md = pack_paint_metas(metas, _dev())
    pj = pack_projections(metas, 'DEPTH', _dev())
    out = paint_points(fd, coords, md, pj, 0.01, (H, W), V)
    ref = torch.cat([r[0] for r in ref_rows])
    go = torch.randn_like(ref)
    ref.backward(go)
    out.backward(go.to(_dev(), dtype))
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    # same pixels selected <=> identical sums (fp32: exact up to summation order)
    _close(out, ref, tol, 'painted features')
    assert float(torch.cat(ref_cnt).float().mean()) > 0.2, 'test scene must have visible points'
    gref = torch.cat([r[1].grad for r in ref_rows])
    _close(fd.grad, gref, 1e-4 if dtype == torch.float32 else 2e-2, 'dfeat')


# ------------------------------------------------------------------------------------------------ head
def _head_scene(seed, n_pts=(6000, 1500, 400, 100)):
    from embodiedscan_b200.synth import synth_scan
    s = synth_scan(seed, n_views=2, H=60, W=80, n_points=200)
    gt = s['data_sample'].gt_instances_3d
    boxes9 = torch.cat((gt.bboxes_3d.gravity_center, gt.bboxes_3d.tensor[:, 3:]), 1)
    g = torch.Generator().manual_seed(seed)
    pts = []
    for l, n in enumerate(n_pts):
        st = 0.08 * 2 ** l
        q = torch.stack([torch.randint(-38, 38, (n, ), generator=g), torch.randint(-38, 38, (n, ), generator=g),
                         torch.randint(0, 35, (n, ), generator=g)], 1)
        q = torch.unique(torch.floor(q * 0.08 / st).to(torch.int32), dim=0)
        pts.append((q * int(round(st * 100))).to(torch.int32) * 0.01)
    return pts, boxes9, gt.labels_3d


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_fcaf3d_targets_bit_exact(seed):
    from embodiedscan_b200.dense_heads import fcaf3d_targets
    from oracle import model_ref as M
    pts, boxes9, labels = _head_scene(seed)
    ct_r, bt_r, kt_r = M.get_targets(pts, boxes9, labels)
    ct, bt, kt = fcaf3d_targets([p.to(_dev()) for p in pts], boxes9.to(_dev()), labels.to(_dev()), 27, 18)
    assert int((kt_r >= 0).sum()) > 20, 'scene must produce positives'
    assert torch.equal(kt.cpu(), kt_r), 'class targets (selection) must be bit-exact'
    assert torch.equal(bt.cpu(), bt_r), 'box targets (selection) must be bit-exact'
    pos = kt_r >= 0
    _close(ct.cpu()[pos], ct_r[pos], 1e-5, 'centerness targets')
    assert torch.equal(ct.cpu()[~pos] >= 0, ct_r[~pos] >= 0)


def test_fcaf3d_targets_batched_matches_per_scan_oracle():
    """Two scans with interleaved rows (the natural order after a coordinate union) in ONE kernel pipeline."""
    from embodiedscan_b200.dense_heads import fcaf3d_targets_batched
    from oracle import model_ref as M
    scenes = [_head_scene(0), _head_scene(1, n_pts=(5000, 1200, 300, 90))]
    g = torch.Generator().manual_seed(9)
    pts_all, batch_all, sizes, back = [], [], [], []
    for l in range(4):
        p = torch.cat([scenes[0][0][l], scenes[1][0][l]])
        b = torch.cat([torch.zeros(len(scenes[0][0][l]), dtype=torch.int32), torch.ones(len(scenes[1][0][l]), dtype=torch.int32)])
        # keep the relative order of each scan's rows (ties break by row index): stable re-sort inside the interleave
        keys = torch.rand(len(p), generator=g)
        order = torch.argsort(keys)
        slots0 = order[: len(scenes[0][0][l])].sort().values
        slots1 = order[len(scenes[0][0][l]):].sort().values
        pl = torch.empty_like(p)
        bl = torch.empty_like(b)
        pl[slots0], bl[slots0] = scenes[0][0][l], 0
        pl[slots1], bl[slots1] = scenes[1][0][l], 1
        pts_all.append(pl); batch_all.append(bl); sizes.append(len(pl)); back.append((slots0, slots1))
    ct, bt, kt = fcaf3d_targets_batched(torch.cat(pts_all).to(_dev()), sizes, torch.cat(batch_all).to(_dev()),
                                        [scenes[0][1].to(_dev()), scenes[1][1].to(_dev())],
                                        [scenes[0][2].to(_dev()), scenes[1][2].to(_dev())], 27, 18)
    ct, bt, kt = ct.cpu(), bt.cpu(), kt.cpu()
    for sidx in range(2):
        ct_r, bt_r, kt_r = M.get_targets(scenes[sidx][0], scenes[sidx][1], scenes[sidx][2])
        off_b, off_r = 0, 0
        for l in range(4):
            sl = back[l][sidx] + off_b
            n = len(scenes[sidx][0][l])
            assert torch.equal(kt[sl], kt_r[off_r:off_r + n]) and torch.equal(bt[sl], bt_r[off_r:off_r + n])
            pos = kt_r[off_r:off_r + n] >= 0
            assert float((ct[sl][pos] - ct_r[off_r:off_r + n][pos]).abs().max() if pos.any() else 0.) < 1e-5
            off_b += sizes[l]
            off_r += n


def test_targets_no_boxes():
    from embodiedscan_b200.dense_heads import fcaf3d_targets
    pts, _, _ = _head_scene(0)
    ct, bt, kt = fcaf3d_targets([p.to(_dev()) for p in pts], torch.zeros((0, 9), device=_dev()),
                                torch.zeros((0, ), dtype=torch.long, device=_dev()), 27, 18)
    assert (kt == -1).all() and ct.abs().sum() == 0 and bt.shape[1] == 9


def test_focal_loss():
    from embodiedscan_b200.dense_heads import FocalLoss
    from oracle import geometry_ref as G
    torch.manual_seed(5)
    n, C = 3000, 284
    x = torch.randn(n, C) * 2 - 3
    t = torch.randint(-1, C, (n, ))
    xr = x.clone().requires_grad_(True)
    lr = G.sigmoid_focal_loss_sum(xr, t) / 37.0
    lr.backward()
    xd = x.to(_dev()).requires_grad_(True)
    l = FocalLoss()(xd, t.to(_dev()), avg_factor=torch.tensor(37.0, device=_dev()))
    l.backward()
    _close(l, lr, 1e-4, 'focal loss')
    _close(xd.grad, xr.grad, 1e-3, 'focal grad')
    # closed form at logit 0: p = .5 -> positives alpha*.25*ln2, negatives (1-alpha)*.25*ln2
    z = torch.zeros(1, 4, device=_dev())
    v = FocalLoss()(z, torch.tensor([2], device=_dev()), avg_factor=torch.tensor(1.0, device=_dev()))
    assert abs(float(v) - (0.25 * 0.25 + 3 * 0.75 * 0.25) * math.log(2)) < 1e-6


# ------------------------------------------------------------------------------------------------ NMS
def _rand_boxes(n, seed, spread=2.0):
    g = np.random.RandomState(seed)
    b = np.zeros((n, 7), dtype=np.float32)
    b[:, :3] = g.uniform(-spread, spread, (n, 3))
    b[:, 3:6] = g.uniform(0.3, 1.5, (n, 3))
    b[:, 6] = g.uniform(-math.pi, math.pi, n)
    return b


def test_iou_bev_closed_forms_and_oracle():
    from embodiedscan_b200 import _ffi
    from oracle import geometry_ref as G
    a = _rand_boxes(40, 1, 1.0)
    b = _rand_boxes(30, 2, 1.0)
    # closed forms: identical box -> 1 ; axis-aligned shifted by half width -> 1/3 ; 45 degree square overlap
    a[0] = [0, 0, 0, 2, 2, 1, 0]; b[0] = [0, 0, 0, 2, 2, 1, 0]
    a[1] = [0, 0, 0, 2, 2, 1, 0]; b[1] = [1, 0, 0, 2, 2, 1, 0]
    a[2] = [0, 0, 0, 2, 2, 1, 0]; b[2] = [0, 0, 0, 2, 2, 1, math.pi / 4]
    out = torch.empty((40, 30), device=_dev())
    ad, bd = torch.from_numpy(a).to(_dev()), torch.from_numpy(b).to(_dev())
    _ffi.call('esb_iou_bev_pairwise', ad.data_ptr(), 40, bd.data_ptr(), 30, 1, out.data_ptr(), _ffi.stream())
    o = out.cpu().numpy()
    assert abs(o[0, 0] - 1.0) < 1e-5 and abs(o[1, 1] - 1.0 / 3.0) < 1e-5
    oct_area = 8 * (math.sqrt(2) - 1)          # regular octagon: two unit-inradius squares at 45 degrees
    assert abs(o[2, 2] - oct_area / (8 - oct_area)) < 1e-4
    ref = np.array([[G.iou_bev(a[i], b[j]) for j in range(30)] for i in range(40)])
    assert np.abs(o - ref).max() < 1e-4


@pytest.mark.parametrize('seed', [0, 1])
def test_multiclass_nms_selection_order(seed):
    from embodiedscan_b200.dense_heads import multiclass_nms_bev
    from oracle import geometry_ref as G
    torch.manual_seed(seed)
    n, C = 300, 12
    boxes = torch.from_numpy(np.concatenate([_rand_boxes(n, seed, 1.5), np.zeros((n, 2), np.float32)], 1))
    scores = torch.rand(n, C) * 0.05
    scores[torch.rand(n, C) < 0.7] = 0.001
    scores[:5, 3] = scores[5:10, 3]                       # exact score ties inside a class
    rb, rs, rl = G.multiclass_nms(boxes, scores, 0.01, 0.5)
    b, s, l = multiclass_nms_bev(boxes.to(_dev()), scores.to(_dev()), 0.01, 0.5)
    assert torch.equal(l.cpu(), rl), 'labels / selection order'
    assert torch.equal(s.cpu(), rs) and torch.equal(b.cpu(), rb)
    assert rl.numel() > 30


def test_box3d_overlap_9dof():
    from embodiedscan_b200.structures import EulerDepthInstance3DBoxes
    from oracle import geometry_ref as G
    g = np.random.RandomState(3)

    def boxes(n, spread):
        b = np.zeros((n, 9), dtype=np.float32)
        b[:, :3] = g.uniform(-spread, spread, (n, 3))
        b[:, 3:6] = g.uniform(0.3, 1.6, (n, 3))
        b[:, 6] = g.uniform(-math.pi, math.pi, n)
        b[:, 7:] = g.normal(0, 0.4, (n, 2))
        return torch.from_numpy(b)
    b1, b2 = boxes(24, 0.8), boxes(18, 0.8)
    b2[0] = b1[0]                                                   # identical pair: IoU 1 despite coplanar faces
    b2[1] = torch.tensor([50., 50., 50., 1., 1., 1., 0., 0., 0.])   # far away: IoU 0
    ref_vol, ref_iou = G.box3d_overlap(G.container_corners(b1).numpy(), G.container_corners(b2).numpy())
    iou = EulerDepthInstance3DBoxes.overlaps(EulerDepthInstance3DBoxes(b1).to(_dev()), EulerDepthInstance3DBoxes(b2).to(_dev()))
    assert iou.shape == (24, 18)
    assert float((iou.cpu().double() - torch.from_numpy(ref_iou)).abs().max()) < 1e-4
    assert abs(float(iou[0, 0]) - 1.0) < 1e-4 and float(iou[:, 1].max()) == 0.0
    assert float((ref_iou > 0.05).mean()) > 0.2, 'the test must exercise real overlaps'


@pytest.mark.parametrize('n_pred,g_max,n_prob', [(256, 12, 84), (32, 32, 9), (700, 5, 4), (7, 1, 3)])
def test_hungarian_batch_equals_scipy(n_pred, g_max, n_prob):
    """One launch for every (layer, sample) problem vs scipy.optimize.linear_sum_assignment per problem (what
    HungarianAssigner3D.assign runs on the host), incl. empty problems, n_gt == n_pred, and NaN/inf costs."""
    from scipy.optimize import linear_sum_assignment
    from embodiedscan_b200.grounding import hungarian_batch
    g = np.random.RandomState(n_pred + g_max)
    cost = g.normal(0, 3, (n_prob, n_pred, g_max)).astype(np.float32)
    cost[0, 0, 0], cost[0, 1, 0], cost[0, 2, 0] = np.nan, np.inf, -np.inf
    n_gt = g.randint(0, g_max + 1, n_prob).astype(np.int32)
    n_gt[0], n_gt[-1] = g_max, 0
    p2g, g2p = hungarian_batch(torch.from_numpy(cost).to(_dev()), torch.from_numpy(n_gt).to(_dev()))
    p2g, g2p = p2g.cpu().numpy(), g2p.cpu().numpy()
    for p in range(n_prob):
        k = int(n_gt[p])
        ref = np.full(n_pred, -1)
        inv = np.full(g_max, -1)
        if k:
            c = np.nan_to_num(cost[p, :, :k].astype(np.float64), nan=100.0, posinf=100.0, neginf=-100.0)
            r, cidx = linear_sum_assignment(c)
            ref[r], inv[cidx] = cidx, r
        assert (p2g[p] == ref).all(), (p, k)
        assert (g2p[p] == inv).all(), (p, k)


# ------------------------------------------------------------------------------------------------ input side
def test_img_normalize_bit_exact():
    from embodiedscan_b200 import Det3DDataPreprocessor
    from oracle import model_ref as M
    g = torch.Generator().manual_seed(6)
    img = torch.randint(0, 256, (2, 3, 3, 50, 70), generator=g, dtype=torch.uint8)
    mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
    ref = M.preprocess_imgs(img, mean, std, True, 32)
    pre = Det3DDataPreprocessor(mean=mean, std=std, bgr_to_rgb=True, pad_size_divisor=32).to(_dev())
    out = pre(dict(inputs=dict(img=[i for i in img])))['inputs']['imgs']
    assert out.shape == ref.shape
    assert torch.equal(out.cpu(), ref), 'fp32 normalisation is a single rounded sub and div per pixel'


def test_unproject_depth():
    from embodiedscan_b200 import _ffi
    from embodiedscan_b200.synth import synth_scan
    V, H, W = 2, 48, 64
    s = synth_scan(3, n_views=V, H=H, W=W, n_points=500)
    depth = s['depth'].to(torch.int16).to(_dev()).contiguous()            # bit pattern of uint16
    meta = s['data_sample'].metainfo['depth2img']
    mats, ref_pts = [], []
    for v in range(V):
        K = torch.from_numpy(meta['intrinsic'][v]).double()
        E = torch.from_numpy(meta['extrinsic'][v]).double()
        mats.append((torch.inverse(E) @ torch.inverse(K)).float())
        d = s['depth'][v].float() / 1000.0
        us, vs = torch.meshgrid(torch.arange(W), torch.arange(H), indexing='xy')
        grid = torch.stack([us * d, vs * d, d, torch.ones_like(d)], -1).view(-1, 4).double()
        nz = torch.nonzero(d.reshape(-1)).squeeze(1)
        ref_pts.append((grid @ (torch.inverse(E) @ torch.inverse(K)).t())[nz, :3].float())
    ref = torch.cat(ref_pts)
    md = torch.stack(mats).to(_dev()).contiguous()
    out = torch.empty((V * H * W, 3), device=_dev())
    cnt = torch.zeros(1, dtype=torch.int32, device=_dev())
    wsb = _ffi.query('esb_unproject_depth_workspace_bytes', V, H, W)
    ws = torch.empty(wsb, dtype=torch.uint8, device=_dev())
    _ffi.call('esb_unproject_depth', depth.data_ptr(), V, H, W, 1000.0, md.data_ptr(), out.data_ptr(), None,
              cnt.data_ptr(), ws.data_ptr(), wsb, _ffi.stream())
    n = int(cnt.item())
    assert n == ref.shape[0], 'zero-depth pixels dropped, row-major order kept'
    _close(out[:n], ref, 1e-5, 'unprojected points')


def test_multiview_depth_to_points_transform():
    from embodiedscan_b200.synth import synth_scan
    from embodiedscan_b200.transforms import MultiViewDepthToPoints, unproject_multiview
    s = synth_scan(4, n_views=3, H=48, W=64, n_points=900)
    meta = s['data_sample'].metainfo['depth2img']
    pts = unproject_multiview(s['depth'].to(_dev()), meta['intrinsic'], meta['extrinsic'])
    assert pts.shape[0] == int((s['depth'] != 0).sum())
    # every synthetic scan point (sampled from the same unprojection in torch) is one of the kernel's points
    d = torch.cdist(s['points'].to(_dev()).double(), pts.double()).min(1).values
    assert float(d.max()) < 1e-4
    out = MultiViewDepthToPoints(num_points=500, points_per_view=300, seed=0)(
        dict(depth_imgs=s['depth'].to(_dev()), depth2img=meta))
    assert out['points'].shape == (500, 3)
    assert float(torch.cdist(out['points'].double(), pts.double()).min(1).values.max()) == 0.0


def test_adamw_and_clip_match_torch():
    from embodiedscan_b200.engine import OptimWrapper
    torch.manual_seed(7)
    net = torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.ReLU(), torch.nn.Linear(53, 11)).to(_dev())
    ref = torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.ReLU(), torch.nn.Linear(53, 11)).to(_dev())
    ref.load_state_dict(net.state_dict())
    opt_ref = torch.optim.AdamW(ref.parameters(), lr=1e-3, weight_decay=1e-4)
    ow = OptimWrapper(net, lr=1e-3, weight_decay=1e-4, max_norm=0.5)
    for step in range(4):
        x = torch.randn(64, 37, device=_dev())
        (ref(x) ** 2).sum().backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.5)
        opt_ref.step(); opt_ref.zero_grad()
        ow.update_params((net(x) ** 2).sum())
    for a, b in zip(net.parameters(), ref.parameters()):
        _close(a, b, 1e-5, 'adamw parameters')


# ------------------------------------------------------------------------------------------------ round-2 kernels
def _run_child(script, *args, timeout=420):
    """First-run tensor-core kernels execute in a child process under a hard timeout (a hang must not take the session)."""
    import json
    import subprocess
    import sys
    p = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), script), *args],
                       capture_output=True, text=True, timeout=timeout)
    rows = [json.loads(l) for l in p.stdout.splitlines() if l.startswith('{')]
    assert p.returncode == 0 and rows, (p.returncode, p.stderr[-800:])
    return rows


def test_conv2d_tma_family_matches_torch():
    """csrc/conv_tma.cu: TMA + wgmma conv2d forward (stride 1 / 2, 32B / 64B / 128B swizzle, fused epilogue), stride-1 and
    stride-2 dgrad (filter read MN-major, parity-class stores), TMA-fed wgrad and the shared-memory-im2col stem, against torch
    fp32 on bf16-rounded operands (1e-2 of the tensor maximum: bf16 output rounding)."""
    rows = _run_child('conv_tma_child.py')
    bad = [r for r in rows if not r.get('ok', True)]
    assert not bad, bad
    kinds = {r['kind'] for r in rows}
    assert {'fwd', 'dgrad', 'wgrad', 'stem', 'conv3d'} <= kinds, kinds


def test_union_add_and_interp_kernels():
    from embodiedscan_b200 import sparse as SP
    from oracle import sparse_ref as R
    torch.manual_seed(3)
    a = R.unique_first(_rand_coords(4000, 10, 2, 21) * np.array([1, 2, 2, 2]))[0]
    b = R.unique_first(_rand_coords(5000, 10, 2, 22) * np.array([1, 2, 2, 2]))[0]
    mgr = SP.CoordinateManager(_dev())
    mgr.batch_size = 2
    ka = mgr.insert_unique(torch.from_numpy(a).to(_dev(), torch.int32), 2)
    kb = mgr.insert_unique(torch.from_numpy(b).to(_dev(), torch.int32), 2)
    for dtype in (torch.float32, torch.bfloat16):
        fa = torch.randn(a.shape[0], 64, device=_dev()).to(dtype).requires_grad_(True)
        fb = torch.randn(b.shape[0], 64, device=_dev()).to(dtype).requires_grad_(True)
        u = SP.SparseTensor(fa, coordinate_map_key=ka, coordinate_manager=mgr) + \
            SP.SparseTensor(fb, coordinate_map_key=kb, coordinate_manager=mgr)
        _, map_b = mgr.union_key(ka, kb)
        n = u.F.shape[0]
        ref = torch.cat([fa.detach(), fa.new_zeros(n - fa.shape[0], 64)], 0).index_add(0, map_b, fb.detach())
        assert torch.equal(u.F.detach(), ref)                       # one addition per element: bit-exact
        g = torch.randn_like(u.F)
        u.F.backward(g)
        assert torch.equal(fa.grad, g[:fa.shape[0]]) and torch.equal(fb.grad, g[map_b])
    # multilinear interpolation at child coordinates: fused kernel (integer queries) vs the eager 8-corner expression
    scores = SP.SparseTensor(torch.randn(a.shape[0], 1, device=_dev()), coordinate_map_key=ka, coordinate_manager=mgr)
    child = mgr.maps[mgr.generative_key(ka)].coords
    fused = scores.features_at_coordinates(child)
    eager = scores.features_at_coordinates(child.float())
    assert torch.equal(fused, eager)
    want = R.features_at_coordinates(a, scores.F.cpu(), 2, child.cpu().numpy().astype(np.int64))
    assert float((fused.cpu() - want).abs().max()) <= 1e-6


def test_rows_gemm_tc_matches_matmul():
    from embodiedscan_b200 import sparse as SP
    torch.manual_seed(5)
    for n, cin, cout in ((5000, 128, 320), (777, 1024, 512), (0, 64, 64)):
        x = (torch.randn(n, cin, device=_dev()) / 4).bfloat16().requires_grad_(True)
        w = (torch.randn(cin, cout, device=_dev()) / math.sqrt(cin)).bfloat16().requires_grad_(True)
        y = SP.rows_gemm(x, w)
        g = torch.randn(n, cout, device=_dev()).bfloat16()
        y.backward(g)
        xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
        yr = xr @ wr
        yr.backward(g.float())
        if n == 0:
            assert y.shape == (0, cout)
            continue
        _close(y, yr, 2e-2, 'rows_gemm fwd')
        _close(x.grad, xr.grad, 2e-2, 'rows_gemm dgrad')
        _close(w.grad, wr.grad, 2e-2, 'rows_gemm wgrad')


def test_fused_batchnorm_bf16_matches_reference():
    """esb_batchnorm_fwd_fused (shifted single-pass statistics + on-the-fly apply) against nn.BatchNorm1d in fp32 on the
    bf16-rounded rows, with a large mean/std ratio (what a naive single-pass variance gets wrong), residual + ELU, backward."""
    from embodiedscan_b200 import sparse as SP
    torch.manual_seed(7)
    for N, C in ((7001, 64), (300, 1024), (129, 192)):
        x = (torch.randn(N, C) * 0.3 + 25.0).bfloat16()
        res = torch.randn(N, C).bfloat16()
        bn = torch.nn.BatchNorm1d(C).to(_dev())
        ref_bn = torch.nn.BatchNorm1d(C)
        with torch.no_grad():
            bn.weight.uniform_(0.5, 1.5); bn.bias.normal_()
            ref_bn.weight.copy_(bn.weight.cpu()); ref_bn.bias.copy_(bn.bias.cpu())
        xr, rr = x.float().requires_grad_(True), res.float().requires_grad_(True)
        zr = torch.nn.functional.elu(ref_bn(xr) + rr)
        g = torch.randn(N, C).bfloat16()
        zr.backward(g.float())
        xd, rd = x.to(_dev()).requires_grad_(True), res.to(_dev()).requires_grad_(True)
        z = SP.batch_norm_rows(xd, bn, True, SP.ACT_ELU, rd)
        z.backward(g.to(_dev()))
        _close(z, zr, 2e-2, 'fused bn fwd')
        _close(xd.grad, xr.grad, 3e-2, 'fused bn dx')
        _close(rd.grad, rr.grad, 2e-2, 'fused bn dres')
        _close(bn.weight.grad, ref_bn.weight.grad, 2e-2, 'fused bn dgamma')
        _close(bn.running_mean, ref_bn.running_mean, 1e-3, 'running mean')
        _close(bn.running_var, ref_bn.running_var, 2e-2, 'running var')


def test_flash_attention_tc_matches_softmax_attention():
    """csrc/attn_tc.cu (wgmma flash attention, forward + dq / dk / dv) against fp32 softmax attention on bf16-rounded
    operands: self-attention, padded keys, 3.5k keys, ragged sizes below one tile."""
    rows = _run_child('attn_child.py')
    bad = [r for r in rows if not r.get('ok', True)]
    assert not bad, bad
    assert sum(r['kind'] == 'attn' for r in rows) >= 6


def test_head_epilogue_kernel_matches_aten_chain():
    """esb_head_split_fwd / _bwd against the slice / bias / Scale / exp / clamp / cat chain of fcaf3d_head.py:1116-1149 on the
    same bf16 head-GEMM output: forward tensors bit-exact (same roundings), gradients to bf16 / fp32-sum tolerance; rows that
    hit the clamp floor pass no gradient; N = 0 and a width that is not the model's."""
    from embodiedscan_b200 import dense_heads as DH
    torch.manual_seed(11)
    for N, n_cls, n_reg, W in ((4099, 284, 12, 320), (37, 18, 12, 64), (0, 284, 12, 320)):
        out = (torch.randn(N, W, device=_dev()) * 2).bfloat16()
        if N:
            out[: N // 3, n_cls + 1:n_cls + 7] -= 30.0         # exp(s x) < 1e-3: the clamp floor, zero gradient
        bias = torch.randn(n_cls, device=_dev())
        scale = torch.tensor(1.3, device=_dev())
        g_cls = torch.randn(N, n_cls, device=_dev()).bfloat16()
        g_ctr = torch.randn(N, 1, device=_dev())
        g_box = torch.randn(N, n_reg, device=_dev())

        o1, b1, s1 = out.clone().requires_grad_(True), bias.clone().requires_grad_(True), scale.clone().requires_grad_(True)
        cls, ctr, box, score = DH._HeadSplit.apply(o1, b1, s1, n_cls, n_reg)
        assert not score.requires_grad
        (cls.float() * g_cls.float()).sum().add((ctr * g_ctr).sum()).add((box * g_box).sum()).backward()

        o2, b2, s2 = out.clone().requires_grad_(True), bias.clone().requires_grad_(True), scale.clone().requires_grad_(True)
        cls_r = o2[:, :n_cls] + b2.to(o2.dtype)
        small = o2[:, n_cls:n_cls + 1 + n_reg].float()
        ctr_r, reg = small[:, :1], small[:, 1:]
        box_r = torch.cat((torch.exp(reg[:, :6] * s2).clamp(min=1e-3), reg[:, 6:]), 1)
        (cls_r.float() * g_cls.float()).sum().add((ctr_r * g_ctr).sum()).add((box_r * g_box).sum()).backward()

        assert cls.shape == (N, n_cls) and ctr.shape == (N, 1) and box.shape == (N, n_reg) and score.shape == (N, 1)
        assert o1.grad.shape == (N, W)
        if N == 0:
            continue
        assert torch.equal(cls, cls_r) and torch.equal(ctr, ctr_r)
        _close(box, box_r, 1e-6, 'head epilogue bbox')
        assert torch.equal(score, cls_r.max(1, keepdim=True).values.float())
        assert float(o1.grad[:, n_cls + 1 + n_reg:].abs().max()) == 0.0
        assert float(o1.grad[: N // 3, n_cls + 1:n_cls + 7].abs().max()) == 0.0
        _close(o1.grad, o2.grad, 1e-2, 'head epilogue dout')
        _close(b1.grad, b2.grad, 1e-2, 'head epilogue dbias')
        _close(s1.grad, s2.grad, 1e-3, 'head epilogue dscale')
