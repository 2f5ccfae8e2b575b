"""Host-side logic of the product exercised without a GPU: the C-ABI call is replaced by a numpy emulation of the ONE
kernel involved, so that batching / padding / bookkeeping code cannot hide a Python
error behind the GPU tests. The emulation lives only here; the product itself never falls back to the CPU."""
import ctypes
import os
import sys

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]


def _emulated_img_normalize(calls):
    def fake_call(name, src_ptr, n_img, H, W, Hp, Wp, mean_p, std_p, conv, channels_last, dst_ptr, dcode, stream):
        assert name == 'esb_img_normalize' and channels_last == 1 and dcode == 0
        calls.append((n_img, H, W, Hp, Wp))
        src = np.ctypeslib.as_array(ctypes.cast(src_ptr, ctypes.POINTER(ctypes.c_ubyte)), shape=(n_img, 3, H, W))
        dst = np.ctypeslib.as_array(ctypes.cast(dst_ptr, ctypes.POINTER(ctypes.c_float)), shape=(n_img, Hp, Wp, 3))
        mean = np.ctypeslib.as_array(ctypes.cast(mean_p, ctypes.POINTER(ctypes.c_float)), shape=(3, ))
        std = np.ctypeslib.as_array(ctypes.cast(std_p, ctypes.POINTER(ctypes.c_float)), shape=(3, ))
        dst[:] = 0
        s = src[:, ::-1] if conv else src
        dst[:, :H, :W, :] = ((s.astype(np.float32) - mean[None, :, None, None]) / std[None, :, None, None]) \
            .transpose(0, 2, 3, 1)
    return fake_call


def test_preprocessor_batching_and_padding(monkeypatch):
    import embodiedscan_b200.detectors as D
    from cases import preprocess_inputs
    from embodiedscan_b200.structures import Det3DDataSample
    from oracle import data_ref as R
    calls = []
    monkeypatch.setattr(D, 'call', _emulated_img_normalize(calls))
    monkeypatch.setattr(D, 'stream', lambda: None)
    gold = np.load(os.path.join(GOLD, 'frontend.npz'))
    pre = D.Det3DDataPreprocessor(mean=MEAN, std=STD, bgr_to_rgb=True, pad_size_divisor=32)
    # mixed view sizes: one launch per scan into its slice of the batch buffer, padded to the batch maximum
    samples = [Det3DDataSample(metainfo={}), Det3DDataSample(metainfo={})]
    out = pre(dict(inputs=dict(img=preprocess_inputs()), data_samples=samples))
    assert torch.equal(out['inputs']['imgs'], torch.from_numpy(gold['pre_imgs']))
    assert calls == [(2, 30, 45, 64, 64), (2, 33, 40, 64, 64)]
    assert [s.metainfo['pad_shape'] for s in samples] == [tuple(r) for r in gold['pre_pad_shape'].tolist()]
    # the usual uniform batch stays ONE launch, whatever container the dataloader hands over
    g = torch.Generator().manual_seed(3)
    five = torch.randint(0, 256, (2, 3, 3, 40, 50), generator=g, dtype=torch.uint8)
    for inp, ref in ((five, list(five)), (list(five), list(five)), (five[:, 0], [x[None] for x in five[:, 0]])):
        calls.clear()
        out = pre(dict(inputs=dict(img=inp)))['inputs']['imgs']
        assert len(calls) == 1 and calls[0][1:] == (40, 50, 64, 64)
        assert torch.equal(out, R.preprocess_multiview(ref, MEAN, STD))
        assert out.shape[2] == 3 and out.stride(2) == 1, 'channels-last memory under a (B,V,3,H,W) view'


def test_preprocessor_batchwise_continuous_inputs(monkeypatch):
    """batchwise_inputs=True: one scan with per-prefix annotation lists -> N samples, nested point lists kept."""
    import embodiedscan_b200.detectors as D
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_golden_cpu import continuous_batch
    calls = []
    monkeypatch.setattr(D, 'call', _emulated_img_normalize(calls))
    monkeypatch.setattr(D, 'stream', lambda: None)
    pre = D.Det3DDataPreprocessor(mean=MEAN, std=STD, bgr_to_rgb=True, pad_size_divisor=32, batchwise_inputs=True)
    data, res = continuous_batch()
    out = pre(data, True)
    assert len(out['data_samples']) == 3 and len(calls) == 1
    assert out['inputs']['imgs'].shape == (1, 3, 3, 256, 320)
    assert [len(p) == 1 and p[0].shape[0] for p in out['inputs']['points']] == [500, 1000, 1500]
    assert all(s.metainfo['pad_shape'] == (256, 320) for s in out['data_samples'])
    assert [len(s.gt_instances_3d.labels_3d) for s in out['data_samples']] == [len(l) for l in res['gt_labels_3d']]


def test_continuous_detector_view_prefix_painting_control_flow(monkeypatch):
    """Embodied3DDetector.extract_feat with the CUDA pieces replaced by recorders: sample idx must be painted from the
    contiguous view-prefix slice feat[:idx+1] with its own meta / projection prefix, rows scattered back in place."""
    import types

    import embodiedscan_b200.detectors as D

    class FakeST:
        def __init__(self, C, F, nb):
            self.C, self.F, self.nb = C, F, nb

        @property
        def decomposition_permutations(self):
            return [torch.nonzero(self.C[:, 0] == b).squeeze(1) for b in range(self.nb)]

        def replace_feature(self, f):
            return FakeST(self.C, f, self.nb)

    g = torch.Generator().manual_seed(0)
    n_prefix, V = 3, 3
    coords = torch.cat([torch.cat([torch.full((n, 1), b), torch.randint(0, 50, (n, 3), generator=g)], 1)
                        for b, n in enumerate((4, 0, 6))]).int()
    coords = coords[torch.randperm(coords.shape[0], generator=g)]            # interleaved rows, one empty prefix
    feats3d = torch.randn(coords.shape[0], 5, generator=g)
    levels = [FakeST(coords, feats3d, n_prefix)]
    calls = []

    def fake_paint(feat, c, metas, proj, voxel_size, pad_hw, n_views):
        assert feat.is_contiguous(memory_format=torch.channels_last) and feat.shape[0] == n_views
        assert proj.shape == (1, n_views, 4, 4) and proj.is_contiguous() and int(c[:, 0].abs().sum()) == 0
        calls.append((n_views, c.shape[0], int(metas[0])))
        return torch.full((c.shape[0], feat.shape[1]), float(n_views))
    monkeypatch.setattr(D, 'paint_points', fake_paint)
    monkeypatch.setattr(D, 'pack_paint_metas', lambda ms, dev: torch.tensor([ms[0]['tag']]))
    monkeypatch.setattr(D, 'pack_projections', lambda ms, ct, dev: torch.zeros(1, V, 4, 4))
    monkeypatch.setattr(D.SP, 'SparseTensor', lambda **kw: None)
    det = D.Embodied3DDetector.__new__(D.Embodied3DDetector)
    torch.nn.Module.__init__(det)
    det.compute_dtype, det.voxel_size, det.coord_type = torch.float32, 0.01, 'DEPTH'
    det.backbone = lambda x: [torch.randn(V, 7, 4, 6).contiguous(memory_format=torch.channels_last)]
    det.backbone_3d = lambda x: levels
    det.voxelize = lambda pts: (torch.zeros(1, 4, dtype=torch.int32), torch.zeros(1, 3))
    samples = [types.SimpleNamespace(metainfo=dict(tag=10 + i)) for i in range(n_prefix)]
    out = det.extract_feat(dict(points=[[torch.zeros(2, 3)] for _ in range(n_prefix)],
                                imgs=torch.zeros(1, V, 3, 32, 32)), samples)
    assert calls == [(1, 4, 10), (3, 6, 12)], calls                          # the empty prefix launches nothing
    f = out[0].F
    assert f.shape == (coords.shape[0], 5 + 7) and torch.equal(f[:, :5], feats3d)
    want = torch.tensor([1., 0., 3.])[coords[:, 0].long()]
    assert torch.equal(f[:, 5:], want[:, None].expand(-1, 7))


def test_morton_row_order_is_stable_and_hierarchical():
    """ESB200_ROW_ORDER=morton (opt-in): one stable sort of the raw voxel coordinates by (scan, Z-order)."""
    from embodiedscan_b200.sparse import _spread3, morton_order
    from oracle import sparse_ref as S
    g = torch.Generator().manual_seed(1)
    v = torch.randint(0, 65536, (200, ), generator=g)
    slow = torch.tensor([sum(((int(x) >> i) & 1) << (3 * i) for i in range(16)) for x in v])
    assert torch.equal(_spread3(v), slow)
    coords = torch.cat([torch.randint(0, 2, (4000, 1), generator=g), torch.randint(-40, 40, (4000, 3), generator=g)], 1).int()
    order = morton_order(coords)
    assert torch.equal(torch.sort(order).values, torch.arange(4000)), 'a permutation'
    sc = coords[order]
    # stable: rows of one voxel keep their input order, so first-occurrence dedup keeps the same point per voxel
    u0, in2out0 = S.unique_first(coords.numpy())
    u1, in2out1 = S.unique_first(sc.numpy())
    first0 = np.full(len(u0), 10 ** 9)
    np.minimum.at(first0, in2out0, np.arange(4000))
    first1 = np.full(len(u1), 10 ** 9)
    np.minimum.at(first1, in2out1, order.numpy())            # original index of the first sorted row of each voxel
    k0 = {tuple(c): f for c, f in zip(u0.tolist(), first0.tolist())}
    k1 = {tuple(c): f for c, f in zip(u1.tolist(), first1.tolist())}
    assert k0 == k1, 'same voxels, same representative point'
    # hierarchical: scans stay contiguous, and the first-occurrence parents at stride 2, 4, 8 are Z-ordered themselves

    def zkey(c):
        c = torch.as_tensor(c).long()
        return (c[:, 0] << 48) | _spread3(c[:, 1] + 32768) | (_spread3(c[:, 2] + 32768) << 1) | (_spread3(c[:, 3] + 32768) << 2)
    cur = u1
    for stride in (2, 4, 8):
        cur = S.unique_first(cur, stride)[0]
        k = zkey(cur)
        assert bool((k[1:] > k[:-1]).all()), f'stride-{stride} parents inherit the order'


def _emulate_conv2d_tc(src, wt, n_img, Hs, Ws, cs, Hr, Wr, cr, kh, kw, stride, pad, r_pad, transposed):
    """Index arithmetic of csrc/conv2d_tc.cu's producer, spelled out per (row pixel, 16-byte piece) in numpy:
    src (n_img,Hs,Ws,cs) NHWC, wt (cr, r_pad) K-major weights -> (n_img*Hr*Wr, cr). Mirrors the kernel's formulas
    line by line (iy0/ix0, tap/ch split of the reduction index, exact-division test of the transposed mode)."""
    M = n_img * Hr * Wr
    A = np.zeros((M, r_pad), np.float32)
    taps = kh * kw
    for m in range(M):
        n, rem = divmod(m, Hr * Wr)
        oy, ox = divmod(rem, Wr)
        iy0 = oy + pad if transposed else oy * stride - pad
        ix0 = ox + pad if transposed else ox * stride - pad
        for r0 in range(0, r_pad, 8):
            tap, ch = divmod(r0, cs)
            ky, kx = divmod(tap, kw)
            ok = tap < taps
            if not transposed:
                iy, ix = iy0 + ky, ix0 + kx
            else:
                ny, nx = iy0 - ky, ix0 - kx
                iy, ix = int(ny / stride), int(nx / stride)          # C division truncates toward zero
                ok = ok and ny >= 0 and nx >= 0 and iy * stride == ny and ix * stride == nx
            ok = ok and 0 <= iy < Hs and 0 <= ix < Ws
            if ok:
                A[m, r0:r0 + 8] = src[n, iy, ix, ch:ch + 8]
    return A @ wt.T


def test_conv2d_tc_index_arithmetic_forward_and_transposed():
    """The gather formulas and the weight packings of the experimental wgmma conv2d (forward and dgrad mode) reproduce
    F.conv2d and its input gradient when evaluated literally on the CPU (the tensor-core plumbing itself needs an H100)."""
    import torch.nn.functional as F
    from embodiedscan_b200.backbones import pack_ohwi
    g = torch.Generator().manual_seed(0)
    for cin, cout, k, stride, pad, hw in ((16, 8, 3, 1, 1, (6, 7)), (8, 16, 3, 2, 1, (7, 9)), (16, 24, 1, 2, 0, (6, 8)),
                                          (8, 8, 7, 2, 3, (12, 10))):
        n = 2
        x = torch.randn(n, cin, *hw, generator=g).bfloat16().float()
        w = torch.randn(cout, cin, k, k, generator=g).bfloat16().float()
        H, W = hw
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        xr = x.clone().requires_grad_(True)
        ref = F.conv2d(xr, w, None, stride, pad)
        wp = pack_ohwi(w).float().numpy()
        out = _emulate_conv2d_tc(x.permute(0, 2, 3, 1).numpy(), wp, n, H, W, cin, Ho, Wo, cout, k, k, stride, pad,
                                 wp.shape[1], False)
        want = ref.detach().permute(0, 2, 3, 1).reshape(-1, cout).numpy()
        assert np.abs(out - want).max() <= 1e-3 * max(np.abs(want).max(), 1), (cin, cout, k, stride)
        dy = torch.randn(ref.shape, generator=g).bfloat16().float()
        ref.backward(dy)
        flat = w.permute(1, 2, 3, 0).reshape(cin, -1)                    # (ci | ky, kx, co), as conv2d_tc_dgrad packs it
        r_pad = (flat.shape[1] + 63) // 64 * 64
        wt = np.zeros((cin, r_pad), np.float32)
        wt[:, :flat.shape[1]] = flat.numpy()
        dx = _emulate_conv2d_tc(dy.permute(0, 2, 3, 1).numpy(), wt, n, Ho, Wo, cout, H, W, cin, k, k, stride, pad, r_pad,
                                True)
        want = xr.grad.permute(0, 2, 3, 1).reshape(-1, cin).numpy()
        assert np.abs(dx - want).max() <= 1e-3 * max(np.abs(want).max(), 1), ('dgrad', cin, cout, k, stride)
        # wgrad: dW^T[r, co] = sum_m A[m, r] dy[m, co] with the forward's implicit A, unpacked like conv2d_tc_wgrad
        wr = w.clone().requires_grad_(True)
        F.conv2d(x, wr, None, stride, pad).backward(dy)
        eye = np.eye(wp.shape[1], dtype=np.float32)                       # identity weights expose A itself
        A = _emulate_conv2d_tc(x.permute(0, 2, 3, 1).numpy(), eye, n, H, W, cin, Ho, Wo, wp.shape[1], k, k, stride, pad,
                               wp.shape[1], False)
        dw_t = A.T @ dy.permute(0, 2, 3, 1).reshape(-1, cout).numpy()
        dw = torch.from_numpy(dw_t[:k * k * cin]).view(k, k, cin, cout).permute(3, 2, 0, 1)
        assert float((dw - wr.grad).abs().max()) <= 1e-3 * max(float(wr.grad.abs().max()), 1), ('wgrad', cin, cout, k)


def test_continuous_occupancy_view_prefix_painting_control_flow(monkeypatch):
    """EmbodiedOccPredictor.extract_feat with the CUDA pieces replaced by recorders: prefix idx paints the whole prior
    grid from feat2d[:idx+1] with its own projection prefix; volumes are stacked per prefix and fused with the sparse
    volume of the same batch size."""
    import types

    import embodiedscan_b200.occupancy as O
    n_prefix, V, C2d, C3d = 3, 3, 6, 5
    n_vox = [4, 4, 2]
    calls = []

    def fake_paint(feat, pts, batch, metas, proj, pad_hw, n_views):
        assert feat.is_contiguous(memory_format=torch.channels_last) and feat.shape[0] == n_views and batch is None
        assert proj.shape == (1, n_views, 4, 4) and proj.is_contiguous() and pts.shape == (32, 3)
        calls.append((n_views, int(metas[0])))
        return torch.full((pts.shape[0], feat.shape[1]), float(n_views))
    monkeypatch.setattr(O, 'paint_float_points', fake_paint)
    monkeypatch.setattr(O, 'pack_paint_metas', lambda ms, dev: torch.tensor([ms[0]['tag']]))
    monkeypatch.setattr(O, 'pack_projections', lambda ms, ct, dev: torch.zeros(1, V, 4, 4))
    m = O.EmbodiedOccPredictor.__new__(O.EmbodiedOccPredictor)
    torch.nn.Module.__init__(m)
    m.compute_dtype, m.coord_type, m.n_voxels = torch.float32, 'DEPTH', n_vox
    m.backbone = lambda x: x
    m.neck = lambda x: [torch.randn(V, C2d, 8, 8).contiguous(memory_format=torch.channels_last)]
    m.prior_generator = types.SimpleNamespace(grid_anchors=lambda sizes, device: [torch.rand(32, 7)])
    seen = {}

    def fake_sparse(points, prior):
        seen['n'] = [p.shape[0] for p in points]
        return torch.ones(len(points), C3d, *n_vox)
    m.sparse_volume = fake_sparse
    m.neck_3d = lambda x: [x]
    samples = [types.SimpleNamespace(metainfo=dict(tag=20 + i, depth2img=dict(origin=[0.1, 0.2, 0.3])))
               for i in range(n_prefix)]
    feats, valid = m.extract_feat(dict(points=[[torch.zeros(5 * (i + 1), 3)] for i in range(n_prefix)],
                                       imgs=torch.zeros(1, V, 3, 32, 32)), samples)
    assert calls == [(1, 20), (2, 21), (3, 22)] and seen['n'] == [5, 10, 15]
    fused = feats[0]
    assert fused.shape == (n_prefix, C2d + C3d, *n_vox) and valid.shape == (n_prefix, 1, *n_vox)
    for i in range(n_prefix):
        assert float(fused[i, :C2d].min()) == float(fused[i, :C2d].max()) == float(i + 1)
    assert float(fused[:, C2d:].min()) == 1.0 and float(valid.min()) == 1.0


def test_optim_wrapper_paramwise_lr_mult_and_gc_schedule():
    """engine.OptimWrapper: mmengine `paramwise_cfg.custom_keys` becomes one per-element multiplier over the arena (longest key
    wins), and the wrapper takes the cyclic collector over (automatic collection off, scheduled young-generation passes)."""
    import gc
    import torch
    from embodiedscan_b200.engine import OptimWrapper
    net = torch.nn.Sequential()
    net.add_module('decoder', torch.nn.Linear(4, 4))
    net.add_module('text_encoder', torch.nn.Linear(4, 2))
    net.add_module('head', torch.nn.Linear(2, 2))
    was = gc.isenabled()
    try:
        ow = OptimWrapper(net, paramwise_cfg=dict(custom_keys={'decoder': dict(lr_mult=0.1), 'text_encoder': dict(lr_mult=0.0),
                                                               'decoder.bias': dict(lr_mult=0.5)}), gc_interval=7)
        assert not gc.isenabled() and ow.gc_interval == 7
        m = ow.optimizer.lr_mult
        for p, o in zip(ow.arena.params, ow.arena.offsets):
            name = {id(q): n for n, q in net.named_parameters()}[id(p)]
            want = 0.5 if name == 'decoder.bias' else 0.1 if name.startswith('decoder') else 0.0 if name.startswith('text') else 1.0
            assert torch.all(m[o:o + p.numel()] == want), (name, want)
        assert OptimWrapper(net, gc_interval=None).optimizer.lr_mult is None
    finally:
        gc.enable() if was else gc.disable()


def test_train_step_log_vars_carry_no_autograd_history():
    """detectors.detach_log_vars: what `train_step` returns must not keep the finished step's graph (and through it the kernel
    maps of the sparse-conv nodes) alive in the caller's hands."""
    import torch
    from embodiedscan_b200.detectors import detach_log_vars, parse_losses
    w = torch.ones(3, requires_grad=True)
    loss, log_vars = parse_losses({'loss_a': (w * 2).sum(), 'loss_b': [(w * 3).sum(), (w * 4).sum()], 'acc': torch.tensor(0.5)})
    assert loss.requires_grad and log_vars['loss'].grad_fn is not None
    out = detach_log_vars(log_vars)
    assert set(out) == set(log_vars)
    assert all(v.grad_fn is None and not v.requires_grad for v in out.values())
    assert float(out['loss']) == float(loss) == 6 + 9 + 12


def _host_view(address, shape, dtype):
    """A torch tensor over raw host memory (the emulated kernels below read and write through the pointers they are given)."""
    n = int(np.prod(shape))
    if n == 0:
        return torch.empty(shape, dtype=dtype)
    ctype = {torch.float32: ctypes.c_float, torch.bfloat16: ctypes.c_uint16}[dtype]
    arr = np.ctypeslib.as_array((ctype * n).from_address(address))
    t = torch.from_numpy(arr)
    return (t.view(torch.bfloat16) if dtype == torch.bfloat16 else t).reshape(shape)


def test_head_epilogue_function_plumbing_with_model_shaped_parameters(monkeypatch):
    """dense_heads._HeadSplit around an emulation of esb_head_split_fwd / _bwd that works through the raw pointers: the host
    side (buffer shapes, (1, n_cls) bias and 0-dim Scale parameters as the model holds them, gradient shapes and dtypes,
    non-differentiable pruning score) against the ATen chain of fcaf3d_head.py:1116-1149. The kernels themselves are checked
    on the GPU (tests/test_kernels_gpu.py)."""
    from embodiedscan_b200 import dense_heads as DH

    def fake_call(name, *a):
        if name == 'esb_head_split_fwd':
            out_p, bias_p, scale_p, N, W, n_cls, n_reg, n_exp, lo, cls_p, ctr_p, box_p, score_p, _ = a
            out = _host_view(out_p, (N, W), torch.bfloat16).float()
            bias = _host_view(bias_p, (n_cls, ), torch.float32).bfloat16().float()
            s = _host_view(scale_p, (1, ), torch.float32)[0]
            cls = (out[:, :n_cls] + bias).bfloat16()
            _host_view(cls_p, (N, n_cls), torch.bfloat16).copy_(cls)
            _host_view(ctr_p, (N, 1), torch.float32).copy_(out[:, n_cls:n_cls + 1])
            reg = out[:, n_cls + 1:n_cls + 1 + n_reg]
            _host_view(box_p, (N, n_reg), torch.float32).copy_(
                torch.cat((torch.exp(reg[:, :n_exp] * s).clamp(min=lo), reg[:, n_exp:]), 1))
            _host_view(score_p, (N, 1), torch.float32).copy_(cls.float().max(1, keepdim=True).values)
        elif name == 'esb_head_split_bwd':
            out_p, dcls_p, dctr_p, dbox_p, scale_p, N, W, n_cls, n_reg, n_exp, lo, dout_p, dbias_p, dscale_p, _ = a
            out = _host_view(out_p, (N, W), torch.bfloat16).float()
            s = _host_view(scale_p, (1, ), torch.float32)[0]
            dcls = _host_view(dcls_p, (N, n_cls), torch.bfloat16)
            dbox = _host_view(dbox_p, (N, n_reg), torch.float32).clone()
            x = out[:, n_cls + 1:n_cls + 1 + n_exp]
            e = torch.exp(x * s)
            live = (e >= lo).float()
            _host_view(dscale_p, (1, ), torch.float32).add_((dbox[:, :n_exp] * e * x * live).sum())
            dbox[:, :n_exp] *= e * s * live
            dout = _host_view(dout_p, (N, W), torch.bfloat16)
            dout.zero_()
            dout[:, :n_cls] = dcls
            dout[:, n_cls:n_cls + 1] = _host_view(dctr_p, (N, 1), torch.float32).bfloat16()
            dout[:, n_cls + 1:n_cls + 1 + n_reg] = dbox.bfloat16()
            _host_view(dbias_p, (n_cls, ), torch.float32).add_(dcls.float().sum(0))
        else:
            raise AssertionError(name)

    monkeypatch.setattr(DH, 'call', fake_call)
    monkeypatch.setattr(DH, 'stream', lambda: None)
    torch.manual_seed(3)
    N, n_cls, n_reg, W = 53, 18, 12, 64
    out = (torch.randn(N, W) * 2).bfloat16()
    out[:9, n_cls + 1:n_cls + 7] -= 30.0
    bias = torch.randn(1, n_cls)                     # MinkowskiConvolution bias layout
    scale = torch.tensor(0.7)                        # mmcv Scale: 0-dim
    g_cls, g_ctr, g_box = torch.randn(N, n_cls).bfloat16(), torch.randn(N, 1), torch.randn(N, n_reg)

    o1, b1, s1 = out.clone().requires_grad_(True), bias.clone().requires_grad_(True), scale.clone().requires_grad_(True)
    cls, ctr, box, score = DH._HeadSplit.apply(o1, b1, s1, n_cls, n_reg)
    assert cls.dtype == torch.bfloat16 and ctr.dtype == box.dtype == score.dtype == torch.float32
    assert not score.requires_grad and cls.requires_grad and box.requires_grad
    (cls.float() * g_cls.float()).sum().add((ctr * g_ctr).sum()).add((box * g_box).sum()).backward()

    o2, b2, s2 = out.clone().requires_grad_(True), bias.clone().requires_grad_(True), scale.clone().requires_grad_(True)
    cls_r = o2[:, :n_cls] + b2.to(o2.dtype)
    small = o2[:, n_cls:n_cls + 1 + n_reg].float()
    reg = small[:, 1:]
    box_r = torch.cat((torch.exp(reg[:, :6] * s2).clamp(min=1e-3), reg[:, 6:]), 1)
    (cls_r.float() * g_cls.float()).sum().add((small[:, :1] * g_ctr).sum()).add((box_r * g_box).sum()).backward()

    assert torch.equal(cls, cls_r) and torch.equal(ctr, small[:, :1]) and torch.equal(box, box_r)
    assert torch.equal(score, cls_r.max(1, keepdim=True).values.float())
    assert b1.grad.shape == bias.shape and s1.grad.shape == scale.shape and o1.grad.shape == out.shape
    assert b1.grad.dtype == torch.float32 and o1.grad.dtype == torch.bfloat16
    assert torch.equal(o1.grad, o2.grad)
    assert float((b1.grad - b2.grad).abs().max()) <= 2e-2 * float(b2.grad.abs().max())      # reference sums in bf16
    assert float((s1.grad - s2.grad).abs()) <= 1e-4 * float(s2.grad.abs())
