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
