"""Occupancy variant of the hot path (SURVEY §8 row a14, BASELINE.json config C3), registered under the reference's
names: ``DenseFusionOccPredictor`` (embodiedscan/models/detectors/dense_fusion_occ.py:26-467), ``IndoorImVoxelNeck``
(models/necks/imvoxel_neck.py:8-143), ``ImVoxelOccHead`` (models/dense_heads/imvoxel_occ_head.py:19-184),
``AlignedAnchor3DRangeGenerator`` (models/task_modules/anchor/anchor_3d_generator.py:241-354), ``mmdet.FPN`` and the
SurroundOcc losses (models/losses/occ_loss.py:7-141).

Shares the front half with the detector — voxel hashing, MinkResNet34 and the point-painting kernel (here on the prior
grid's fp32 voxel centres) all run in libesb200.so. The dense Conv3d FPN is the one tensor-core-bound stage of the named
configs (~4 TFLOP/scan); this round it is evaluated by the library convolution (cuDNN) in channels-last-3d bf16 — the
wgmma implicit-GEMM Conv3d is listed in DESIGN.md §7.
"""
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import sparse as SP
from .detectors import detach_log_vars, parse_losses
from .fusion import pack_paint_metas, pack_projections, paint_float_points
from .registry import MODELS, TASK_UTILS


@TASK_UTILS.register_module()
class AlignedAnchor3DRangeGenerator:
    """Only what the occupancy model uses: voxel-centre priors of one range (anchor_3d_generator.py:271-354)."""

    def __init__(self, ranges, sizes=((3.9, 1.6, 1.56), ), scales=(1, ), rotations=(0, 1.5707963), custom_values=(),
                 reshape_out=True, size_per_range=True, align_corner=False):
        self.ranges, self.sizes, self.scales, self.rotations = ranges, sizes, scales, list(rotations)
        self.align_corner = align_corner

    def grid_anchors(self, featmap_sizes, device='cuda'):
        out = []
        for fs in featmap_sizes:                      # fs = (D, H, W) = (z, y, x)
            r = torch.tensor(self.ranges[0], device=device)
            axes = []
            for lo, hi, n in ((r[2], r[5], fs[0]), (r[1], r[4], fs[1]), (r[0], r[3], fs[2])):
                c = torch.linspace(lo, hi, n + 1, device=device)
                if not self.align_corner:
                    c = c + (c[1] - c[0]) / 2
                axes.append(c[:n])
            z, y, x = axes
            n_anchor = len(self.rotations) * len(self.sizes)
            zz, yy, xx = torch.meshgrid(z, y, x, indexing='ij')          # z slowest, x fastest (the reference's permute)
            ctr = torch.stack([xx, yy, zz], -1).reshape(-1, 1, 3).repeat(1, n_anchor, 1).reshape(-1, 3)
            out.append(torch.cat([ctr, ctr.new_zeros((ctr.shape[0], 4))], 1))
        return out


@MODELS.register_module(name=['mmdet.FPN', 'FPN'])
class FPN(nn.Module):
    """mmdet.FPN (†upstream) for num_outs == len(in_channels), no norm / activation, nearest top-down upsampling."""

    def __init__(self, in_channels, out_channels, num_outs, **kwargs):
        super().__init__()
        assert num_outs == len(in_channels)
        self.lateral_convs = nn.ModuleList([_ConvOnly(c, out_channels, 1) for c in in_channels])
        self.fpn_convs = nn.ModuleList([_ConvOnly(out_channels, out_channels, 3, padding=1) for _ in in_channels])
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.xavier_uniform_(m.weight)
                nn.init.zeros_(m.bias)

    def forward(self, inputs):
        lat = [l(x) for l, x in zip(self.lateral_convs, inputs)]
        for i in range(len(lat) - 1, 0, -1):
            lat[i - 1] = lat[i - 1] + F.interpolate(lat[i], size=lat[i - 1].shape[2:], mode='nearest')
        return tuple(c(x) for c, x in zip(self.fpn_convs, lat))


class _ConvOnly(nn.Module):
    """mmcv ConvModule without norm/act: parameters live under `.conv`."""

    def __init__(self, cin, cout, k, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, padding=padding)

    def forward(self, x):
        return F.conv2d(x, self.conv.weight.to(x.dtype), self.conv.bias.to(x.dtype), 1, self.conv.padding)


def _tma3d_ok(x, conv) -> bool:
    """The dense 3-D stack runs on the library's TMA + wgmma kernels (csrc/conv_tma.cu, rank-5 tensor maps) when the
    activations are bf16 on the GPU and the channel counts tile (16, 32, multiples of 64; outputs a power of two <= 256 or a
    multiple of 256); anything else (fp32 parity arithmetic, toy widths) stays on the library convolution."""
    import os
    if not (x.is_cuda and x.dtype == torch.bfloat16 and os.environ.get('ESB200_CONV3D', 'own') == 'own'):
        return False
    cin, cout = (conv.in_channels, conv.out_channels)

    def ok(c):
        return c in (16, 32) or (c >= 64 and c % 64 == 0)

    def ok_out(c):
        return (c <= 256 and c & (c - 1) == 0 and c >= 16) or (c > 256 and c % 256 == 0)

    if isinstance(conv, nn.ConvTranspose3d):
        return cin % 64 == 0 and (8 * cout) % 64 == 0 and tuple(conv.kernel_size) == (2, 2, 2) and tuple(conv.stride) == (2, 2, 2)
    k, st, pd = conv.kernel_size, conv.stride, conv.padding
    return (ok(cin) and ok(cout) and ok_out(cout) and ok_out(cin) and k[0] == k[1] == k[2] and k[0] in (1, 3)
            and st[0] == st[1] == st[2] and st[0] in (1, 2) and pd[0] == pd[1] == pd[2])


class _Conv3dTMA(torch.autograd.Function):
    """nn.Conv3d (bias-free) on NDHWC bf16 volumes with the library's kernels, all three passes (esb_conv3d_tma_*)."""

    @staticmethod
    def forward(ctx, x, w, stride, pad):
        from . import _ffi
        N, cin, D, H, W = x.shape
        cout, _, k = w.shape[0], w.shape[1], w.shape[2]
        if not x.is_contiguous(memory_format=torch.channels_last_3d):
            x = x.contiguous(memory_format=torch.channels_last_3d)
        w_odhwi = w.detach().permute(0, 2, 3, 4, 1).contiguous()
        Do, Ho, Wo = ((D + 2 * pad - k) // stride + 1, (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1)
        y = torch.empty((N, cout, Do, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last_3d)
        _ffi.call('esb_conv3d_tma_fwd', x.data_ptr(), w_odhwi.data_ptr(), None, None, y.data_ptr(), N, D, H, W, cin, cout, k,
                  stride, pad, 0, _ffi.stream())
        ctx.save_for_backward(x, w_odhwi)
        ctx.geom = (stride, pad)
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import _ffi
        x, w_odhwi = ctx.saved_tensors
        stride, pad = ctx.geom
        N, cin, D, H, W = x.shape
        cout, k = w_odhwi.shape[0], w_odhwi.shape[1]
        if not dy.is_contiguous(memory_format=torch.channels_last_3d):
            dy = dy.contiguous(memory_format=torch.channels_last_3d)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _ffi.call('esb_conv3d_tma_dgrad', dy.data_ptr(), w_odhwi.data_ptr(), dx.data_ptr(), N, D, H, W, cin, cout, k, stride,
                      pad, _ffi.stream())
        if ctx.needs_input_grad[1]:
            dw_t = torch.zeros((k * k * k * cin, cout), dtype=torch.float32, device=x.device)
            _ffi.call('esb_conv3d_tma_wgrad', x.data_ptr(), dy.data_ptr(), dw_t.data_ptr(), N, D, H, W, cin, cout, k, stride, pad,
                      _ffi.stream())
            dw = dw_t.view(k, k, k, cin, cout).permute(4, 3, 0, 1, 2).to(x.dtype)
        return dx, dw, None, None


def _bn3d(bn, x, act=0, res=None):
    """BatchNorm3d (+ residual) (+ ReLU) on an NDHWC volume through the row kernels of the sparse path (one segment)."""
    if x.is_cuda and x.is_contiguous(memory_format=torch.channels_last_3d) and x.dtype in (torch.float32, torch.bfloat16) \
            and x.shape[1] % 8 == 0:
        N, C, D, H, W = x.shape
        rows = x.permute(0, 2, 3, 4, 1).reshape(-1, C)
        rres = res.contiguous(memory_format=torch.channels_last_3d).permute(0, 2, 3, 4, 1).reshape(-1, C) if res is not None else None
        y = SP.batch_norm_rows(rows, bn, bn.training, act, rres)
        return y.view(N, D, H, W, C).permute(0, 4, 1, 2, 3)
    y = bn(x)
    if res is not None:
        y = y + res
    return F.relu(y) if act == SP.ACT_RELU else y


class ResModule(nn.Module):

    def __init__(self, in_channels, out_channels, stride=1):
        super().__init__()
        self.stride = stride
        self.conv1 = nn.Conv3d(in_channels, out_channels, 3, stride, 1, bias=False)
        self.norm1 = nn.BatchNorm3d(out_channels)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv3d(out_channels, out_channels, 3, 1, 1, bias=False)
        self.norm2 = nn.BatchNorm3d(out_channels)
        if self.stride != 1:
            self.downsample = nn.Sequential(nn.Conv3d(in_channels, out_channels, 1, stride, bias=False),
                                            nn.BatchNorm3d(out_channels))

    def forward(self, x):
        identity = x
        out = _bn3d(self.norm1, _conv3d(self.conv1, x), SP.ACT_RELU)
        out = _conv3d(self.conv2, out)
        if self.stride != 1:
            identity = _bn3d(self.downsample[1], _conv3d(self.downsample[0], x))
        return _bn3d(self.norm2, out, SP.ACT_RELU, res=identity)          # relu(norm2(out) + identity), one pass


def _conv3d(conv, x):
    if _tma3d_ok(x, conv):
        w = SP.weight_operand(conv.weight, x.dtype)
        if isinstance(conv, nn.ConvTranspose3d):
            # k2 s2 transpose = a dense GEMM (voxels, Cin) x (Cin, 8*Cout) on the tensor-core rows kernel, then the 2x2x2
            # children interleave into the fine grid
            N, cin, D, H, W = x.shape
            cout = conv.out_channels
            rows = x.contiguous(memory_format=torch.channels_last_3d).permute(0, 2, 3, 4, 1).reshape(-1, cin)
            wm = w.permute(0, 2, 3, 4, 1).reshape(cin, 8 * cout)                # (ci | i, j, k, co)
            y = SP.rows_gemm(rows, wm).view(N, D, H, W, 2, 2, 2, cout)
            y = y.permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(N, 2 * D, 2 * H, 2 * W, cout)
            return y.permute(0, 4, 1, 2, 3)                                     # NCDHW view of NDHWC memory
        return _Conv3dTMA.apply(x, w, conv.stride[0], conv.padding[0])
    if isinstance(conv, nn.ConvTranspose3d):
        return F.conv_transpose3d(x, conv.weight.to(x.dtype), None, conv.stride)
    return F.conv3d(x, conv.weight.to(x.dtype), None, conv.stride, conv.padding)


class _Seq3d(nn.Sequential):
    """Sequential whose convolutions run in the activation dtype (bf16) while parameters stay fp32 masters; a BatchNorm3d
    followed by a ReLU is one fused row-kernel pass."""

    def forward(self, x):
        mods = list(self)
        i = 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, (nn.Conv3d, nn.ConvTranspose3d)):
                x = _conv3d(m, x)
            elif isinstance(m, nn.BatchNorm3d) and i + 1 < len(mods) and isinstance(mods[i + 1], nn.ReLU):
                x = _bn3d(m, x, SP.ACT_RELU)
                i += 1
            else:
                x = m(x)
            i += 1
        return x


@MODELS.register_module()
class IndoorImVoxelNeck(nn.Module):

    def __init__(self, in_channels, out_channels, n_blocks):
        super().__init__()
        self.n_scales = len(n_blocks)
        n_channels = in_channels
        for i in range(len(n_blocks)):
            stride = 1 if i == 0 else 2
            setattr(self, f'down_layer_{i}', self._make_layer(stride, n_channels, n_blocks[i]))
            n_channels = n_channels * stride
            if i > 0:
                setattr(self, f'up_block_{i}', self._make_up_block(n_channels, n_channels // 2))
            setattr(self, f'out_block_{i}', self._make_block(n_channels, out_channels))

    def forward(self, x):
        down_outs = []
        for i in range(self.n_scales):
            x = getattr(self, f'down_layer_{i}')(x)
            down_outs.append(x)
        outs = []
        for i in range(self.n_scales - 1, -1, -1):
            if i < self.n_scales - 1:
                x = getattr(self, f'up_block_{i + 1}')(x)
                x = down_outs[i] + x
            outs.append(getattr(self, f'out_block_{i}')(x))
        return outs[::-1]

    @staticmethod
    def _make_layer(stride, n_channels, n_blocks):
        blocks = []
        for i in range(n_blocks):
            if i == 0 and stride != 1:
                blocks.append(ResModule(n_channels, n_channels * 2, stride))
                n_channels = n_channels * 2
            else:
                blocks.append(ResModule(n_channels, n_channels))
        return nn.Sequential(*blocks)

    @staticmethod
    def _make_block(in_channels, out_channels):
        return _Seq3d(nn.Conv3d(in_channels, out_channels, 3, 1, 1, bias=False), nn.BatchNorm3d(out_channels),
                      nn.ReLU(inplace=True))

    @staticmethod
    def _make_up_block(in_channels, out_channels):
        return _Seq3d(nn.ConvTranspose3d(in_channels, out_channels, 2, 2, bias=False), nn.BatchNorm3d(out_channels),
                      nn.ReLU(inplace=True), nn.Conv3d(out_channels, out_channels, 3, 1, 1, bias=False),
                      nn.BatchNorm3d(out_channels), nn.ReLU(inplace=True))


# ---- SurroundOcc losses (occ_loss.py) -------------------------------------------------------------------------------
def occ_multiscale_supervision(gt_occ, ratio, gt_shape, gt_occupancy_masks=None):
    """occ_loss.py:7-29. At ratio > 1 several fine voxels land in one coarse cell; the reference's indexed assignment
    leaves the winner to the device's write order. Frozen here to the sequential (CPU) order: the last row wins."""
    B, X, Y, Z = gt_shape[0], gt_shape[2], gt_shape[3], gt_shape[4]
    gt = torch.zeros([B, X * Y * Z], dtype=torch.long, device=gt_occ[0].device)
    for i in range(B):
        occ = gt_occ[i].long()
        c = torch.div(occ[:, :3], ratio, rounding_mode='trunc')
        lin = (c[:, 0] * Y + c[:, 1]) * Z + c[:, 2]
        last = torch.full((X * Y * Z, ), -1, dtype=torch.long, device=occ.device)
        last.scatter_reduce_(0, lin, torch.arange(occ.shape[0], device=occ.device), reduce='amax')
        gt[i] = torch.where(last >= 0, occ[last.clamp(min=0), 3], gt[i])
    gt = gt.view(B, X, Y, Z)
    if gt_occupancy_masks is not None:
        for i in range(B):
            gt[i][~gt_occupancy_masks[i]] = 255
    return gt


def _nlog(x):
    """F.binary_cross_entropy(x, ones): -max(log x, -100) with the library's bounded gradient at x == 0 (a scale whose
    target set is empty yields exactly 0 there). The clamp guards the op's [0, 1] domain check against a 1-ulp overshoot."""
    x = x.clamp(0., 1.)
    return F.binary_cross_entropy(x, torch.ones_like(x), reduction='none')


def geo_scal_loss(pred, ssc_target, semantic=True):
    if semantic:
        empty_probs = F.softmax(pred, dim=1)[:, 0]
    else:
        empty_probs = 1 - torch.sigmoid(pred)
    nonempty_probs = 1 - empty_probs
    mask = (ssc_target != 255).float()
    nonempty_target = (ssc_target != 0).float() * mask
    eps = 1e-6
    intersection = (nonempty_target * nonempty_probs).sum()
    precision = intersection / ((nonempty_probs * mask).sum() + eps)
    recall = intersection / (nonempty_target.sum() + eps)
    empty_target = (1 - (ssc_target != 0).float()) * mask
    spec = (empty_target * empty_probs).sum() / (empty_target.sum() + eps)
    return _nlog(precision) + _nlog(recall) + _nlog(spec)


def sem_scal_loss(pred, ssc_target):
    """occ_loss.py:83-141 with the 81-iteration class loop (3 host syncs per class) folded into per-class reductions."""
    p = F.softmax(pred, dim=1)                                       # (B,C,X,Y,Z)
    C = p.shape[1]
    mask = (ssc_target != 255)
    pm = p.permute(1, 0, 2, 3, 4)[:, mask]                           # (C, M)
    tgt = ssc_target[mask]                                           # (M,)
    onehot = (tgt[None] == torch.arange(C, device=pred.device)[:, None]).to(pm.dtype)   # (C, M)
    n_tgt = onehot.sum(1)
    sum_p = pm.sum(1)
    nominator = (pm * onehot).sum(1)
    n_not = (1 - onehot).sum(1)
    present = n_tgt > 0
    one = torch.ones_like(sum_p)
    # absent classes are skipped by the reference's loop: route them through log(1) so no inf/nan reaches autograd
    ratio = lambda a, b, on: torch.where(on & (b > 0), a / torch.where(b > 0, b, one), one)
    loss_c = _nlog(ratio(nominator, sum_p, present)) + _nlog(ratio(nominator, n_tgt, present)) + \
        _nlog(ratio(((1 - pm) * (1 - onehot)).sum(1), n_not, present))
    count = present.float().sum()
    total = torch.where(present, loss_c, torch.zeros_like(loss_c)).sum()
    return torch.where(count > 0, total / torch.clamp(count, min=1.), total * 0)


@MODELS.register_module()
class ImVoxelOccHead(nn.Module):

    def __init__(self, *args, num_classes=21, volume_h=40, volume_w=40, volume_z=16, in_channels=128, use_semantic=True,
                 train_cfg=None, test_cfg=None, **kwargs):
        super().__init__()
        self.num_classes, self.in_channels, self.use_semantic = num_classes, in_channels, use_semantic
        self.occ = nn.ModuleList([nn.Conv3d(c, num_classes if use_semantic else 1, 1, bias=False) for c in in_channels])

    def forward(self, mlvl_feats, input_metas=None):
        return [_conv3d(self.occ[i], mlvl_feats[i]) for i in range(len(mlvl_feats))]

    def predict(self, x, batch_data_samples):
        pred = self.forward(x)[0].float()
        if self.use_semantic:
            return torch.max(torch.softmax(pred, dim=1), dim=1)[1]
        return torch.sigmoid(pred[:, 0])

    def loss(self, x, batch_data_samples):
        occ_preds = self.forward(x)
        gt_occupancy = [ds.gt_occupancy for ds in batch_data_samples]
        masks = [ds.gt_occupancy_masks for ds in batch_data_samples] if 'gt_occupancy_masks' in batch_data_samples[0] \
            else None
        loss_dict = {}
        for i, pred in enumerate(occ_preds):
            pred = pred.float()
            ratio = 2 ** i
            pooled = None
            if masks is not None:
                pooled = [F.max_pool3d(m.float()[None], ratio, stride=ratio)[0].bool() for m in masks]
            gt = occ_multiscale_supervision(gt_occupancy, ratio, pred.shape, pooled)
            if self.use_semantic:
                li = F.cross_entropy(pred, gt, ignore_index=255) + sem_scal_loss(pred, gt) + geo_scal_loss(pred, gt)
            else:
                li = F.binary_cross_entropy_with_logits(pred[:, 0], gt.float()) + geo_scal_loss(pred[:, 0], gt, False)
            loss_dict[f'loss_occ_{i}'] = li * (0.5 ** i)
        return loss_dict


@MODELS.register_module()
class DenseFusionOccPredictor(nn.Module):

    def __init__(self, backbone, backbone_3d, neck, neck_3d, bbox_head, prior_generator, n_voxels, coord_type,
                 use_valid_mask=True, use_xyz_feat=False, point_cloud_range=None, train_cfg=None, test_cfg=None,
                 data_preprocessor=None, init_cfg=None, compute_dtype=torch.float32):
        super().__init__()
        self.compute_dtype = compute_dtype
        if isinstance(data_preprocessor, dict):
            data_preprocessor = dict(data_preprocessor, compute_dtype=compute_dtype)
            data_preprocessor.setdefault('type', 'Det3DDataPreprocessor')
        self.data_preprocessor = MODELS.build(data_preprocessor) if data_preprocessor is not None else None
        self.backbone = MODELS.build(backbone)
        self.backbone_3d = MODELS.build(backbone_3d)
        self.neck = MODELS.build(neck) if neck is not None else None
        self.neck_3d = MODELS.build(neck_3d) if neck_3d is not None else None
        bbox_head = dict(bbox_head, train_cfg=train_cfg, test_cfg=test_cfg)
        self.bbox_head = MODELS.build(bbox_head)
        self.n_voxels = list(n_voxels)
        self.point_cloud_range = point_cloud_range
        pr = prior_generator['ranges'][0]
        self.voxel_stride = 2 ** 6 if backbone_3d['type'] == 'MinkResNet' else 1
        self.voxel_size = [(pr[3] - pr[0]) / self.n_voxels[0] / self.voxel_stride,
                           (pr[4] - pr[1]) / self.n_voxels[1] / self.voxel_stride,
                           (pr[5] - pr[2]) / self.n_voxels[2] / self.voxel_stride]
        self.prior_generator = TASK_UTILS.build(prior_generator)
        self.coord_type, self.use_valid_mask, self.use_xyz_feat = coord_type, use_valid_mask, use_xyz_feat
        self.train_cfg, self.test_cfg = train_cfg, test_cfg

    def extract_feat(self, batch_inputs_dict, batch_data_samples):
        img = batch_inputs_dict['imgs']
        metas_list = [ds.metainfo for ds in batch_data_samples]
        B, V = img.shape[:2]
        dev = img.device
        img4 = img.reshape([-1] + list(img.shape)[2:]).to(self.compute_dtype)
        if not img4.is_contiguous(memory_format=torch.channels_last):
            img4 = img4.contiguous(memory_format=torch.channels_last)
        feat2d = self.neck(self.backbone(img4))[0]                     # (B*V, 256, H/4, W/4)

        prior = self.prior_generator.grid_anchors([self.n_voxels[::-1]], device=dev)[0][:, :3]
        if 'origin' in metas_list[0]['depth2img']:
            assert len(metas_list) == 1, 'only support batch_size=1 here'
            prior = prior + prior.new_tensor(np.asarray(metas_list[0]['depth2img']['origin'], dtype=np.float32))
        n_prior = prior.shape[0]
        pts = prior.repeat(B, 1).contiguous()
        pb = torch.arange(B, dtype=torch.int32, device=dev).repeat_interleave(n_prior)
        metas = pack_paint_metas(metas_list, dev)
        proj = pack_projections(metas_list, self.coord_type, dev)
        vol = paint_float_points(feat2d, pts, pb, metas, proj, tuple(img.shape[-2:]), V)        # (B*n_prior, C)
        img_volume = vol.view([B] + self.n_voxels[::-1] + [-1]).permute(0, 4, 3, 2, 1)          # (B, C, X, Y, Z)
        valid_preds = ~torch.all(img_volume == 0, dim=1, keepdim=True)

        # sparse branch: ((p - range_min) / voxel_size) floored, clamped into the grid (dense_fusion_occ.py:224-245)
        points = batch_inputs_dict['points']
        assert len(points) == 1, 'Only support batch size 1 for now!!'
        vs = prior.new_tensor(self.voxel_size)
        lo = prior.new_tensor(self.point_cloud_range[:3])
        coords, feats = [], []
        for b, p in enumerate(points):
            q = torch.floor((p[:, :3].float() - lo) / vs).to(torch.int32)
            hi = torch.tensor([n * self.voxel_stride - 1 for n in self.n_voxels], dtype=torch.int32, device=dev)
            q = torch.minimum(torch.clamp(q, min=0), hi)
            coords.append(torch.cat([torch.full((q.shape[0], 1), b, dtype=torch.int32, device=dev), q], 1))
            feats.append(p.float() if self.use_xyz_feat else p[:, 3:].float())
        x = SP.SparseTensor(coordinates=torch.cat(coords), features=torch.cat(feats).to(self.compute_dtype),
                            batch_size=len(points))
        last = self.backbone_3d(x)[-1]
        point_volume, _, _ = last.dense((1, last.F.shape[-1], *self.n_voxels), min_coordinate=[0, 0, 0])
        fused = torch.cat([img_volume.to(self.compute_dtype), point_volume], dim=1)
        return self.neck_3d(fused.contiguous(memory_format=torch.channels_last_3d)), valid_preds.float()

    def sparse_volume(self, points, prior):
        """MinkResNet over the clamped voxel grid -> dense (B, C, X, Y, Z) volume of its coarsest level."""
        dev = prior.device
        vs = prior.new_tensor(self.voxel_size)
        lo = prior.new_tensor(self.point_cloud_range[:3])
        coords, feats = [], []
        for b, p in enumerate(points):
            q = torch.floor((p[:, :3].float() - lo) / vs).to(torch.int32)
            hi = torch.tensor([n * self.voxel_stride - 1 for n in self.n_voxels], dtype=torch.int32, device=dev)
            q = torch.minimum(torch.clamp(q, min=0), hi)
            coords.append(torch.cat([torch.full((q.shape[0], 1), b, dtype=torch.int32, device=dev), q], 1))
            feats.append(p.float() if self.use_xyz_feat else p[:, 3:].float())
        x = SP.SparseTensor(coordinates=torch.cat(coords), features=torch.cat(feats).to(self.compute_dtype),
                            batch_size=len(points))
        last = self.backbone_3d(x)[-1]
        return last.dense((len(points), last.F.shape[-1], *self.n_voxels), min_coordinate=[0, 0, 0])[0]

    def loss(self, batch_inputs_dict, batch_data_samples, **kwargs):
        x, valid = self.extract_feat(batch_inputs_dict, batch_data_samples)
        return self.bbox_head.loss(x, batch_data_samples)

    def predict(self, batch_inputs_dict, batch_data_samples, **kwargs):
        x, valid = self.extract_feat(batch_inputs_dict, batch_data_samples)
        pred = self.bbox_head.predict(x, batch_data_samples)
        for i, ds in enumerate(batch_data_samples):
            ds.pred_occupancy = pred[i]
        return batch_data_samples

    def forward(self, inputs, data_samples=None, mode='tensor', **kwargs):
        if self.compute_dtype == torch.float32:
            # fp32 = the parity arithmetic: library contractions stay out of TF32 in forward AND backward
            from .precision import fence_losses, fp32_exact
            with fp32_exact():
                return fence_losses(self._forward(inputs, data_samples, mode, **kwargs))
        return self._forward(inputs, data_samples, mode, **kwargs)

    def _forward(self, inputs, data_samples, mode, **kwargs):
        if mode == 'loss':
            return self.loss(inputs, data_samples, **kwargs)
        if mode == 'predict':
            return self.predict(inputs, data_samples, **kwargs)
        raise RuntimeError(f'Invalid mode "{mode}". Only supports loss and predict mode')

    def train_step(self, data, optim_wrapper):
        data = self.data_preprocessor(data, True)
        loss, log_vars = parse_losses(self(**data, mode='loss'))
        optim_wrapper.update_params(loss)
        return detach_log_vars(log_vars)

    @torch.no_grad()
    def val_step(self, data):
        data = self.data_preprocessor(data, False)
        return self(**data, mode='predict')

    test_step = val_step


@MODELS.register_module()
class EmbodiedOccPredictor(DenseFusionOccPredictor):
    """Continuous (1..N frames) occupancy predictor (embodiedscan/models/detectors/embodied_occ.py:118-247): the batch is
    ONE scan seen through its N growing frame prefixes; prefix ``idx`` paints the prior grid from views 0..idx only and
    voxelises the points of frames 0..idx. Same kernels as the multi-view predictor; painting runs once per prefix on a
    contiguous view-prefix slice of the FPN map."""

    def extract_feat(self, batch_inputs_dict, batch_data_samples):
        img = batch_inputs_dict['imgs']
        metas_list = [ds.metainfo for ds in batch_data_samples]
        assert img.dim() == 5 and img.shape[0] == 1, 'one scan: (1, n_views, C, H, W)'
        V, dev = img.shape[1], img.device
        n_prefix = len(metas_list)
        assert n_prefix <= V
        img4 = img.reshape([-1] + list(img.shape)[2:]).to(self.compute_dtype)
        if not img4.is_contiguous(memory_format=torch.channels_last):
            img4 = img4.contiguous(memory_format=torch.channels_last)
        feat2d = self.neck(self.backbone(img4))[0]                      # (V, C, H/4, W/4)
        if not feat2d.is_contiguous(memory_format=torch.channels_last):
            feat2d = feat2d.contiguous(memory_format=torch.channels_last)
        prior = self.prior_generator.grid_anchors([self.n_voxels[::-1]], device=dev)[0][:, :3]
        if 'origin' in metas_list[0]['depth2img']:
            prior = prior + prior.new_tensor(np.asarray(metas_list[0]['depth2img']['origin'], dtype=np.float32))
        prior = prior.contiguous()
        vols = []
        for idx, meta in enumerate(metas_list):
            proj = pack_projections([meta], self.coord_type, dev)[:, :idx + 1].contiguous()
            vol = paint_float_points(feat2d[:idx + 1], prior, None, pack_paint_metas([meta], dev), proj,
                                     tuple(img.shape[-2:]), idx + 1)
            vols.append(vol.view(self.n_voxels[::-1] + [-1]).permute(3, 2, 1, 0))
        img_volume = torch.stack(vols)                                   # (N, C, X, Y, Z)
        valid_preds = ~torch.all(img_volume == 0, dim=1, keepdim=True)
        points = batch_inputs_dict['points']
        assert all(isinstance(p, (list, tuple)) and len(p) == 1 for p in points), 'only support batch_size=1 for now!'
        point_volume = self.sparse_volume([p[0] for p in points], prior)
        fused = torch.cat([img_volume.to(self.compute_dtype), point_volume], dim=1)
        return self.neck_3d(fused.contiguous(memory_format=torch.channels_last_3d)), valid_preds.float()
