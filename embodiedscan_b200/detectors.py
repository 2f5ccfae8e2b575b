"""``SparseFeatureFusionSingleStage3DDetector`` and ``Det3DDataPreprocessor`` under the reference's registry names
(embodiedscan/models/detectors/sparse_featfusion_single_stage.py:28-426,
embodiedscan/models/data_preprocessors/data_preprocessor.py:23-339) — same constructor arguments and
``forward(inputs, data_samples, mode)`` contract, so mmengine's ``train_step / val_step / test_step`` (mirrored
here for the mmengine-less image) drive it unchanged. ``MultiModal3DModel`` holds that contract and the input front half
for the detector, occupancy and grounding models alike.
"""
from typing import Dict, List, Optional, Union

import math
import numpy as np
import torch
import torch.nn as nn

from . import _ffi
from . import sparse as SP
from ._ffi import call, ptr, stream
from .fusion import pack_paint_metas, pack_projections, paint_points
from .precision import fence_losses, fp32_exact
from .registry import MODELS
from .structures import Det3DDataSample, InstanceData


@MODELS.register_module()
class Det3DDataPreprocessor(nn.Module):
    """Image path of the reference preprocessor as one kernel: BGR->RGB, (x-mean)/std, right/bottom pad to a multiple
    of ``pad_size_divisor``, multi-view stack; points pass through (``voxel=False`` is the only configured mode)."""

    def __init__(self, mean=None, std=None, bgr_to_rgb=False, rgb_to_bgr=False, pad_size_divisor=1, pad_value=0,
                 voxel=False, non_blocking=False, compute_dtype=torch.float32, batchwise_inputs=False, **kwargs):
        super().__init__()
        assert not voxel, 'mmcv voxelisation wrappers are not on any configured path (SURVEY N14)'
        assert not (bgr_to_rgb and rgb_to_bgr)
        self.channel_conversion = bgr_to_rgb or rgb_to_bgr
        self.mean = [float(m) for m in (mean or [0., 0., 0.])]
        self.std = [float(s) for s in (std or [1., 1., 1.])]
        self.pad_size_divisor, self.pad_value = pad_size_divisor, pad_value
        self.compute_dtype = compute_dtype
        self.batchwise_inputs = batchwise_inputs
        self.register_buffer('_dev', torch.zeros(1), persistent=False)

    @property
    def device(self):
        return self._dev.device

    @staticmethod
    def split_batchwise(data_samples):
        """`batchwise_inputs=True` (data_preprocessor.py:172-205): ONE scan whose annotations are lists over its 1..N
        frame prefixes becomes N data samples sharing the scan's metainfo (continuous 3D perception)."""
        first = data_samples[0]
        gt = first.gt_instances_3d
        labels = gt.labels_3d
        assert isinstance(labels, list), 'continuous inputs carry per-prefix lists (ConstructMultiSweeps)'
        boxes = gt.bboxes_3d if 'bboxes_3d' in gt else None
        masks = list(first.gt_occupancy_masks) if 'gt_occupancy_masks' in first else None
        ann = first.eval_ann_info if 'eval_ann_info' in first and first.eval_ann_info is not None else None
        out = []
        for idx in range(len(labels)):
            ds = Det3DDataSample(metainfo=dict(first.metainfo))
            for k in first.keys():
                if k not in ('gt_instances_3d', 'gt_occupancy_masks', 'eval_ann_info'):
                    setattr(ds, k, getattr(first, k))
            inst = InstanceData()
            if boxes is not None:
                inst.bboxes_3d = boxes[idx]
            inst.labels_3d = labels[idx]
            ds.gt_instances_3d = inst
            if masks is not None:
                ds.gt_occupancy_masks = masks[idx]
            if 'eval_ann_info' in first:
                ds.eval_ann_info = None if ann is None else dict(gt_bboxes_3d=ann['gt_bboxes_3d'][idx],
                                                                 gt_labels_3d=ann['gt_labels_3d'][idx])
            out.append(ds)
        return out

    def forward(self, data: dict, training: bool = False) -> dict:
        inputs, data_samples = data['inputs'], data.get('data_samples')
        if self.batchwise_inputs and data_samples is not None:
            data_samples = self.split_batchwise(data_samples)
        dev = self.device
        out = {}
        if 'points' in inputs:      # continuous inputs arrive pseudo-collated: points[idx] = [tensor] (batch size 1)
            out['points'] = [[q.to(dev, non_blocking=True) for q in p] if isinstance(p, (list, tuple))
                             else p.to(dev, non_blocking=True) for p in inputs['points']]
        if 'img' in inputs:
            imgs = inputs['img']
            if isinstance(imgs, torch.Tensor):                      # default_collate: one (B,[V,]3,H,W) tensor, one copy
                imgs = imgs.to(dev, non_blocking=True)
                imgs = list(imgs[:, None] if imgs.dim() == 4 else imgs)
            imgs = [i[None] if i.dim() == 3 else i for i in imgs]   # (V,3,H,W) per scan
            assert all(i.dtype == torch.uint8 for i in imgs), 'images arrive as uint8 CHW (Pack3DDetInputs)'
            assert len({i.shape[0] for i in imgs}) == 1, 'scans of a batch carry the same number of views'
            assert self.pad_value == 0, 'the pad region is written as 0 in normalised space (configs use pad_value=0)'
            B, V = len(imgs), imgs[0].shape[0]
            d = self.pad_size_divisor
            # multiview_img_stack_batch (utils.py:9-63): every scan is right/bottom padded to the batch maximum,
            # rounded up to the divisor; `pad_shape` stays per scan (data_preprocessor.py:_get_pad_shape)
            Hp = int(math.ceil(max(i.shape[-2] for i in imgs) / d) * d)
            Wp = int(math.ceil(max(i.shape[-1] for i in imgs) / d) * d)
            buf = torch.empty((B * V, Hp, Wp, 3), dtype=self.compute_dtype, device=dev)
            import ctypes
            mean = (ctypes.c_float * 3)(*self.mean)
            std = (ctypes.c_float * 3)(*self.std)
            uniform = len({tuple(i.shape) for i in imgs}) == 1
            groups = [(torch.stack([i.to(dev, non_blocking=True) for i in imgs]), buf)] if uniform else \
                [(i.to(dev, non_blocking=True), buf[b * V:(b + 1) * V]) for b, i in enumerate(imgs)]
            for src, dst in groups:                                 # one launch for the usual uniform batch
                H, W = src.shape[-2:]
                call('esb_img_normalize', ptr(src.contiguous()), dst.shape[0], H, W, Hp, Wp,
                     ctypes.cast(mean, ctypes.c_void_p), ctypes.cast(std, ctypes.c_void_p),
                     1 if self.channel_conversion else 0, 1, ptr(dst), _ffi.dtype_code(self.compute_dtype), stream())
            out['imgs'] = buf.view(B, V, Hp, Wp, 3).permute(0, 1, 4, 2, 3)   # (B,V,3,Hp,Wp), channels-last memory
            if data_samples is not None:
                per_sample = imgs if len(imgs) == len(data_samples) else [imgs[0]] * len(data_samples)
                for ds, i in zip(data_samples, per_sample):       # batchwise: every prefix shares the scan's images
                    ds.set_metainfo({'batch_input_shape': (Hp, Wp),
                                     'pad_shape': (int(math.ceil(i.shape[-2] / d) * d),
                                                   int(math.ceil(i.shape[-1] / d) * d))})
        elif 'imgs' in inputs:
            out['imgs'] = inputs['imgs'].to(dev)
        if data_samples is not None:
            for ds in data_samples:
                if 'gt_instances_3d' in ds:
                    ds.gt_instances_3d.to(dev)
                for k in ('gt_occupancy', 'gt_occupancy_masks'):
                    if k in ds:
                        setattr(ds, k, getattr(ds, k).to(dev))
        return {'inputs': out, 'data_samples': data_samples}


def preprocessor_cfg(data_preprocessor: Optional[dict], compute_dtype) -> Optional[dict]:
    """A model's preprocessor config: a copy that writes images in the model's compute dtype, ``Det3DDataPreprocessor``
    unless the config names another type."""
    if isinstance(data_preprocessor, dict):
        data_preprocessor = dict(data_preprocessor, compute_dtype=compute_dtype)
        data_preprocessor.setdefault('type', 'Det3DDataPreprocessor')
    return data_preprocessor


class MultiModal3DModel(nn.Module):
    """What the detector, occupancy and grounding models share: mmengine's ``BaseModel`` contract (``forward(mode=...)``,
    ``train_step / val_step / test_step``), the multi-view image batch, and the sparse front half of the detector and the
    grounder (voxelise -> MinkResNet -> paint every level from the scan's views). Subclasses set ``compute_dtype`` and
    ``data_preprocessor`` and implement ``loss`` / ``predict``."""

    def forward(self, inputs: Union[dict, List[dict]], data_samples=None, mode: str = 'tensor', **kwargs):
        if self.compute_dtype == torch.float32:
            # fp32 = the parity arithmetic: library contractions stay out of TF32 in forward AND backward
            with fp32_exact():
                return fence_losses(self._forward(inputs, data_samples, mode, **kwargs))
        return self._forward(inputs, data_samples, mode, **kwargs)

    def _forward(self, inputs, data_samples, mode, **kwargs):
        if mode == 'loss':
            return self.loss(inputs, data_samples, **kwargs)
        if mode == 'predict':
            return self.predict(inputs, data_samples, **kwargs)
        raise RuntimeError(f'Invalid mode "{mode}". Only supports loss and predict mode')

    # ---- mmengine BaseModel contract (†upstream) -------------------------------------------------------------
    def train_step(self, data, optim_wrapper):
        with optim_wrapper.optim_context(self):
            data = self.data_preprocessor(data, True)
            losses = self(**data, mode='loss')
        loss, log_vars = parse_losses(losses)
        optim_wrapper.update_params(loss)
        return detach_log_vars(log_vars)

    @torch.no_grad()
    def val_step(self, data):
        data = self.data_preprocessor(data, False)
        return self(**data, mode='predict')

    test_step = val_step

    # ---- shared feature extraction (sparse_featfusion_single_stage.py:86-221) --------------------------------
    def view_batch(self, img: torch.Tensor) -> torch.Tensor:
        """(B, V, 3, H, W) images -> the (B*V, 3, H, W) batch of the 2D backbone, channels-last, in the compute dtype."""
        img4 = img.reshape([-1] + list(img.shape)[2:]).to(self.compute_dtype)
        if not img4.is_contiguous(memory_format=torch.channels_last):
            img4 = img4.contiguous(memory_format=torch.channels_last)
        return img4

    def voxelize(self, points: List[torch.Tensor]):
        dev = points[0].device
        n_tot = sum(p.shape[0] for p in points)
        coords = torch.empty((n_tot, 4), dtype=torch.int32, device=dev)
        inv = float(np.float32(1.) / np.float32(self.voxel_size))
        off = 0
        feats = []
        for b, p in enumerate(points):
            p = p.float().contiguous()
            call('esb_voxelize_points', ptr(p), p.shape[0], p.shape[1], b, inv, ptr(coords[off:]), stream())
            off += p.shape[0]
            feats.append(p if self.use_xyz_feat else p[:, 3:])
        return coords, torch.cat(feats)

    def sparse_levels(self, points: List[torch.Tensor]) -> List[SP.SparseTensor]:
        """Voxelise the point clouds (one sample each) and run the sparse 3D backbone: its levels, fine -> coarse."""
        coordinates, features = self.voxelize(points)
        x = SP.SparseTensor(coordinates=coordinates, features=features.to(self.compute_dtype), batch_size=len(points))
        return self.backbone_3d(x)

    def paint_levels(self, x: List[SP.SparseTensor], img_features, img: torch.Tensor, batch_img_metas) -> None:
        """Append to every level's features the image features its voxels project onto, over all V views of each scan."""
        dev = img.device
        metas = pack_paint_metas(batch_img_metas, dev)
        proj = pack_projections(batch_img_metas, self.coord_type, dev)
        pad_hw = tuple(img.shape[-2:])
        for level_idx in range(len(x)):
            painted = paint_points(img_features[level_idx], x[level_idx].C, metas, proj, self.voxel_size, pad_hw,
                                   img.shape[1])
            x[level_idx] = x[level_idx].replace_feature(torch.cat([x[level_idx].F, painted.to(x[level_idx].F.dtype)], 1))


@MODELS.register_module()
class SparseFeatureFusionSingleStage3DDetector(MultiModal3DModel):

    def __init__(self, backbone, backbone_3d, bbox_head, neck=None, neck_3d=None, coord_type: str = 'CAMERA',
                 train_cfg: Optional[dict] = None, test_cfg: Optional[dict] = None,
                 data_preprocessor: Optional[dict] = None, use_xyz_feat: bool = False, init_cfg: Optional[dict] = None,
                 compute_dtype=torch.float32):
        super().__init__()
        assert neck is None and neck_3d is None, 'no configured hot-path model uses neck / neck_3d here'
        self.compute_dtype = compute_dtype
        data_preprocessor = preprocessor_cfg(data_preprocessor, compute_dtype)
        self.data_preprocessor = MODELS.build(data_preprocessor) if data_preprocessor is not None else None
        self.backbone = MODELS.build(backbone)
        self.backbone_3d = MODELS.build(backbone_3d)
        bbox_head = dict(bbox_head)
        bbox_head.update(train_cfg=train_cfg)
        bbox_head.update(test_cfg=test_cfg)
        self.bbox_head = MODELS.build(bbox_head)
        self.coord_type = coord_type
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.voxel_size = bbox_head['voxel_size']
        self.use_xyz_feat = use_xyz_feat
        self.overlap_2d_3d = True
        self._side_stream = None

    def extract_feat(self, batch_inputs_dict: Dict[str, torch.Tensor], batch_data_samples) -> List[SP.SparseTensor]:
        img = batch_inputs_dict['imgs']
        assert img.dim() == 5, 'multi-view input (B, n_views, C, H, W)'
        img4 = self.view_batch(img)

        # Two streams: the dense per-view 2D backbone runs on a side stream while the main stream builds the coordinate
        # plan (whose row-count read-backs synchronise only the main stream) and runs the sparse 3D backbone; they
        # join before point painting. Autograd replays the same stream assignment in backward.
        side = None
        if img4.is_cuda and self.overlap_2d_3d:
            main = torch.cuda.current_stream()
            if self._side_stream is None or self._side_stream.device != img4.device:
                self._side_stream = torch.cuda.Stream(device=img4.device)
                from .engine import register_grad_stream
                register_grad_stream(self._side_stream)   # its backward writes 2D-backbone gradients into the arena
            side = self._side_stream
            side.wait_stream(main)
            with torch.cuda.stream(side):
                img_features = self.backbone(img4)
        else:
            img_features = self.backbone(img4)

        x = self.sparse_levels(batch_inputs_dict['points'])
        if side is not None:
            main.wait_stream(side)
            for f in img_features:
                f.record_stream(main)
        self.paint_levels(x, img_features, img, [ds.metainfo for ds in batch_data_samples])
        return x

    def loss(self, batch_inputs_dict, batch_data_samples, **kwargs):
        x = self.extract_feat(batch_inputs_dict, batch_data_samples)
        return self.bbox_head.loss(x, batch_data_samples, **kwargs)

    def predict(self, batch_inputs_dict, batch_data_samples, **kwargs):
        x = self.extract_feat(batch_inputs_dict, batch_data_samples)
        results_list = self.bbox_head.predict(x, batch_data_samples, **kwargs)
        return self.add_pred_to_datasample(batch_data_samples, results_list)

    @staticmethod
    def add_pred_to_datasample(data_samples, data_instances_3d=None, data_instances_2d=None):
        assert data_instances_3d is not None or data_instances_2d is not None
        if data_instances_2d is None:
            data_instances_2d = [InstanceData() for _ in range(len(data_instances_3d))]
        if data_instances_3d is None:
            data_instances_3d = [InstanceData() for _ in range(len(data_instances_2d))]
        for i, ds in enumerate(data_samples):
            ds.pred_instances_3d = data_instances_3d[i]
            ds.pred_instances = data_instances_2d[i]
        return data_samples


@MODELS.register_module()
class Embodied3DDetector(SparseFeatureFusionSingleStage3DDetector):
    """Continuous (1..N frames) detector (embodiedscan/models/detectors/embodied_det3d.py:90-207): the batch is ONE scan
    seen through its N growing frame prefixes. Sample ``idx`` holds the points of frames 0..idx and is painted from the
    image features of views 0..idx only; everything else is the multi-view detector. Same kernels: the sparse backbone
    and the head see an N-sample batch, painting runs once per (prefix, level) on a view-prefix slice of the feature map
    (the slice is contiguous, so no copy and no new kernel)."""

    def __init__(self, *args, neck_lidar=None, **kwargs):
        assert neck_lidar is None, 'no configured continuous model uses neck_lidar'
        super().__init__(*args, **kwargs)

    def extract_feat(self, batch_inputs_dict, batch_data_samples):
        points = batch_inputs_dict['points']
        assert all(isinstance(p, (list, tuple)) and len(p) == 1 for p in points), 'only support batch_size=1 for now!'
        points = [p[0] for p in points]
        img = batch_inputs_dict['imgs']
        assert img.dim() == 5 and img.shape[0] == 1, 'one scan: (1, n_views, C, H, W)'
        batch_img_metas = [ds.metainfo for ds in batch_data_samples]
        assert len(points) == len(batch_img_metas) <= img.shape[1]
        img_features = self.backbone(self.view_batch(img))               # per level (V, C, Hf, Wf)
        x = self.sparse_levels(points)
        dev = img.device
        pad_hw = tuple(img.shape[-2:])
        metas = [pack_paint_metas([m], dev) for m in batch_img_metas]
        projs = [pack_projections([m], self.coord_type, dev) for m in batch_img_metas]       # (1, V, 4, 4) each
        for level_idx in range(len(x)):
            lv = x[level_idx]
            feat = img_features[level_idx]
            painted = lv.F.new_zeros((lv.F.shape[0], feat.shape[1]))
            for idx, rows in enumerate(lv.decomposition_permutations):
                if rows.numel() == 0:
                    continue
                c = lv.C[rows].clone()
                c[:, 0] = 0                                              # one "scan" per launch: the prefix itself
                out = paint_points(feat[:idx + 1], c.contiguous(), metas[idx], projs[idx][:, :idx + 1].contiguous(),
                                   self.voxel_size, pad_hw, idx + 1)
                painted = painted.index_copy(0, rows, out.to(painted.dtype))
            x[level_idx] = lv.replace_feature(torch.cat([lv.F, painted], 1))
        return x


def detach_log_vars(log_vars: dict) -> dict:
    """What `train_step` hands back: the logged values WITHOUT their autograd history. A caller that keeps the dict until the
    next step (every logging loop does) would otherwise keep the whole graph of the finished step alive through the loss
    tensors' grad_fn — including the kernel maps and coordinate tables the sparse-conv nodes hold (hundreds of MB) — so the
    next step could not reuse that memory and the allocator had to map new segments (a 100-300 ms stall, measured)."""
    return {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in log_vars.items()}


def parse_losses(losses: dict):
    """mmengine BaseModel.parse_losses: total = sum of every entry whose key contains 'loss'."""
    log_vars = {k: (v.mean() if isinstance(v, torch.Tensor) else sum(x.mean() for x in v)) for k, v in losses.items()}
    loss = sum(v for k, v in log_vars.items() if 'loss' in k)
    log_vars['loss'] = loss
    return loss, log_vars
