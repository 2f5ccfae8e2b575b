"""Grounding variant of the hot path (SURVEY §8 row a15, BASELINE.json config C4), registered under the reference's
names: ``SparseFeatureFusion3DGrounder`` (embodiedscan/models/detectors/sparse_featfusion_grounder.py:30-766),
``MinkNeck`` (models/necks/mink_neck.py:17-244), ``SparseFeatureFusionTransformerDecoder[Layer]`` and
``PositionEmbeddingLearned`` (models/layers/ground_transformer/decoder.py:20-297), ``GroundingHead`` /
``ContrastiveEmbed`` (models/dense_heads/grounding_head.py:22-824), ``HungarianAssigner3D``
(models/task_modules/assigners/hungarian_assigner.py:17-138) and the match costs (models/losses/match_cost.py).

What is H100-native here:
* the front half (voxel hashing, MinkResNet, painting, the pruned sparse FPN) runs in libesb200.so like the detector;
* target assignment is ONE device launch for all decoder layers x samples (``esb_hungarian_batch``) fed by batched
  cost tensors and the exact 9-DoF IoU kernel (``esb_box3d_overlap``) — the reference does 7 x batch D2H copies,
  scipy calls and H2D copies per iteration; the loss needs no host synchronisation (matched pairs are addressed
  through the inverse map, their count is known from the ground truth);
* the text encoder runs without autograd when it is frozen (the reference trains it with lr_mult = 0).
The attention / FFN contractions are library calls (``nn.MultiheadAttention`` -> SDPA / cuBLAS), as in the reference.
"""
import math
import re
import warnings
import zlib
from typing import Dict, List, Optional

import numpy as np
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import sparse as SP
from ._ffi import call, ptr, stream
from .dense_heads import FCAF3DHeadRotMat
from .detectors import SparseFeatureFusionSingleStage3DDetector, detach_log_vars, parse_losses
from .fusion import pack_paint_metas, pack_projections, paint_points
from .geometry import (bbox_to_corners, box3d_overlap, box_corners_container, chamfer_l1_src,
                       matrix_to_euler_angles_zxy, ortho_6d_2_mat, rotation_3d_in_euler)
from .registry import MODELS, TASK_UTILS
from .structures import EulerDepthInstance3DBoxes, InstanceData


# ======================================================================================================= text side
class _Encoding(dict):
    """The slice of ``transformers.BatchEncoding`` the grounder uses: mapping protocol for ``model(**enc)``,
    attribute access, ``.to(device)`` and ``char_to_token``."""

    def __init__(self, data, spans):
        super().__init__(data)
        self._spans = spans

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def to(self, device):
        return _Encoding({k: v.to(device) for k, v in self.items()}, self._spans)

    def char_to_token(self, batch_idx, char_idx):
        for t, (a, b) in enumerate(self._spans[batch_idx]):
            if a <= char_idx < b:
                return t + 1              # +1: <s>
        return None


class SimpleTokenizer:
    """Stand-in for ``RobertaTokenizerFast`` when the 'roberta-base' vocabulary is not on disk (no network here):
    words and punctuation marks become one token each, ids are a stable hash into the RoBERTa id range, <s>=0,
    <pad>=1, </s>=2. Same call surface as the real tokenizer for the two calls the grounder makes."""

    def __init__(self, vocab_size=50265):
        self.vocab_size = vocab_size

    def batch_encode_plus(self, texts, padding='longest', return_tensors='pt'):
        ids, spans = [], []
        for t in texts:
            sp = [(m.start(), m.end()) for m in re.finditer(r'\w+|[^\w\s]', t)]
            spans.append(sp)
            ids.append([0] + [4 + zlib.crc32(t[a:b].lower().encode()) % (self.vocab_size - 4) for a, b in sp] + [2])
        L = max(len(i) for i in ids)
        input_ids = torch.ones((len(ids), L), dtype=torch.long)
        mask = torch.zeros((len(ids), L), dtype=torch.long)
        for r, i in enumerate(ids):
            input_ids[r, :len(i)] = torch.tensor(i)
            mask[r, :len(i)] = 1
        return _Encoding(dict(input_ids=input_ids, attention_mask=mask), spans)


def build_text_modules(t_type='roberta-base'):
    """RoBERTa-base tokenizer + encoder (sparse_featfusion_grounder.py:107-110), loaded like the reference does
    (`from_pretrained`, which downloads when the files are not cached). Only when ESB200_TEXT_RANDOM_INIT=1 is set — the
    synthetic benchmarks and the parity tests, which need shapes and not the checkpoint — a failure to resolve the files
    falls back to the same architecture with random weights and the stand-in tokenizer; otherwise the error propagates (a
    grounder silently training on a random frozen text encoder is worse than one that refuses to start)."""
    from transformers import RobertaConfig, RobertaModel
    try:
        from transformers import RobertaTokenizerFast
        offline = os.environ.get('HF_HUB_OFFLINE') == '1' or os.environ.get('ESB200_TEXT_RANDOM_INIT') == '1'
        tok = RobertaTokenizerFast.from_pretrained(t_type, local_files_only=offline)
        enc = RobertaModel.from_pretrained(t_type, local_files_only=offline)
    except Exception:
        if os.environ.get('ESB200_TEXT_RANDOM_INIT') != '1':
            raise
        warnings.warn(f"'{t_type}' is not available: ESB200_TEXT_RANDOM_INIT=1 -> random-init RobertaModel + SimpleTokenizer")
        cfg = RobertaConfig(vocab_size=50265, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                            bos_token_id=0, eos_token_id=2, layer_norm_eps=1e-5)
        tok, enc = SimpleTokenizer(cfg.vocab_size), RobertaModel(cfg)
    return tok, enc


# ======================================================================================================= decoder
class PositionEmbeddingLearned(nn.Module):

    def __init__(self, input_channel, embed_dims=256):
        super().__init__()
        self.position_embedding_head = nn.Sequential(nn.Conv1d(input_channel, embed_dims, kernel_size=1),
                                                     nn.BatchNorm1d(embed_dims), nn.ReLU(inplace=True),
                                                     nn.Conv1d(embed_dims, embed_dims, kernel_size=1))

    def forward(self, xyz):
        return self.position_embedding_head(xyz.transpose(1, 2).contiguous()).transpose(1, 2).contiguous()


class _FlashAttention(torch.autograd.Function):
    """softmax(q k^T * scale + key padding) v for 32-channel heads on the library's wgmma flash-attention tiles
    (csrc/attn_tc.cu), forward and backward. q (B,H,Lq,32), k / v (B,H,Lk,32) bf16 contiguous; key_pad (B,Lk) bool or None."""

    @staticmethod
    def forward(ctx, q, k, v, key_pad, scale):
        from . import _ffi
        B, H, Lq, D = q.shape
        Lk = k.shape[2]
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        pad = key_pad.to(torch.uint8).contiguous() if key_pad is not None else None
        o = torch.empty_like(q)
        lse = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device)
        _ffi.call('esb_attn_fwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), _ffi.ptr(pad), o.data_ptr(), lse.data_ptr(), B, H, Lq,
                  Lk, float(scale), _ffi.stream())
        ctx.save_for_backward(q, k, v, o, lse, pad)
        ctx.scale = float(scale)
        return o

    @staticmethod
    def backward(ctx, do):
        from . import _ffi
        q, k, v, o, lse, pad = ctx.saved_tensors
        B, H, Lq, D = q.shape
        Lk = k.shape[2]
        do = do.contiguous()
        dq = torch.zeros((B, H, Lq, D), dtype=torch.float32, device=q.device)
        dk, dv = torch.empty_like(k), torch.empty_like(v)
        delta = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device)
        _ffi.call('esb_attn_bwd', q.data_ptr(), k.data_ptr(), v.data_ptr(), _ffi.ptr(pad), o.data_ptr(), do.data_ptr(),
                  lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, H, Lq, Lk, ctx.scale,
                  _ffi.stream())
        return dq.to(q.dtype), dk, dv, None, None


def flash_attention(q, k, v, key_pad=None, scale=None):
    return _FlashAttention.apply(q, k, v, key_pad, scale if scale is not None else q.shape[-1] ** -0.5)


class MultiheadAttention(nn.Module):
    """mmcv.cnn.bricks.transformer.MultiheadAttention (†upstream) with batch_first=True, no dropout: positional
    encodings are added to query / key (never to value), the result is added to ``identity`` (= the un-encoded query)."""

    def __init__(self, embed_dims, num_heads, dropout=0.0, batch_first=True, **kwargs):
        super().__init__()
        assert batch_first and dropout == 0.0
        self.embed_dims, self.num_heads = embed_dims, num_heads
        self.attn = nn.MultiheadAttention(embed_dims, num_heads, 0.0, batch_first=True)

    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_pos=None, attn_mask=None,
                key_padding_mask=None):
        key = query if key is None else key
        value = key if value is None else value
        identity = query if identity is None else identity
        if key_pos is None and query_pos is not None and query_pos.shape == key.shape:
            key_pos = query_pos
        if query_pos is not None:
            query = query + query_pos
        if key_pos is not None:
            key = key + key_pos
        E, H = self.embed_dims, self.num_heads
        if (query.is_cuda and attn_mask is None and E // H == 32 and torch.is_autocast_enabled()
                and torch.get_autocast_gpu_dtype() == torch.bfloat16 and os.environ.get('ESB200_ATTN', 'own') == 'own'):
            # the projections are plain library GEMMs; the attention core runs on the library's wgmma flash tiles
            W, bias = self.attn.in_proj_weight, self.attn.in_proj_bias
            B, Lq, Lk = query.shape[0], query.shape[1], key.shape[1]
            q = F.linear(query, W[:E], bias[:E]).view(B, Lq, H, 32).transpose(1, 2)
            k = F.linear(key, W[E:2 * E], bias[E:2 * E]).view(B, Lk, H, 32).transpose(1, 2)
            v = F.linear(value, W[2 * E:], bias[2 * E:]).view(B, Lk, H, 32).transpose(1, 2)
            o = flash_attention(q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16), key_padding_mask)
            out = F.linear(o.transpose(1, 2).reshape(B, Lq, E), self.attn.out_proj.weight, self.attn.out_proj.bias)
            return identity + out
        out = self.attn(query, key, value, attn_mask=attn_mask, key_padding_mask=key_padding_mask, need_weights=False)[0]
        return identity + out


class FFN(nn.Module):
    """mmcv FFN (†upstream): Linear-ReLU-Linear with the identity added; parameters under ``layers.0.0`` / ``layers.1``."""

    def __init__(self, embed_dims=256, feedforward_channels=1024, num_fcs=2, ffn_drop=0., **kwargs):
        super().__init__()
        assert num_fcs == 2 and ffn_drop == 0.
        self.layers = nn.Sequential(nn.Sequential(nn.Linear(embed_dims, feedforward_channels), nn.ReLU(inplace=True),
                                                  nn.Dropout(0.)), nn.Linear(feedforward_channels, embed_dims),
                                    nn.Dropout(0.))

    def forward(self, x):
        return x + self.layers(x)


class SparseFeatureFusionTransformerDecoderLayer(nn.Module):

    def __init__(self, self_attn_cfg=dict(embed_dims=256, num_heads=8, dropout=0.0),
                 cross_attn_cfg=dict(embed_dims=256, num_heads=8, dropout=0.0),
                 cross_attn_text_cfg=dict(embed_dims=256, num_heads=8, dropout=0.0),
                 ffn_cfg=dict(embed_dims=256, feedforward_channels=1024, num_fcs=2, ffn_drop=0.), norm_cfg=dict(type='LN'),
                 init_cfg=None):
        super().__init__()
        self.self_attn = MultiheadAttention(**dict(self_attn_cfg, batch_first=True))
        self.cross_attn_text = MultiheadAttention(**dict(cross_attn_text_cfg, batch_first=True))
        self.cross_attn = MultiheadAttention(**dict(cross_attn_cfg, batch_first=True))
        self.embed_dims = self.self_attn.embed_dims
        self.ffn = FFN(**ffn_cfg)
        self.norms = nn.ModuleList([nn.LayerNorm(self.embed_dims) for _ in range(4)])
        self.self_posembed = PositionEmbeddingLearned(3, self.embed_dims)      # present in checkpoints, unused in forward

    def forward(self, query, key=None, value=None, query_pos=None, key_pos=None, self_attn_mask=None,
                cross_attn_mask=None, key_padding_mask=None, memory_text=None, text_attention_mask=None):
        query = self.self_attn(query=query, key=query, value=query, query_pos=query_pos, key_pos=query_pos,
                               attn_mask=self_attn_mask)
        query = self.norms[0](query)
        query = self.cross_attn_text(query=query, query_pos=query_pos, key=memory_text, value=memory_text,
                                     key_padding_mask=text_attention_mask)
        query = self.norms[1](query)
        query = self.cross_attn(query=query, key=key, value=value, query_pos=query_pos, key_pos=key_pos,
                                attn_mask=cross_attn_mask, key_padding_mask=key_padding_mask)
        query = self.norms[2](query)
        query = self.ffn(query)
        return self.norms[3](query)


class SparseFeatureFusionTransformerDecoder(nn.Module):

    def __init__(self, num_layers, layer_cfg, post_norm_cfg=dict(type='LN'), return_intermediate=True, init_cfg=None):
        super().__init__()
        if post_norm_cfg is not None:
            raise ValueError('There is not post_norm in SparseFeatureFusionTransformerDecoder')
        self.num_layers, self.return_intermediate = num_layers, return_intermediate
        self.layers = nn.ModuleList([SparseFeatureFusionTransformerDecoderLayer(**layer_cfg) for _ in range(num_layers)])
        self.embed_dims = self.layers[0].embed_dims
        self.self_posembed = PositionEmbeddingLearned(9, self.embed_dims)
        self.cross_posembed = PositionEmbeddingLearned(3, self.embed_dims)
        self.norm = nn.LayerNorm(self.embed_dims)

    def forward(self, query, key, value, key_padding_mask, self_attn_mask, cross_attn_mask, query_coords, key_coords,
                pred_bboxes, text_feats, text_attention_mask, bbox_head):
        intermediate, intermediate_bboxes = [], []
        for lid, layer in enumerate(self.layers):
            query_pos = self.self_posembed(pred_bboxes)
            key_pos = self.cross_posembed(key_coords)
            query = layer(query=query, key=key, value=value, query_pos=query_pos, key_pos=key_pos,
                          memory_text=text_feats, self_attn_mask=self_attn_mask, cross_attn_mask=cross_attn_mask,
                          key_padding_mask=key_padding_mask, text_attention_mask=text_attention_mask)
            new_pred_bboxes = bbox_head._bbox_pred_to_bbox(query_coords, bbox_head.reg_branches[lid](query))
            pred_bboxes = new_pred_bboxes.detach().clone()
            if self.return_intermediate:
                intermediate.append(self.norm(query))
                intermediate_bboxes.append(new_pred_bboxes)
        if self.return_intermediate:
            return torch.stack(intermediate), torch.stack(intermediate_bboxes)
        return query, new_pred_bboxes


# ======================================================================================================= head
class ContrastiveEmbed(nn.Module):

    def __init__(self, max_text_len=256, log_scale=None, bias=False):
        super().__init__()
        self.max_text_len = max_text_len
        self.log_scale = log_scale
        if isinstance(log_scale, float):
            self.log_scale = nn.Parameter(torch.Tensor([float(log_scale)]), requires_grad=True)
        elif log_scale not in ['auto', 'none', None]:
            raise ValueError(f'log_scale should be one of "auto", "none", None, but got {log_scale}')
        self.bias = None
        if bias:
            self.bias = nn.Parameter(torch.Tensor([-math.log((1 - 0.01) / 0.01)]), requires_grad=True)

    def forward(self, visual_feat, text_feat, text_token_mask, visual_feat_mask=None):
        """visual (..., b, n, d), text (b, L, d) -> (..., b, n, max_text_len) with -inf on padded text / visual rows."""
        res = visual_feat @ text_feat.transpose(-1, -2)
        if isinstance(self.log_scale, nn.Parameter):
            res = res * self.log_scale.exp()
        elif self.log_scale == 'auto':
            res = res / math.sqrt(visual_feat.shape[-1])
        if self.bias is not None:
            res = res + self.bias
        res = res.masked_fill(~text_token_mask[:, None, :], float('-inf'))
        if visual_feat_mask is not None:
            res = res.masked_fill(~visual_feat_mask[:, :, None], float('-inf'))
        return F.pad(res, (0, self.max_text_len - res.shape[-1]), value=float('-inf'))


class BaseMatchCost:

    def __init__(self, weight=1.):
        self.weight = weight


@TASK_UTILS.register_module()
class BBox3DL1Cost(BaseMatchCost):

    def __call__(self, pred_instances, gt_instances, **kwargs):
        return torch.cdist(pred_instances.bboxes_3d.tensor, gt_instances.bboxes_3d.tensor, p=1) * self.weight


@TASK_UTILS.register_module()
class IoU3DCost:

    def __init__(self, weight):
        self.weight = weight

    def __call__(self, pred_instances, gt_instances, **kwargs):
        pred = EulerDepthInstance3DBoxes(pred_instances.bboxes_3d.tensor, origin=(0.5, 0.5, 0.5))
        gt = EulerDepthInstance3DBoxes(gt_instances.bboxes_3d.tensor, origin=(0.5, 0.5, 0.5))
        return -pred.overlaps(pred, gt) * self.weight


@TASK_UTILS.register_module()
class BinaryFocalLossCost(BaseMatchCost):

    def __init__(self, alpha=0.25, gamma=2, eps=1e-12, binary_input=False, weight=1.):
        super().__init__(weight)
        self.alpha, self.gamma, self.eps = alpha, gamma, eps

    def _focal_loss_cost(self, cls_pred, gt_labels):
        """cls_pred (..., n, T) logits (-inf on padding is fine: sigmoid -> 0 and the matching label is 0),
        gt_labels (..., g, T) in {0,1} -> (..., n, g)."""
        gt_labels = gt_labels.float()
        p = cls_pred.float().sigmoid()
        neg_cost = -(1 - p + self.eps).log() * (1 - self.alpha) * p.pow(self.gamma)
        pos_cost = -(p + self.eps).log() * self.alpha * (1 - p).pow(self.gamma)
        cost = pos_cost @ gt_labels.transpose(-1, -2) + neg_cost @ (1 - gt_labels).transpose(-1, -2)
        return cost * self.weight

    def __call__(self, pred_instances, gt_instances, **kwargs):
        tm = torch.nonzero(gt_instances.text_token_mask[0]).squeeze(-1)
        return self._focal_loss_cost(pred_instances.scores_3d[:, tm], gt_instances.positive_maps[:, tm])


class AssignResult:

    def __init__(self, num_gts, gt_inds, max_overlaps, labels):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = num_gts, gt_inds, max_overlaps, labels


def hungarian_batch(cost: torch.Tensor, n_gt: torch.Tensor):
    """cost (P, n_pred, G) fp32 on the device, n_gt (P,) int32 -> (pred_to_gt (P, n_pred), gt_to_pred (P, G)) int32."""
    P, n_pred, G = cost.shape
    cost = cost.float().contiguous()
    p2g = torch.empty((P, n_pred), dtype=torch.int32, device=cost.device)
    g2p = torch.empty((P, G), dtype=torch.int32, device=cost.device)
    call('esb_hungarian_batch', ptr(cost), ptr(n_gt), P, n_pred, G, ptr(p2g), ptr(g2p), stream())
    return p2g, g2p


@TASK_UTILS.register_module()
class HungarianAssigner3D:
    """Reference interface (one sample): ``assign(pred_instances_3d, gt_instances_3d) -> AssignResult`` with 1-based
    ``gt_inds`` (0 = background). The costs are the registered callables; the matching itself runs on the device."""

    def __init__(self, match_costs):
        if isinstance(match_costs, dict):
            match_costs = [match_costs]
        assert len(match_costs) > 0, 'match_costs must not be a empty list.'
        self.match_costs = [TASK_UTILS.build(c) for c in match_costs]

    def assign(self, pred_instances_3d, gt_instances_3d, eps=1e-7):
        num_gts, num_preds = len(gt_instances_3d), len(pred_instances_3d)
        gt_labels = gt_instances_3d.labels_3d
        device = gt_labels.device
        gt_inds = torch.full((num_preds, ), -1, dtype=torch.long, device=device)
        labels = torch.full((num_preds, ), -1, dtype=torch.long, device=device)
        if num_gts == 0 or num_preds == 0:
            if num_gts == 0:
                gt_inds[:] = 0
            return AssignResult(num_gts, gt_inds, None, labels)
        cost = torch.stack([c(pred_instances=pred_instances_3d, gt_instances=gt_instances_3d)
                            for c in self.match_costs]).sum(dim=0).detach()
        if num_gts > num_preds:           # more targets than queries: solve the transposed problem
            g2p, _ = hungarian_batch(cost.t()[None], torch.tensor([num_preds], dtype=torch.int32, device=device))
            p2g = torch.full((num_preds, ), -1, dtype=torch.int32, device=device)
            sel = g2p[0] >= 0
            p2g[g2p[0][sel].long()] = torch.nonzero(sel).squeeze(1).int()
        else:
            p2g = hungarian_batch(cost[None], torch.tensor([num_gts], dtype=torch.int32, device=device))[0][0]
        gt_inds = (p2g + 1).long()
        labels = torch.where(p2g >= 0, gt_labels[p2g.clamp(min=0).long()], labels)
        return AssignResult(num_gts, gt_inds, None, labels)


@MODELS.register_module()
class GroundingHead(nn.Module):

    def __init__(self, num_classes, embed_dims=256, num_pred_layer=7, num_reg_fcs=2, num_reg=9, box_coder='baseline',
                 sync_cls_avg_factor=False, decouple_bbox_loss=False, decouple_groups=3, decouple_weights=None,
                 norm_decouple_loss=False, loss_cls=dict(type='mmdet.FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25),
                 loss_bbox=dict(type='BBoxCDLoss', mode='l1', loss_weight=1.0, group='g8'),
                 train_cfg=dict(assigner=dict(type='HungarianAssigner3D', match_costs=[
                     dict(type='BinaryFocalLossCost', weight=1.0), dict(type='BBox3DL1Cost', weight=2.0),
                     dict(type='IoU3DCost', weight=2.0)])),
                 contrastive_cfg=dict(max_text_len=256), share_pred_layer=False, test_cfg=None, init_cfg=None):
        super().__init__()
        self.contrastive_cfg = dict(contrastive_cfg)
        self.max_text_len = contrastive_cfg.get('max_text_len', 256)
        self.share_pred_layer, self.num_pred_layer = share_pred_layer, num_pred_layer
        self.bg_cls_weight = 0
        self.sync_cls_avg_factor = sync_cls_avg_factor
        self.decouple_bbox_loss, self.decouple_groups = decouple_bbox_loss, decouple_groups
        self.norm_decouple_loss = norm_decouple_loss
        assert not norm_decouple_loss, 'hot-path configuration: norm_decouple_loss=False'
        self.decouple_weights = decouple_weights or [1.0 / decouple_groups] * decouple_groups
        self.num_reg, self.box_coder = num_reg, box_coder
        assert box_coder in ('baseline', 'FCAF')
        if train_cfg:
            assert 'assigner' in train_cfg, 'assigner should be provided when train_cfg is set.'
            self.assigner = TASK_UTILS.build(train_cfg['assigner'])
        self.num_classes, self.embed_dims, self.num_reg_fcs = num_classes, embed_dims, num_reg_fcs
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.loss_cls = MODELS.build(loss_cls)
        self.loss_bbox = MODELS.build(loss_bbox)
        self.process_group = None
        self._init_layers()
        self.init_weights()

    def _init_layers(self):
        import copy
        fc_cls = ContrastiveEmbed(**self.contrastive_cfg)
        reg = []
        for _ in range(self.num_reg_fcs):
            reg += [nn.Linear(self.embed_dims, self.embed_dims), nn.ReLU()]
        reg.append(nn.Linear(self.embed_dims, self.num_reg))
        reg = nn.Sequential(*reg)
        if self.share_pred_layer:
            self.cls_branches = nn.ModuleList([fc_cls for _ in range(self.num_pred_layer)])
            self.reg_branches = nn.ModuleList([reg for _ in range(self.num_pred_layer)])
        else:
            self.cls_branches = nn.ModuleList([copy.deepcopy(fc_cls) for _ in range(self.num_pred_layer)])
            self.reg_branches = nn.ModuleList([copy.deepcopy(reg) for _ in range(self.num_pred_layer)])

    def init_weights(self):
        for m in self.reg_branches:
            nn.init.constant_(m[-1].weight, 0)
            nn.init.constant_(m[-1].bias, 0)
        nn.init.constant_(self.reg_branches[0][-1].bias.data[2:], -2.0)

    def _bbox_pred_to_bbox(self, points, bbox_pred):
        """grounding_head.py:267-363: (B, nq, 3) anchor points + (B, nq, 9|12) regression -> (B, nq, 9) boxes."""
        assert points.dim() == bbox_pred.dim() == 3
        B, nq = points.shape[:2]
        points, bbox_pred = points.float(), bbox_pred.float()
        if self.box_coder == 'baseline':
            center = bbox_pred[..., :3] + points
            size = torch.exp(bbox_pred[..., 3:6]).clamp(min=2e-2)
            if bbox_pred.shape[-1] == 9:
                euler = bbox_pred[..., 6:]
            elif bbox_pred.shape[-1] == 12:
                rot = ortho_6d_2_mat(bbox_pred[..., 6:9].reshape(-1, 3), bbox_pred[..., 9:].reshape(-1, 3))
                euler = matrix_to_euler_angles_zxy(rot).view(B, nq, 3)
            else:
                raise NotImplementedError
            return torch.cat((center, size, euler), dim=-1)
        pts = points.reshape(-1, 3)
        bp = bbox_pred.reshape(-1, bbox_pred.shape[-1])
        if bp.shape[0] == 0:
            return bbox_pred
        d = torch.exp(bp[:, :6]).clamp(min=2e-2)
        shift = torch.stack(((d[:, 1] - d[:, 0]) / 2, (d[:, 3] - d[:, 2]) / 2, (d[:, 5] - d[:, 4]) / 2), -1).view(-1, 1, 3)
        if bp.shape[-1] == 9:
            euler = bp[:, 6:]
        elif bp.shape[-1] == 12:
            euler = matrix_to_euler_angles_zxy(ortho_6d_2_mat(bp[:, 6:9], bp[:, 9:]))
        else:
            raise NotImplementedError
        center = pts + rotation_3d_in_euler(shift, euler)[:, 0, :]
        size = torch.stack((d[:, 0] + d[:, 1], d[:, 2] + d[:, 3], d[:, 4] + d[:, 5]), -1)
        return torch.cat((center, size, euler), -1).view(B, nq, -1)

    def forward(self, hidden_states, text_feats, text_token_mask):
        return (torch.stack([self.cls_branches[l](hidden_states[l], text_feats, text_token_mask)
                             for l in range(hidden_states.shape[0])]), )

    # ---- prediction -----------------------------------------------------------------------------------------------
    def predict(self, hidden_states, all_layers_pred_bboxes, text_feats, text_token_mask, batch_data_samples):
        cls_scores = self(hidden_states, text_feats, text_token_mask)[0][-1]
        bbox_preds = all_layers_pred_bboxes[-1]
        out = []
        for b in range(len(batch_data_samples)):
            scores = cls_scores[b].float().sigmoid().max(-1)[0]
            r = InstanceData()
            r.bboxes_3d = EulerDepthInstance3DBoxes(bbox_preds[b].float())
            r.scores_3d = scores
            r.target_scores_3d = scores
            out.append(r)
        return out

    # ---- loss -------------------------------------------------------------------------------------------------------
    def _batched_costs(self, cls_scores, pred_bboxes, gt_boxes, pos_maps, n_gt_host):
        """All decoder layers x samples at once. cls_scores (Ly,B,nq,T), pred_bboxes (Ly,B,nq,9), gt_boxes (B,G,9) zero
        padded, pos_maps (B,G,T) -> cost (Ly,B,nq,G) fp32 (columns >= n_gt[b] are never read by the solver)."""
        Ly, B, nq, T = cls_scores.shape
        G = gt_boxes.shape[1]
        cost = cls_scores.new_zeros((Ly, B, nq, G), dtype=torch.float32)
        for c in self.assigner.match_costs:
            if isinstance(c, BinaryFocalLossCost):
                cost += c._focal_loss_cost(cls_scores, pos_maps[None])
            elif isinstance(c, BBox3DL1Cost):
                cost += torch.cdist(pred_bboxes.float(), gt_boxes[None].expand(Ly, -1, -1, -1).float(), p=1) * c.weight
            elif isinstance(c, IoU3DCost):
                for b in range(B):
                    g = n_gt_host[b]
                    if g == 0:
                        continue
                    pc = box_corners_container(pred_bboxes[:, b].reshape(-1, 9).float())
                    gc = box_corners_container(gt_boxes[b, :g].float())
                    iou = box3d_overlap(pc, gc)[1]
                    cost[:, b, :, :g] -= iou.view(Ly, nq, g) * c.weight
            else:
                raise NotImplementedError(type(c))
        return cost

    def loss(self, hidden_states, all_layers_pred_bboxes, text_feats, text_token_mask, batch_data_samples):
        cls_scores = self(hidden_states, text_feats, text_token_mask)[0].float()    # (Ly,B,nq,T)
        return self.loss_by_feat(cls_scores, all_layers_pred_bboxes, text_token_mask,
                                 [ds.gt_instances_3d for ds in batch_data_samples])

    def loss_by_feat(self, cls_scores, pred_bboxes, text_token_mask, batch_gt_instances_3d):
        Ly, B, nq, T = cls_scores.shape
        dev = cls_scores.device
        n_gt_host = [len(g.bboxes_3d) for g in batch_gt_instances_3d]
        assert max(n_gt_host) <= nq, 'more targets than queries: use HungarianAssigner3D.assign per sample'
        G = max(max(n_gt_host), 1)
        gt_boxes = torch.zeros((B, G, 9), dtype=torch.float32, device=dev)
        pos_maps = torch.zeros((B, G, T), dtype=torch.float32, device=dev)
        for b, g in enumerate(batch_gt_instances_3d):
            if n_gt_host[b]:
                gt_boxes[b, :n_gt_host[b]] = g.bboxes_3d.tensor.float()
                pos_maps[b, :n_gt_host[b]] = g.positive_maps.float()
        n_gt = torch.tensor(n_gt_host * Ly, dtype=torch.int32, device=dev)           # problem p = layer * B + b
        with torch.no_grad():
            cost = self._batched_costs(cls_scores.detach(), pred_bboxes.detach(), gt_boxes, pos_maps, n_gt_host)
            p2g, g2p = hungarian_batch(cost.view(Ly * B, nq, G), n_gt)
            p2g = p2g.view(Ly, B, nq).long()
            labels = torch.gather(pos_maps[None].expand(Ly, -1, -1, -1), 2,
                                  p2g.clamp(min=0)[..., None].expand(-1, -1, -1, T))
            labels = labels * (p2g >= 0)[..., None]
            # matched pairs through the inverse map: (layer, sample, gt) -> query; count known on the host
            bi = torch.tensor([b for b in range(B) for _ in range(n_gt_host[b])], dtype=torch.long, device=dev)
            gi = torch.tensor([g for b in range(B) for g in range(n_gt_host[b])], dtype=torch.long, device=dev)
            qi = g2p.view(Ly, B, G).long()[:, bi, gi]                                  # (Ly, Npos)
        num_total_pos = float(sum(n_gt_host))
        cls_avg_factor = num_total_pos * 1.0 + (B * nq - num_total_pos) * self.bg_cls_weight
        if self.sync_cls_avg_factor and torch.distributed.is_available() and torch.distributed.is_initialized():
            t = torch.tensor([cls_avg_factor], device=dev)
            torch.distributed.all_reduce(t, group=self.process_group)
            cls_avg_factor = float(t) / torch.distributed.get_world_size(self.process_group)
        cls_avg_factor = max(cls_avg_factor, 1)

        # token-level focal loss on the valid text tokens (masked_select in the reference; a mask product here)
        tmask = F.pad(text_token_mask, (0, T - text_token_mask.shape[1]))[None, :, None, :].expand(Ly, -1, nq, -1)
        logits = torch.where(tmask, cls_scores.float(), torch.zeros_like(cls_scores, dtype=torch.float32))
        losses_cls = [self.loss_cls(logits[l], labels[l], tmask[l].float(), avg_factor=cls_avg_factor) for l in range(Ly)]

        n_pos = bi.numel()
        if n_pos:
            tgt = gt_boxes[bi, gi]                                                    # (Npos, 9)
            pred = pred_bboxes.float()[torch.arange(Ly, device=dev)[:, None], bi[None], qi]   # (Ly, Npos, 9)
            tgt_l = tgt[None].expand(Ly, -1, -1)
            if self.decouple_bbox_loss:
                assert self.decouple_groups in (3, 4), 'Only support groups=3 or 4 with stable performance.'
                variants = [torch.cat((pred[..., :3], tgt_l[..., 3:]), -1),
                            torch.cat((tgt_l[..., :3], pred[..., 3:6], tgt_l[..., 6:]), -1),
                            torch.cat((tgt_l[..., :6], pred[..., 6:]), -1)]
                if self.decouple_groups == 4:
                    variants.append(pred)
                src = torch.stack(variants, 1)                                         # (Ly, Gp, Npos, 9)
                Gp = src.shape[1]
                cd = chamfer_l1_src(bbox_to_corners(src.reshape(-1, 9)),
                                    bbox_to_corners(tgt_l[:, None].expand(-1, Gp, -1, -1).reshape(-1, 9)))
                per = cd.view(Ly, Gp, -1).mean(-1) * self.loss_bbox.loss_weight        # mean over pairs x 8 corners
                w = per.new_tensor(self.decouple_weights[:Gp])
                losses_bbox = list((per * w).sum(1))
            else:
                cd = chamfer_l1_src(bbox_to_corners(pred.reshape(-1, 9)), bbox_to_corners(tgt_l.reshape(-1, 9)))
                losses_bbox = list(cd.view(Ly, -1).mean(-1) * self.loss_bbox.loss_weight)
        else:
            losses_bbox = [pred_bboxes[l].sum() * 0 for l in range(Ly)]
        loss_dict = dict(loss_cls=losses_cls[-1], loss_bbox=losses_bbox[-1])
        for l in range(Ly - 1):
            loss_dict[f'd{l}.loss_cls'] = losses_cls[l]
            loss_dict[f'd{l}.loss_bbox'] = losses_bbox[l]
        return loss_dict


# ======================================================================================================= sparse neck
@MODELS.register_module()
class MinkNeck(nn.Module):
    """Sparse FPN with score-driven pruning (mink_neck.py:133-244); per-scan outputs are concatenated coarse -> fine."""

    _make_block = staticmethod(FCAF3DHeadRotMat._make_block)
    _make_up_block = staticmethod(FCAF3DHeadRotMat._make_up_block)
    _run_block = FCAF3DHeadRotMat._run_block
    _prune = FCAF3DHeadRotMat._prune

    def __init__(self, num_classes, in_channels, out_channels, voxel_size, pts_prune_threshold, train_cfg=None,
                 test_cfg=None, init_cfg=None):
        super().__init__()
        self.voxel_size, self.pts_prune_threshold = voxel_size, pts_prune_threshold
        self.pruning = SP.MinkowskiPruning()
        for i in range(len(in_channels)):
            if i > 0:
                setattr(self, f'up_block_{i}', self._make_up_block(in_channels[i], in_channels[i - 1]))
            setattr(self, f'out_block_{i}', self._make_block(in_channels[i], out_channels))
        self.conv_cls = SP.MinkowskiConvolution(out_channels, num_classes, kernel_size=1, bias=True, dimension=3)
        nn.init.normal_(self.conv_cls.kernel, std=.01)
        nn.init.constant_(self.conv_cls.bias, -4.59511985013459)

    def forward(self, x: List[SP.SparseTensor], batch_size: int):
        feats, scores, points = [], [], []
        inputs = x
        x = inputs[-1]
        prune_score = None
        for i in range(len(inputs) - 1, -1, -1):
            if i < len(inputs) - 1:
                x = self._run_block(getattr(self, f'up_block_{i + 1}'), x)
                x = inputs[i] + x
                x = self._prune(x, prune_score)
            out = self._run_block(getattr(self, f'out_block_{i}'), x)
            f = out.F
            cls = torch.addmm(self.conv_cls.bias.to(f.dtype), f, self.conv_cls.kernel.to(f.dtype))
            prune_score = out.replace_feature(cls.max(dim=1, keepdim=True).values.float())
            perms = out.decomposition_permutations
            pts = out.C[:, 1:] * self.voxel_size
            feats.append([f[p] for p in perms])
            scores.append([cls[p] for p in perms])
            points.append([pts[p] for p in perms])
        cat = lambda lv: [torch.cat([l[b] for l in lv], 0) for b in range(batch_size)]
        return cat(feats), cat(scores), cat(points)


# ======================================================================================================= the model
@MODELS.register_module()
class SparseFeatureFusion3DGrounder(nn.Module):

    def __init__(self, backbone, backbone_3d, bbox_head, neck=None, neck_3d=None, decoder=None, voxel_size=0.01,
                 num_queries=512, max_num_entities=256, coord_type='CAMERA', train_cfg=None, test_cfg=None,
                 data_preprocessor=None, use_xyz_feat=False, init_cfg=None, compute_dtype=torch.float32,
                 freeze_text_encoder=True):
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
        self.bbox_head = MODELS.build(dict(bbox_head, train_cfg=train_cfg, test_cfg=test_cfg))
        self.coord_type, self.train_cfg, self.test_cfg = coord_type, train_cfg, test_cfg
        self.num_queries = num_queries
        self.max_num_entities = self.bbox_head.contrastive_cfg.get('max_text_len', max_num_entities)
        self.voxel_size, self.use_xyz_feat = voxel_size, use_xyz_feat
        self.freeze_text_encoder = freeze_text_encoder       # cfg: paramwise lr_mult=0 for 'text_encoder'
        self.tokenizer, self.text_encoder = build_text_modules('roberta-base')
        if freeze_text_encoder:        # keeps the encoder out of the optimiser arena (no weight decay on frozen weights)
            self.text_encoder.requires_grad_(False)
        self.decoder = SparseFeatureFusionTransformerDecoder(**decoder)
        self.embed_dims = self.decoder.embed_dims
        self.text_feat_map = nn.Linear(self.text_encoder.config.hidden_size, self.embed_dims, bias=True)

    # ---- features ---------------------------------------------------------------------------------------------------
    voxelize = SparseFeatureFusionSingleStage3DDetector.voxelize

    def extract_feat(self, batch_inputs_dict, batch_data_samples):
        points = batch_inputs_dict['points']
        img = batch_inputs_dict['imgs']
        metas_list = [ds.metainfo for ds in batch_data_samples]
        dev = points[0].device
        B, V = img.shape[:2]
        img4 = img.reshape([-1] + list(img.shape)[2:]).to(self.compute_dtype)
        if not img4.is_contiguous(memory_format=torch.channels_last):
            img4 = img4.contiguous(memory_format=torch.channels_last)
        img_features = self.backbone(img4)
        coords, feats = self.voxelize(points)
        x = SP.SparseTensor(coordinates=coords, features=feats.to(self.compute_dtype), batch_size=len(points))
        x = self.backbone_3d(x)
        metas = pack_paint_metas(metas_list, dev)
        proj = pack_projections(metas_list, self.coord_type, dev)
        for li in range(len(x)):
            painted = paint_points(img_features[li], x[li].C, metas, proj, self.voxel_size, tuple(img.shape[-2:]), V)
            x[li] = x[li].replace_feature(torch.cat([x[li].F, painted.to(x[li].F.dtype)], 1))
        return self.neck_3d(x, B)

    # ---- text -------------------------------------------------------------------------------------------------------
    def create_positive_map(self, tokenized, tokens_positive, batch_idx):
        pm = torch.zeros((len(tokens_positive), self.max_num_entities), dtype=torch.float)
        for j, tok_list in enumerate(tokens_positive):
            for (beg, end) in tok_list:
                beg_pos = tokenized.char_to_token(batch_idx, beg)
                end_pos = tokenized.char_to_token(batch_idx, end - 1)
                if beg_pos is None:
                    beg_pos = tokenized.char_to_token(batch_idx, beg + 1)
                    if beg_pos is None:
                        beg_pos = tokenized.char_to_token(batch_idx, beg + 2)
                if end_pos is None:
                    end_pos = tokenized.char_to_token(batch_idx, end - 2)
                    if end_pos is None:
                        end_pos = tokenized.char_to_token(batch_idx, end - 3)
                if beg_pos is None or end_pos is None:
                    continue
                pm[j, beg_pos:end_pos + 1].fill_(1)
        return pm / (pm.sum(-1)[:, None] + 1e-6)

    def get_positive_map(self, tokenized, tokens_positive):
        return [self.create_positive_map(tokenized, tp, i) for i, tp in enumerate(tokens_positive)]

    def encode_text(self, batch_data_samples, dev):
        texts = [ds.text for ds in batch_data_samples]
        if 'tokens_positive' in batch_data_samples[0]:
            tokens_positive = [ds.tokens_positive for ds in batch_data_samples]
        else:
            tokens_positive = [[[0, 1]] for _ in batch_data_samples]
        tokenized = self.tokenizer.batch_encode_plus(texts, padding='longest', return_tensors='pt')
        positive_maps = self.get_positive_map(tokenized, tokens_positive)
        tokenized = tokenized.to(dev)
        if self.freeze_text_encoder:
            with torch.no_grad():
                hidden = self.text_encoder(**tokenized).last_hidden_state
        else:
            hidden = self.text_encoder(**tokenized).last_hidden_state
        text_feats = self.text_feat_map(hidden.float())
        text_token_mask = tokenized.attention_mask.bool()
        for i, ds in enumerate(batch_data_samples):
            pm = positive_maps[i].to(dev).bool().float()
            ds.gt_instances_3d.positive_maps = pm
            ds.gt_instances_3d.text_token_mask = text_token_mask[i].unsqueeze(0).repeat(len(pm), 1)
        return dict(text_feats=text_feats, text_token_mask=text_token_mask)

    # ---- transformer ------------------------------------------------------------------------------------------------
    def pre_decoder(self, feats_list, scores_list, xyz_list, text_feats, text_token_mask):
        B = len(feats_list)
        lens = [f.shape[0] for f in feats_list]
        n_max, n_min = max(lens), min(lens)
        C = feats_list[0].shape[1]
        dev = feats_list[0].device
        feats = torch.zeros((B, n_max, C), dtype=torch.float32, device=dev)
        coords = torch.zeros((B, n_max, 3), dtype=torch.float32, device=dev)
        feats_mask = torch.zeros((B, n_max), dtype=torch.bool, device=dev)
        for b in range(B):
            feats[b, :lens[b]] = feats_list[b].float()
            coords[b, :lens[b]] = xyz_list[b].float()
            feats_mask[b, :lens[b]] = True
        head = self.bbox_head
        enc_cls = head.cls_branches[self.decoder.num_layers](feats, text_feats, text_token_mask, feats_mask)
        topk = min(self.num_queries, n_min)
        # torch.topk leaves ties unspecified; frozen like the prune rule: descending score, lowest row first
        order = torch.sort(enc_cls.max(-1)[0], dim=1, descending=True, stable=True).indices[:, :topk]
        bbox_preds = head.reg_branches[self.decoder.num_layers](feats)
        boxes = head._bbox_pred_to_bbox(coords, bbox_preds)
        gather = lambda t: torch.gather(t, 1, order.unsqueeze(-1).expand(-1, -1, t.shape[-1]))
        dec_in = dict(query=gather(feats), feats=feats, feats_attention_mask=~feats_mask, query_coords=gather(coords),
                      feats_coords=coords, pred_bboxes=gather(boxes).detach().clone(), text_feats=text_feats,
                      text_attention_mask=~text_token_mask)
        return dec_in, dict(text_feats=text_feats, text_token_mask=text_token_mask)

    def forward_decoder(self, query, feats, feats_attention_mask, query_coords, feats_coords, pred_bboxes, text_feats,
                        text_attention_mask):
        inter, boxes = self.decoder(query=query, key=feats, value=feats, key_padding_mask=feats_attention_mask,
                                    self_attn_mask=None, cross_attn_mask=None, query_coords=query_coords,
                                    key_coords=feats_coords, pred_bboxes=pred_bboxes, text_feats=text_feats,
                                    text_attention_mask=text_attention_mask, bbox_head=self.bbox_head)
        return dict(hidden_states=inter, all_layers_pred_bboxes=boxes)

    def forward_transformer(self, point_feats, scores, point_xyz, text_dict, batch_data_samples=None):
        # bf16 compute: the attention / FFN / contrastive contractions autocast to bf16 (LayerNorm and softmax stay fp32,
        # box decoding and the losses are fp32 below); fp32 compute leaves the decoder in fp32 (the parity arithmetic)
        amp = self.compute_dtype == torch.bfloat16 and point_feats[0].is_cuda
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=amp):
            dec_in, head_in = self.pre_decoder(point_feats, scores, point_xyz, **text_dict)
            head_in.update(self.forward_decoder(**dec_in))
        return head_in

    # ---- entry points -----------------------------------------------------------------------------------------------
    def loss(self, batch_inputs_dict, batch_data_samples, **kwargs):
        text_dict = self.encode_text(batch_data_samples, batch_inputs_dict['points'][0].device)
        feats, scores, xyz = self.extract_feat(batch_inputs_dict, batch_data_samples)
        head_in = self.forward_transformer(feats, scores, xyz, text_dict, batch_data_samples)
        return self.bbox_head.loss(**head_in, batch_data_samples=batch_data_samples)

    def predict(self, batch_inputs_dict, batch_data_samples, **kwargs):
        feats, scores, xyz = self.extract_feat(batch_inputs_dict, batch_data_samples)
        text_dict = self.encode_text(batch_data_samples, batch_inputs_dict['points'][0].device)
        head_in = self.forward_transformer(feats, scores, xyz, text_dict, batch_data_samples)
        results = self.bbox_head.predict(**head_in, batch_data_samples=batch_data_samples)
        for ds, r in zip(batch_data_samples, results):
            ds.pred_instances_3d = r
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
        raise RuntimeError(f'Invalid mode "{mode}". Only supports loss, predict and tensor mode')

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
