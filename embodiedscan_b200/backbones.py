"""Backbones of the hot path, registered under the reference's names.

* ``MinkResNet`` — sparse 3D ResNet (embodiedscan/models/backbones/mink_resnet.py:20-140) over ``esb200.sparse``.
  Depth 14 = (BasicBlock, (1,1,1,1)) is added for BASELINE.json config C1 (SURVEY H9).
* ``ResNet`` (registered as ``mmdet.ResNet``) — the per-view 2D backbone named by the config
  (configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py:24-34): pytorch-style ResNet with
  ``base_channels``, ``frozen_stages`` and ``norm_eval``. The BatchNorms are frozen (requires_grad=False, eval), so each
  conv+BN pair is evaluated as ONE convolution with folded scale/shift, in channels-last bf16/fp32; the dense
  contraction itself is the library conv (cuDNN) in this round — see DESIGN.md "2D backbone".
"""
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import sparse as SP
from .registry import MODELS


@MODELS.register_module()
class MinkResNet(nn.Module):
    arch_settings = {
        14: (SP.BasicBlock, (1, 1, 1, 1)),
        18: (SP.BasicBlock, (2, 2, 2, 2)),
        34: (SP.BasicBlock, (3, 4, 6, 3)),
        50: (SP.Bottleneck, (3, 4, 6, 3)),
        101: (SP.Bottleneck, (3, 4, 23, 3)),
        152: (SP.Bottleneck, (3, 8, 36, 3)),
    }

    def __init__(self, depth: int, in_channels: int, num_stages: int = 4, pool: bool = True):
        super().__init__()
        if depth not in self.arch_settings:
            raise KeyError(f'invalid depth {depth} for resnet')
        assert 4 >= num_stages >= 1
        block, stage_blocks = self.arch_settings[depth]
        stage_blocks = stage_blocks[:num_stages]
        self.num_stages, self.pool = num_stages, pool
        self.inplanes = 64
        self.conv1 = SP.MinkowskiConvolution(in_channels, self.inplanes, kernel_size=3, stride=2, dimension=3)
        self.norm1 = SP.MinkowskiInstanceNorm(self.inplanes)
        self.relu = SP.MinkowskiReLU(inplace=True)
        if self.pool:
            self.maxpool = SP.MinkowskiMaxPooling(kernel_size=2, stride=2, dimension=3)
        for i in range(len(stage_blocks)):
            setattr(self, f'layer{i + 1}', self._make_layer(block, 64 * 2 ** i, stage_blocks[i], stride=2))
        self.init_weights()

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, SP.MinkowskiConvolution):
                SP.kaiming_normal_(m.kernel, mode='fan_out', nonlinearity='relu')
            if isinstance(m, SP.MinkowskiBatchNorm):
                nn.init.constant_(m.bn.weight, 1)
                nn.init.constant_(m.bn.bias, 0)

    def _make_layer(self, block, planes, blocks, stride):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                SP.MinkowskiConvolution(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride,
                                        dimension=3), SP.MinkowskiBatchNorm(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride=stride, downsample=downsample, dimension=3)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, stride=1, dimension=3))
        return nn.Sequential(*layers)

    def forward(self, x: SP.SparseTensor) -> List[SP.SparseTensor]:
        x = self.conv1(x)
        x = self.norm1(x, act=SP.ACT_RELU)      # InstanceNorm + ReLU fused
        if self.pool:
            x = self.maxpool(x)
        outs = []
        for i in range(self.num_stages):
            x = getattr(self, f'layer{i + 1}')(x)
            outs.append(x)
        return outs


# ------------------------------------------------------------------------------------------------------------
# 2D ResNet (mmdet.ResNet semantics)
# ------------------------------------------------------------------------------------------------------------
def _fold(conv_w, bn: nn.BatchNorm2d, dtype):
    scale = bn.weight * torch.rsqrt(bn.running_var + bn.eps)
    w = conv_w * scale[:, None, None, None]
    b = bn.bias - bn.running_mean * scale
    return w.to(dtype), b.to(dtype)


class _BiasResAct(torch.autograd.Function):
    """y = act(conv_out + bias[c] (+ res)) in ONE pass over the NHWC activation, written in place of conv_out."""

    @staticmethod
    def forward(ctx, conv_out, bias, res, act):
        from . import _ffi
        assert conv_out.is_contiguous(memory_format=torch.channels_last)
        N, C, H, W = conv_out.shape
        if res is not None and not res.is_contiguous(memory_format=torch.channels_last):
            res = res.contiguous(memory_format=torch.channels_last)
        _ffi.call('esb_bias_act_fwd', conv_out.data_ptr(), bias.data_ptr(), _ffi.ptr(res), conv_out.data_ptr(), N * H * W, C,
                  act, _ffi.dtype_code(conv_out.dtype), _ffi.stream())
        ctx.mark_dirty(conv_out)
        ctx.act, ctx.has_res = act, res is not None
        if act != SP.ACT_NONE:
            ctx.save_for_backward(conv_out)
        return conv_out

    @staticmethod
    def backward(ctx, dy):
        from . import _ffi
        if ctx.act != SP.ACT_NONE:
            (y, ) = ctx.saved_tensors
            dy = dy.contiguous(memory_format=torch.channels_last)
            g = torch.empty_like(y)
            _ffi.call('esb_act_bwd', dy.data_ptr(), y.data_ptr(), g.data_ptr(), y.numel(), ctx.act,
                      _ffi.dtype_code(y.dtype), _ffi.stream())
        else:
            g = dy
        # the bias is the folded BN shift beta - mean * scale: it needs a gradient whenever the BN affine is trainable
        db = g.sum((0, 2, 3), dtype=torch.float32) if ctx.needs_input_grad[1] else None
        return g, db, (g if ctx.has_res else None), None


def ohwi(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, kh, kw) -> contiguous (Cout, kh, kw, Cin) bf16: the filter matrix of csrc/conv_tma.cu (a channels_last
    filter already is this memory: no copy then)."""
    return w.detach().to(torch.bfloat16).permute(0, 2, 3, 1).contiguous()


def tma_channels_ok(c: int) -> bool:
    return c in (16, 32, 64, 128, 256) or (c > 256 and c % 256 == 0)


def conv2d_tma(x: torch.Tensor, w_ohwi: torch.Tensor, bias, res, relu: bool, stride: int, pad: int) -> torch.Tensor:
    """conv + bias + residual + ReLU in ONE persistent TMA + wgmma launch (csrc/conv_tma.cu). x (N,Cin,H,W) bf16 in
    channels_last memory; w_ohwi (Cout,kh,kw,Cin) bf16 from :func:`ohwi`; bias (Cout,) fp32 or None; res like the output."""
    from . import _ffi
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last)
    N, cin, H, W = x.shape
    cout, kh, kw, _ = w_ohwi.shape
    Ho, Wo = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    y = torch.empty((N, cout, Ho, Wo), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    if res is not None:
        assert res.shape == y.shape and res.dtype == torch.bfloat16
        if not res.is_contiguous(memory_format=torch.channels_last):
            res = res.contiguous(memory_format=torch.channels_last)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    _ffi.call('esb_conv2d_tma_fwd', x.data_ptr(), w_ohwi.data_ptr(), _ffi.ptr(bias), _ffi.ptr(res), y.data_ptr(), N, H, W,
              cin, cout, kh, kw, stride, pad, 1 if relu else 0, _ffi.stream())
    return y


def conv2d_tma_wgrad(x: torch.Tensor, dy: torch.Tensor, w_shape, stride: int, pad: int) -> torch.Tensor:
    """dL/dw of ``F.conv2d(x, w, stride, pad)`` with TMA-fed MN-major operands (csrc/conv_tma.cu::conv_tma_wgrad_kernel);
    x (N,Cin,H,W), dy (N,Cout,Ho,Wo) bf16 channels_last -> (Cout,Cin,kh,kw) fp32 view of the (kh*kw*Cin, Cout) accumulator."""
    from . import _ffi
    cout, cin, kh, kw = w_shape
    assert x.dtype == dy.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last) \
        and dy.is_contiguous(memory_format=torch.channels_last)
    dw_t = torch.zeros((kh * kw * cin, cout), dtype=torch.float32, device=x.device)
    _ffi.call('esb_conv2d_tma_wgrad', x.data_ptr(), dy.data_ptr(), dw_t.data_ptr(), x.shape[0], x.shape[2], x.shape[3], cin,
              cout, kh, kw, stride, pad, _ffi.stream())
    return dw_t.view(kh, kw, cin, cout).permute(3, 2, 0, 1)


def conv2d_tma_dgrad(dy: torch.Tensor, w_ohwi: torch.Tensor, in_hw, pad: int, stride: int = 1) -> torch.Tensor:
    """dL/dx of ``F.conv2d(x, w, stride, pad)`` (stride 1 or 2) with the same kernel: flipped taps, filter read MN-major;
    stride 2 = one launch per parity class of dx (strided TMA stores)."""
    from . import _ffi
    assert dy.is_cuda and dy.dtype == torch.bfloat16 and dy.is_contiguous(memory_format=torch.channels_last)
    cout, kh, kw, cin = w_ohwi.shape
    H, W = in_hw
    dx = torch.empty((dy.shape[0], cin, H, W), dtype=torch.bfloat16, device=dy.device, memory_format=torch.channels_last)
    _ffi.call('esb_conv2d_tma_dgrad', dy.data_ptr(), w_ohwi.data_ptr(), dx.data_ptr(), dy.shape[0], H, W, cin, cout, kh, kw,
              stride, pad, _ffi.stream())
    return dx


class _ConvBlock2D(torch.autograd.Function):
    """out = act(conv2d(x, w) + bias + res) of the image backbone on the library's own kernels, all three passes:
      bf16, tensor-core channel counts -> csrc/conv_tma.cu (TMA + wgmma; fused epilogue), its stride-1 / stride-2 dgrad
                                         and its wgrad; the dgrad of larger strides -> csrc/conv2d_direct.cu
      fp32 (the parity arithmetic) / the 3-channel stem -> csrc/conv2d_direct.cu (fp32 FMA)
    x channels_last; w (Cout,Cin,kh,kw) in channels_last memory (= OHWI); bias fp32 (Cout,) constant; res like the output."""

    @staticmethod
    def forward(ctx, x, w, bias, res, relu, stride, pad):
        from . import _ffi
        N, cin, H, W = x.shape
        cout, _, kh, kw = w.shape
        w_ohwi = w.detach().permute(0, 2, 3, 1)
        if not w_ohwi.is_contiguous():
            w_ohwi = w_ohwi.contiguous()
        tma = x.dtype == torch.bfloat16 and tma_channels_ok(cin) and tma_channels_ok(cout)
        stem = (x.dtype == torch.bfloat16 and (cin, cout, kh, kw, stride, pad) == (3, 16, 7, 7, 2, 3) and res is None
                and bias is not None and (W * 3) % 2 == 0)
        if tma:
            y = conv2d_tma(x, w_ohwi, bias, res, relu, stride, pad)
        elif stem:       # wgmma with the im2col rows built in shared memory (csrc/conv_tma.cu::stem7x7_tc_kernel)
            Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
            y = torch.empty((N, cout, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
            _ffi.call('esb_stem7x7_tc', x.data_ptr(), w_ohwi.data_ptr(), bias.data_ptr(), y.data_ptr(), N, H, W,
                      1 if relu else 0, _ffi.stream())
        else:
            Ho, Wo = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
            y = torch.empty((N, cout, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
            if res is not None and not res.is_contiguous(memory_format=torch.channels_last):
                res = res.contiguous(memory_format=torch.channels_last)
            _ffi.call('esb_conv2d_direct_fwd', x.data_ptr(), w_ohwi.data_ptr(), _ffi.ptr(bias), _ffi.ptr(res), y.data_ptr(),
                      N, H, W, cin, cout, kh, kw, stride, pad, 1 if relu else 0, _ffi.dtype_code(x.dtype), _ffi.stream())
        ctx.save_for_backward(x, w_ohwi, y if relu else None)
        ctx.geom = (stride, pad, relu, res is not None, tma)
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import _ffi
        x, w_ohwi, y = ctx.saved_tensors
        stride, pad, relu, has_res, tma = ctx.geom
        N, cin, H, W = x.shape
        cout, kh, kw, _ = w_ohwi.shape
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        if relu:
            g = torch.empty_like(y)
            _ffi.call('esb_act_bwd', dy.data_ptr(), y.data_ptr(), g.data_ptr(), y.numel(), SP.ACT_RELU,
                      _ffi.dtype_code(y.dtype), _ffi.stream())
        else:
            g = dy
        code = _ffi.dtype_code(x.dtype)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            if tma and stride in (1, 2):
                dx = conv2d_tma_dgrad(g, w_ohwi, (H, W), pad, stride)
            else:
                dx = torch.empty_like(x)
                _ffi.call('esb_conv2d_direct_dgrad', g.data_ptr(), w_ohwi.data_ptr(), dx.data_ptr(), N, H, W, cin, cout, kh,
                          kw, stride, pad, code, _ffi.stream())
        if ctx.needs_input_grad[1]:
            if tma:
                dw = conv2d_tma_wgrad(x, g, (cout, cin, kh, kw), stride, pad)         # (Cout,Cin,kh,kw) view, fp32
            else:
                dwo = torch.zeros((cout, kh, kw, cin), dtype=torch.float32, device=x.device)
                _ffi.call('esb_conv2d_direct_wgrad', x.data_ptr(), g.data_ptr(), dwo.data_ptr(), N, H, W, cin, cout, kh, kw,
                          stride, pad, code, _ffi.stream())
                dw = dwo.permute(0, 3, 1, 2)
            dw = dw.to(x.dtype)
        return dx, dw, None, (g if has_res else None), None, None, None


def maxpool2d(x: torch.Tensor, k: int, stride: int, pad: int) -> torch.Tensor:
    """F.max_pool2d on a channels_last activation with the library's kernel when no gradient flows (the frozen stem)."""
    if (x.is_cuda and x.dtype in (torch.float32, torch.bfloat16) and x.is_contiguous(memory_format=torch.channels_last)
            and not (torch.is_grad_enabled() and x.requires_grad)):
        from . import _ffi
        N, C, H, W = x.shape
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        y = torch.empty((N, C, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        _ffi.call('esb_maxpool2d_nhwc', x.data_ptr(), y.data_ptr(), N, H, W, C, k, stride, pad, _ffi.dtype_code(x.dtype),
                  _ffi.stream())
        return y
    return F.max_pool2d(x, kernel_size=k, stride=stride, padding=pad)


class _ConvBN(nn.Module):
    """Conv2d(bias=False) followed by a BatchNorm2d; evaluated folded when the norm is in eval mode."""

    def __init__(self, cin, cout, k, stride=1, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(cout)
        self._fold_key, self._fold_cache, self._const_w = None, None, {}

    def _folded_constants(self):
        """scale = gamma / sqrt(var + eps) (C,1,1,1) and shift = beta - mean * scale (C,), cached while the frozen BN
        tensors are unchanged (norm_eval + requires_grad=False: they never change during training)."""
        bn = self.bn
        key = (bn.weight._version, bn.bias._version, bn.running_mean._version, bn.running_var._version,
               bn.weight.data_ptr(), bn.weight.device)
        if self._fold_key != key or bn.weight.requires_grad or bn.bias.requires_grad:
            scale = bn.weight * torch.rsqrt(bn.running_var + bn.eps)
            shift = (bn.bias - bn.running_mean * scale).float()
            if bn.weight.requires_grad or bn.bias.requires_grad:
                return scale[:, None, None, None], shift          # trainable affine: keep the autograd graph, no cache
            self._fold_cache = (scale.detach()[:, None, None, None].contiguous(), shift.detach().contiguous())
            self._fold_key = key
            self._const_w = {}
        return self._fold_cache

    def forward(self, x, relu, res=None):
        if x.dtype == torch.float32 and x.is_cuda and torch.backends.cudnn.allow_tf32:
            # fp32 is the parity arithmetic: keep cuDNN out of TF32 (10-bit mantissa breaks the 1e-3 bound)
            with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
                return self._forward(x, relu, res)
        return self._forward(x, relu, res)

    def _forward(self, x, relu, res):
        conv, bn = self.conv, self.bn
        if bn.training:
            y = bn(F.conv2d(x, conv.weight.to(x.dtype), None, conv.stride, conv.padding))
            y = y + res if res is not None else y
            return F.relu(y, inplace=True) if relu else y
        scale4, b = self._folded_constants()
        if conv.weight.requires_grad:
            w = (conv.weight * scale4).to(x.dtype)
        else:                       # frozen stage: the folded bf16/fp32 kernel is a constant too
            w = self._const_w.get(x.dtype)
            if w is None:
                w = self._const_w[x.dtype] = (conv.weight.detach() * scale4).to(x.dtype)
        if (x.is_cuda and x.dtype in (torch.float32, torch.bfloat16) and not b.requires_grad
                and conv.stride[0] == conv.stride[1] and conv.padding[0] == conv.padding[1]):
            # the library's own kernels, all three passes (conv + bias + residual + ReLU fused into one launch)
            if not x.is_contiguous(memory_format=torch.channels_last):
                x = x.contiguous(memory_format=torch.channels_last)
            if w.requires_grad:
                w = w.contiguous(memory_format=torch.channels_last)
            else:
                wc = self._const_w.get(('cl', x.dtype))
                if wc is None:
                    wc = self._const_w[('cl', x.dtype)] = w.contiguous(memory_format=torch.channels_last)
                w = wc
            return _ConvBlock2D.apply(x, w, b, res, relu, conv.stride[0], conv.padding[0])
        y = F.conv2d(x, w, None, conv.stride, conv.padding)
        if y.is_cuda and y.shape[1] % 8 == 0 and y.is_contiguous(memory_format=torch.channels_last):
            return _BiasResAct.apply(y, b, res, SP.ACT_RELU if relu else SP.ACT_NONE)   # bias + residual + ReLU fused
        y = y + b.to(y.dtype).view(1, -1, 1, 1)
        y = y + res if res is not None else y
        return F.relu(y, inplace=True) if relu else y


class _Bottleneck2D(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=False):
        super().__init__()
        self.cb1 = _ConvBN(inplanes, planes, 1)
        self.cb2 = _ConvBN(planes, planes, 3, stride=stride, padding=1)     # style='pytorch': stride on the 3x3
        self.cb3 = _ConvBN(planes, planes * 4, 1)
        self.ds = _ConvBN(inplanes, planes * 4, 1, stride=stride) if downsample else None

    def forward(self, x):
        idt = self.ds(x, False) if self.ds is not None else x
        return self.cb3(self.cb2(self.cb1(x, True), True), True, res=idt)


class _BasicBlock2D(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=False):
        super().__init__()
        self.cb1 = _ConvBN(inplanes, planes, 3, stride=stride, padding=1)
        self.cb2 = _ConvBN(planes, planes, 3, padding=1)
        self.ds = _ConvBN(inplanes, planes, 1, stride=stride) if downsample else None

    def forward(self, x):
        idt = self.ds(x, False) if self.ds is not None else x
        return self.cb2(self.cb1(x, True), True, res=idt)


class _GraphShim(nn.Module):
    """What torch.cuda.make_graphed_callables needs of a module (parameters, buffers, training flag, a patchable forward)
    for ONE input shape of a ResNet, without registering the net as a child (no reference cycle in the module tree)."""

    def __init__(self, net):
        super().__init__()
        self.__dict__['_net'] = net
        self.training = net.training

    def parameters(self, recurse=True):
        return self.__dict__['_net'].parameters(recurse)

    def buffers(self, recurse=True):
        return self.__dict__['_net'].buffers(recurse)

    def forward(self, x):
        return self.__dict__['_net']._forward_impl(x)


# state_dict names follow mmdet/torchvision: conv1/bn1, layer{i}.{j}.conv{k}/bn{k}, downsample.0/.1
_RENAME = {'cb1.conv': 'conv1', 'cb1.bn': 'bn1', 'cb2.conv': 'conv2', 'cb2.bn': 'bn2', 'cb3.conv': 'conv3',
           'cb3.bn': 'bn3', 'ds.conv': 'downsample.0', 'ds.bn': 'downsample.1', 'stem.conv': 'conv1', 'stem.bn': 'bn1'}


@MODELS.register_module(name=['mmdet.ResNet', 'ResNet'])
class ResNet(nn.Module):
    arch_settings = {18: (_BasicBlock2D, (2, 2, 2, 2)), 34: (_BasicBlock2D, (3, 4, 6, 3)),
                     50: (_Bottleneck2D, (3, 4, 6, 3)), 101: (_Bottleneck2D, (3, 4, 23, 3))}

    def __init__(self, depth, in_channels=3, stem_channels=None, base_channels=64, num_stages=4,
                 strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3), style='pytorch',
                 frozen_stages=-1, norm_cfg=None, norm_eval=True, init_cfg=None, **kwargs):
        super().__init__()
        assert style == 'pytorch' and tuple(dilations) == (1, 1, 1, 1)
        block, stage_blocks = self.arch_settings[depth]
        stem_channels = stem_channels or base_channels
        self.out_indices, self.frozen_stages, self.norm_eval = tuple(out_indices), frozen_stages, norm_eval
        self.norm_requires_grad = (norm_cfg or {}).get('requires_grad', True)
        self.stem = _ConvBN(in_channels, stem_channels, 7, stride=2, padding=3)
        inplanes = stem_channels
        self.num_stages = num_stages
        for i in range(num_stages):
            planes = base_channels * 2 ** i
            blocks = []
            for j in range(stage_blocks[i]):
                stride = strides[i] if j == 0 else 1
                ds = j == 0 and (stride != 1 or inplanes != planes * block.expansion)
                blocks.append(block(inplanes, planes, stride=stride, downsample=ds))
                inplanes = planes * block.expansion
            setattr(self, f'layer{i + 1}', nn.Sequential(*blocks))
        self.out_channels = [base_channels * 2 ** i * block.expansion for i in range(num_stages)]
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
        self._freeze()
        self._register_state_dict_hook(ResNet._rename_hook)

    def _freeze(self):
        if not self.norm_requires_grad:
            for m in self.modules():
                if isinstance(m, nn.BatchNorm2d):
                    for p in m.parameters():
                        p.requires_grad = False
        if self.frozen_stages >= 0:
            for p in self.stem.parameters():
                p.requires_grad = False
            for i in range(1, self.frozen_stages + 1):
                for p in getattr(self, f'layer{i}').parameters():
                    p.requires_grad = False

    def train(self, mode=True):
        super().train(mode)
        if mode:
            if self.frozen_stages >= 0:
                self.stem.eval()
                for i in range(1, self.frozen_stages + 1):
                    getattr(self, f'layer{i}').eval()
            if self.norm_eval:
                for m in self.modules():
                    if isinstance(m, nn.BatchNorm2d):
                        m.eval()
        return self

    def forward(self, x):
        if self._graphable(x):
            return self._graphed_forward(x)
        return self._forward_impl(x)

    def _forward_impl(self, x):
        x = self.stem(x, True)
        x = maxpool2d(x, 3, 2, 1)
        outs = []
        for i in range(self.num_stages):
            x = getattr(self, f'layer{i + 1}')(x)
            if i in self.out_indices:
                outs.append(x)
        return tuple(outs)

    # ---- CUDA graphs: the image branch has static shapes (views x H x W), so its ~60 forward launches and ~150 backward
    # launches replay as TWO graph launches per step; the host thread is free for the data-dependent 3D plan (SURVEY §7 H2/H7).
    def _graph_lists(self):
        c = self.__dict__.get('_graph_cache')
        if c is None:        # module / tensor lists are walked once (named_modules costs milliseconds per step otherwise)
            c = self.__dict__['_graph_cache'] = dict(bns=[m for m in self.modules() if isinstance(m, nn.BatchNorm2d)],
                                                     params=list(self.parameters()), buffers=list(self.buffers()))
        return c

    def _graphable(self, x):
        import os
        c = self._graph_lists()
        return (x.is_cuda and self.training and torch.is_grad_enabled() and x.dtype == torch.bfloat16
                and os.environ.get('ESB200_GRAPH2D', '1') != '0'
                and not torch.cuda.is_current_stream_capturing()
                and all(not b.training for b in c['bns']) and any(p.requires_grad for p in c['params']))

    def _graph_signature(self):
        # frozen tensors are baked into the captured constants (folded filters): any in-place change invalidates the graph
        c = self._graph_lists()
        return tuple(t._version for t in c['buffers']) + tuple(p._version for p in c['params'] if not p.requires_grad) \
            + tuple(p.data_ptr() for p in c['params'] if p.requires_grad)

    def _graphed_forward(self, x):
        graphs = self.__dict__.setdefault('_graphs', {})
        key = (tuple(x.shape), x.device.index)
        sig = self._graph_signature()
        entry = graphs.get(key)
        if entry is None or entry[0] != sig:
            if len(graphs) >= 4:
                graphs.clear()
            from . import _ffi
            shim = _GraphShim(self)
            sample = torch.empty_like(x).copy_(x)
            k0 = _ffi.launch_counter['kernels']
            fn = torch.cuda.make_graphed_callables(shim, (sample, ), num_warmup_iters=3, allow_unused_input=True)
            # kernels of one forward + backward pair of the branch (3 warm-up iterations + 1 capture ran through _ffi.call):
            # a replay launches them without passing through Python, so the launch counter is advanced by hand below
            per_pair = (_ffi.launch_counter['kernels'] - k0) // 4
            entry = graphs[key] = (sig, fn, per_pair)
        from . import _ffi
        _ffi.launch_counter['kernels'] += entry[2]
        return entry[1](x)

    # checkpoint compatibility with mmdet / torchvision parameter names: a state-dict hook (not a `state_dict` override,
    # which nn.Module ignores for nested modules) so `detector.state_dict()` carries `backbone.layer1.0.conv1.weight`
    @staticmethod
    def _rename_hook(module, sd, prefix, local_metadata):
        items = list(sd.items())
        sd.clear()                                   # rebuilt in place so the key order is kept
        for k, v in items:
            if k.startswith(prefix):
                tail = k[len(prefix):]
                for a, b in _RENAME.items():
                    tail = tail.replace(a, b)
                k = prefix + tail
            sd[k] = v
        return sd

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        inv = {b: a for a, b in _RENAME.items() if not a.startswith('stem.')}     # stem handled explicitly below
        own = {prefix + k for k, _ in list(self.named_parameters()) + list(self.named_buffers())}
        for k in list(state_dict.keys()):
            if not k.startswith(prefix) or k in own:
                continue
            tail = k[len(prefix):]
            parts = tail.split('.')
            new = None
            if parts[0] in ('conv1', 'bn1') and len(parts) == 2:
                new = 'stem.' + ('conv' if parts[0] == 'conv1' else 'bn') + '.' + parts[1]
            elif parts[0].startswith('layer') and len(parts) >= 4:
                mid = '.'.join(parts[2:-1])
                if mid in inv:
                    new = '.'.join(parts[:2] + [inv[mid], parts[-1]])
            if new is not None:
                state_dict[prefix + new] = state_dict.pop(k)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
