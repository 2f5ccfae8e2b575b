"""End-to-end parity of the registered detector (built from the reference-shaped config dict) against the CPU oracle
on BASELINE.json config C1 (1-2 scans x 2 views 240x320, 2k points, ResNet-18/16 + MinkResNet14), fp32."""
import numpy as np
import pytest
import torch

# state dicts carry the reference's (mmdet) names; named_parameters() the module structure's
OWN = {'backbone.layer2.0.conv1.weight': 'backbone.layer2.0.cb1.conv.weight'}
pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _setup(n_scans=1, augment=False, variant='C1', seed=0, cls_bias=None):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    from oracle import model_ref as M
    torch.manual_seed(seed)
    cfg = mv_det3d_config(variant)
    model = MODELS.build(cfg).to(DEV)
    if cls_bias is not None:
        with torch.no_grad():
            model.bbox_head.conv_cls.bias.fill_(cls_bias)
    batch = synth_batch(1, n_scans, n_views=2, H=240, W=320, n_points=2000, augment=augment)
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    imgs = M.preprocess_imgs(torch.stack(batch['inputs']['img']), cfg['data_preprocessor']['mean'],
                             cfg['data_preprocessor']['std'])
    return cfg, model, batch, sd, imgs


@pytest.mark.parametrize('n_scans,augment', [(1, False), (2, True)])
def test_loss_and_gradients_match_oracle(n_scans, augment):
    from oracle import model_ref as M
    cfg, model, batch, sd, imgs = _setup(n_scans, augment)
    model.train()
    watch = ['bbox_head.conv_cls.kernel', 'bbox_head.conv_reg.kernel', 'bbox_head.out_block_0.0.kernel',
             'bbox_head.up_block_1.0.kernel', 'backbone_3d.conv1.kernel', 'backbone_3d.layer2.0.conv1.kernel',
             'backbone_3d.layer1.0.norm1.bn.weight', 'backbone.layer2.0.conv1.weight', 'bbox_head.scales.1.scale']
    for k in watch:
        sd[k] = sd[k].clone().requires_grad_(True)
    ref = M.detector_loss(sd, cfg, batch['inputs']['points'], imgs, batch['data_samples'])
    sum(ref.values()).backward()
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    losses = model(**data, mode='loss')
    sum(losses.values()).backward()
    for k in ('loss_center', 'loss_bbox', 'loss_cls'):
        a, b = float(losses[k]), float(ref[k])
        assert abs(a - b) <= 1e-3 * max(abs(b), 1e-3), (k, a, b)
    assert float(ref['loss_bbox']) > 0, 'the scene must contain positives'
    params = dict(model.named_parameters())
    report = {}
    for k in watch:
        g, gr = params[OWN.get(k, k)].grad.cpu(), sd[k].grad
        report[k] = (float((g - gr).abs().max()) / max(float(gr.abs().max()), 1e-9),
                     float((g - gr).norm()) / max(float(gr.norm()), 1e-9))
    print('gradient parity (max-rel, l2-rel):', report)
    for k, (mx, l2) in report.items():
        assert mx <= 2e-3 and l2 <= 2e-3, (k, mx, l2)


def test_predict_matches_oracle():
    from oracle import model_ref as M
    cfg, model, batch, sd, imgs = _setup(1, False)
    # three classes clear the score threshold (the oracle NMS is a scalar python loop), top-50 per level exercises topk
    with torch.no_grad():
        bias = torch.full((284, ), -9.0)
        bias[[3, 77, 200]] = -1.5
        model.bbox_head.conv_cls.bias.copy_(bias.view(1, -1))
        model.bbox_head.conv_cls.kernel.mul_(20.)
        model.bbox_head.conv_center.kernel.mul_(20.)
    sd['bbox_head.conv_cls.bias'] = model.bbox_head.conv_cls.bias.detach().cpu().clone()
    sd['bbox_head.conv_cls.kernel'] = model.bbox_head.conv_cls.kernel.detach().cpu().clone()
    sd['bbox_head.conv_center.kernel'] = model.bbox_head.conv_center.kernel.detach().cpu().clone()
    cfg = dict(cfg, test_cfg=dict(nms_pre=50, iou_thr=.5, score_thr=.01))
    model.bbox_head.test_cfg = cfg['test_cfg']
    model.eval()
    with torch.no_grad():
        ref = M.detector_predict(sd, cfg, batch['inputs']['points'], imgs, batch['data_samples'])
        out = model.val_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']))
    rb, rs, rl = ref[0]
    pred = out[0].pred_instances_3d
    assert rl.numel() > 10, 'the test must exercise NMS'
    assert torch.equal(pred.labels_3d.cpu(), rl), 'NMS selection order must be identical'
    assert float((pred.scores_3d.cpu() - rs).abs().max()) < 1e-4
    box = pred.bboxes_3d.tensor.cpu()
    assert box.shape[1] == 9 and float(box[:, 7:].abs().max()) == 0.0      # 9-DoF -> 7 -> padded back (SURVEY H4)
    assert float((box[:, :7] - rb).abs().max()) <= 1e-3 * float(rb.abs().max())


def test_bf16_step_tracks_fp32():
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    torch.manual_seed(0)
    cfg = mv_det3d_config('C1')
    m32 = MODELS.build(cfg).to(DEV).train()
    m16 = MODELS.build(dict(cfg, compute_dtype=torch.bfloat16)).to(DEV).train()
    m16.load_state_dict(m32.state_dict())
    batch = synth_batch(1, 1, n_views=2, H=240, W=320, n_points=2000)
    out = []
    for m in (m32, m16):
        data = m.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
        out.append({k: float(v) for k, v in m(**data, mode='loss').items()})
    for k in out[0]:
        assert abs(out[0][k] - out[1][k]) <= 0.05 * max(abs(out[0][k]), 1e-2), (k, out)


def test_train_steps_reduce_loss():
    from embodiedscan_b200.engine import OptimWrapper
    cfg, model, batch, sd, imgs = _setup(1, True)
    model.train()
    ow = OptimWrapper(model, lr=1e-3)
    hist = []
    for _ in range(6):
        logs = model.train_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), ow)
        hist.append(float(logs['loss']))
    assert all(np.isfinite(hist)) and hist[-1] < hist[0], hist


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_arena_direct_gradients_equal_autograd(dtype):
    """engine.FlatArena lets the wgrad / BatchNorm-backward kernels accumulate straight into the flat gradient buffer
    (and, in bf16, feeds them the arena's bf16 shadow weights): every gradient must equal the plain autograd path.
    fp32: tight bound (the 2D branch's fp32 atomics differ run to run). bf16: bit-equal, parameter by parameter. The bf16
    step is deterministic, the shadow is the same round-to-nearest cast the plain path makes, and the direct path adds the
    same partials in the same order onto a zeroed slot that autograd's fresh gradient starts from."""
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import FlatArena
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    torch.manual_seed(0)
    cfg = dict(mv_det3d_config('C2' if dtype == torch.bfloat16 else 'C1'), compute_dtype=dtype)
    models = [MODELS.build(cfg).to(DEV).train() for _ in range(3)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    arena = FlatArena(models[2])
    arena.zero_grad()
    batch = synth_batch(1, 2, n_views=2, H=240, W=320, n_points=2000, augment=True)
    losses = []
    for m in models:
        data = m.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
        out = m(**data, mode='loss')
        losses.append(float(sum(out.values()).detach()))
        sum(out.values()).backward()
    assert abs(losses[2] - losses[0]) <= (1e-5 if dtype == torch.float32 else 2e-2) * abs(losses[0])

    def rel_err(ma, mb, check=None):
        num = den = 0.
        for (n1, p1), (n2, p2) in zip(ma.named_parameters(), mb.named_parameters()):
            if p1.grad is None:
                assert not p2.requires_grad or p2.grad is None or float(p2.grad.abs().sum()) == 0.
                continue
            num += float((p1.grad - p2.grad).norm()) ** 2
            den += float(p1.grad.norm()) ** 2
            if check is not None:
                scale = max(float(p1.grad.abs().max()), 1e-8)
                assert float((p1.grad - p2.grad).abs().max()) / scale <= check, n1
        return (num / max(den, 1e-30)) ** 0.5

    if dtype == torch.float32:
        # (2D-backbone gradients pass through fp32 atomics in paint-bwd and cuDNN wgrad: run-to-run noise ~3e-4)
        assert rel_err(models[0], models[2], check=2e-3) <= 1e-3
    else:
        assert losses[2] == losses[0] == losses[1], losses
        differ = []
        for (name, p0), p1, p2 in zip(models[0].named_parameters(), models[1].parameters(), models[2].parameters()):
            if p0.grad is None:
                assert p2.grad is None or not bool(p2.grad.any()), name
                continue
            assert torch.equal(p0.grad, p1.grad), f'{name}: two plain runs differ'
            if not torch.equal(p0.grad, p2.grad):
                differ.append(name)
        assert not differ, f'arena gradients differ from autograd: {differ}'


# ---- occupancy (SURVEY §8 a14): DenseFusionOccPredictor on an 8x8x4 grid against oracle/occ_ref.py -------------------
def _setup_occ(seed=0):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_occ_config, synth_batch, synth_occupancy
    from oracle import model_ref as M
    torch.manual_seed(seed)
    cfg = mv_occ_config('C3-small')
    model = MODELS.build(cfg).to(DEV)
    batch = synth_batch(1, 1, n_views=2, H=240, W=320, n_points=4000)
    for ds in batch['data_samples']:
        ds.gt_occupancy = synth_occupancy(ds, cfg['point_cloud_range'], cfg['n_voxels'])
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    imgs = M.preprocess_imgs(torch.stack(batch['inputs']['img']), cfg['data_preprocessor']['mean'],
                             cfg['data_preprocessor']['std'])
    return cfg, model, batch, sd, imgs


def test_occupancy_loss_and_gradients_match_oracle():
    from oracle import occ_ref as R
    cfg, model, batch, sd, imgs = _setup_occ()
    model.train()
    watch = ['bbox_head.occ.0.weight', 'bbox_head.occ.2.weight', 'neck_3d.down_layer_1.0.conv1.weight',
             'neck_3d.up_block_1.0.weight', 'neck.lateral_convs.0.conv.weight', 'neck.lateral_convs.3.conv.bias',
             'backbone_3d.layer4.0.conv1.kernel', 'backbone_3d.conv1.kernel', 'backbone.layer2.0.conv1.weight']
    for k in watch:
        sd[k] = sd[k].clone().requires_grad_(True)
    ref = R.occ_loss(sd, cfg, batch['inputs']['points'], imgs, batch['data_samples'])
    sum(ref.values()).backward()
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the backward pass reads the global flag
    try:
        losses = model(**data, mode='loss')
        sum(losses.values()).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert int((batch['data_samples'][0].gt_occupancy[:, 3] > 1).sum()) > 0, 'the grid must contain object voxels'
    for k in ('loss_occ_0', 'loss_occ_1', 'loss_occ_2'):
        a, b = float(losses[k]), float(ref[k])
        assert abs(a - b) <= 1e-3 * max(abs(b), 1e-3), (k, a, b)
    params = dict(model.named_parameters())
    report = {}
    for k in watch:
        g, gr = params[OWN.get(k, k)].grad.cpu(), sd[k].grad
        report[k] = (float((g - gr).abs().max()) / max(float(gr.abs().max()), 1e-9),
                     float((g - gr).norm()) / max(float(gr.norm()), 1e-9))
    print('occupancy gradient parity (max-rel, l2-rel):', report)
    for k, (mx, l2) in report.items():
        assert mx <= 5e-3 and l2 <= 5e-3, (k, mx, l2)


def test_occupancy_predict_matches_oracle():
    from oracle import occ_ref as R
    cfg, model, batch, sd, imgs = _setup_occ(seed=1)
    model.eval()
    ref = R.occ_predict(sd, cfg, batch['inputs']['points'], imgs, batch['data_samples'])
    out = model.val_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']))
    pred = out[0].pred_occupancy.cpu()
    assert pred.shape == tuple(cfg['n_voxels'])
    agree = float((pred == ref[0]).float().mean())
    assert agree >= 0.99, agree      # argmax over 81 near-tied random-init logits: allow isolated fp32 tie flips


# ---- grounding (SURVEY §8 a15): SparseFeatureFusion3DGrounder against oracle/ground_ref.py -------------------------
def _setup_ground(seed=0):
    import warnings
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import add_grounding_prompt, mv_grounding_config, synth_batch
    from oracle import model_ref as M
    torch.manual_seed(seed)
    cfg = mv_grounding_config('C4-small')
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        model = MODELS.build(cfg).to(DEV)
    with torch.no_grad():          # the reference zero-initialises the last regression layer: make it informative
        for p in model.bbox_head.reg_branches[0][-1].parameters():
            p.normal_(0, 0.05)
    batch = synth_batch(1, 2, n_views=2, H=240, W=320, n_points=2000)
    for i, ds in enumerate(batch['data_samples']):
        add_grounding_prompt(ds, 1 + 2 * i, seed=i)
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    imgs = M.preprocess_imgs(torch.stack(batch['inputs']['img']), cfg['data_preprocessor']['mean'],
                             cfg['data_preprocessor']['std'])
    return cfg, model, batch, sd, imgs


def test_grounder_loss_and_gradients_match_oracle():
    from oracle import ground_ref as R
    cfg, model, batch, sd, imgs = _setup_ground()
    model.train()
    model.text_encoder.eval()      # RoBERTa's dropout is random in training mode (as in the reference): pin it here
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the backward pass reads the global flag
    try:
        losses = model(**data, mode='loss')
        sum(losses.values()).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    # the text encoder is a library model on both sides: its hidden states are the oracle's input
    with torch.no_grad():
        tok = model.tokenizer.batch_encode_plus([d.text for d in batch['data_samples']], padding='longest').to(DEV)
        hidden = model.text_encoder(**tok).last_hidden_state.float().cpu()
    tmask = tok.attention_mask.bool().cpu()
    pos_maps = [d.gt_instances_3d.positive_maps.cpu() for d in batch['data_samples']]
    watch = ['bbox_head.reg_branches.0.4.weight', 'bbox_head.cls_branches.0.bias', 'text_feat_map.weight',
             'decoder.layers.0.cross_attn.attn.in_proj_weight', 'decoder.layers.1.ffn.layers.1.weight',
             'decoder.cross_posembed.position_embedding_head.0.weight', 'neck_3d.out_block_0.0.kernel',
             'neck_3d.up_block_2.0.kernel', 'backbone_3d.conv1.kernel', 'backbone.layer2.0.conv1.weight']
    for k in watch:
        sd[k] = sd[k].clone().requires_grad_(True)
    for i in range(1, 3):              # shared prediction layers: every index aliases entry 0
        for k in list(sd):
            if k.startswith(f'bbox_head.reg_branches.{i}.') or k.startswith(f'bbox_head.cls_branches.{i}.'):
                sd[k] = sd[k.replace(f'_branches.{i}.', '_branches.0.')]
    ref, ref_inds = R.grounder_loss(sd, cfg, [p.cpu() for p in batch['inputs']['points']], imgs, batch['data_samples'],
                                    hidden, tmask, pos_maps)
    sum(ref.values()).backward()
    assert set(ref) == set(losses)
    for k in ref:
        a, b = float(losses[k].detach()), float(ref[k].detach())
        assert abs(a - b) <= 1e-3 * max(abs(b), 1e-3), (k, a, b)
    params = dict(model.named_parameters())
    report = {}
    for k in watch:
        g, gr = params[OWN.get(k, k)].grad.cpu(), sd[k].grad
        report[k] = (float((g - gr).abs().max()) / max(float(gr.abs().max()), 1e-9),
                     float((g - gr).norm()) / max(float(gr.norm()), 1e-9))
    print('grounding gradient parity (max-rel, l2-rel):', report)
    for k, (mx, l2) in report.items():
        assert mx <= 5e-3 and l2 <= 5e-3, (k, mx, l2)


def test_grounder_predict_matches_oracle():
    from oracle import ground_ref as R
    cfg, model, batch, sd, imgs = _setup_ground(seed=1)
    model.eval()
    out = model.val_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']))
    with torch.no_grad():
        tok = model.tokenizer.batch_encode_plus([d.text for d in batch['data_samples']], padding='longest').to(DEV)
        hidden = model.text_encoder(**tok).last_hidden_state.float().cpu()
    cls, boxes = R.grounder_forward(sd, cfg, [p.cpu() for p in batch['inputs']['points']], imgs, batch['data_samples'],
                                    hidden, tok.attention_mask.bool().cpu(), False)
    for b, ds in enumerate(out):
        ref_scores = cls[-1][b].sigmoid().max(-1)[0]
        assert torch.allclose(ds.pred_instances_3d.scores_3d.cpu(), ref_scores, atol=1e-4)
        assert torch.allclose(ds.pred_instances_3d.bboxes_3d.tensor.cpu(), boxes[-1][b], atol=1e-3, rtol=1e-3)


def test_c2_shaped_bf16_step_matches_oracle():
    """Parity AT THE HEADLINE SHAPE: one C2 scan (20 views 480x640, 100k points, ResNet-50/16 + MinkResNet34) against the fp32
    CPU oracle on the same weights and inputs, through (a) the fp32 parity arithmetic of the CUDA path and (b) the bf16
    throughput path (wgmma / TMA kernels, CUDA-graphed 2D branch, fused BatchNorm).
    Losses: (a) 1e-3, (b) 2e-3 relative (measured 1e-4). Gradients: (a) must match the oracle in direction and size on every
    watched tensor; (b) must match on the head's classifier, whose gradient is well conditioned — deeper tensors are reported
    only: with batch statistics over one scan a round-off perturbation of the weights is amplified ~x300 on its way into the
    gradient (measured on the C1 fixture, tests/test_a_golden_gpu.py), which at bf16's 2^-8 is an O(1) relative change, so the
    first layers' bf16 gradients are noise-dominated at random initialisation (cosine 0.05-0.6 against fp32) while the losses
    agree to 1e-4."""
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    from oracle import model_ref as M
    torch.manual_seed(0)
    cfg = mv_det3d_config('C2')
    m32 = MODELS.build(cfg).to(DEV).train()
    batch = synth_batch(7, 1, n_views=20, H=480, W=640, n_points=100000, augment=True)
    sd = {k: v.detach().cpu().clone().float() for k, v in m32.state_dict().items()}
    watch = ['bbox_head.conv_cls.kernel', 'bbox_head.out_block_0.0.kernel', 'bbox_head.up_block_3.0.kernel',
             'backbone_3d.layer3.0.conv1.kernel', 'backbone_3d.conv1.kernel', 'backbone.layer3.0.conv2.weight']
    own = {'backbone.layer3.0.conv2.weight': 'backbone.layer3.0.cb2.conv.weight'}
    for k in watch:
        sd[k] = sd[k].clone().requires_grad_(True)
    imgs = M.preprocess_imgs(torch.stack(batch['inputs']['img']), cfg['data_preprocessor']['mean'],
                             cfg['data_preprocessor']['std'])
    ref = M.detector_loss(sd, cfg, [p.cpu() for p in batch['inputs']['points']], imgs, batch['data_samples'])
    sum(ref.values()).backward()

    def run(model):
        data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
        losses = model(**data, mode='loss')
        sum(losses.values()).backward()
        rep = {k: (float(losses[k]), float(ref[k])) for k in ref}
        params = dict(model.named_parameters())
        for k in watch:
            g, gr = params[own.get(k, k)].grad.float().cpu().flatten(), sd[k].grad.flatten()
            rep[k] = (float(torch.dot(g, gr) / (g.norm() * gr.norm() + 1e-30)), float(g.norm() / (gr.norm() + 1e-30)))
        return rep

    r32 = run(m32)
    print('C2-shaped fp32 CUDA path vs oracle: losses (cuda, oracle), gradients (cosine, norm ratio):', r32)
    for k in ref:
        assert abs(r32[k][0] - r32[k][1]) <= 1e-3 * max(abs(r32[k][1]), 1e-3), (k, r32)
    for k in watch:
        assert r32[k][0] >= 0.995 and 0.98 <= r32[k][1] <= 1.02, (k, r32)
    m16 = MODELS.build(dict(cfg, compute_dtype=torch.bfloat16)).to(DEV).train()
    m16.load_state_dict(m32.state_dict())
    del m32
    r16 = run(m16)
    print('C2-shaped bf16 path vs oracle: losses (cuda, oracle), gradients (cosine, norm ratio):', r16)
    for k in ref:
        assert abs(r16[k][0] - r16[k][1]) <= 2e-3 * max(abs(r16[k][1]), 1e-3), (k, r16)
    cos, ratio = r16['bbox_head.conv_cls.kernel']
    assert cos >= 0.999 and 0.99 <= ratio <= 1.01, r16
    for k in watch:
        assert np.isfinite(r16[k][0]) and np.isfinite(r16[k][1]), (k, r16)
