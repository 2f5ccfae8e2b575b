"""GPU: ``inference_scan`` on the grounder, C4-small (max_text_len = 32 tokens) on a small synthetic scan, fp32 and bf16
compute. K prompts share one visual pass and one decoder batch; the reference's test loop (``predict`` on K samples that
each hold the scan and one prompt) runs the visual branch over K scans.

One prompt gives bit for bit what ``predict`` gives on one sample. For K > 1 the visual branch runs at batch size 1 here
and at K there, and two of its operations round differently at the two batch sizes:
* fp32: the cuBLAS GEMMs of ``MinkNeck`` (``sparse.rows_gemm`` of the generative transposed convolution and the class
  projection's ``torch.addmm`` in ``MinkNeck._level``) choose their kernel by row count;
* bf16: ``MinkResNet``'s first ``MinkowskiInstanceNorm`` takes the fused single-pass statistics kernel for a batch of one
  scan (``esb_batchnorm_fwd_fused``) and the segmented two-pass kernel (``esb_norm_fwd``) for several.
``test_batch_size_dependent_ops_are_the_only_difference`` makes those operations batch-size independent and gets the two
routes bit for bit equal. The other tests compare query by query and hold the results to TOL (fp32: the project's fp32
bar; bf16: two bf16 ulps, against a largest difference of 0.34 % measured on these scans). A query is found by its
anchor point: in bf16, near-tied encoder scores may put two of the queries ``pre_decoder`` selects in swapped slots."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for d in (HERE, os.path.join(HERE, 'golden')):
    if d not in sys.path:
        sys.path.insert(0, d)

from ground_inference_util import PROMPTS, grounder, predict_route, scan_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
KW = dict(num_points=2000, points_per_view=1500, seed=5)
DTYPES = {'fp32': torch.float32, 'bf16': torch.bfloat16}
TOL = {torch.float32: 1e-3, torch.bfloat16: 2 ** -7}


@pytest.fixture(scope='module', params=list(DTYPES))
def model(request):
    return grounder(compute_dtype=DTYPES[request.param], device=DEV)


def _run(model, scan, prompts, **kw):
    from embodiedscan_b200.inference import inference_scan
    return inference_scan(model, scan['imgs'], scan['depth'], scan['intrinsic'], scan['extrinsics'], prompts=prompts,
                          **KW, **kw)


def _reference(model, scan, prompts):
    return predict_route(model, *scan_inputs(scan['depth'], scan['extrinsics'], scan['intrinsic'], scan['img_chw'], **KW),
                         prompts)


@pytest.fixture(scope='module')
def scan():
    from embodiedscan_b200.synth import synth_scan
    s = synth_scan(3, n_views=2, H=240, W=320, n_points=2000, device=DEV)
    pm = s['data_sample'].metainfo['depth2img']
    return dict(img_chw=s['img'], imgs=s['img'].permute(0, 2, 3, 1).contiguous(), depth=s['depth'],
                intrinsic=pm['intrinsic'][0], extrinsics=pm['extrinsic'])


class _Counter:
    """Wraps ``model.extract_feat``: the number of calls and the number of scans each call saw."""

    def __init__(self, model):
        self.model, self.fn, self.scans = model, model.extract_feat, []

    def __enter__(self):
        def counted(inputs, samples):
            self.scans.append(len(inputs['points']))
            return self.fn(inputs, samples)
        self.model.extract_feat = counted
        return self

    def __exit__(self, *exc):
        del self.model.extract_feat


def _same(a, b):
    pa, pb = a.pred_instances_3d, b.pred_instances_3d
    return (torch.equal(pa.bboxes_3d.tensor, pb.bboxes_3d.tensor) and torch.equal(pa.scores_3d, pb.scores_3d)
            and torch.equal(pa.target_scores_3d, pb.target_scores_3d))


class _Queries:
    """Records the anchor points of the queries ``pre_decoder`` selects, (K, nq, 3) per call."""

    def __init__(self, model):
        self.model, self.fn, self.coords = model, model.pre_decoder, []

    def __enter__(self):
        def recorded(*args, **kwargs):
            dec_in, head_in = self.fn(*args, **kwargs)
            self.coords.append(dec_in['query_coords'].cpu())
            return dec_in, head_in
        self.model.pre_decoder = recorded
        return self

    def __exit__(self, *exc):
        del self.model.pre_decoder


def _match(mine, theirs):
    """Per prompt, the reference's slot of each query of ours (same anchor point). Near-tied encoder scores may leave
    two queries in swapped slots; both routes must select the same queries."""
    perms = []
    for a, b in zip(mine, theirs):
        slot = {tuple(p): j for j, p in enumerate(b.tolist())}
        assert set(slot) == {tuple(p) for p in a.tolist()}, 'the two routes select different queries'
        perms.append(torch.tensor([slot[tuple(p)] for p in a.tolist()]))
    return perms


def _close(results, ref, perms, tol):
    """Query by query: scores within `tol` relative, box entries within `tol` * max(|b|, 1), and the same ranked query
    wherever the reference scores of the two ranked queries are more than `tol` apart. Returns the largest differences
    and the number of queries in swapped slots."""
    worst = [0., 0., 0]
    for r, q, perm in zip(results, ref, perms):
        a, b = r.pred_instances_3d, q.pred_instances_3d
        sb, bb = b.scores_3d[perm.to(DEV)], b.bboxes_3d.tensor[perm.to(DEV)]      # the reference, in our slots
        ds = ((a.scores_3d - sb).abs() / sb.abs()).max().item()
        db = ((a.bboxes_3d.tensor - bb).abs() / bb.abs().clamp(min=1)).max().item()
        assert ds <= tol and db <= tol, (ds, db, tol)
        assert torch.equal(a.target_scores_3d, a.scores_3d)
        s_ref = sb.cpu().numpy()
        mine = np.argsort(-a.scores_3d.cpu().numpy(), kind='stable')[:10]
        theirs = np.argsort(-s_ref, kind='stable')[:10]
        gap = np.abs(s_ref[mine] - s_ref[theirs])
        assert np.all((mine == theirs) | (gap <= tol * np.abs(s_ref[theirs]))), (mine, theirs)
        worst = [max(worst[0], ds), max(worst[1], db), worst[2] + int((perm != torch.arange(len(perm))).sum())]
    return worst


def _check_ranked(results, ranked, topk):
    for r, (boxes, scores) in zip(results, ranked):
        s = r.pred_instances_3d.scores_3d.cpu().numpy()
        order = np.argsort(-s, kind='stable')[:topk]              # host-side stable descending sort
        assert boxes.is_cuda and scores.is_cuda and boxes.shape == (len(order), 9)
        assert np.array_equal(scores.cpu().numpy(), s[order])
        assert np.array_equal(boxes.cpu().numpy(), r.pred_instances_3d.bboxes_3d.tensor.cpu().numpy()[order])


@pytest.mark.parametrize('K', [1, 3, 12])
def test_shared_visual_pass_equals_predict(model, scan, K):
    prompts = PROMPTS[:K] if K > 1 else [PROMPTS[2]]
    with _Counter(model) as shared, _Queries(model) as q_shared:
        results, ranked = _run(model, scan, prompts)
    with _Counter(model) as per_sample, _Queries(model) as q_ref:
        ref = _reference(model, scan, prompts)
    assert shared.scans == [1] and per_sample.scans == [K], 'one visual pass at B = 1; predict: one pass over K scans'
    assert len(results) == len(ranked) == K
    nq = model.num_queries
    for r, q, p in zip(results, ref, prompts):
        assert r.text == p
        for k in ('img_shape', 'scale_factor', 'ori_shape', 'pad_shape', 'batch_input_shape'):
            assert r.metainfo[k] == q.metainfo[k], k
        assert r.pred_instances_3d.bboxes_3d.tensor.shape == (nq, 9) and r.pred_instances_3d.scores_3d.shape == (nq, )
    if K == 1:
        assert _same(results[0], ref[0])
    else:
        print(f'{model.compute_dtype} K={K}: largest score (relative) and box differences, queries in swapped slots',
              _close(results, ref, _match(q_shared.coords[0], q_ref.coords[0]), TOL[model.compute_dtype]))
    _check_ranked(results, ranked, 10)
    # every query ranked; and the prompts' scores differ, so the prompts reach the prediction
    _check_ranked(results, _run(model, scan, prompts, topk=10 ** 6)[1], nq)
    if K > 1:
        assert not torch.equal(results[0].pred_instances_3d.scores_3d, results[1].pred_instances_3d.scores_3d)


@pytest.mark.parametrize('K', [3, 12])
def test_batch_size_dependent_ops_are_the_only_difference(model, scan, K, monkeypatch):
    """With the fp32 GEMMs computed in fp64 (correctly rounded to fp32 whatever kernel runs them) and a one-scan
    InstanceNorm sent through the segmented kernel, the two routes agree bit for bit at any K."""
    from embodiedscan_b200 import sparse as SP
    rows_gemm, addmm, seg_norm = SP.rows_gemm, torch.addmm, SP.seg_norm

    def rows_gemm64(x, w):
        return (x.double() @ w.double()).float() if x.dtype == torch.float32 else rows_gemm(x, w)

    def addmm64(b, x, w, **kw):
        return (b.double() + x.double() @ w.double()).float() if x.dtype == torch.float32 and not kw else \
            addmm(b, x, w, **kw)

    def seg_norm_segmented(x, gamma, beta, seg_off, row_seg, S, max_rows, eps, act=SP.ACT_NONE, res=None,
                           running_mean=None, running_var=None, momentum=0.1):
        if S == 1 and seg_off is not None and running_mean is None:      # InstanceNorm of one scan: add an empty scan
            seg_off, S = torch.cat([seg_off, seg_off[-1:]]), 2
        return seg_norm(x, gamma, beta, seg_off, row_seg, S, max_rows, eps, act, res, running_mean, running_var, momentum)

    monkeypatch.setattr(SP, 'rows_gemm', rows_gemm64)
    monkeypatch.setattr(torch, 'addmm', addmm64)
    monkeypatch.setattr(SP, 'seg_norm', seg_norm_segmented)
    prompts = PROMPTS[:K]
    results, _ = _run(model, scan, prompts)
    for r, q in zip(results, _reference(model, scan, prompts)):
        assert _same(r, q)


def test_rank_queries_ties():
    from embodiedscan_b200.inference import _rank_queries
    s = torch.tensor([.5, .9, .5, .1, .9, .5, .9], device=DEV)
    assert _rank_queries(s, 10).tolist() == [1, 4, 6, 0, 2, 5, 3]
    assert _rank_queries(s, 4).tolist() == [1, 4, 6, 0]
    g = torch.Generator().manual_seed(0)
    s = torch.randint(0, 6, (5000, ), generator=g).float() / 5           # 6 values over 5000 queries: ties everywhere
    got = _rank_queries(s.to(DEV), 300).cpu().numpy()
    assert np.array_equal(got, np.argsort(-s.numpy(), kind='stable')[:300])


def test_resize_equals_pipeline_route(model):
    """img_scale=(480, 480) on 640x480 frames equals the cv2-resized frames with mmcv Resize's meta: bit for bit for one
    prompt, within TOL for three (see the module docstring)."""
    from embodiedscan_b200.inference import inference_scan
    from embodiedscan_b200.synth import synth_scan
    from oracle import resize_ref as R
    from resize_cases import frames
    V = 3
    s = synth_scan(3, n_views=V, H=480, W=640, n_points=2000, device=DEV)
    pm = s['data_sample'].metainfo['depth2img']
    imgs = frames('scannet_640x480', V)
    imgs_chw = torch.from_numpy(R.resize_linear_u8(imgs, (480, 480))).permute(0, 3, 1, 2).contiguous().to(DEV)
    prompts = PROMPTS[:3]
    with _Queries(model) as q_ref:
        ref = predict_route(model, *scan_inputs(s['depth'], pm['extrinsic'], pm['intrinsic'][0], imgs_chw,
                                                img_shape=(480, 480), scale_factor=(0.75, 1.0), **KW), prompts)
    imgs_dev = torch.from_numpy(imgs).to(DEV)
    with _Queries(model) as q_shared:
        results, ranked = inference_scan(model, imgs_dev, s['depth'], pm['intrinsic'][0], pm['extrinsic'],
                                         img_scale=(480, 480), prompts=prompts, **KW)
    for r in results:
        assert r.metainfo['img_shape'] == (480, 480) and r.metainfo['scale_factor'] == (0.75, 1.0)
    print(f'{model.compute_dtype} resize: largest score (relative) and box differences, queries in swapped slots',
          _close(results, ref, _match(q_shared.coords[0], q_ref.coords[0]), TOL[model.compute_dtype]))
    _check_ranked(results, ranked, 10)
    one, _ = inference_scan(model, imgs_dev, s['depth'], pm['intrinsic'][0], pm['extrinsic'], img_scale=(480, 480),
                            prompts=prompts[:1], **KW)
    assert _same(one[0], predict_route(model, *scan_inputs(s['depth'], pm['extrinsic'], pm['intrinsic'][0], imgs_chw,
                                                           img_shape=(480, 480), scale_factor=(0.75, 1.0), **KW),
                                       prompts[:1])[0])
    # the frames reach the prediction: the native-size route (no Resize) predicts other boxes
    native, _ = inference_scan(model, imgs_dev, s['depth'], pm['intrinsic'][0], pm['extrinsic'], prompts=prompts, **KW)
    assert not all(_same(a, b) for a, b in zip(native, results))
