"""What ``inference_scan`` refuses, checked before any device work: prompts on a detector, missing / empty / non-string
/ too long prompts on the grounder, and models that predict no boxes. Plus the query ranking and the token counts of the
test prompts (tests/ground_inference_util.py)."""
import os
import sys
import warnings

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ground_inference_util import PROMPTS, grounder  # noqa: E402

ARGS = (None, None, None, None)
KW = dict(num_points=1, points_per_view=1)


@pytest.fixture(scope='module')
def model():
    return grounder(device='cpu')


def _tokens(model, prompts):
    return model.tokenizer.batch_encode_plus(prompts, padding='longest')['attention_mask'].sum(1).tolist()


def test_prompts_fit_the_head(model):
    assert model.bbox_head.max_text_len == 32
    n = _tokens(model, PROMPTS)
    assert max(n) == 32 and len(set(n[:3])) == 3, n       # the longest fills max_text_len; the first three differ


@pytest.mark.parametrize('prompts, match', [
    (None, 'needs prompts'), ([], 'empty'), ('find the chair', 'not one string'), (['a chair', 7], r'prompts\[1\] is a int'),
    ([PROMPTS[0], 'chair ' * 31], "prompt 'chair chair .* is 33 tokens long.*max_text_len = 32"),
])
def test_grounder_rejects_prompts(model, prompts, match):
    from embodiedscan_b200.inference import inference_scan
    with pytest.raises(ValueError, match=match):
        inference_scan(model, *ARGS, prompts=prompts, **KW)


def test_grounder_rejects_detector_arguments(model):
    from embodiedscan_b200.inference import inference_scan
    with pytest.raises(ValueError, match='not filtered'):
        inference_scan(model, *ARGS, prompts=['a chair'], filter=dict(iou_thr=.5), **KW)
    with pytest.raises(ValueError, match='topk must be >= 1'):
        inference_scan(model, *ARGS, prompts=['a chair'], topk=0, **KW)


def test_detector_rejects_prompts():
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.inference import inference_scan
    from embodiedscan_b200.synth import mv_det3d_config
    det = MODELS.build(mv_det3d_config('C1'))
    for kw in (dict(prompts=['a chair']), dict(topk=5)):
        with pytest.raises(ValueError, match='for the grounder'):
            inference_scan(det, *ARGS, **kw, **KW)


@pytest.mark.parametrize('prompts', [None, ['a chair']])
def test_models_without_boxes(prompts):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.inference import inference_scan
    from embodiedscan_b200.synth import mv_occ_config
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        occ = MODELS.build(mv_occ_config('C3-small'))
    for m in (occ, torch.nn.Linear(1, 1)):
        with pytest.raises(TypeError, match='predicts no boxes'):
            inference_scan(m, *ARGS, prompts=prompts, **KW)


def test_rank_queries():
    from embodiedscan_b200.inference import _rank_queries
    s = torch.tensor([.5, .9, .5, .1, .9, .5, .9])
    assert _rank_queries(s, 10).tolist() == [1, 4, 6, 0, 2, 5, 3]      # ties: lower query index first
    assert _rank_queries(s, 2).tolist() == [1, 4]
