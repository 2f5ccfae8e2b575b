"""What the grounding inference tests and tests/ground_inference_bench.py share: the grounder, the prompts, and the
reference's route, where every (scan, prompt) pair is a sample of its own and ``predict`` runs the visual branch for each."""
import warnings

import numpy as np
import torch

# SimpleTokenizer counts one token per word or punctuation mark, plus <s> and </s>: token lengths 6, 11, 16, 32, 5, ...;
# the 30-word prompt fills C4-small's max_text_len = 32 exactly
PROMPTS = ['find the chair.',
           'the lamp that is close to the wall.',
           'the table between the sofa and the shelf, next to the window.',
           ' '.join(['chair', 'table', 'lamp', 'sofa', 'shelf', 'box'] * 5),
           'a box.', 'the monitor on the desk.', 'the plant near the door, left of the bed.', 'the cabinet.',
           'the bed', 'the shelf above the box on the floor.', 'sofa', 'the big lamp in the corner of the room.']


def grounder(variant='C4-small', compute_dtype=torch.float32, device='cuda:0', seed=0):
    """The grounder in eval mode. The last regression layer, which the reference initialises to zero, is drawn at random
    so that the queries' boxes differ."""
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_grounding_config
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')       # the random-init text encoder warns that the RoBERTa files are absent
        model = MODELS.build(dict(mv_grounding_config(variant), compute_dtype=compute_dtype))
    with torch.no_grad():
        for p in model.bbox_head.reg_branches[0][-1].parameters():
            p.normal_(0, 0.05)
    return model.to(device).eval()


def scan_inputs(depth, extrinsics, intrinsic, img_chw, *, num_points, points_per_view, seed, img_shape=None,
                scale_factor=(1.0, 1.0)):
    """A scan the way the configs' test pipeline builds it: seeded ``MultiViewDepthToPoints`` points, (V,3,h,w) uint8
    frames as given, and the scan's metainfo. Returns ``(points, img_chw, meta)``."""
    from embodiedscan_b200.structures import EulerDepthInstance3DBoxes
    from embodiedscan_b200.transforms import MultiViewDepthToPoints
    V, H, W = depth.shape
    K = np.asarray(intrinsic, dtype=np.float32)
    K4 = np.eye(4, dtype=np.float32)
    K4[:K.shape[0], :K.shape[1]] = K
    extr = [np.asarray(e, dtype=np.float32).reshape(4, 4) for e in extrinsics]
    meta = dict(img_shape=(H, W) if img_shape is None else img_shape, ori_shape=(H, W), scale_factor=scale_factor,
                flip=False, transformation_3d_flow=[],
                depth2img=dict(extrinsic=extr, intrinsic=[K4] * V, origin=np.array([.0, .0, .5], dtype=np.float32)),
                box_type_3d=EulerDepthInstance3DBoxes)
    points = MultiViewDepthToPoints(num_points, points_per_view, seed=seed)(
        dict(depth_imgs=depth, depth2img=meta['depth2img']))['points']
    return points, img_chw, meta


def predict_route(model, points, img_chw, meta, prompts):
    """The reference's test loop: one sample per prompt, each holding the same scan, through ``data_preprocessor`` and
    ``model.forward(mode='predict')`` as one batch of K samples. Each sample names its whole prompt as its phrase, as
    ``inference_scan`` does: ``predict`` needs a ``tokens_positive``."""
    from embodiedscan_b200.structures import Det3DDataSample, InstanceData
    samples = []
    for p in prompts:
        ds = Det3DDataSample(metainfo=meta)
        ds.text = p
        ds.tokens_positive = [[[0, len(p)]]]
        ds.gt_instances_3d = InstanceData()
        samples.append(ds)
    K = len(prompts)
    with torch.no_grad():
        data = model.data_preprocessor(dict(inputs=dict(points=[points] * K, img=[img_chw] * K), data_samples=samples),
                                       False)
        return model(**data, mode='predict')
