"""esb200 — H100-native implementation of the EmbodiedScan multi-view 3D perception hot path.

Host side mirrors the reference's registry / module interface; every hot operator runs in ``libesb200.so``
(hand-written sm_90a CUDA behind the C ABI of ``include/esb200.h``). There is no CPU fallback.
"""
from .registry import MODELS, TASK_UTILS  # noqa: F401
from . import sparse  # noqa: F401
from .backbones import MinkResNet, ResNet  # noqa: F401
from .dense_heads import (BBoxCDLoss, ChamferDistance, FCAF3DHead, FCAF3DHeadRotMat, RotatedIoU3DLoss,  # noqa: F401
                          chamfer_distance, rotated_iou_3d)
from .detectors import Det3DDataPreprocessor, SparseFeatureFusionSingleStage3DDetector  # noqa: F401
from .grounding import GroundingHead, MinkNeck, SparseFeatureFusion3DGrounder  # noqa: F401
from .occupancy import DenseFusionOccPredictor, ImVoxelOccHead, IndoorImVoxelNeck  # noqa: F401
from .structures import Det3DDataSample, EulerDepthInstance3DBoxes, InstanceData  # noqa: F401

__version__ = '0.1.0'
