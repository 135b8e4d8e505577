"""H100-native (sm_90a) implementation of ORB-SLAM3's per-frame hot path behind the reference's own
ORBextractor / ORBmatcher / Optimizer interfaces.  See DESIGN.md."""
from ._native import OrbError, build, lib, KP_DTYPE  # noqa: F401
from .extractor import ORBextractor  # noqa: F401
from .mappoint import ComputeDistinctiveDescriptors, UpdateNormalAndDepth  # noqa: F401
from .vocabulary import ORBVocabulary, synthetic_vocabulary  # noqa: F401
from .matcher import ORBmatcher, camera, isInFrustum, isInFrustumDevice, knnMatch2  # noqa: F401
from .optimizer import Optimizer, InertialOptimizer, PoseOptimization, PoseOptimizationDevice, PoseEdgesDevice, PoseOptimizationFrames  # noqa: F401
