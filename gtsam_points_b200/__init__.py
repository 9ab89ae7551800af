"""gtsam_points_b200 -- H100-native (sm_90a) scan-matching linearization behind gtsam_points' factor interface.

Only the hot path of koide3/gtsam_points is implemented here (SURVEY.md section 8): voxel-hash / kd-tree
correspondence search, SE(3) transform, Mahalanobis residual and Jacobians, and the reduction into each factor's
H and b.  The compute lives in lib/libb2points.so (hand-written CUDA, C ABI in include/b2points.h); this package is
the thin host-side mirror of the reference's interface.  There is no CPU fallback.
"""
from . import capi  # noqa: F401
from .capi import B2Error  # noqa: F401
from .factors import (  # noqa: F401
    HessianFactor,
    IntegratedGICPFactor,
    IntegratedICPFactor,
    IntegratedPointToPlaneICPFactor,
    IntegratedMatchingCostFactor,
    IntegratedVGICPFactor,
    IntegratedVGICPFactorGPU,
    NonlinearFactorSetGPU,
    pose_inverse,
)
from .occupancy import FastOccupancyGrid, raycast  # noqa: F401
from .optimize import (GraphOptimizationResult, LevenbergMarquardtExtParams, PoseOptimizationResult, PriorFactorPose3, optimize_graph_gpu,  # noqa: F401
                       optimize_pose_gpu)
from .registration import Features, GNCParams, RANSACParams, RegistrationResult, estimate_fpfh, estimate_pfh, estimate_pose_gnc, estimate_pose_ransac  # noqa: F401
from .segmentation import MinCutParams, MinCutResult, RegionGrowing, RegionGrowingParams, min_cut, region_growing_init, region_growing_update  # noqa: F401
from .types import (  # noqa: F401
    Context,
    GaussianVoxelMapGPU,
    KdTree,
    OffloadableGPU,
    PointCloud,
    current_access_time,
    default_context,
    estimate_covariances,
    estimate_normals,
    find_inlier_points,
    iVox,
    iVoxCovarianceEstimation,
    merge_frames_gpu,
    overlap_gpu,
    random_sampling,
    randomgrid_sampling,
    remove_outliers,
    sample,
    transform_gpu,
    voxelgrid_sampling,
)

__version__ = "0.1.0"
