"""lumixengine_b200 — H100-native implementation of LumixEngine's per-frame ECS hot path.

  culling.CullingSystem      <- src/renderer/culling_system.h:58-77  (CullingSystem::cull on the GPU)
  hierarchy.Hierarchy        <- src/engine/world.cpp:255-282         (World::transformEntity, batched)
  animation.AnimationSystem  <- src/animation/animation_module.cpp:439-472 + pipeline.cpp:2680-2745 + model.cpp:103-137
  sortkeys.SortKeys          <- src/renderer/pipeline.cpp:3789-4144  (createSortKeys + radixSort: the consumer of the visible list)
  clusters.Clusters          <- src/renderer/pipeline.cpp:3327-3684  (fillClusters: light records, atlas candidates, froxel binning)

Everything computes in liblumix_b200.so (hand-written sm_90a CUDA behind the C-ABI of include/lumix_b200.h).
There is no CPU fallback: importing works anywhere, creating a Context without a GPU raises NoDeviceError.
"""
from ._lib import (Context, LumixB200Error, NoDeviceError, PALETTE_DUAL_QUAT, PALETTE_MATRIX, PALETTE_POSE, TYPE_ALL, device_count)  # noqa: F401
from .culling import CullingSystem, CullResult, frustum_from_viewport, frustum_ortho, frustum_perspective  # noqa: F401
from .hierarchy import Hierarchy, TRANSFORM_DTYPE  # noqa: F401
from .animation import AnimationClip, AnimationSystem, SkinnedMesh, Skeleton  # noqa: F401
from .sortkeys import SortKeys, radix_sort  # noqa: F401
from . import sortkeys  # noqa: F401
from .clusters import Clusters  # noqa: F401
