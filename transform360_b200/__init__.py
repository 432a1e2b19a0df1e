"""transform360_b200: H100-native (sm_90a) implementation of Transform360's projection-remap hot path.

The product is ``lib/libTransform360.so`` (C-ABI of the reference's VideoFrameTransformHandler.h, sm_90a
CUDA kernels inside); this package is its Python binding plus the build script.  No CPU fallback exists.
"""
from .handler import (CUBIC, LANCZOS4, LAYOUT_BARREL, LAYOUT_BARREL_SPLIT, LAYOUT_CUBEMAP_23_OFFCENTER,  # noqa: F401
                      LAYOUT_CUBEMAP_32, LAYOUT_EAC_32, LAYOUT_EQUIRECT, LAYOUT_FLAT_FIXED, LINEAR, NEAREST,
                      STEREO_FORMAT_GUESS, STEREO_FORMAT_LR, STEREO_FORMAT_MONO, STEREO_FORMAT_TB,
                      FrameTransformContext, HostPlan, VideoFrameTransform, device_count, kernel_launch_count, load,
                      make_context, remap_table, weight_image, deal_lanes)
