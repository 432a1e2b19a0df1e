"""transform360_b200: H100-native (sm_90a) implementation of Transform360's projection-remap hot path.

The product is ``lib/libTransform360.so`` (C-ABI of the reference's VideoFrameTransformHandler.h, sm_90a
CUDA kernels inside); this package is its Python binding plus the build script.  No CPU fallback exists.
"""
from .handler import (BORDER_TRANSPARENT, BORDER_WRAP, CUBIC, LANCZOS4, LAYOUT_BARREL, LAYOUT_BARREL_SPLIT, LAYOUT_CUBEMAP_23_OFFCENTER,  # noqa: F401
                      LAYOUT_CUBEMAP_32, LAYOUT_EAC_32, LAYOUT_EQUIRECT, LAYOUT_FLAT_FIXED, LINEAR, NEAREST,
                      STEREO_FORMAT_GUESS, STEREO_FORMAT_LR, STEREO_FORMAT_MONO, STEREO_FORMAT_TB, T360_CAMERA_EQUIDISTANT, T360_CAMERA_PANNINI,
                      T360_CAMERA_EQUIRECT, T360_CAMERA_PINHOLE, T360_CAMERA_STEREOGRAPHIC,
                      FrameTransformContext, HostPlan, T360Camera, T360Lens, T360LensPhotometry, T360Minify, T360LensRig, T360RigPhotometry, T360LensReadout, T360RigMotion, T360Orientation, T360Pose, T360View, VideoFrameTransform, device_count, kernel_launch_count,
                      camera_map, camera_aniso_maps, camera_mip_maps, camera_motion_maps, camera_photo_maps, lens_motion_maps, rig_motion, lens_blend_maps, lens_map, lens_photo_maps, load, make_context, oriented_samples, pose_samples, rectilinear_map, remap_table, stereo_camera_maps,
                      mip_level_sizes, square_pixel_vfov, view_samples, weight_image, deal_lanes)
