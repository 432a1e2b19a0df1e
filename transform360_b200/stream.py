"""Frame-stream driver: shards the frames of a stream over the GPUs of one box (SURVEY.md 8e).

One process per GPU (torchrun).  The path has no inter-GPU pixel traffic: rank 0 broadcasts the 112-byte
FrameTransformContext plus the plane dimensions once (NCCL on GPUs, gloo in the CPU tests), every rank
plans locally and then transforms frames k with k mod world_size == rank.  Per-frame work goes through
the product's C-ABI (device-pointer extension for resident frames, the four reference entry points for
host frames).  torch is used for device buffers and torch.distributed only.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import handler as H


@dataclass
class StreamSpec:
    """What a stream needs besides the context: luma size in, luma size out, chroma subsampling shifts."""
    in_w: int
    in_h: int
    out_w: int
    out_h: int
    log2_chroma_w: int = 1
    log2_chroma_h: int = 1
    num_planes: int = 3

    def plane_dims(self, plane: int):
        """(in_w, in_h, out_w, out_h, plan_index) like the reference filter's per-plane loop (vf_transform360.c:368-381)."""
        if plane == 0:
            return self.in_w, self.in_h, self.out_w, self.out_h, 0
        cw, ch = self.log2_chroma_w, self.log2_chroma_h
        r = lambda v, s: -((-v) >> s)  # FF_CEIL_RSHIFT
        return r(self.in_w, cw), r(self.in_h, ch), r(self.out_w, cw), r(self.out_h, ch), 1

    def input_pixels_per_frame(self) -> int:
        return sum(self.plane_dims(p)[0] * self.plane_dims(p)[1] for p in range(self.num_planes))

    def output_pixels_per_frame(self) -> int:
        return sum(self.plane_dims(p)[2] * self.plane_dims(p)[3] for p in range(self.num_planes))

    def to_ints(self):
        return [self.in_w, self.in_h, self.out_w, self.out_h, self.log2_chroma_w, self.log2_chroma_h, self.num_planes]

    @staticmethod
    def from_ints(v):
        return StreamSpec(*[int(x) for x in v])


def bind_to_gpu_numa_node(gpu_index: int):
    """Pins the calling process to the CPUs of the NUMA node the GPU hangs off (PCI sysfs), BEFORE it allocates the
    page-locked frame buffers, so that they are first-touched on that node.  On a 2-socket host a pinned host
    plane on the far socket is DMA'd more slowly than one on the GPU's node, and 8 ranks without affinity fight over the
    inter-socket link.  Returns (node, cpus bound) or None when the topology cannot be read."""
    import os
    import subprocess
    try:
        bus = subprocess.run(["nvidia-smi", "-i", str(gpu_index), "--query-gpu=pci.bus_id", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().lower()
        if bus.startswith("0000"):
            bus = bus[4:]
        base = f"/sys/bus/pci/devices/{bus}/"
        node = int(open(base + "numa_node").read())
        cpus = set()
        for part in open(base + "local_cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if node < 0 or not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return node, len(cpus)
    except Exception:
        return None


def frames_for_rank(num_frames: int, rank: int, world_size: int):
    """Round-robin sharding: frame k goes to GPU k mod N."""
    return range(rank, num_frames, world_size)


def broadcast_parameters(ctx: H.FrameTransformContext | None, spec: StreamSpec | None, rank: int, world_size: int,
                         device="cpu"):
    """Rank 0 holds (ctx, spec); every rank returns identical copies.  The only collective of the path."""
    if world_size == 1:
        return ctx, spec
    import torch
    import torch.distributed as dist
    nbytes = C.sizeof(H.FrameTransformContext)
    payload = torch.zeros(nbytes + 7 * 4, dtype=torch.uint8)
    if rank == 0:
        raw = bytes(ctx) + np.asarray(spec.to_ints(), np.int32).tobytes()
        payload = torch.frombuffer(bytearray(raw), dtype=torch.uint8).clone()
    payload = payload.to(device)
    dist.broadcast(payload, src=0)
    raw = payload.cpu().numpy().tobytes()
    out_ctx = H.FrameTransformContext.from_buffer_copy(raw[:nbytes])
    out_spec = StreamSpec.from_ints(np.frombuffer(raw[nbytes:], np.int32))
    return out_ctx, out_spec


class FrameTransformer:
    """Per-rank worker: one VideoFrameTransform handle with both plans generated (luma, chroma)."""

    def __init__(self, ctx: H.FrameTransformContext, spec: StreamSpec):
        self.ctx, self.spec = ctx, spec
        self.vft = H.VideoFrameTransform(ctx)
        for idx, plane in ((0, 0), (1, 1)):
            if plane >= spec.num_planes:
                break
            iw, ih, ow, oh, _ = spec.plane_dims(plane)
            if not self.vft.generateMapForPlane(iw, ih, ow, oh, idx):
                raise RuntimeError(f"generateMapForPlane failed for plan {idx} (message on stdout)")

    def close(self):
        self.vft.close()

    def _dims(self):
        """(in_w, in_h, out_w, out_h) of every plane, as the frame calls take them."""
        return [self.spec.plane_dims(p)[:4] for p in range(self.spec.num_planes)]

    def frame_call(self, in_planes, out_planes):
        """Prebuilt whole-frame call (T360B200_transformFrameAsync) for one (input, output) buffer pair:
        in_planes / out_planes are per plane (device_address, pitch).  Returns f(stream) -> bool."""
        return self.vft.make_frame_call(in_planes, out_planes, self._dims())

    def view_frame_call(self, in_planes, out_planes):
        """Prebuilt whole-frame call with a per-frame view (T360B200_transformFrameViewAsync, FLAT_FIXED contexts) for one
        (input, output) buffer pair.  Returns f(view, stream) -> bool; view: T360View or (yaw, pitch, hfov, vfov)."""
        return self.vft.make_view_frame_call(in_planes, out_planes, self._dims())

    def oriented_frame_call(self, in_planes, out_planes):
        """Prebuilt whole-frame call with a per-frame orientation (T360B200_transformFrameOrientedAsync: cube-map, EAC and
        equirect outputs) for one (input, output) buffer pair.  Returns f(orientation, stream) -> bool; orientation:
        T360Orientation or (yaw, pitch, roll)."""
        return self.vft.make_oriented_frame_call(in_planes, out_planes, self._dims())

    def pose_frame_call(self, in_planes, out_planes):
        """Prebuilt whole-frame call with a per-frame pose (T360B200_transformFramePoseAsync: every output layout) for one
        (input, output) buffer pair.  Returns f(pose, stream) -> bool; pose: T360Pose or (yaw, pitch, roll, hfov, vfov)."""
        return self.vft.make_pose_frame_call(in_planes, out_planes, self._dims())

    def remap_frame_call(self, in_planes, out_planes, border: int = H.BORDER_WRAP):
        """Prebuilt whole-frame call through per-frame warp maps (T360B200_remapFrameAsync: one device map per plane, the size
        of its output plane) for one (input, output) buffer pair.  Returns f(maps, stream) -> bool; maps: per plane a CUDA
        float32 tensor [out_h][out_w][2], a (device address, pitch) pair or the device address of a dense map."""
        return self.vft.make_remap_frame_call(in_planes, out_planes, self._dims(), border)

    def transform_frame_device(self, in_planes, out_planes, stream: int = 0):
        """in_planes / out_planes: per plane (device_address, pitch).  Asynchronous on `stream`; the planes of
        the frame run concurrently on the transform's internal lanes."""
        if not self.frame_call(in_planes, out_planes)(stream):
            raise RuntimeError("T360B200_transformFrameAsync failed (message on stdout)")

    def transform_frame_host(self, in_planes, out_planes):
        """in_planes / out_planes: per plane (host_address, pitch).  The reference-facing, synchronous path."""
        for p in range(self.spec.num_planes):
            iw, ih, ow, oh, idx = self.spec.plane_dims(p)
            (src, sp), (dst, dp) = in_planes[p], out_planes[p]
            if not self.vft.transformFramePlane(src, dst, iw, ih, sp, ow, oh, dp, idx, p):
                raise RuntimeError("VideoFrameTransform_transformFramePlane failed (message on stdout)")
