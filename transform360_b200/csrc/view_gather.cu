// sm_90a kernel of the per-frame paths: every plane of a frame in one launch, with the per-frame constants (a view, an
// orientation, a map, a lens rig, a camera) as launch parameters instead of a sampling plan.
//
// One kernel template, perFrameGatherKernel<K, FLAG, Positions>, serves every source (kernels.cuh: PerFrameSource).  Its
// persistent tile loop (gatherViewTiles): a CTA takes tiles of 32 columns x viewTileRows(k) rows over the planes of the
// frame, a thread takes one column of a tile and walks down kViewRowsPerThread rows of it.  The taps go through the
// read-only path with gatherPixel (gather_common.cuh): whole aligned words for interior windows, per-tap wrapping
// (BORDER_WRAP) for windows that cross the seam or a plane edge, or BORDER_TRANSPARENT.  The weight table is staged once
// per CTA (stageWeights).  Where the sources differ is where a pixel's sampling record comes from, the Positions policy:
//   - FLAT_FIXED (FlatPositions): the source column and its phase depend only on the output column (and on the pole fold
//     and the eye), the source row and its phase only on the output row (flat_view.h).  So per tile the CTA computes a
//     column table (32 columns x fold x eye) and a row table (rows x eye) in shared memory and each pixel combines them.
//   - sphere outputs (SpherePositions): the rotation mixes both axes, so every pixel runs the whole chain
//     (oriented_view.h: sphereSample), with the plan's per-column / per-row tables for the view-independent libm steps.
//   - a caller's warp map (MapPositions): the pixel's map entry, quantised by quantizeAxis.
//   - a fisheye lens rig (LensPositions): the output half of the sphere chain, then the lens model (oriented_view.h:
//     lensSample), quantised like a map entry.
//   - a two-lens rig with a feathered seam (LensBlendPositions): both lenses' records and a weight (lensBlendSample); the
//     tile loop gathers the second record only where the weight blends the two.
//   - a camera view (RectilinearPositions): the camera model's ray per pixel (a pinhole launch in a loop of its own),
//     rotated, then the context's input lookup or the lens model (oriented_view.h: rectilinearSample);
//   - an anti-aliased camera view (MipCameraPositions): the same chain, the pixel's footprint from ray differentials, and
//     two records at adjacent levels of the plane's input pyramid, blended by the footprint's weight (mipCameraSample);
//   - a lens rig with photometry (LensPhotoPositions): both lenses' records and gains (lensPhotoSample); the tile loop
//     corrects each sample, combines them by the seam and accumulates the overlap's statistics;
//   - a camera view of a lens rig with photometry (CameraPhotoPositions): the camera view's ray, then both lenses' records,
//     levels and gains (cameraPhotoSample); each lens's sample is the blend of its two levels, then the tile loop goes on
//     as for LensPhotoPositions;
//   - a camera view of a stereo rig (StereoCameraPositions): the same, with the output eye picking the lens;
//   - a lens rig or a camera view of one with photometry and a rig motion over the readout (LensMotionPositions,
//     CameraMotionPositions): the photometric records with each lens's M following the readout time of its point
//     (lensMotionSample, cameraMotionSample);
//   - an anisotropic camera view (AnisoCameraPositions): the anti-aliased view's footprint once per pixel, then up to 16
//     probes along its longer axis, each probe's records at the pixel's two levels (anisoFootprint, anisoCameraSample).
// In all thirteen, the records come from the same host/device functions the planner (or its host twin) uses: bit-identical.
#include "gather_common.cuh"

#include <algorithm>
#include <type_traits>

namespace t360 {
namespace {

// One pixel of record {col0, rowPhase}: its value, or -1 where BORDER_TRANSPARENT leaves it alone
template <int K, bool TRANSPARENT>
__device__ __forceinline__ int viewPixel(const SrcView& s, const unsigned char* smem, int col0, int rowPhase) {
  if constexpr (K == 1) {  // nearest: the rounded position, wrapped like cv::remap's BORDER_WRAP
    if constexpr (TRANSPARENT) {
      const int sx = col0, sy = rowPhase >> 10;
      if ((unsigned)sx >= (unsigned)s.w || (unsigned)sy >= (unsigned)s.h) return -1;
      return __ldg(s.bytes + (size_t)sy * s.pitch + sx);
    } else {
      return __ldg(s.bytes + (size_t)wrapIndex(rowPhase >> 10, s.h) * s.pitch + wrapIndex(col0, s.w));
    }
  } else {
    return gatherPixel<K, TRANSPARENT, 16384>(s, smem, col0, rowPhase);
  }
}

// Level l >= 1 of a plane's pyramid as a source
__device__ __forceinline__ SrcView mipView(const PerFrameGatherParams::MipLevel& l) {
  SrcView s;
  s.bytes = l.bytes;
  s.misalign = (int)(reinterpret_cast<uintptr_t>(l.bytes) & 3);
  s.words = reinterpret_cast<const uint32_t*>(l.bytes - s.misalign);
  s.w = l.w; s.h = l.h; s.pitch = l.pitch;
  return s;
}
// a and b blended by b's weight w (0..256), rounded; where BORDER_TRANSPARENT skipped one of the two (-1) the other stands
// alone, -1 where it skipped both
__device__ __forceinline__ int blendPixels(int a, int b, int w) {
  return a < 0 ? b : (b < 0 ? a : (a * (256 - w) + b * w + 128) >> 8);
}
// Pyramid level `level` of a plane as a source (0: the plane's src s; levels[l - 1]: level l)
__device__ __forceinline__ SrcView levelView(const PerFrameGatherParams::MipLevel* levels, const SrcView& s, int level) {
  return level ? mipView(levels[level - 1]) : s;
}
// A pixel at a level (its view lo) and, where w > 0, at the next one (levels[level]), blended by w (0..255)
template <int K, bool TRANSPARENT>
__device__ __forceinline__ int levelPixel(const SrcView& lo, const PerFrameGatherParams::MipLevel* levels, const unsigned char* smem,
                                          int level, const int32_t* rec0, const int32_t* rec1, int w) {
  int value = viewPixel<K, TRANSPARENT>(lo, smem, rec0[0], rec0[1]);
  if (w > 0) value = blendPixels(value, viewPixel<K, TRANSPARENT>(mipView(levels[level]), smem, rec1[0], rec1[1]), w);
  return value;
}

// TRANSPARENT (barrel layouts): BORDER_TRANSPARENT, a pixel whose anchor tap lies outside the source keeps its byte.
// Positions::kMip: record() returns the pixel's pyramid level and hands over its record there, the record at the next
// level and that level's weight w (0..255); the next level is gathered only where w > 0 (levelPixel).
// Positions::kAniso: footprint() gives the pixel's level, next-level weight w and probe count N = 2^e, and probe() probe
// k's records at those levels, computed in registers as the loop reaches them.  Each probe is gathered as kMip gathers a
// pixel; the pixel is the rounded mean (sum + n / 2) / n of the n probes BORDER_TRANSPARENT does not skip (all N under
// BORDER_WRAP), and keeps its byte where it skips them all.
// Positions::kBlend: its record() hands over two records and the weight w (0..256) of the second; the first is gathered
// for every pixel, the second only where 0 < w < 256, and the two values are blended (PerFrameSource::kLensBlend).
// Positions::kPhoto (the photometric sources): record() hands over both lenses' records, their gains and w, and the
// policy's pixel() gathers a lens's sample from them.  Lens 0 is gathered where w < 256, lens 1 where w > 0, and, with
// statistics, both wherever both cover the pixel; each sample is corrected (photoCorrect) before w combines them (as
// kBlend combines its two values).  A thread sums its overlap pixels' six values over its rows of the tile,
// its warp reduces them (__reduce_add_sync over the warp's live columns), and one lane adds them to the plane's sums with
// one 64-bit atomic each.  Whether statistics are taken and which seam is used are launch-uniform branches.
template <int K, bool TRANSPARENT, class Positions>
__device__ __forceinline__ void gatherViewTiles(const PerFrameGatherParams& p, int numTiles, unsigned char* smem, Positions& pos) {
  constexpr int kRows = viewTileRows(K);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
    const int pl = (p.numPlanes > 2 && tile >= p.plane[2].firstTile) ? 2 : ((p.numPlanes > 1 && tile >= p.plane[1].firstTile) ? 1 : 0);
    const auto& v = p.plane[pl];
    const int t = tile - v.firstTile, ty = t / v.tilesX;
    const int x0 = (t - ty * v.tilesX) * 32, y0 = ty * kRows;
    pos.beginTile(p, v, x0, y0);  // (synchronises the CTA where it builds tables)

    const int j = x0 + lane;
    if (j >= v.geometry.mapW) continue;
    SrcView s;
    s.bytes = v.src;
    s.misalign = (int)(reinterpret_cast<uintptr_t>(v.src) & 3);
    s.words = reinterpret_cast<const uint32_t*>(v.src - s.misalign);
    s.w = v.geometry.inW; s.h = v.geometry.inH; s.pitch = v.srcPitch;
    pos.beginColumn(lane);
    const int r0 = warp * kViewRowsPerThread;
    [[maybe_unused]] uint32_t sums[kPhotoStats] = {};  // (kPhoto: this thread's overlap sums over its rows of the tile)
#pragma unroll 1
    for (int r = r0; r < r0 + kViewRowsPerThread; ++r) {
      const int i = y0 + r;
      if (i >= v.geometry.mapH) break;
      int col0, rowPhase;
      int value;
      if constexpr (Positions::kPhoto) {
        int32_t rec0[2], rec1[2];
        int g0, g1;
        bool overlap;
        const int w = pos.record(p, v, pl, i, j, rec0, rec1, &g0, &g1, &overlap);
        const LensPhotoPlane& c = p.photo.plane[pl];
        const bool stats = p.photo.stats && overlap;
        int a = -1, b = -1;
        if (w < 256 || stats) {
          a = pos.template pixel<K, TRANSPARENT>(p, pl, s, smem, 0, rec0);
          if (a >= 0) a = photoCorrect(a, g0, c.offset[0], c.pivot);
        }
        if (w > 0 || stats) {
          b = pos.template pixel<K, TRANSPARENT>(p, pl, s, smem, 1, rec1);
          if (b >= 0) b = photoCorrect(b, g1, c.offset[1], c.pivot);
        }
        if (stats && a >= 0 && b >= 0) {
          sums[0] += 1; sums[1] += a; sums[2] += b;
          sums[3] += a * a; sums[4] += b * b; sums[5] += a * b;
        }
        value = w == 0 ? a : (w == 256 ? b : blendPixels(a, b, w));
        if (value < 0) continue;
      } else if constexpr (Positions::kMip) {
        int32_t rec0[2], rec1[2];
        int w;
        const int level = pos.record(p, v, pl, i, j, rec0, rec1, &w);
        value = levelPixel<K, TRANSPARENT>(levelView(p.mip[pl].level, s, level), p.mip[pl].level, smem, level, rec0, rec1, w);
        if (TRANSPARENT && value < 0) continue;
      } else if constexpr (Positions::kAniso) {
        const AnisoFootprint f = pos.footprint(p, v, pl, i, j);
        const SrcView lo = levelView(p.mip[pl].level, s, f.level);
        int sum = 0, n = 0;
#pragma unroll 1
        for (int k = 0; k < (1 << f.e); ++k) {
          int32_t rec0[2], rec1[2];
          pos.probe(p, v, pl, f, k, rec0, rec1);
          const int a = levelPixel<K, TRANSPARENT>(lo, p.mip[pl].level, smem, f.level, rec0, rec1, f.w);
          if (a >= 0) {
            sum += a;
            ++n;
          }
        }
        if (TRANSPARENT && n == 0) continue;
        value = (sum + n / 2) / n;
      } else if constexpr (Positions::kBlend) {
        int col1, rowPhase1, w;
        pos.record(p, v, lane, r, i, j, &col0, &rowPhase, &col1, &rowPhase1, &w);
        value = viewPixel<K, TRANSPARENT>(s, smem, col0, rowPhase);
        if (w > 0 && w < 256) value = blendPixels(value, viewPixel<K, TRANSPARENT>(s, smem, col1, rowPhase1), w);
        if (value < 0) continue;
      } else {
        pos.record(p, v, lane, r, i, j, &col0, &rowPhase);
        if constexpr (K == 1 && TRANSPARENT) {  // (nearest: the bounds test skips the store directly, without viewPixel's -1)
          const int sx = col0, sy = rowPhase >> 10;
          if ((unsigned)sx >= (unsigned)s.w || (unsigned)sy >= (unsigned)s.h) continue;
          value = __ldg(s.bytes + (size_t)sy * s.pitch + sx);
        } else {
          value = viewPixel<K, TRANSPARENT>(s, smem, col0, rowPhase);
          if (TRANSPARENT && value < 0) continue;
        }
      }
      v.dst[(size_t)i * v.dstPitch + j] = (uint8_t)value;
    }
    if constexpr (Positions::kPhoto) {
      if (p.photo.stats) {  // (every lane of the warp's live columns gets here: a row bound breaks the whole warp)
        const int live = v.geometry.mapW - x0;
        const unsigned mask = live >= 32 ? 0xffffffffu : (1u << live) - 1u;
        if (__reduce_add_sync(mask, sums[0])) {
          unsigned long long* out = p.photo.stats + pl * kPhotoStats;
#pragma unroll
          for (int k = 0; k < kPhotoStats; ++k) {
            const unsigned total = __reduce_add_sync(mask, sums[k]);
            if (lane == 0) atomicAdd(out + k, (unsigned long long)total);
          }
        }
      }
    }
  }
}

// The policies below take K and the launch's compile-time flag (launchPerFrameGather) as template arguments.  kTransparent:
// BORDER_TRANSPARENT instead of BORDER_WRAP.  kTableBytes: the shared memory of the per-tile tables, after the weights.

// Positions without per-tile tables
struct NoTables {
  static constexpr int kTableBytes = 0;
  static constexpr bool kBlend = false, kMip = false, kAniso = false, kPhoto = false;
  __device__ explicit NoTables(unsigned char*) {}
  __device__ void beginTile(const PerFrameGatherParams&, const PerFramePlane&, int, int) {}
  __device__ void beginColumn(int) {}
};

// FLAT_FIXED: per-tile column and row tables in shared memory, after the weights
template <int K, bool>
struct FlatPositions {
  static constexpr int kRows = viewTileRows(K);
  static constexpr int kTableBytes = 4 * 32 * (int)sizeof(FlatColumn) + 2 * kRows * (int)sizeof(FlatRow) + 32;
  static constexpr bool kBlend = false, kMip = false, kAniso = false, kPhoto = false, kTransparent = false;
  FlatColumn* colTab;  // [eye][fold][32]
  FlatRow* rowTab;     // [column eye][kRows]
  bool* colEye;        // [32]
  const FlatRow* rows;
  __device__ explicit FlatPositions(unsigned char* tables)
      : colTab(reinterpret_cast<FlatColumn*>(tables)), rowTab(reinterpret_cast<FlatRow*>(colTab + 4 * 32)),
        colEye(reinterpret_cast<bool*>(rowTab + 2 * kRows)), rows(nullptr) {}
  __device__ void beginTile(const PerFrameGatherParams& p, const PerFramePlane& v, int x0, int y0) {
    const SphereGeometry& g = v.geometry;
    __syncthreads();  // (the previous tile's tables have been read; the first time: the weights are staged)
    for (int e = threadIdx.x; e < 4 * 32 + 2 * kRows + 32; e += blockDim.x) {
      if (e < 4 * 32) {
        const int j = x0 + (e & 31);
        if (j < g.mapW) colTab[e] = flatColumn(p.view, g, j, (e >> 5) & 1, e >> 6);
      } else if (e < 4 * 32 + 2 * kRows) {
        const int r = e - 4 * 32, i = y0 + r % kRows;
        if (i < g.mapH) rowTab[r] = flatRow(p.view, g, i, r >= kRows);
      } else {
        const int j = x0 + e - (4 * 32 + 2 * kRows);
        colEye[j - x0] = j < g.mapW && flatColumnEye(g, j);
      }
    }
    __syncthreads();
  }
  __device__ void beginColumn(int lane) { rows = rowTab + (colEye[lane] ? kRows : 0); }
  __device__ void record(const PerFrameGatherParams&, const PerFramePlane&, int lane, int r, int, int, int* col0, int* rowPhase) const {
    const FlatRow row = rows[r];
    const FlatColumn c = colTab[(row.eye ? 64 : 0) + (row.fold ? 32 : 0) + lane];
    *col0 = c.col0;
    *rowPhase = row.rowPart + c.fracX;
  }
};

// Sphere and barrel outputs (BARREL: the barrel layouts' positions and BORDER_TRANSPARENT): the whole chain per pixel
template <int, bool BARREL>
struct SpherePositions : NoTables {
  static constexpr bool kTransparent = BARREL;
  using NoTables::NoTables;
  __device__ void record(const PerFrameGatherParams& p, const PerFramePlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    sphereSample<BARREL>(v.geometry, p.rotation, v.colTable, v.rowTable, i, j, col0, rowPhase);
  }
};

// A caller's warp map: the pixel's (x, y) from the map (a warp's lanes read 32 consecutive entries of a row: one coalesced
// 256-byte load), quantised as quantizeWarpMap quantises a planned map, NaN, infinities and out-of-range values included.
// TRANSPARENT: the caller's border, BORDER_TRANSPARENT instead of BORDER_WRAP
template <int K, bool TRANSPARENT>
struct MapPositions : NoTables {
  static constexpr bool kTransparent = TRANSPARENT;
  using NoTables::NoTables;
  __device__ void record(const PerFrameGatherParams&, const PerFramePlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    const float2 m = __ldg(v.map + (size_t)i * v.mapPitch + j);
    int row0, fracX, fracY;
    quantizeAxis(m.x, K, col0, &fracX);
    quantizeAxis(m.y, K, &row0, &fracY);
    *rowPhase = row0 * 1024 + fracY * 32 + fracX;
  }
};

// A fisheye lens rig: the whole chain per pixel; BARREL: the barrel layouts' positions (dead zones included); always
// BORDER_TRANSPARENT
template <int, bool BARREL>
struct LensPositions : NoTables {
  static constexpr bool kTransparent = true;
  using NoTables::NoTables;
  __device__ void record(const PerFrameGatherParams& p, const PerFramePlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    lensSample<BARREL>(v.geometry, p.rotation, p.rig, v.colTable, v.rowTable, i, j, col0, rowPhase);
  }
};

// A two-lens rig with a feathered seam: both lenses' records and lens 1's weight per pixel (lensBlendSample).  The first
// record is the lens that carries the pixel: lens 1 where w = 256, lens 0 everywhere else (also where neither lens covers
// the pixel: its NaN record is skipped by BORDER_TRANSPARENT).  So a warp gathers twice only for its belt pixels.
template <int, bool BARREL>
struct LensBlendPositions : NoTables {
  static constexpr bool kBlend = true, kTransparent = true;
  using NoTables::NoTables;
  __device__ void record(const PerFrameGatherParams& p, const PerFramePlane& v, int, int, int i, int j, int* col0, int* rowPhase, int* col1,
                         int* rowPhase1, int* w) const {
    int32_t rec0[2], rec1[2];
    *w = lensBlendSample<BARREL>(v.geometry, p.rotation, p.rig, p.seamScale, v.colTable, v.rowTable, i, j, rec0, rec1);
    *col0 = *w == 256 ? rec1[0] : rec0[0];
    *rowPhase = *w == 256 ? rec1[1] : rec0[1];
    *col1 = rec1[0];
    *rowPhase1 = rec1[1];
  }
};

// A camera view: the camera model's ray, the rotation and the input lookup per pixel, no tables.  LENS: the rig's lenses
// (rectilinearSample<true>) with BORDER_TRANSPARENT instead of the context's input with BORDER_WRAP.  ANY_MODEL = false:
// the launch's camera is a pinhole.
template <bool LENS, bool ANY_MODEL>
struct CameraPositions : NoTables {
  static constexpr bool kTransparent = LENS;
  using NoTables::NoTables;
  __device__ void record(const PerFrameGatherParams& p, const PerFramePlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    rectilinearSample<LENS, ANY_MODEL>(v.geometry, p.camera, p.rig, i, j, col0, rowPhase);
  }
};
// The kernel runs a pinhole launch (the rectilinear views) through its own tile loop, Pinhole, so the model switch costs
// those views nothing per pixel; the other models take the loop with the switch.
template <int, bool LENS>
struct RectilinearPositions : CameraPositions<LENS, true> {
  using Pinhole = CameraPositions<LENS, false>;
  using CameraPositions<LENS, true>::CameraPositions;
};
// An anti-aliased camera view (kCameraMip): the camera view's chain and the pixel's footprint (mipCameraSample) give its
// pyramid level, its record there and, where the next level has weight, the record at the next level.  Every model in one
// loop (no pinhole loop of its own).  LENS as for CameraPositions.
template <int, bool LENS>
struct MipCameraPositions : NoTables {
  static constexpr bool kMip = true, kTransparent = LENS;
  using NoTables::NoTables;
  __device__ int record(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j, int32_t* rec0, int32_t* rec1,
                        int* w) const {
    return mipCameraSample<LENS>(v.geometry, p.camera, p.rig, p.mip[pl].geometry, p.mipBias, i, j, rec0, rec1, w);
  }
};

// An anisotropic camera view (kCameraAniso): MipCameraPositions' chain, footprint and levels, with the footprint's probe
// count from cameraAniso (log2 maxProbes).  footprint() takes the centre ray's footprint (anisoFootprint), probe() one
// probe's records (anisoCameraSample).  LENS as for CameraPositions.
template <int, bool LENS>
struct AnisoCameraPositions : NoTables {
  static constexpr bool kAniso = true, kTransparent = LENS;
  using NoTables::NoTables;
  __device__ AnisoFootprint footprint(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j) const {
    return anisoFootprint<LENS>(v.geometry, p.camera, p.rig, p.mip[pl].geometry, p.mipBias, p.cameraAniso, i, j);
  }
  __device__ void probe(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, const AnisoFootprint& f, int k, int32_t* rec0,
                        int32_t* rec1) const {
    anisoCameraSample<LENS>(v.geometry, p.camera, p.rig, p.mip[pl].geometry, f, k, rec0, rec1);
  }
};

// A lens rig with photometry (kLensPhoto): both lenses' records, their gains, the overlap and w per pixel
// (lensPhotoSample); BARREL as for LensPositions.  With the hard seam and no statistics only the closer lens is projected.
template <int, bool BARREL>
struct LensPhotoPositions : NoTables {
  static constexpr bool kPhoto = true, kTransparent = true;
  using NoTables::NoTables;
  __device__ int record(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j, int32_t* rec0, int32_t* rec1, int* g0,
                        int* g1, bool* overlap) const {
    return lensPhotoSample<BARREL>(v.geometry, p.rotation, p.rig, p.seamScale, p.photo.stats != nullptr, p.photo.plane[pl], v.colTable,
                                   v.rowTable, i, j, rec0, rec1, g0, g1, overlap);
  }
  template <int K, bool TRANSPARENT>
  __device__ int pixel(const PerFrameGatherParams&, int, const SrcView& s, const unsigned char* smem, int, const int32_t* rec) const {
    return viewPixel<K, TRANSPARENT>(s, smem, rec[0], rec[1]);
  }
};

// A camera view of a lens rig with photometry (kCameraPhoto): the camera view's ray, then both lenses' records, levels and
// gains, the overlap and w per pixel (cameraPhotoSample).  record() keeps each lens's records, level and level weight in
// the policy, and pixel() gathers lens l's sample from them: the blend of its two levels (levelPixel).  MIP = false: no
// pyramid, level 0 alone (a launch whose planes all have top level 0).  Every model in one loop; always
// BORDER_TRANSPARENT.  With the hard seam and no statistics only the closer lens is projected.
template <int, bool MIP>
struct CameraPhotoPositions : NoTables {
  static constexpr bool kPhoto = true, kTransparent = true;
  CameraPhotoRecords lens[2];
  using NoTables::NoTables;
  __device__ int record(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j, int32_t*, int32_t*, int* g0, int* g1,
                        bool* overlap) {
    const int w = cameraPhotoSample<MIP>(v.geometry, p.camera, p.rig, p.mip[pl].geometry, p.mipBias, p.seamScale, p.photo.stats != nullptr,
                                         p.photo.plane[pl], i, j, lens, overlap);
    *g0 = lens[0].gain;
    *g1 = lens[1].gain;
    return w;
  }
  template <int K, bool TRANSPARENT>
  __device__ int pixel(const PerFrameGatherParams& p, int pl, const SrcView& s, const unsigned char* smem, int l, const int32_t*) const {
    const CameraPhotoRecords& r = lens[l];
    if constexpr (MIP) {
      return levelPixel<K, TRANSPARENT>(levelView(p.mip[pl].level, s, r.level), p.mip[pl].level, smem, r.level, r.rec0, r.rec1, r.w);
    } else {
      return viewPixel<K, TRANSPARENT>(s, smem, r.rec0[0], r.rec0[1]);
    }
  }
};

// A camera view of a stereo rig (kStereoCamera): CameraPhotoPositions with the output eye's lens in place of the closer
// lens (cameraPhotoSample<MIP, true>): eye e's pixels gather lens e alone, and with statistics the other lens too.  The
// launch's seamScale is 0.
template <int K, bool MIP>
struct StereoCameraPositions : CameraPhotoPositions<K, MIP> {
  using CameraPhotoPositions<K, MIP>::CameraPhotoPositions;
  __device__ int record(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j, int32_t*, int32_t*, int* g0, int* g1,
                        bool* overlap) {
    CameraPhotoRecords* lens = this->lens;
    const int w = cameraPhotoSample<MIP, true>(v.geometry, p.camera, p.rig, p.mip[pl].geometry, p.mipBias, 0.0f, p.photo.stats != nullptr,
                                               p.photo.plane[pl], i, j, lens, overlap);
    *g0 = lens[0].gain;
    *g1 = lens[1].gain;
    return w;
  }
};

// A lens rig with photometry and a rig motion (kLensMotion): LensPhotoPositions with each lens's M following the readout
// time of the point it projects (lensMotionSample).  The motion's sample table is read with read-only global loads: at
// most 1152 bytes and the same for every pixel of the launch, it stays in L1 (DESIGN.md section 5).
template <int K, bool BARREL>
struct LensMotionPositions : LensPhotoPositions<K, BARREL> {
  using LensPhotoPositions<K, BARREL>::LensPhotoPositions;
  __device__ int record(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j, int32_t* rec0, int32_t* rec1, int* g0,
                        int* g1, bool* overlap) const {
    return lensMotionSample<BARREL>(v.geometry, p.rotation, p.rig, p.motion, p.seamScale, p.photo.stats != nullptr, p.photo.plane[pl],
                                    v.colTable, v.rowTable, i, j, rec0, rec1, g0, g1, overlap);
  }
};

// A camera view of a lens rig with photometry and a rig motion (kCameraMotion): CameraPhotoPositions' levels and pixel
// blend, the records from cameraMotionSample.  The table as for LensMotionPositions.
template <int K, bool MIP>
struct CameraMotionPositions : CameraPhotoPositions<K, MIP> {
  using CameraPhotoPositions<K, MIP>::CameraPhotoPositions;
  __device__ int record(const PerFrameGatherParams& p, const PerFramePlane& v, int pl, int i, int j, int32_t*, int32_t*, int* g0, int* g1,
                        bool* overlap) {
    CameraPhotoRecords* lens = this->lens;
    const int w = cameraMotionSample<MIP>(v.geometry, p.camera, p.rig, p.motion, p.mip[pl].geometry, p.mipBias, p.seamScale,
                                          p.photo.stats != nullptr, p.photo.plane[pl], i, j, lens, overlap);
    *g0 = lens[0].gain;
    *g1 = lens[1].gain;
    return w;
  }
};

template <class Pos, class = void>
struct HasPinholeLoop : std::false_type {};
template <class Pos>
struct HasPinholeLoop<Pos, std::void_t<typename Pos::Pinhole>> : std::true_type {};

// The weights are staged first.  A policy with per-tile tables publishes them with its first beginTile __syncthreads;
// without tables no tile synchronises, so the kernel does it here.
template <int K, bool FLAG, template <int, bool> class Positions>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4)
perFrameGatherKernel(const __grid_constant__ PerFrameGatherParams p, int numTiles) {
  using Pos = Positions<K, FLAG>;
  extern __shared__ __align__(16) unsigned char smem[];
  Pos pos(smem + (K >= 2 ? weightBytes<K>() : 0));
  if constexpr (K >= 2) {
    stageWeights<K>(p.weights, smem);
    if constexpr (Pos::kTableBytes == 0) __syncthreads();
  }
  if constexpr (HasPinholeLoop<Pos>::value) {
    if (p.camera.model == kCameraPinhole) {
      typename Pos::Pinhole pinhole(smem + (K >= 2 ? weightBytes<K>() : 0));
      gatherViewTiles<K, Pos::kTransparent>(p, numTiles, smem, pinhole);
      return;
    }
  }
  gatherViewTiles<K, Pos::kTransparent>(p, numTiles, smem, pos);
}

// Positions<K, FLAG> for K = p.kernelSize, one CTA per tile up to the occupancy the __launch_bounds__ allow; its shared
// memory is the weight table and the policy's per-tile tables.  flag: a bool, or std::false_type where the source has no
// flag (one instantiation per K)
template <template <int, bool> class Positions, class Flag>
cudaError_t launchPositions(const PerFrameGatherParams& p, Flag flag, int numTiles, int numSMs, cudaStream_t stream) {
  auto launch = [&](auto k, auto f) {
    constexpr int K = decltype(k)::value;
    constexpr auto Kern = perFrameGatherKernel<K, decltype(f)::value, Positions>;
    static DeviceLaunchCfg cfgs;  // per kernel instantiation, one entry per device
    constexpr int threads = gatherThreads(K);
    constexpr int smemBytes = (K >= 2 ? weightBytes<K>() : 0) + Positions<K, decltype(f)::value>::kTableBytes;
    LaunchCfg cfg;
    cudaError_t err = prepare<Kern>(cfgs, threads, smemBytes, cfg);
    if (err != cudaSuccess) return err;
    const int grid = std::min(numSMs * cfg.perSM, numTiles);
    Kern<<<grid, threads, smemBytes, stream>>>(p, numTiles);
    gLaunches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
  };
  auto withFlag = [&](auto k) {
    if constexpr (std::is_same_v<Flag, bool>) return flag ? launch(k, std::true_type{}) : launch(k, std::false_type{});
    else return launch(k, flag);
  };
  switch (p.kernelSize) {
    case 1: return withFlag(std::integral_constant<int, 1>{});
    case 2: return withFlag(std::integral_constant<int, 2>{});
    case 4: return withFlag(std::integral_constant<int, 4>{});
    case 8: return withFlag(std::integral_constant<int, 8>{});
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t launchPerFrameGather(PerFrameGatherParams p, PerFrameSource source, int numSMs, cudaStream_t stream) {
  if (p.numPlanes < 1 || p.numPlanes > kMaxFramePlanes) return cudaErrorInvalidValue;
  // tiles of every plane, in plane order
  const int rows = viewTileRows(p.kernelSize);
  int numTiles = 0;
  for (int i = 0; i < p.numPlanes; ++i) {
    PerFramePlane& v = p.plane[i];
    v.tilesX = (v.geometry.mapW + 31) / 32;
    v.firstTile = numTiles;
    numTiles += v.tilesX * ((v.geometry.mapH + rows - 1) / rows);
  }
  if (numTiles <= 0) return cudaSuccess;
  const bool barrel = barrelLayout(p.plane[0].geometry.outputLayout);
  switch (source) {
    case PerFrameSource::kView: return launchPositions<FlatPositions>(p, std::false_type{}, numTiles, numSMs, stream);
    case PerFrameSource::kSphere: return launchPositions<SpherePositions>(p, barrel, numTiles, numSMs, stream);
    case PerFrameSource::kMap: return launchPositions<MapPositions>(p, p.transparent, numTiles, numSMs, stream);
    case PerFrameSource::kLens: return launchPositions<LensPositions>(p, barrel, numTiles, numSMs, stream);
    case PerFrameSource::kLensBlend: return launchPositions<LensBlendPositions>(p, barrel, numTiles, numSMs, stream);
    case PerFrameSource::kRectilinear: return launchPositions<RectilinearPositions>(p, p.lens, numTiles, numSMs, stream);
    case PerFrameSource::kCameraMip: return launchPositions<MipCameraPositions>(p, p.lens, numTiles, numSMs, stream);
    case PerFrameSource::kCameraAniso: return launchPositions<AnisoCameraPositions>(p, p.lens, numTiles, numSMs, stream);
    case PerFrameSource::kLensPhoto: return launchPositions<LensPhotoPositions>(p, barrel, numTiles, numSMs, stream);
    case PerFrameSource::kLensMotion: return launchPositions<LensMotionPositions>(p, barrel, numTiles, numSMs, stream);
    case PerFrameSource::kCameraPhoto:
    case PerFrameSource::kStereoCamera:
    case PerFrameSource::kCameraMotion: {
      bool mip = false;  // (a level table only where some plane has a pyramid)
      for (int i = 0; i < p.numPlanes; ++i) mip = mip || p.mip[i].geometry.top > 0;
      if (source == PerFrameSource::kStereoCamera) return launchPositions<StereoCameraPositions>(p, mip, numTiles, numSMs, stream);
      if (source == PerFrameSource::kCameraMotion) return launchPositions<CameraMotionPositions>(p, mip, numTiles, numSMs, stream);
      return launchPositions<CameraPhotoPositions>(p, mip, numTiles, numSMs, stream);
    }
  }
  return cudaErrorInvalidValue;
}

}  // namespace t360
