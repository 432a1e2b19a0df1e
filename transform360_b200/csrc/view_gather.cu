// sm_90a kernels of the per-frame paths: every plane of a frame in one launch, with the view (FLAT_FIXED) or the
// orientation (cube maps, EAC, equirect, barrel) as a launch parameter instead of a sampling plan.
//
// Both share one persistent tile loop (gatherViewTiles): a CTA takes tiles of 32 columns x viewTileRows(k) rows over the
// planes of the frame, a thread takes one column of a tile and walks down kViewRowsPerThread rows of it.  The taps go
// through the read-only path with gatherPixel (gather_common.cuh): whole aligned words for interior windows, per-tap
// wrapping (BORDER_WRAP) for windows that cross the seam or a plane edge, or BORDER_TRANSPARENT for the barrel layouts.  The
// weight table is staged once per CTA (stageWeights).  Where the kernels differ is where a pixel's sampling record comes
// from:
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
//   - a rectilinear view (RectilinearPositions): a pinhole ray per pixel, rotated, then the context's input lookup or the
//     lens model (oriented_view.h: rectilinearSample).
// In all six, the records come from the same host/device functions the planner (or its host twin) uses: bit-identical.
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

// TRANSPARENT (barrel layouts): BORDER_TRANSPARENT, a pixel whose anchor tap lies outside the source keeps its byte.
// Positions::kBlend: its record() hands over two records and the weight w (0..256) of the second; the first is gathered
// for every pixel, the second only where 0 < w < 256, and the two values are blended (LensBlendGatherParams).  Where
// BORDER_TRANSPARENT skips one of the two, the other stands alone.
template <int K, bool TRANSPARENT, class Params, class Positions>
__device__ __forceinline__ void gatherViewTiles(const Params& p, int numTiles, unsigned char* smem, Positions& pos) {
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
#pragma unroll 1
    for (int r = r0; r < r0 + kViewRowsPerThread; ++r) {
      const int i = y0 + r;
      if (i >= v.geometry.mapH) break;
      int col0, rowPhase;
      int value;
      if constexpr (Positions::kBlend) {
        int col1, rowPhase1, w;
        pos.record(p, v, lane, r, i, j, &col0, &rowPhase, &col1, &rowPhase1, &w);
        value = viewPixel<K, TRANSPARENT>(s, smem, col0, rowPhase);
        if (w > 0 && w < 256) {
          const int b = viewPixel<K, TRANSPARENT>(s, smem, col1, rowPhase1);
          value = value < 0 ? b : (b < 0 ? value : (value * (256 - w) + b * w + 128) >> 8);
        }
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
  }
}

// FLAT_FIXED: per-tile column and row tables in shared memory, after the weights
template <int K>
struct FlatPositions {
  static constexpr int kRows = viewTileRows(K);
  static constexpr int kTableBytes = 4 * 32 * (int)sizeof(FlatColumn) + 2 * kRows * (int)sizeof(FlatRow) + 32;
  static constexpr bool kBlend = false;
  FlatColumn* colTab;  // [eye][fold][32]
  FlatRow* rowTab;     // [column eye][kRows]
  bool* colEye;        // [32]
  const FlatRow* rows;
  __device__ explicit FlatPositions(unsigned char* tables)
      : colTab(reinterpret_cast<FlatColumn*>(tables)), rowTab(reinterpret_cast<FlatRow*>(colTab + 4 * 32)),
        colEye(reinterpret_cast<bool*>(rowTab + 2 * kRows)), rows(nullptr) {}
  __device__ void beginTile(const ViewGatherParams& p, const ViewPlane& v, int x0, int y0) {
    const FlatGeometry& g = v.geometry;
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
  __device__ void record(const ViewGatherParams&, const ViewPlane&, int lane, int r, int, int, int* col0, int* rowPhase) const {
    const FlatRow row = rows[r];
    const FlatColumn c = colTab[(row.eye ? 64 : 0) + (row.fold ? 32 : 0) + lane];
    *col0 = c.col0;
    *rowPhase = row.rowPart + c.fracX;
  }
};

// Sphere and barrel outputs: the whole chain per pixel, no shared tables
template <bool BARREL>
struct SpherePositions {
  static constexpr int kTableBytes = 0;
  static constexpr bool kBlend = false;
  __device__ void beginTile(const OrientedGatherParams&, const OrientedPlane&, int, int) {}
  __device__ void beginColumn(int) {}
  __device__ void record(const OrientedGatherParams& p, const OrientedPlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    sphereSample<BARREL>(v.geometry, p.rotation, v.colTable, v.rowTable, i, j, col0, rowPhase);
  }
};

// A caller's warp map: the pixel's (x, y) from the map (a warp's lanes read 32 consecutive entries of a row: one coalesced
// 256-byte load), quantised as quantizeWarpMap quantises a planned map, NaN, infinities and out-of-range values included
template <int K>
struct MapPositions {
  static constexpr int kTableBytes = 0;
  static constexpr bool kBlend = false;
  __device__ void beginTile(const MapGatherParams&, const MapPlane&, int, int) {}
  __device__ void beginColumn(int) {}
  __device__ void record(const MapGatherParams&, const MapPlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    const float2 m = __ldg(v.map + (size_t)i * v.mapPitch + j);
    int row0, fracX, fracY;
    quantizeAxis(m.x, K, col0, &fracX);
    quantizeAxis(m.y, K, &row0, &fracY);
    *rowPhase = row0 * 1024 + fracY * 32 + fracX;
  }
};

// A fisheye lens rig: the whole chain per pixel, no shared tables
template <bool BARREL>
struct LensPositions {
  static constexpr int kTableBytes = 0;
  static constexpr bool kBlend = false;
  __device__ void beginTile(const LensGatherParams&, const OrientedPlane&, int, int) {}
  __device__ void beginColumn(int) {}
  __device__ void record(const LensGatherParams& p, const OrientedPlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    lensSample<BARREL>(v.geometry, p.rotation, p.rig, v.colTable, v.rowTable, i, j, col0, rowPhase);
  }
};

// A two-lens rig with a feathered seam: both lenses' records and lens 1's weight per pixel (lensBlendSample).  The first
// record is the lens that carries the pixel: lens 1 where w = 256, lens 0 everywhere else (also where neither lens covers
// the pixel: its NaN record is skipped by BORDER_TRANSPARENT).  So a warp gathers twice only for its belt pixels.
template <bool BARREL>
struct LensBlendPositions {
  static constexpr int kTableBytes = 0;
  static constexpr bool kBlend = true;
  __device__ void beginTile(const LensBlendGatherParams&, const OrientedPlane&, int, int) {}
  __device__ void beginColumn(int) {}
  __device__ void record(const LensBlendGatherParams& p, const OrientedPlane& v, int, int, int i, int j, int* col0, int* rowPhase, int* col1,
                         int* rowPhase1, int* w) const {
    int32_t rec0[2], rec1[2];
    *w = lensBlendSample<BARREL>(v.geometry, p.rotation, p.rig, p.seamScale, v.colTable, v.rowTable, i, j, rec0, rec1);
    *col0 = *w == 256 ? rec1[0] : rec0[0];
    *rowPhase = *w == 256 ? rec1[1] : rec0[1];
    *col1 = rec1[0];
    *rowPhase1 = rec1[1];
  }
};

// A rectilinear view: the pinhole ray, the rotation and the input lookup per pixel, no shared tables.  LENS: the rig's
// lenses (rectilinearSample<true>) instead of the context's input
template <bool LENS>
struct RectilinearPositions {
  static constexpr int kTableBytes = 0;
  static constexpr bool kBlend = false;
  __device__ void beginTile(const RectilinearGatherParams&, const OrientedPlane&, int, int) {}
  __device__ void beginColumn(int) {}
  __device__ void record(const RectilinearGatherParams& p, const OrientedPlane& v, int, int, int i, int j, int* col0, int* rowPhase) const {
    rectilinearSample<LENS>(v.geometry, p.camera, p.rig, i, j, col0, rowPhase);
  }
};

template <int K>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) viewGatherKernel(const __grid_constant__ ViewGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int kWeightBytes = K >= 2 ? weightBytes<K>() : 0;
  FlatPositions<K> pos(smem + kWeightBytes);
  if constexpr (K >= 2) stageWeights<K>(p.weights, smem);  // (the first tile's __syncthreads publishes them)
  gatherViewTiles<K, false>(p, numTiles, smem, pos);
}

// TRANSPARENT: the barrel layouts, with their positions and BORDER_TRANSPARENT; the other layouts use BORDER_WRAP
template <int K, bool TRANSPARENT>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) orientedGatherKernel(const __grid_constant__ OrientedGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  SpherePositions<TRANSPARENT> pos;
  if constexpr (K >= 2) {
    stageWeights<K>(p.weights, smem);
    __syncthreads();  // (no tile synchronises after this)
  }
  gatherViewTiles<K, TRANSPARENT>(p, numTiles, smem, pos);
}

// TRANSPARENT: the caller's border, BORDER_TRANSPARENT instead of BORDER_WRAP
template <int K, bool TRANSPARENT>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) mapGatherKernel(const __grid_constant__ MapGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  MapPositions<K> pos;
  if constexpr (K >= 2) {
    stageWeights<K>(p.weights, smem);
    __syncthreads();  // (no tile synchronises after this)
  }
  gatherViewTiles<K, TRANSPARENT>(p, numTiles, smem, pos);
}

// BARREL: the barrel layouts' positions (dead zones included); always BORDER_TRANSPARENT
template <int K, bool BARREL>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) lensGatherKernel(const __grid_constant__ LensGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  LensPositions<BARREL> pos;
  if constexpr (K >= 2) {
    stageWeights<K>(p.weights, smem);
    __syncthreads();  // (no tile synchronises after this)
  }
  gatherViewTiles<K, true>(p, numTiles, smem, pos);
}

// BARREL: as lensGatherKernel
template <int K, bool BARREL>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) lensBlendGatherKernel(const __grid_constant__ LensBlendGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  LensBlendPositions<BARREL> pos;
  if constexpr (K >= 2) {
    stageWeights<K>(p.weights, smem);
    __syncthreads();  // (no tile synchronises after this)
  }
  gatherViewTiles<K, true>(p, numTiles, smem, pos);
}

// LENS: a lens rig's input with BORDER_TRANSPARENT; else the context's input with BORDER_WRAP
template <int K, bool LENS>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) rectilinearGatherKernel(const __grid_constant__ RectilinearGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  RectilinearPositions<LENS> pos;
  if constexpr (K >= 2) {
    stageWeights<K>(p.weights, smem);
    __syncthreads();  // (no tile synchronises after this)
  }
  gatherViewTiles<K, LENS>(p, numTiles, smem, pos);
}

// Instantiation Kern of kernel size K, one CTA per tile up to the occupancy the __launch_bounds__ allow; its shared memory
// is the weight table and the per-tile tables of its Positions
template <int K, auto Kern, class Positions, class Params>
cudaError_t launchPositionsK(const Params& p, int numTiles, int numSMs, cudaStream_t stream) {
  static DeviceLaunchCfg cfgs;  // per kernel instantiation, one entry per device
  constexpr int threads = gatherThreads(K);
  constexpr int smemBytes = (K >= 2 ? weightBytes<K>() : 0) + Positions::kTableBytes;
  LaunchCfg cfg;
  cudaError_t err = prepare<Kern>(cfgs, threads, smemBytes, cfg);
  if (err != cudaSuccess) return err;
  const int grid = std::min(numSMs * cfg.perSM, numTiles);
  Kern<<<grid, threads, smemBytes, stream>>>(p, numTiles);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

// tiles of every plane, in plane order
template <class Params>
int assignTiles(Params& p) {
  const int rows = viewTileRows(p.kernelSize);
  int numTiles = 0;
  for (int i = 0; i < p.numPlanes; ++i) {
    auto& v = p.plane[i];
    v.tilesX = (v.geometry.mapW + 31) / 32;
    v.firstTile = numTiles;
    numTiles += v.tilesX * ((v.geometry.mapH + rows - 1) / rows);
  }
  return numTiles;
}

// The tiles of every plane of p, in one launch of launch(K, FLAG, numTiles): K = p.kernelSize and FLAG = flag as
// compile-time constants (std::integral_constant / std::bool_constant)
template <class Params, class Launch>
cudaError_t launchTiles(Params& p, bool flag, Launch&& launch) {
  if (p.numPlanes < 1 || p.numPlanes > kMaxFramePlanes) return cudaErrorInvalidValue;
  const int numTiles = assignTiles(p);
  if (numTiles <= 0) return cudaSuccess;
  auto withFlag = [&](auto k) { return flag ? launch(k, std::true_type{}, numTiles) : launch(k, std::false_type{}, numTiles); };
  switch (p.kernelSize) {
    case 1: return withFlag(std::integral_constant<int, 1>{});
    case 2: return withFlag(std::integral_constant<int, 2>{});
    case 4: return withFlag(std::integral_constant<int, 4>{});
    case 8: return withFlag(std::integral_constant<int, 8>{});
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t launchViewGather(ViewGatherParams p, int numSMs, cudaStream_t stream) {
  return launchTiles(p, false, [&](auto k, auto, int numTiles) {
    constexpr int K = decltype(k)::value;
    return launchPositionsK<K, viewGatherKernel<K>, FlatPositions<K>>(p, numTiles, numSMs, stream);
  });
}

// (every plane of a frame has the same layout)
cudaError_t launchOrientedGather(OrientedGatherParams p, int numSMs, cudaStream_t stream) {
  return launchTiles(p, barrelLayout(p.plane[0].geometry.outputLayout), [&](auto k, auto barrel, int numTiles) {
    constexpr int K = decltype(k)::value;
    constexpr bool B = decltype(barrel)::value;
    return launchPositionsK<K, orientedGatherKernel<K, B>, SpherePositions<B>>(p, numTiles, numSMs, stream);
  });
}

cudaError_t launchMapGather(MapGatherParams p, int numSMs, cudaStream_t stream) {
  return launchTiles(p, p.transparent, [&](auto k, auto transparent, int numTiles) {
    constexpr int K = decltype(k)::value;
    return launchPositionsK<K, mapGatherKernel<K, decltype(transparent)::value>, MapPositions<K>>(p, numTiles, numSMs, stream);
  });
}

cudaError_t launchLensGather(LensGatherParams p, int numSMs, cudaStream_t stream) {
  return launchTiles(p, barrelLayout(p.plane[0].geometry.outputLayout), [&](auto k, auto barrel, int numTiles) {
    constexpr int K = decltype(k)::value;
    constexpr bool B = decltype(barrel)::value;
    return launchPositionsK<K, lensGatherKernel<K, B>, LensPositions<B>>(p, numTiles, numSMs, stream);
  });
}

cudaError_t launchLensBlendGather(LensBlendGatherParams p, int numSMs, cudaStream_t stream) {
  return launchTiles(p, barrelLayout(p.plane[0].geometry.outputLayout), [&](auto k, auto barrel, int numTiles) {
    constexpr int K = decltype(k)::value;
    constexpr bool B = decltype(barrel)::value;
    return launchPositionsK<K, lensBlendGatherKernel<K, B>, LensBlendPositions<B>>(p, numTiles, numSMs, stream);
  });
}

cudaError_t launchRectilinearGather(RectilinearGatherParams p, int numSMs, cudaStream_t stream) {
  return launchTiles(p, p.lens, [&](auto k, auto lens, int numTiles) {
    constexpr int K = decltype(k)::value;
    constexpr bool L = decltype(lens)::value;
    return launchPositionsK<K, rectilinearGatherKernel<K, L>, RectilinearPositions<L>>(p, numTiles, numSMs, stream);
  });
}

}  // namespace t360
