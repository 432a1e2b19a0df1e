// sm_90a kernel of the per-view FLAT_FIXED path: every plane of a frame in one launch, with the view as a launch
// parameter instead of a sampling plan.
//
// In FLAT_FIXED the source column and its phase depend only on the output column (and on the pole fold and the eye),
// the source row and its phase only on the output row (flat_view.h).  So a CTA computes, per tile of 32 columns x
// viewTileRows(k) rows, a column table (32 columns x fold x eye) and a row table (rows x eye) in shared memory, with the
// same host/device functions the planner uses -- bit-identical records -- and then a thread takes one column and walks
// down kViewRowsPerThread rows of it.  The taps go through the read-only path with gatherPixel (gather_common.cuh):
// whole aligned words for interior windows, per-tap wrapping (BORDER_WRAP, the only border mode FLAT_FIXED uses) for
// windows that cross the seam or a plane edge.  The weight table is staged once per CTA (stageWeights); the grid is
// persistent over the tiles of all planes.
#include "gather_common.cuh"

#include <algorithm>

namespace t360 {
namespace {

template <int K>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4) viewGatherKernel(const __grid_constant__ ViewGatherParams p, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int kRows = viewTileRows(K);
  constexpr int kWeightBytes = K >= 2 ? weightBytes<K>() : 0;
  FlatColumn* colTab = reinterpret_cast<FlatColumn*>(smem + kWeightBytes);  // [eye][fold][32]
  FlatRow* rowTab = reinterpret_cast<FlatRow*>(colTab + 4 * 32);             // [column eye][kRows]
  bool* colEye = reinterpret_cast<bool*>(rowTab + 2 * kRows);                // [32]
  if constexpr (K >= 2) stageWeights<K>(p.weights, smem);

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
    const int pl = (p.numPlanes > 2 && tile >= p.plane[2].firstTile) ? 2 : ((p.numPlanes > 1 && tile >= p.plane[1].firstTile) ? 1 : 0);
    const ViewPlane& v = p.plane[pl];
    const FlatGeometry& g = v.geometry;
    const int t = tile - v.firstTile, ty = t / v.tilesX;
    const int x0 = (t - ty * v.tilesX) * 32, y0 = ty * kRows;
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

    const int j = x0 + lane;
    if (j >= g.mapW) continue;
    SrcView s;
    s.bytes = v.src;
    s.misalign = (int)(reinterpret_cast<uintptr_t>(v.src) & 3);
    s.words = reinterpret_cast<const uint32_t*>(v.src - s.misalign);
    s.w = g.inW; s.h = g.inH; s.pitch = v.srcPitch;
    const FlatRow* rows = rowTab + (colEye[lane] ? kRows : 0);
    const int r0 = warp * kViewRowsPerThread;
#pragma unroll 1
    for (int r = r0; r < r0 + kViewRowsPerThread; ++r) {
      const int i = y0 + r;
      if (i >= g.mapH) break;
      const FlatRow row = rows[r];
      const FlatColumn c = colTab[(row.eye ? 64 : 0) + (row.fold ? 32 : 0) + lane];
      int value;
      if constexpr (K == 1) {  // nearest: the rounded position, wrapped like cv::remap's BORDER_WRAP
        value = __ldg(s.bytes + (size_t)wrapIndex(row.rowPart >> 10, s.h) * s.pitch + wrapIndex(c.col0, s.w));
      } else {
        value = gatherPixel<K, false, 16384>(s, smem, c.col0, row.rowPart + c.fracX);
      }
      v.dst[(size_t)i * v.dstPitch + j] = (uint8_t)value;
    }
  }
}

template <int K>
cudaError_t launchViewK(const ViewGatherParams& p, int numTiles, int numSMs, cudaStream_t stream) {
  static DeviceLaunchCfg cfgs;  // per kernel instantiation, one entry per device
  constexpr int threads = gatherThreads(K);
  constexpr int smemBytes = (K >= 2 ? weightBytes<K>() : 0) + 4 * 32 * (int)sizeof(FlatColumn) + 2 * viewTileRows(K) * (int)sizeof(FlatRow) + 32;
  LaunchCfg cfg;
  cudaError_t err = prepare<viewGatherKernel<K>>(cfgs, threads, smemBytes, cfg);
  if (err != cudaSuccess) return err;
  const int grid = std::min(numSMs * cfg.perSM, numTiles);
  viewGatherKernel<K><<<grid, threads, smemBytes, stream>>>(p, numTiles);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launchViewGather(ViewGatherParams p, int numSMs, cudaStream_t stream) {
  if (p.numPlanes < 1 || p.numPlanes > kMaxFramePlanes) return cudaErrorInvalidValue;
  const int rows = viewTileRows(p.kernelSize);
  int numTiles = 0;
  for (int i = 0; i < p.numPlanes; ++i) {
    ViewPlane& v = p.plane[i];
    v.tilesX = (v.geometry.mapW + 31) / 32;
    v.firstTile = numTiles;
    numTiles += v.tilesX * ((v.geometry.mapH + rows - 1) / rows);
  }
  if (numTiles <= 0) return cudaSuccess;
  switch (p.kernelSize) {
    case 1: return launchViewK<1>(p, numTiles, numSMs, stream);
    case 2: return launchViewK<2>(p, numTiles, numSMs, stream);
    case 4: return launchViewK<4>(p, numTiles, numSMs, stream);
    case 8: return launchViewK<8>(p, numTiles, numSMs, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace t360
