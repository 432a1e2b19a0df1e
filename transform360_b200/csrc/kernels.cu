// sm_90a kernels of the projection-remap hot path, part 1: everything except the persistent frame gather
// (gather_frame.cu).
//
//   gatherKernel<K>        replace cv::remap as the reference calls it (VideoFrameTransform.cpp:748-754) for whole
//   nearestKernel          planes the frame kernel cannot take (BORDER_TRANSPARENT plans, nearest neighbour, planes
//                          TMA cannot describe): taps through L1, every border case.
//   blurStripKernel<HY>    replace cv::sepFilter2D over the reference's tiles (cpp:173-204, 579-704):
//   blurTileKernel         separable Gaussian, float32, fused multiply-add chain in the order cv2 4.13 uses
//   blurDirectKernel       (see oracle/t360_oracle.c for the model and its pin), round-half-even, u8.
//   areaResizeKernel       replaces cv::resize(INTER_AREA) (cpp:770-776).
#include "gather_common.cuh"

#include <algorithm>
#include <atomic>
#include <cstring>

namespace t360 {

std::atomic<unsigned long long> gLaunches{0};  // all kernels of the library (also counted in gather_frame.cu)

namespace {

template <int K, bool TRANSPARENT>
__global__ void __launch_bounds__(gatherThreads(K), K == 8 ? 1 : 4)
gatherKernel(GatherParams p, int tilesX, int numTiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  stageWeights<K>(p.weights, smem);
  __syncthreads();

  SrcView s;
  s.bytes = p.src;
  s.misalign = (int)(reinterpret_cast<uintptr_t>(p.src) & 3);
  s.words = reinterpret_cast<const uint32_t*>(p.src - s.misalign);
  s.w = p.srcW; s.h = p.srcH; s.pitch = p.srcPitch;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  for (int tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
    const int ty = tile / tilesX, tx = tile - ty * tilesX;
    const int y0 = ty * gatherTileH(K) + warp * kRowsPerThread;
    const int segX = tx * kGatherTileW;
    if (y0 >= p.dstH || segX + lane >= p.dstW) continue;  // records exist for every pixel of the plane, in lane order
    int2 rec[kRowsPerThread];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      rec[j] = loadPlan(p.samples + ((size_t)tile * gatherTileH(K) + warp * kRowsPerThread + j) * kGatherTileW + lane);
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      if (y0 + j >= p.dstH) break;
      const int v = gatherPixel<K, TRANSPARENT, 16384>(s, smem, recordCol0(rec[j].x), rec[j].y);
      if (!TRANSPARENT || v >= 0) p.dst[(size_t)(y0 + j) * p.dstPitch + segX + recordColumn(rec[j].x)] = (uint8_t)v;
    }
  }
}

template <bool TRANSPARENT>
__global__ void __launch_bounds__(256, 4) nearestKernel(GatherParams p, int tilesX, int numTiles) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
    const int ty = tile / tilesX, tx = tile - ty * tilesX;
    const int y0 = ty * gatherTileH(1) + warp * kRowsPerThread;
    const int segX = tx * kGatherTileW;
    if (y0 >= p.dstH || segX + lane >= p.dstW) continue;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      if (y0 + j >= p.dstH) break;
      const int2 rec = loadPlan(p.samples + ((size_t)tile * gatherTileH(1) + warp * kRowsPerThread + j) * kGatherTileW + lane);
      const int x = segX + recordColumn(rec.x);
      int sx = recordCol0(rec.x), sy = rec.y >> 10;
      const bool inside = (unsigned)sx < (unsigned)p.srcW && (unsigned)sy < (unsigned)p.srcH;
      if (!inside && TRANSPARENT) continue;
      if (!inside) { sx = wrapIndex(sx, p.srcW); sy = wrapIndex(sy, p.srcH); }
      p.dst[(size_t)(y0 + j) * p.dstPitch + x] = __ldg(p.src + (size_t)sy * p.srcPitch + sx);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Segmented low-pass.  One CTA per job (a <= 64 x 32 rectangle inside one plan segment).
//   stage 0: source bytes of the rectangle grown by the kernel half-sizes -> shared (edge-replicated
//            against the PLANE border only: tiles see their real neighbours, reference cpp:184-197)
//   stage 1: horizontal pass -> float rows in shared:  s = kx[0]*p[0]; s = fma(kx[i], p[i], s)
//   stage 2: vertical pass, symmetric pairs:  s = ky[h]*R[y]; s = fma(ky[h+i], R[y+i] + R[y-i], s)
//            -> round-half-even, saturate, store
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) blurTileKernel(BlurParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  const BlurJob job = p.jobs[blockIdx.x];
  const int hx = job.kxCount >> 1, hy = job.kyCount >> 1;
  const int rows = job.h + 2 * hy;
  const int srcStride = (job.w + 2 * hx + 3) & ~3;
  uint8_t* tile = smem;
  float* R = reinterpret_cast<float*>(smem + rows * srcStride);
  const float* __restrict__ kx = p.taps + job.kxOffset;
  const float* __restrict__ ky = p.taps + job.kyOffset;

  const int cols = job.w + 2 * hx;
  for (int i = threadIdx.x; i < rows * cols; i += blockDim.x) {
    const int r = i / cols, c = i - r * cols;
    const int sy = min(max(job.y0 - hy + r, 0), p.height - 1);
    const int sx = min(max(job.x0 - hx + c, 0), p.width - 1);
    tile[r * srcStride + c] = __ldg(p.src + (size_t)sy * p.srcPitch + sx);
  }
  __syncthreads();

  for (int i = threadIdx.x; i < rows * job.w; i += blockDim.x) {
    const int r = i / job.w, x = i - r * job.w;
    const uint8_t* t = tile + r * srcStride + x;
    float s = __fmul_rn(__ldg(kx), (float)t[0]);
    for (int k = 1; k < job.kxCount; ++k) s = __fmaf_rn(__ldg(kx + k), (float)t[k], s);
    R[i] = s;
  }
  __syncthreads();

  for (int i = threadIdx.x; i < job.h * job.w; i += blockDim.x) {
    const int y = i / job.w, x = i - y * job.w;
    const float* c = R + (y + hy) * job.w + x;
    float s = __fmul_rn(__ldg(ky + hy), c[0]);
    for (int k = 1; k <= hy; ++k) s = __fmaf_rn(__ldg(ky + hy + k), __fadd_rn(c[k * job.w], c[-k * job.w]), s);
    const int v = __float2int_rn(s);
    p.dst[(size_t)(job.y0 + y) * p.dstPitch + job.x0 + x] = (uint8_t)min(max(v, 0), 255);
  }
}

// ---------------------------------------------------------------------------------------------------
// Register-resident low-pass (the fast path; vertical half-size HY <= 3, any horizontal size).
// One WARP per job, no shared memory, no barriers.  Lane L owns columns x0 + 8L .. x0 + 8L + 7 and marches
// down the rows of the strip:
//   horizontal: the 8 running sums advance together through the taps in chunks of 4; the source bytes they
//     need form a sliding window kept as floats in a 12-register ring (3 groups of 4).  Each chunk issues
//     the 32 scalar multiply-adds, converts one new group of 4 bytes (I2F.U8 with a byte selector: exact, one XU
//     instruction each) fetched as one aligned 32-bit word and aligned with a funnel shift, and reads 4 taps as one
//     128-bit uniform load.
//     Tap arrays are zero-padded to a multiple of 4: fma(0, p, s) == s exactly, and starting the chain from
//     +0 makes the first fma equal the reference's plain multiply, so the bits match the oracle's order.
//   vertical: the last 2*HY+1 row results stay in a register ring; the symmetric-pair FMA chain of the oracle
//     produces one output row per input row; rounding is the 1.5*2^23 magic add (round-half-even), and the low
//     mantissa bytes of 8 results are packed into one 64-bit store.
//   sm_90 has no packed single-precision FFMA2 / FADD2 / FMUL2: every operation is a scalar round-to-nearest
//   instruction, in the oracle's order.
// ---------------------------------------------------------------------------------------------------
#ifndef T360_BLUR_I2F
#define T360_BLUR_I2F 1
#endif
#ifndef T360_BLUR_L2_AHEAD
#define T360_BLUR_L2_AHEAD 2
#endif

__device__ __forceinline__ float byteToFloat(uint32_t word, int k) {
#if T360_BLUR_I2F == 1
  return __uint2float_rn((word >> (8 * k)) & 0xFFu);  // I2F.U8 with a byte selector: one instruction, on the XU pipe
#elif T360_BLUR_I2F == 2
  if (k & 1) return __uint2float_rn((word >> (8 * k)) & 0xFFu);
  return __uint_as_float(__byte_perm(word, 0x4B000000u, 0x7440 | k)) - 8388608.0f;
#else
  // (float)byte k of word: place it in the low mantissa byte of 8388608.0f, subtract 8388608.0f
  return __uint_as_float(__byte_perm(word, 0x4B000000u, 0x7440 | k)) - 8388608.0f;
#endif
}

// Source bytes of one strip row as seen by one lane.  Interior strips read aligned 32-bit words through the
// read-only path; edge strips replicate the plane's left/right border byte by byte (BORDER_REPLICATE against the
// parent plane, reference cpp:197).
template <bool EDGE>
struct StripRowReader {
  const uint8_t* rowBytes;
  const uint32_t* rowWords;
  int firstByte, sh, width;

  __device__ __forceinline__ StripRowReader(const StripParams& p, int y, int firstByte_) : firstByte(firstByte_), width(p.width) {
    rowBytes = p.src + (size_t)min(max(y, 0), p.height - 1) * p.srcPitch;
    const uintptr_t a = reinterpret_cast<uintptr_t>(rowBytes) + firstByte;
    rowWords = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    sh = (int)(a & 3) * 8;
  }
  // raw[0..3]: what the first three groups (window positions 0..11) are made of
  __device__ __forceinline__ void head(uint32_t (&raw)[4]) const {
    if (EDGE) {
#pragma unroll
      for (int g = 0; g < 3; ++g) raw[g] = bytes(g);
      raw[3] = 0;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) raw[i] = __ldg(rowWords + i);
    }
  }
  __device__ __forceinline__ uint32_t bytes(int group) const {
    uint32_t g = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) g |= (uint32_t)__ldg(rowBytes + min(max(firstByte + group * 4 + b, 0), width - 1)) << (8 * b);
    return g;
  }
  // group `group` (>= 3) given the previous aligned word
  __device__ __forceinline__ uint32_t next(int group, uint32_t& prevWord) const {
    if (EDGE) return bytes(group);
    const uint32_t w = __ldg(rowWords + group + 1);
    const uint32_t g = __funnelshift_r(prevWord, w, sh);
    prevWord = w;
    return g;
  }
};

// One chunk of 4 taps: 32 FMAs on the ring, then ring slots 4u..4u+3 take the next group of source bytes.
template <bool EDGE, int U, bool LAST>
__device__ __forceinline__ void stripChunk(const StripRowReader<EDGE>& rd, const float4* __restrict__ taps, int c, uint32_t& prev,
                                           float (&ring)[12], float (&s)[8]) {
  const float4 k4 = __ldg(taps + c);
  uint32_t grp = 0;
  if (!LAST) grp = rd.next(c + 3, prev);  // the group that replaces the 4 oldest window positions
  const float k[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
  for (int t = 0; t < 4; ++t)
#pragma unroll
    for (int m = 0; m < 8; ++m) s[m] = __fmaf_rn(k[t], ring[(4 * U + m + t) % 12], s[m]);
  if (!LAST) {
#pragma unroll
    for (int b = 0; b < 4; ++b) ring[4 * U + b] = byteToFloat(grp, b);
  }
}

template <bool EDGE>
__device__ __forceinline__ void stripRow(const StripParams& p, const StripJob& job, const StripRowReader<EDGE>& rd,
                                         const uint32_t (&raw)[4], float (&s)[8]) {
  float ring[12];
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    const uint32_t grp = EDGE ? raw[g] : __funnelshift_r(raw[g], raw[g + 1], rd.sh);
#pragma unroll
    for (int b = 0; b < 4; ++b) ring[g * 4 + b] = byteToFloat(grp, b);
  }
  uint32_t prev = raw[3];
#pragma unroll
  for (int m = 0; m < 8; ++m) s[m] = 0.0f;
  const float4* taps = reinterpret_cast<const float4*>(p.taps + job.kxOffset);
  // 3-, 5-, 7-, 9-tap kernels (1-3 chunks) cover most of a plane: straight-line code for them (warp-uniform switch)
  switch (job.kxChunks) {
    case 1:
      stripChunk<EDGE, 0, true>(rd, taps, 0, prev, ring, s);
      return;
    case 2:
      stripChunk<EDGE, 0, false>(rd, taps, 0, prev, ring, s);
      stripChunk<EDGE, 1, true>(rd, taps, 1, prev, ring, s);
      return;
    case 3:
      stripChunk<EDGE, 0, false>(rd, taps, 0, prev, ring, s);
      stripChunk<EDGE, 1, false>(rd, taps, 1, prev, ring, s);
      stripChunk<EDGE, 2, true>(rd, taps, 2, prev, ring, s);
      return;
    default:
      break;
  }
  for (int c = 0; c < job.kxChunks; c += 3) {  // the ring is back in phase every 3 chunks
    stripChunk<EDGE, 0, false>(rd, taps, c, prev, ring, s);
    if (c + 1 < job.kxChunks) stripChunk<EDGE, 1, false>(rd, taps, c + 1, prev, ring, s);
    if (c + 2 < job.kxChunks) stripChunk<EDGE, 2, false>(rd, taps, c + 2, prev, ring, s);
  }
}

template <int HY, bool EDGE>
__device__ __forceinline__ void stripBody(const StripParams& p, const StripJob& job, int lane) {
  constexpr int L = 2 * HY + 1;
  const int hx = job.kxCount >> 1;
  const int lx = job.x0 + lane * kStripLanePx;
  if (lane * kStripLanePx >= job.w) return;
  const int firstByte = lx - hx;  // column of window position 0
  const float* __restrict__ ky = p.taps + job.kyOffset;
  float kv[HY + 1];
#pragma unroll
  for (int i = 0; i <= HY; ++i) kv[i] = __ldg(ky + HY + i);
  const int nValid = min(kStripLanePx, job.w - lane * kStripLanePx);
  const bool wide = nValid == 8 && ((reinterpret_cast<uintptr_t>(p.dst) | (unsigned)p.dstPitch | (unsigned)lx) & 7) == 0;

  float R[L][8];
  const int rowsTotal = job.h + 2 * HY;
  // software pipeline over rows: the head of row j+1 is requested before row j is computed (rows are first
  // touches of DRAM lines; without this every row start exposes the full memory latency)
  uint32_t rawNext[4];
  StripRowReader<EDGE>(p, job.y0 - HY, firstByte).head(rawNext);
  for (int jb = 0; jb < rowsTotal; jb += L) {
#pragma unroll
    for (int u = 0; u < L; ++u) {
      const int j = jb + u;
      if (j < rowsTotal) {
        const StripRowReader<EDGE> rd(p, job.y0 - HY + j, firstByte);
        uint32_t raw[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) raw[i] = rawNext[i];
        if (j + 1 < rowsTotal) StripRowReader<EDGE>(p, job.y0 - HY + j + 1, firstByte).head(rawNext);
#if T360_BLUR_L2_AHEAD > 0
        {  // rows further down are first touches of DRAM lines as well: ask L2 for them now (no register is held)
          const int yAhead = min(max(job.y0 - HY + j + 1 + T360_BLUR_L2_AHEAD, 0), p.height - 1);
          const uint8_t* ahead = p.src + (size_t)yAhead * p.srcPitch + max(firstByte, 0);
          asm volatile("prefetch.global.L2 [%0];" ::"l"(ahead));
        }
#endif
        stripRow<EDGE>(p, job, rd, raw, R[u]);
        if (j >= 2 * HY) {
          // centre row is the one computed HY steps ago: ring slot (u - HY) mod L
          constexpr int kBig = 4 * L;
          float o[8];
#pragma unroll
          for (int m = 0; m < 8; ++m) {
            float acc = __fmul_rn(kv[0], R[(u - HY + kBig) % L][m]);
#pragma unroll
            for (int i = 1; i <= HY; ++i)
              acc = __fmaf_rn(kv[i], __fadd_rn(R[(u - HY + i + kBig) % L][m], R[(u - HY - i + kBig) % L][m]), acc);
            o[m] = __fadd_rn(acc, 12582912.0f);  // low mantissa byte = rint(acc), half-even
          }
          const int y = job.y0 + j - 2 * HY;
          uint8_t* out = p.dst + (size_t)y * p.dstPitch + lx;
          const uint32_t lo = __byte_perm(__byte_perm(__float_as_uint(o[0]), __float_as_uint(o[1]), 0x0040),
                                          __byte_perm(__float_as_uint(o[2]), __float_as_uint(o[3]), 0x0040), 0x5410);
          const uint32_t hi = __byte_perm(__byte_perm(__float_as_uint(o[4]), __float_as_uint(o[5]), 0x0040),
                                          __byte_perm(__float_as_uint(o[6]), __float_as_uint(o[7]), 0x0040), 0x5410);
          if (wide) {
            *reinterpret_cast<uint2*>(out) = make_uint2(lo, hi);
          } else {
#pragma unroll
            for (int m = 0; m < 8; ++m)
              if (m < nValid) out[m] = (uint8_t)((m < 4 ? lo >> (8 * m) : hi >> (8 * (m - 4))) & 0xFF);
          }
        }
      }
    }
  }
}

template <int HY>
#ifndef T360_BLUR_PDL
#define T360_BLUR_PDL 0
#endif
#ifndef T360_BLUR_MINBLOCKS
#define T360_BLUR_MINBLOCKS 6  // H100 at 700 W: 80 registers (with spills), 142.4 us per cfg3 frame; 4 blocks 144.4 us, 3 blocks 157.2 us
#endif
__global__ void __launch_bounds__(128, T360_BLUR_MINBLOCKS) blurStripKernel(StripParams p) {
  const int job = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (job >= p.numJobs) return;
  const StripJob j = p.jobs[job];
  if (j.edge) stripBody<HY, true>(p, j, threadIdx.x & 31);
  else stripBody<HY, false>(p, j, threadIdx.x & 31);
}

template <int HY>
__global__ void __launch_bounds__(128, T360_BLUR_MINBLOCKS) blurFrameStripKernel(const __grid_constant__ FrameStripParams fp) {
#if T360_BLUR_PDL
  // the frame gather that follows on the stream may place its CTAs on SMs this grid has already left and run its
  // prologue there (it waits for this grid's completion before it touches the planes)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
  const int job = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (job >= fp.numJobs) return;
  const StripJob j = fp.jobs[job];
  const int pl = j.edge >> kStripPlaneShift;
  const FrameStripParams::Plane &a = fp.plane[0], &b = fp.plane[1], &c = fp.plane[2];
#define T360_PICK(f) (pl == 0 ? a.f : (pl == 1 ? b.f : c.f))
  const StripParams p{T360_PICK(src), T360_PICK(dst), T360_PICK(width), T360_PICK(height), T360_PICK(srcPitch), T360_PICK(dstPitch),
                      fp.jobs, fp.numJobs, fp.taps};
#undef T360_PICK
  if (j.edge & 1) stripBody<HY, true>(p, j, threadIdx.x & 31);
  else stripBody<HY, false>(p, j, threadIdx.x & 31);
}

// Fallback for kernels too large for a shared-memory tile (sigma can reach half the plane width):
// every thread evaluates its pixel's whole separable sum straight from global memory.  Same order.
__global__ void __launch_bounds__(256) blurDirectKernel(BlurParams p) {
  const BlurJob job = p.jobs[blockIdx.x];
  const int hx = job.kxCount >> 1, hy = job.kyCount >> 1;
  const float* __restrict__ kx = p.taps + job.kxOffset;
  const float* __restrict__ ky = p.taps + job.kyOffset;
  for (int i = threadIdx.x; i < job.h * job.w; i += blockDim.x) {
    const int y = job.y0 + i / job.w, x = job.x0 + i % job.w;
    auto rowSum = [&](int yy) {
      const uint8_t* rowp = p.src + (size_t)min(max(yy, 0), p.height - 1) * p.srcPitch;
      float s = __fmul_rn(__ldg(kx), (float)__ldg(rowp + min(max(x - hx, 0), p.width - 1)));
      for (int k = 1; k < job.kxCount; ++k)
        s = __fmaf_rn(__ldg(kx + k), (float)__ldg(rowp + min(max(x - hx + k, 0), p.width - 1)), s);
      return s;
    };
    float s = __fmul_rn(__ldg(ky + hy), rowSum(y));
    for (int k = 1; k <= hy; ++k) s = __fmaf_rn(__ldg(ky + hy + k), __fadd_rn(rowSum(y + k), rowSum(y - k)), s);
    const int v = __float2int_rn(s);
    p.dst[(size_t)y * p.dstPitch + x] = (uint8_t)min(max(v, 0), 255);
  }
}

// ---------------------------------------------------------------------------------------------------
// cv::resize(INTER_AREA) shrink (reference cpp:770-776, only when *_scale_factor != 1).  Not on the hot
// configurations: a straightforward one-thread-per-output-pixel kernel that follows OpenCV's order of
// operations (separate multiply and add, float32) so that the result is bit-exact.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) areaResizeKernel(AreaParams p) {
  const int dx = blockIdx.x * 32 + (threadIdx.x & 31), dy = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (dx >= p.dstW || dy >= p.dstH) return;
  int v;
  if (p.cellW > 0) {
    int sum = 0;
    for (int y = 0; y < p.cellH; ++y) {
      const uint8_t* row = p.src + (size_t)(dy * p.cellH + y) * p.srcPitch + dx * p.cellW;
      for (int x = 0; x < p.cellW; ++x) sum += __ldg(row + x);
    }
    if (p.cellW == 2 && p.cellH == 2) v = (sum + 2) >> 2;
    else v = __float2int_rn(__fmul_rn((float)sum, 1.f / (float)(p.cellW * p.cellH)));
  } else {
    const int x0 = __ldg(p.xFirst + dx), x1 = __ldg(p.xFirst + dx + 1);
    const int y0 = __ldg(p.yFirst + dy), y1 = __ldg(p.yFirst + dy + 1);
    float sum = 0.f;
    for (int j = y0; j < y1; ++j) {
      const int2 ty = __ldg(p.yTaps + j);
      const uint8_t* row = p.src + (size_t)ty.x * p.srcPitch;
      float buf = 0.f;
      for (int k = x0; k < x1; ++k) {
        const int2 tx = __ldg(p.xTaps + k);
        buf = __fadd_rn(buf, __fmul_rn((float)__ldg(row + tx.x), __int_as_float(tx.y)));
      }
      const float term = __fmul_rn(__int_as_float(ty.y), buf);
      sum = j == y0 ? term : __fadd_rn(sum, term);
    }
    v = __float2int_rn(sum);
  }
  p.dst[(size_t)dy * p.dstPitch + dx] = (uint8_t)min(max(v, 0), 255);
}

template <int K, bool T>
cudaError_t launchGatherK(const GatherParams& p, int numSMs, cudaStream_t stream) {
  static DeviceLaunchCfg cfgs;  // per kernel instantiation, one entry per device
  constexpr int threads = gatherThreads(K), smemBytes = weightBytes<K>();
  LaunchCfg cfg;
  cudaError_t err = prepare<gatherKernel<K, T>>(cfgs, threads, smemBytes, cfg);
  if (err != cudaSuccess) return err;
  const int tilesX = (p.dstW + kGatherTileW - 1) / kGatherTileW;
  const int tilesY = (p.dstH + gatherTileH(K) - 1) / gatherTileH(K);
  const int numTiles = tilesX * tilesY;
  if (numTiles <= 0) return cudaSuccess;
  const int grid = std::min(numSMs * cfg.perSM, numTiles);  // whole waves: a multiple of the SM count
  gatherKernel<K, T><<<grid, threads, smemBytes, stream>>>(p, tilesX, numTiles);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

template <bool T>
cudaError_t launchNearest(const GatherParams& p, int numSMs, cudaStream_t stream) {
  static DeviceLaunchCfg cfgs;
  LaunchCfg cfg;
  cudaError_t err = prepare<nearestKernel<T>>(cfgs, 256, 0, cfg);
  if (err != cudaSuccess) return err;
  const int tilesX = (p.dstW + kGatherTileW - 1) / kGatherTileW;
  const int tilesY = (p.dstH + gatherTileH(1) - 1) / gatherTileH(1);
  const int grid = std::min(numSMs * cfg.perSM, tilesX * tilesY);
  nearestKernel<T><<<grid, 256, 0, stream>>>(p, tilesX, tilesX * tilesY);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

// cv::resize(INTER_AREA) with an enlarging axis (scale factors below 1): OpenCV's 8-bit fixed-point bilinear kernel with
// "area mode" weights (sampling.cpp: areaLinearAxis), horizontal pass in 11-bit fixed point, vertical pass with the
// shifts of VResizeLinear<uchar>.  Integer arithmetic: bit-exact.
__global__ void __launch_bounds__(256) areaEnlargeKernel(AreaParams p) {
  const int dx = blockIdx.x * 32 + (threadIdx.x & 31), dy = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (dx >= p.dstW || dy >= p.dstH) return;
  const int2 tx = __ldg(p.xLinear + dx), ty = __ldg(p.yLinear + dy);
  const int a0 = (int16_t)(tx.y & 0xffff), a1 = tx.y >> 16, b0 = (int16_t)(ty.y & 0xffff), b1 = ty.y >> 16;
  int H[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int sy = min(max(ty.x + k, 0), p.srcH - 1);
    const uint8_t* S = p.src + (size_t)sy * p.srcPitch;
    H[k] = dx < p.xMax ? __ldg(S + tx.x) * a0 + __ldg(S + tx.x + 1) * a1 : __ldg(S + tx.x) * 2048;
  }
  const int v = (((b0 * (H[0] >> 4)) >> 16) + ((b1 * (H[1] >> 4)) >> 16) + 2) >> 2;
  p.dst[(size_t)dy * p.dstPitch + dx] = (uint8_t)min(max(v, 0), 255);
}

}  // namespace

cudaError_t launchGather(const GatherParams& p, int numSMs, cudaStream_t stream) {
  if (p.dstW <= 0 || p.dstH <= 0) return cudaSuccess;
  const bool t = p.transparent != 0;
  switch (p.kernelSize) {
    case 1: return t ? launchNearest<true>(p, numSMs, stream) : launchNearest<false>(p, numSMs, stream);
    case 2: return t ? launchGatherK<2, true>(p, numSMs, stream) : launchGatherK<2, false>(p, numSMs, stream);
    case 4: return t ? launchGatherK<4, true>(p, numSMs, stream) : launchGatherK<4, false>(p, numSMs, stream);
    case 8: return t ? launchGatherK<8, true>(p, numSMs, stream) : launchGatherK<8, false>(p, numSMs, stream);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launchAreaResize(const AreaParams& p, cudaStream_t stream) {
  if (p.dstW <= 0 || p.dstH <= 0) return cudaSuccess;
  const dim3 grid((p.dstW + 31) / 32, (p.dstH + 7) / 8);
  if (p.cellW < 0) areaEnlargeKernel<<<grid, 256, 0, stream>>>(p);
  else areaResizeKernel<<<grid, 256, 0, stream>>>(p);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

cudaError_t launchBlurStrips(const StripParams& p, int hy, cudaStream_t stream) {
  if (p.numJobs <= 0) return cudaSuccess;
  const int grid = (p.numJobs + 3) / 4;
  switch (hy) {
    case 0: case 1: blurStripKernel<1><<<grid, 128, 0, stream>>>(p); break;  // hy == 0: one tap, padded with two zeros
    case 2: blurStripKernel<2><<<grid, 128, 0, stream>>>(p); break;
    case 3: blurStripKernel<3><<<grid, 128, 0, stream>>>(p); break;
    default: return cudaErrorInvalidValue;
  }
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

cudaError_t launchBlurFrameStrips(const FrameStripParams& p, int hy, cudaStream_t stream) {
  if (p.numJobs <= 0) return cudaSuccess;
  const int grid = (p.numJobs + 3) / 4;
  switch (hy) {
    case 0: case 1: blurFrameStripKernel<1><<<grid, 128, 0, stream>>>(p); break;
    case 2: blurFrameStripKernel<2><<<grid, 128, 0, stream>>>(p); break;
    case 3: blurFrameStripKernel<3><<<grid, 128, 0, stream>>>(p); break;
    default: return cudaErrorInvalidValue;
  }
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

cudaError_t launchBlur(const BlurParams& p, cudaStream_t stream) {
  if (p.numJobs <= 0) return cudaSuccess;
  if (p.tileSmemBytes > 48 * 1024) {  // the opt-in is per device: cached per device ordinal
    static DeviceLaunchCfg cfgs;
    LaunchCfg cfg;
    cudaError_t err = prepare<blurTileKernel>(cfgs, 256, kBlurMaxSmem, cfg);
    if (err != cudaSuccess) return err;
  }
  blurTileKernel<<<p.numJobs, 256, p.tileSmemBytes, stream>>>(p);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

cudaError_t launchBlurDirect(const BlurParams& p, cudaStream_t stream) {
  if (p.numJobs <= 0) return cudaSuccess;
  blurDirectKernel<<<p.numJobs, 256, 0, stream>>>(p);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

unsigned long long kernelLaunchCount() { return gLaunches.load(std::memory_order_relaxed); }
void countKernelLaunches(long long n) { gLaunches.fetch_add(static_cast<unsigned long long>(n), std::memory_order_relaxed); }

}  // namespace t360
