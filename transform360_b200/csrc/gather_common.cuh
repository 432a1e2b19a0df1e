// Device helpers shared by the gather kernels (kernels.cu: whole-plane general kernels; gather_frame.cu: the
// persistent frame kernel).  The arithmetic is OpenCV's cv::remap fixed-point path (SURVEY.md Appendix A):
// K x K window of 8-bit samples x 15-bit table weights, (sum + 16384) >> 15, saturate.
#pragma once

#include "kernels.cuh"

#include <atomic>
#include <mutex>

namespace t360 {

extern std::atomic<unsigned long long> gLaunches;  // kernels.cu

namespace {

// Launch configuration of one kernel instantiation: the opt-in to large dynamic shared memory and the occupancy are
// properties of (kernel, DEVICE), so they are cached per device ordinal (a thread may drive several GPUs).
struct LaunchCfg {
  bool ready = false;
  int perSM = 0;
};
struct DeviceLaunchCfg {
  static constexpr int kMaxDevices = 64;
  std::mutex mu;
  LaunchCfg perDevice[kMaxDevices];
};
template <auto Kern>
cudaError_t prepare(DeviceLaunchCfg& cfgs, int threads, int smemBytes, LaunchCfg& out) {
  int dev = 0;
  cudaError_t err = cudaGetDevice(&dev);
  if (err != cudaSuccess) return err;
  if (dev < 0 || dev >= DeviceLaunchCfg::kMaxDevices) return cudaErrorInvalidDevice;
  std::lock_guard<std::mutex> lock(cfgs.mu);
  LaunchCfg& cfg = cfgs.perDevice[dev];
  if (!cfg.ready) {
    if (smemBytes > 48 * 1024) {
      err = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smemBytes);
      if (err != cudaSuccess) return err;
    }
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cfg.perSM, Kern, threads, smemBytes);
    if (err != cudaSuccess) return err;
    if (cfg.perSM < 1) return cudaErrorLaunchOutOfResources;
    cfg.ready = true;
  }
  out = cfg;
  return cudaSuccess;
}

constexpr int kRowsPerThread = 4;

__device__ __forceinline__ int dp2aLo(uint32_t w, uint32_t b, int acc) {
  int d;
  asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(w), "r"(b), "r"(acc));
  return d;
}
__device__ __forceinline__ int dp2aHi(uint32_t w, uint32_t b, int acc) {
  int d;
  asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(w), "r"(b), "r"(acc));
  return d;
}

// the sampling plan is streamed once per frame: read-only path, do not allocate in L1
__device__ __forceinline__ int2 loadPlan(const int2* p) {
  int2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}

__device__ __forceinline__ int recordColumn(int word0) { return (int)((unsigned)word0 >> kRecordColumnShift); }
__device__ __forceinline__ int recordCol0(int word0) { return (word0 << (32 - kRecordColumnShift)) >> (32 - kRecordColumnShift); }

__device__ __forceinline__ int wrapIndex(int p, int n) {  // cv::borderInterpolate(BORDER_WRAP)
  if ((unsigned)p < (unsigned)n) return p;
  p %= n;
  return p < 0 ? p + n : p;
}
__device__ __forceinline__ int reflect101(int p, int n) {  // what remap uses for taps under BORDER_TRANSPARENT
  if (n == 1) return 0;
  while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

template <int K>
__host__ __device__ constexpr int weightBytes() { return 1024 * K * K * 2; }

template <int K>
__device__ __forceinline__ int weightSlot(int phase) { return weightSlotOf(K, phase); }

// Copies the [1024][K][K] int16 table into shared memory as [K*K/8][1024] 16-byte vectors (K >= 4) or
// [1024] 8-byte vectors (K == 2), slot-permuted by weightSlot().
template <int K>
__device__ __forceinline__ void stageWeights(const int16_t* __restrict__ g, unsigned char* smem) {
  if constexpr (K == 2) {
    const uint2* src = reinterpret_cast<const uint2*>(g);
    uint2* dst = reinterpret_cast<uint2*>(smem);
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) dst[weightSlot<K>(i)] = __ldg(src + i);
  } else {
    constexpr int kVec = K * K / 8;  // uint4 per phase
    const uint4* src = reinterpret_cast<const uint4*>(g);
    uint4* dst = reinterpret_cast<uint4*>(smem);
    for (int i = threadIdx.x; i < 1024 * kVec; i += blockDim.x) dst[(i % kVec) * 1024 + weightSlot<K>(i / kVec)] = __ldg(src + i);
  }
}

// K x K window in GLOBAL memory (read-only path) whose rows are `pitch` bytes apart, starting at byte offset `off`
// of a 4-byte aligned base.  No bounds handling: the caller guarantees the window (plus the tail of its last
// aligned word) is readable.
template <int K, int VSTRIDE, bool DIAG = false>
__device__ __forceinline__ int foldWindow(const uint32_t* __restrict__ words, int off, int pitch,
                                          const unsigned char* wsmem, int phase) {
  phase = weightSlot<K>(phase);
  auto ld = [&](int wordIndex) -> uint32_t { return __ldg(words + wordIndex); };
  int acc = 0;
  if constexpr (K == 2) {
    const uint2 wt = reinterpret_cast<const uint2*>(wsmem)[phase];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const uint32_t b = __funnelshift_r(ld(off >> 2), ld((off >> 2) + 1), (off & 3) * 8);
      acc = dp2aLo(r == 0 ? wt.x : wt.y, b, acc);
      off += pitch;
    }
  } else if constexpr (K == 4) {
    const uint4* tab = reinterpret_cast<const uint4*>(wsmem);
    const uint4 wa = tab[phase], wb = tab[VSTRIDE / 16 + phase];
    const uint32_t w01[4] = {wa.x, wa.z, wb.x, wb.z}, w23[4] = {wa.y, wa.w, wb.y, wb.w};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint32_t b = __funnelshift_r(ld(off >> 2), ld((off >> 2) + 1), (off & 3) * 8);
      acc = dp2aLo(w01[r], b, acc);
      acc = dp2aHi(w23[r], b, acc);
      off += pitch;
    }
  } else {
    const uint4* tab = reinterpret_cast<const uint4*>(wsmem);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint4 wt = tab[r * (VSTRIDE / 16) + (DIAG ? phase ^ r : phase)];
      const uint32_t q0 = ld(off >> 2), q1 = ld((off >> 2) + 1), q2 = ld((off >> 2) + 2);
      const int sh = (off & 3) * 8;
      const uint32_t b0 = __funnelshift_r(q0, q1, sh), b1 = __funnelshift_r(q1, q2, sh);
      acc = dp2aLo(wt.x, b0, acc);
      acc = dp2aHi(wt.y, b0, acc);
      acc = dp2aLo(wt.z, b1, acc);
      acc = dp2aHi(wt.w, b1, acc);
      off += pitch;
    }
  }
  return acc;
}

__device__ __forceinline__ int roundToByte(int acc) {  // FixedPtCast<int, uchar, 15>
  return min(max((acc + (1 << 14)) >> 15, 0), 255);
}

struct SrcView {
  const uint32_t* words;  // source plane base rounded down to 4 bytes
  const uint8_t* bytes;   // true base
  int misalign;           // bytes - words
  int w, h, pitch;
};

// One output pixel through L1, any border case.  Returns the 8-bit value, or -1 when BORDER_TRANSPARENT
// leaves the pixel untouched.
template <int K, bool TRANSPARENT, int VSTRIDE, bool DIAG = false>
__device__ __forceinline__ int gatherPixel(const SrcView& s, const unsigned char* wsmem, int col0, int rowPhase) {
  const int row0 = rowPhase >> 10, phase = rowPhase & 1023;
  // interior: no wrapping, and the aligned word reads (2 words for K <= 4, 3 for K = 8, starting at col0 & ~3) stay
  // inside the row even when the pitch equals the width
  const bool interior = col0 >= 0 && row0 >= 0 && col0 + (K == 2 ? 8 : K + 4) <= s.w && row0 + K <= s.h;
  if (interior)
    return roundToByte(foldWindow<K, VSTRIDE, DIAG>(s.words, row0 * s.pitch + col0 + s.misalign, s.pitch, wsmem, phase));

  // window touches an edge: per-tap addressing.  BORDER_WRAP wraps columns AND rows (reference cpp:719).
  const int slot = weightSlot<K>(phase);
  const int16_t* wt = reinterpret_cast<const int16_t*>(wsmem) + (DIAG ? 0 : slot * (K == 2 ? 4 : 8));
  if (TRANSPARENT) {
    // every interpolator leaves the pixel alone when its anchor sample lies outside the source
    const int ax = col0 + (K / 2 - 1), ay = row0 + (K / 2 - 1);
    if ((unsigned)ax >= (unsigned)s.w || (unsigned)ay >= (unsigned)s.h) return -1;
    if (K == 2) {
      // bilinear, anchor inside but the 2x2 window sticks out on the last row / column: OpenCV blends the taps
      // that exist and renormalises by their weight, rounding half up (oracle/t360_oracle.c)
      int num = 0, den = 0;
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (col0 + c < s.w && row0 + r < s.h) {
            num += wt[r * 2 + c] * (int)__ldg(s.bytes + (size_t)(row0 + r) * s.pitch + col0 + c);
            den += wt[r * 2 + c];
          }
      return den > 0 ? (2 * num + den) / (2 * den) : -1;
    }
  }
  // border columns once, then every load of a row (of the whole window for K <= 4) before the first use: a warp that
  // straddles the +-180 degree seam waits for its few border lanes, so their latency is the tile's latency
  int acc = 0;
  int xs[K];
#pragma unroll
  for (int c = 0; c < K; ++c) xs[c] = TRANSPARENT ? reflect101(col0 + c, s.w) : wrapIndex(col0 + c, s.w);
#pragma unroll(K <= 4 ? K : 1)
  for (int r = 0; r < K; ++r) {
    const int yy = TRANSPARENT ? reflect101(row0 + r, s.h) : wrapIndex(row0 + r, s.h);
    const uint8_t* rowp = s.bytes + (size_t)yy * s.pitch;
    int px[K];
#pragma unroll
    for (int c = 0; c < K; ++c) px[c] = __ldg(rowp + xs[c]);
#pragma unroll
    for (int c = 0; c < K; ++c) {
      const int e = r * K + c;  // element (r, c) lives in vector e / 8, lane e % 8 of the transposed table
      // (the diagonal image keeps vector e / 8 of the slot at position slot ^ (e / 8) of its plane)
      acc += (K == 2 ? wt[e] : wt[(e >> 3) * (VSTRIDE / 2) + (DIAG ? (slot ^ (e >> 3)) * 8 : 0) + (e & 7)]) * px[c];
    }
  }
  return roundToByte(acc);
}


}  // namespace
}  // namespace t360
