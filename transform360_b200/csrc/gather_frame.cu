// sm_90a kernels of the projection-remap hot path, part 2: the persistent frame gather.
//
//   gatherFrameKernel<K, COPIES, GROUPS>   replaces cv::remap as the reference calls it (VideoFrameTransform.cpp:748-754)
//   for all planes of a frame in ONE launch: per output pixel a K x K window of the 8-bit source is weighted with
//   OpenCV's 15-bit fixed-point table and rounded with (sum + 16384) >> 15.  Bit-exact by construction: same table
//   (host-built, sampling.cpp), same integer arithmetic.
//
// This is a gather, not a contraction: no tensor cores.  What the design is built around (formats: kernels.cuh):
//   * One CTA per SM: GROUPS consumer groups of 8 warps + one producer warp per group, ONE weight-table image in shared
//     memory for all of them (brought in by cp.async.bulk), so that the cubic table can be kept twice (bank-group
//     balancing by the host: 4.5-5.0 wavefronts per 128-bit weight load instead of 6.3-7.5) and Lanczos4's 128 KB table
//     serves two groups.
//   * Producer: claims a job, waits for a free stage of its group's two-stage ring, and issues ONE
//     cp.async.bulk.tensor.2d (TMA) box load of the job's source window from the pitch-linear plane plus ONE
//     cp.async.bulk of its compact sampling records; both complete on the stage's "full" mbarrier.  Consumers wait for
//     "full", compute out of shared memory and arrive on "empty": no global load, no claim, no CTA barrier on their side.
//   * Taps are read as aligned 32-bit shared-memory words and aligned with a funnel shift; every window row is folded
//     with IDP.2A (two s16 x u8 multiply-adds per instruction).
//   * Share jobs (64 x 32 pixels, 3/5 of a cube map): a thread slides one K-row register window down its output column
//     and fetches only the 1-2 new source rows per pixel, branch-free; 2.5 bytes of plan per pixel.
//   * Tile jobs (32 x 32 or one 16 x 16 quadrant): a window per pixel, lanes cover 8 x 4 patches, 4 bytes of plan per
//     pixel; seam jobs OR two boxes together.
//   * Pole-cap jobs (the pixels no tile's box holds, grouped by source position into class-0 boxes): a window per pixel,
//     8 bytes of plan per pixel with its output position.  Only the few pixels whose window wraps around a plane border
//     (border jobs) read their taps through L1.
//   * Programmatic dependent launch lets the next frame's prologue run under this frame's tail; the job counter re-arms
//     itself.
#include "gather_common.cuh"

#include <cuda.h>  // CUtensorMap (type only; no libcuda symbol is referenced)

#include <algorithm>
#include <cstring>
#include <utility>

namespace t360 {

namespace {

template <class F, int... I>
__device__ __forceinline__ void staticForImpl(F&& f, std::integer_sequence<int, I...>) {
  (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F>
__device__ __forceinline__ void staticFor(F&& f) {  // f(integral_constant<int, 0>) ... f(integral_constant<int, N-1>)
  staticForImpl(f, std::make_integer_sequence<int, N>{});
}

// shared-memory loads with immediate offsets (one address register per pixel / per column)
template <int IMM>
__device__ __forceinline__ uint32_t ldsWordImm(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(IMM));
  return v;
}
template <int IMM>
__device__ __forceinline__ uint4 ldsVecImm(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4+%5];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr), "n"(IMM));
  return v;
}
template <int IMM>
__device__ __forceinline__ uint2 ldsVec2Imm(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2+%3];" : "=r"(v.x), "=r"(v.y) : "r"(addr), "n"(IMM));
  return v;
}

__device__ __forceinline__ uint32_t smemAddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbarInit(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(arrivals));
}
__device__ __forceinline__ void mbarExpectTx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarWait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smemAddr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tmaLoadBox(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smemAddr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smemAddr(bar)) : "memory");
}
__device__ __forceinline__ void bulkCopyToShared(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smemAddr(dst)), "l"(src), "r"(bytes), "r"(smemAddr(bar)) : "memory");
}
__device__ __forceinline__ void groupBarrier(int group) {  // the 8 warps of one job pipeline
  asm volatile("bar.sync %0, %1;" ::"r"(group + 1), "n"(kGroupThreads) : "memory");
}

// ---- window arithmetic -------------------------------------------------------------------------------------------
template <int K>
struct RowBytes {
  uint32_t b[K == 8 ? 2 : 1];  // the K source bytes of one window row, already aligned (K = 2: the low two bytes)
};

// row at byte offset IMM from the (word-aligned) address; sh = 8 * (byte offset of the window inside its first word)
template <int K, int IMM>
__device__ __forceinline__ RowBytes<K> loadRow(uint32_t addr, int sh) {
  RowBytes<K> o;
  const uint32_t q0 = ldsWordImm<IMM>(addr), q1 = ldsWordImm<IMM + 4>(addr);
  o.b[0] = __funnelshift_r(q0, q1, sh);
  if constexpr (K == 8) o.b[1] = __funnelshift_r(q1, ldsWordImm<IMM + 8>(addr), sh);
  return o;
}

// sum + 16384 over the window; slotAddr = shared address of the slot's first weight vector (VS bytes between vectors)
template <int K, int VS>
__device__ __forceinline__ int foldRows(const RowBytes<K> (&W)[K], uint32_t slotAddr) {
  int acc = 1 << 14;  // the rounding constant of FixedPtCast<int, uchar, 15>
  if constexpr (K == 2) {
    const uint2 w = ldsVec2Imm<0>(slotAddr);
    acc = dp2aLo(w.x, W[0].b[0], acc);
    acc = dp2aLo(w.y, W[1].b[0], acc);
  } else if constexpr (K == 4) {
    const uint4 wa = ldsVecImm<0>(slotAddr), wb = ldsVecImm<VS>(slotAddr);
    acc = dp2aLo(wa.x, W[0].b[0], acc); acc = dp2aHi(wa.y, W[0].b[0], acc);
    acc = dp2aLo(wa.z, W[1].b[0], acc); acc = dp2aHi(wa.w, W[1].b[0], acc);
    acc = dp2aLo(wb.x, W[2].b[0], acc); acc = dp2aHi(wb.y, W[2].b[0], acc);
    acc = dp2aLo(wb.z, W[3].b[0], acc); acc = dp2aHi(wb.w, W[3].b[0], acc);
  } else {
    staticFor<8>([&](auto R) {
      constexpr int r = decltype(R)::value;
      const uint4 wt = ldsVecImm<r * VS>(slotAddr);
      acc = dp2aLo(wt.x, W[r].b[0], acc); acc = dp2aHi(wt.y, W[r].b[0], acc);
      acc = dp2aLo(wt.z, W[r].b[1], acc); acc = dp2aHi(wt.w, W[r].b[1], acc);
    });
  }
  return acc;
}
// K = 2 slots are 8 bytes: the record's slot field (slot << 4) is halved
template <int K>
__device__ __forceinline__ uint32_t slotOffset(uint32_t field) { return K == 2 ? field >> 1 : field; }

// Lanczos4: the same sum with the vectors fetched in the lane's own XOR-rotated order (kernels.cuh: "XOR-DIAGONAL").
// field = the record's slot field (slot << 4).
template <int VS>
__device__ __forceinline__ int foldRowsRotated(const RowBytes<8> (&W)[8], uint32_t wAddr, uint32_t field) {
  static_assert(VS == 16384, "one copy of the table");
  const uint32_t r = ((field >> 4) ^ threadIdx.x) & 7u;
  const uint32_t first = field ^ (r * (uint32_t)kDiagonalStep);  // bank group bits: lane & 7; plane bits: r
  const bool p0 = (r & 1u) != 0, p1 = (r & 2u) != 0, p2 = (r & 4u) != 0;
  RowBytes<8> A[8], B[8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) A[i].b[h] = p0 ? W[i ^ 1].b[h] : W[i].b[h];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) B[i].b[h] = p1 ? A[i ^ 2].b[h] : A[i].b[h];
  int acc = 1 << 14;
  staticFor<8>([&](auto V) {
    constexpr int v = decltype(V)::value;
    // row v ^ r of the window meets vector v ^ r of the slot
    const uint4 wt = ldsVecImm<0>(wAddr + (first ^ (uint32_t)(v * kDiagonalStep)));
    const uint32_t b0 = p2 ? B[v ^ 4].b[0] : B[v].b[0], b1 = p2 ? B[v ^ 4].b[1] : B[v].b[1];
    acc = dp2aLo(wt.x, b0, acc); acc = dp2aHi(wt.y, b0, acc);
    acc = dp2aLo(wt.z, b1, acc); acc = dp2aHi(wt.w, b1, acc);
  });
  return acc;
}
// the fold of a staged or general-interior pixel, whatever the table's layout
template <int K, int VS>
__device__ __forceinline__ int foldPixel(const RowBytes<K> (&W)[K], uint32_t wAddr, uint32_t field) {
  if constexpr (K == 8) return foldRowsRotated<VS>(W, wAddr, field);
  else return foldRows<K, VS>(W, wAddr + slotOffset<K>(field));
}
__device__ __forceinline__ int biasedToByte(int acc) { return min(max(acc >> 15, 0), 255); }  // acc already holds + 16384


// ---- share job: one register window per output column, slid down ROWS rows -------------------------------------------
// Consecutive pixels of a column start 1 or 2 source rows apart (bit 0 of the pixel record: the second row).  The part
// of the window's address that is known at compile time (one row per pixel) lives in the immediate offsets of the
// loads; `base` only takes up the second rows.  No branch: the row that only a two-row step needs is a predicated load.
__device__ __forceinline__ uint32_t packBytes(int hi, int lo) {  // sat_u8(hi) << 8 | sat_u8(lo): I2IP.U8.S32.SAT
  uint32_t r;
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(hi), "r"(lo), "r"(0));
  return r;
}

template <int K, int PITCH, int VS, int ROWS, bool ZERO>
__device__ __forceinline__ void computeShareJob(uint8_t* dst, int dstPitch, uint32_t stageAddr, const uint4 (&rec)[ROWS / 8],
                                                uint32_t header, uint32_t wAddr) {
  static_assert(PITCH % 4 == 0 && (K == 4 || K == 8) && ROWS % 8 == 0, "");
  uint32_t base = stageAddr + (header & 0x7ffcu);
  const int sh = (int)(header << 3);  // the funnel shift takes the low five bits: 8 * (offset & 3)
  RowBytes<K> W[K];
  staticFor<K>([&](auto R) { W[decltype(R)::value] = loadRow<K, decltype(R)::value * PITCH>(base, sh); });
  int accPrev = 0;
  staticFor<ROWS>([&](auto J) {
    constexpr int j = decltype(J)::value;
    const uint4& block = rec[j >> 3];
    const uint32_t word = ((j >> 1) & 3) == 0 ? block.x : (((j >> 1) & 3) == 1 ? block.y : (((j >> 1) & 3) == 2 ? block.z : block.w));
    const uint32_t r = (j & 1) ? word >> 16 : word;
    if constexpr (j > 0 && !ZERO) {
      const bool two = (r & 1u) != 0;
      // the previous window starts at base + (j - 1) * PITCH; this one 1 (+ 1) rows below
      const RowBytes<K> below = loadRow<K, (j - 1 + K) * PITCH>(base, sh);
      RowBytes<K> below2 = below;
      if (two) below2 = loadRow<K, (j + K) * PITCH>(base, sh);
#pragma unroll
      for (int q = 0; q + 2 < K; ++q)
#pragma unroll
        for (int i = 0; i < (K == 8 ? 2 : 1); ++i) W[q].b[i] = two ? W[q + 2].b[i] : W[q + 1].b[i];
#pragma unroll
      for (int i = 0; i < (K == 8 ? 2 : 1); ++i) W[K - 2].b[i] = two ? below.b[i] : W[K - 1].b[i];
      W[K - 1] = below2;
      if (two) base += PITCH;
    }
    if constexpr (j > 0 && ZERO) {
      // the variant for blocks in which a window may also stay where it is (d = 0, 1 or 2 in bits 0-1 of the record): no
      // static part in the addresses, three-way selects
      const uint32_t d = r & 3u;
      RowBytes<K> below = W[K - 1], below2 = W[K - 1];
      if (d != 0) below = loadRow<K, K * PITCH>(base, sh);
      if (d == 2) below2 = loadRow<K, (K + 1) * PITCH>(base, sh);
#pragma unroll
      for (int q = 0; q + 2 < K; ++q)
#pragma unroll
        for (int i = 0; i < (K == 8 ? 2 : 1); ++i) W[q].b[i] = d == 0 ? W[q].b[i] : (d == 1 ? W[q + 1].b[i] : W[q + 2].b[i]);
#pragma unroll
      for (int i = 0; i < (K == 8 ? 2 : 1); ++i) {
        W[K - 2].b[i] = d == 0 ? W[K - 2].b[i] : (d == 1 ? W[K - 1].b[i] : below.b[i]);
        W[K - 1].b[i] = d == 0 ? W[K - 1].b[i] : (d == 1 ? below.b[i] : below2.b[i]);
      }
      base += d * PITCH;
    }
    const int acc = foldPixel<K, VS>(W, wAddr, r & kSlotFieldMask) >> 15;
    if constexpr (j & 1) {
      const uint32_t pair = packBytes(acc, accPrev);
      dst[(size_t)(j - 1) * dstPitch] = (uint8_t)pair;
      dst[(size_t)j * dstPitch] = (uint8_t)(pair >> 8);
    } else {
      accPrev = acc;
    }
  });
}

// ---- 32 x 32 staged job: a window per pixel, four pixels per thread (one of each 8 x 4 patch of the warp's rows) --------
template <int K, int PITCH, int VS>
__device__ __forceinline__ void computeTileJob(const PlaneView& pv, uint32_t stageAddr, int outX, int outY, const uint4& rec,
                                               uint32_t wAddr, int warp) {
  static_assert(PITCH % 4 == 0, "");
  const int y0 = outY + warp * kTilePatchH;
  const int dstPitch = pv.dstPitch, dstW = pv.dstW, dstH = pv.dstH;
  uint8_t* const dstRow = pv.dst + (size_t)y0 * dstPitch + outX;
  const uint32_t words[4] = {rec.x, rec.y, rec.z, rec.w};
  staticFor<kRowsPerPatchStep>([&](auto J) {
    constexpr int j = decltype(J)::value;
    const uint32_t w = words[j];
    const int col = kTilePatchW * j + ((int)(w >> 16) & (kTilePatchW - 1)), row = (int)(w >> 19) & (kTilePatchH - 1);
    if (!(w & kRecordSkip) && outX + col < dstW && y0 + row < dstH) {
      const uint32_t rowAddr = stageAddr + (w & 0x7ffcu);
      const int sh = (int)(w << 3);
      RowBytes<K> W[K];
      staticFor<K>([&](auto R) { W[decltype(R)::value] = loadRow<K, decltype(R)::value * PITCH>(rowAddr, sh); });
      const int acc = foldPixel<K, VS>(W, wAddr, (w >> 17) & kSlotFieldMask);
      dstRow[(size_t)row * dstPitch + col] = (uint8_t)biasedToByte(acc);
    }
  });
}

// ---- pole-cap job: a class-0 box of pixels grouped by source position, each with its own output position -----------
// Warp w takes steps w, w + 8, .. of the job's `steps` (kernels.cuh: "cap job").
template <int K, int PITCH, int VS>
__device__ __forceinline__ void computeCapJob(const PlaneView& pv, uint32_t stageAddr, uint32_t recAddr, int steps, uint32_t wAddr,
                                              int warp, int lane) {
  static_assert(PITCH % 4 == 0, "");
  for (int s = warp; s < steps; s += kGroupWarps) {
    const uint2 r = ldsVec2Imm<0>(recAddr + s * kCapStepBytes + lane * 8);
    if (r.x & kRecordSkip) continue;
    const uint32_t rowAddr = stageAddr + (r.x & 0x7ffcu);
    const int sh = (int)(r.x << 3);
    RowBytes<K> W[K];
    staticFor<K>([&](auto R) { W[decltype(R)::value] = loadRow<K, decltype(R)::value * PITCH>(rowAddr, sh); });
    const int acc = foldPixel<K, VS>(W, wAddr, (r.x >> 17) & kSlotFieldMask);
    pv.dst[(size_t)(r.y >> 16) * pv.dstPitch + (r.y & 0xffffu)] = (uint8_t)biasedToByte(acc);
  }
}

// ---- border job: pixels whose window leaves the plane (BORDER_WRAP), one tap at a time through L1 ------------------
template <int K, int VS>
__device__ __forceinline__ void computeBorderJob(const PlaneView& pv, uint32_t recAddr, int n, const unsigned char* wsmem, int warp, int lane) {
  SrcView sv;
  sv.bytes = pv.src;
  sv.misalign = (int)(reinterpret_cast<uintptr_t>(pv.src) & 3);
  sv.words = reinterpret_cast<const uint32_t*>(pv.src - sv.misalign);
  sv.w = pv.srcW; sv.h = pv.srcH; sv.pitch = pv.srcPitch;
  for (int i = warp * 32 + lane; i < n; i += kGroupThreads) {
    const uint4 r = ldsVecImm<0>(recAddr + i * kBorderPixelBytes);
    const int v = gatherPixel<K, false, VS, weightDiagonal(K)>(sv, wsmem, (int)r.x, (int)r.y);
    pv.dst[(size_t)(r.z >> 16) * pv.dstPitch + (r.z & 0xffffu)] = (uint8_t)v;
  }
}

template <int K>
struct FrameTensorMaps {
  CUtensorMap map[kMaxFramePlanes][boxMaps(K)];  // (only the box shapes of kernel size K: fewer kernel-parameter bytes)
};

__device__ __forceinline__ void mbarArrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smemAddr(bar)) : "memory");
}
__device__ __forceinline__ uint4 ldsVec(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t ldsWord(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// shared-memory layout: weights | per group {boxes of all stages, records of all stages} | planes | barriers
template <int K, int COPIES, int GROUPS>
struct FrameLayout {
  static constexpr int kStages = gatherStages(K);
  static constexpr int kWeights = weightImageBytes(K, COPIES);
  static constexpr int kStage = stageBytesOf(K), kRec = stageRecordBytes(K);
  static constexpr int kGroupBytes = kStages * (kStage + kRec);
  static constexpr int kPlanes = kWeights + GROUPS * kGroupBytes;
  static constexpr int kBars = kPlanes + 256;  // per group: full[kStages], empty[kStages]; then the weight barrier
  static constexpr int kTotal = kBars + GROUPS * kStages * 16 + 16;
  static_assert(kTotal <= 232448, "227 KB of shared memory per CTA");
  static_assert(sizeof(PlaneView) * kMaxFramePlanes <= 256, "");
  static_assert(kStage % 128 == 0 && kRec % 128 == 0 && kWeights % 128 == 0, "TMA / bulk-copy destinations");
};

template <int K, int COPIES, int GROUPS>
__global__ void __launch_bounds__(GROUPS * (kGroupWarps + 1) * 32, 1)
gatherFrameKernel(const __grid_constant__ FrameGatherParams p, StagedParams jobs, const __grid_constant__ FrameTensorMaps<K> maps) {
  using L = FrameLayout<K, COPIES, GROUPS>;
  constexpr int VS = weightVectorStride(K, COPIES), kStage = L::kStage, kRec = L::kRec, S = L::kStages;
  constexpr uint32_t kBox0 = stageBoxW(K, 0) * stageBoxH(K, 0), kBox1 = stageBoxW(K, 1) * stageBoxH(K, 1),
                     kBoxShare = stageBoxW(K, 2) * stageBoxH(K, 2);
  static_assert(kBox1 + 64 <= 2 * kStage && kBox0 + 64 <= kStage && kBoxShare + 64 <= kStage, "boxes must fit their stage buffers");
  static_assert(boxVariantRows(K, 0, kBoxVariants - 1) > 0 && boxVariantRows(K, 2, kBoxVariants - 1) > 0, "");
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* wsmem = smem;
  PlaneView* planes = reinterpret_cast<PlaneView*>(smem + L::kPlanes);
  uint64_t* barBase = reinterpret_cast<uint64_t*>(smem + L::kBars);  // group g: full[S], empty[S]
  uint64_t* weightBar = barBase + GROUPS * 2 * S;
  const int warpId = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kProducerWarp = GROUPS * kGroupWarps;

  // Programmatic dependent launch: the next launch on the stream (the next frame's gather) may place its CTAs as soon
  // as ours retire, and run its prologue -- which touches only constant data: weights, job list -- under our tail.
  // Everything an earlier kernel may have written or may still read (the planes, the scheduler counters) is only
  // touched after griddepcontrol.wait below.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) {
    for (int g = 0; g < GROUPS; ++g)
      for (int st = 0; st < S; ++st) {
        mbarInit(barBase + g * 2 * S + st, 1);
        mbarInit(barBase + g * 2 * S + S + st, kGroupWarps);
      }
    mbarInit(weightBar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < kMaxFramePlanes * (int)(sizeof(PlaneView) / 4))
    reinterpret_cast<uint32_t*>(planes)[threadIdx.x] = reinterpret_cast<const uint32_t*>(p.plane)[threadIdx.x];
  __syncthreads();

  if (warpId >= kProducerWarp) {
    // =================================== producers: one warp per group ==============================================
    const int g = warpId - kProducerWarp;
    if (g == 0 && lane == 0) {  // the weight image (host-permuted, both copies) in four bulk copies
      mbarExpectTx(weightBar, L::kWeights);
      constexpr int kChunk = L::kWeights / 4;
      for (int i = 0; i < 4; ++i)
        bulkCopyToShared(wsmem + i * kChunk, reinterpret_cast<const unsigned char*>(p.weightImage) + i * kChunk, kChunk, weightBar);
    }
    // Jobs are claimed one at a time: the first two jobs of a producer are static, every further one comes from the
    // global counter.  Lane 0 holds the headers of the current and the next job.  The claim runs two jobs ahead and the
    // header load one, so neither the atomic nor the loads are waited for.  (Asking L2 for a job's records and source
    // box a job ahead with cp.async.bulk.prefetch paid while a job's box was the whole stage buffer; with the boxes cut
    // to the rows a job needs the copies are not waited for either, and the prefetches only add producer work.)
    const int producer = blockIdx.x * GROUPS + g, dynamicBase = gridDim.x * GROUPS * 2;
    auto loadJob = [&](int i) {
      int4 h = make_int4(0, kJobExit << kJobKindShift, 0, 0);
      if (lane == 0 && i < jobs.numTiles) h = __ldg(reinterpret_cast<const int4*>(jobs.tiles) + i);
      return h;
    };
    // (the first TWO jobs are static, so that the first job is not held up by the round trip of an atomic)
    int4 header = loadJob(producer * 2);
    int4 headerNext = loadJob(producer * 2 + 1);
    asm volatile("griddepcontrol.wait;" ::: "memory");  // earlier kernels on the stream are complete and visible from here on
    int claimed = 0;  // lane 0: the claim for the job after next, issued one job before it is looked at
    if (lane == 0) claimed = atomicAdd(jobs.claimCounter, 1);
    unsigned char* groupBase = smem + L::kWeights + g * L::kGroupBytes;
    uint64_t* full = barBase + g * 2 * S;
    uint64_t* empty = full + S;
    uint32_t st = 0, phase = 0;  // the stage the next job goes to, and the parity of its use count
    auto advance = [&]() { if (++st == S) { st = 0; phase ^= 1; } };
    auto postEmptyJob = [&](int kind) {  // header only (lane 0)
      *reinterpret_cast<int4*>(groupBase + S * kStage + st * kRec) = make_int4(0, kind << kJobKindShift, 0, 0);
      mbarArrive(full + st);
    };
    for (;;) {
      int4 h;
      h.x = __shfl_sync(0xffffffffu, header.x, 0); h.y = __shfl_sync(0xffffffffu, header.y, 0);
      h.z = __shfl_sync(0xffffffffu, header.z, 0); h.w = __shfl_sync(0xffffffffu, header.w, 0);
      const int kind = (h.y >> kJobKindShift) & kJobKindMask;
      mbarWait(empty + st, phase ^ 1);
      const bool twoStages = kind == kJobClass1 || kind == kJobSeam;
      if (twoStages) {
        // its box(es) span two stage buffers: they must be adjacent (not the last and the first) and both free; no-op
        // jobs stand for the stages that carry no job of their own
        if (st == S - 1) {
          if (lane == 0) postEmptyJob(kJobNop);
          advance();
          mbarWait(empty + st, phase ^ 1);
        }
        mbarWait(empty + st + 1, phase ^ 1);  // (st + 1 < S: the same round of the ring)
      }
      if (lane == 0) {
        unsigned char* rec = groupBase + S * kStage + st * kRec;
        *reinterpret_cast<int4*>(rec) = h;
        if (kind == kJobExit) {
          mbarArrive(full + st);  // end of the list: the header is all there is
        } else {
          const int pl = h.y >> kJobPlaneShift;
          const uint32_t recBytes = (uint32_t)jobRecordBytes(K, kind, h.x);
          if (kind == kJobBorder) {  // records only: its taps are read through L1
            mbarExpectTx(full + st, recBytes);
          } else {
            // the source box: the lowest variant of its class that holds the rows the job's windows span, for a class-0
            // job also the narrowest width that holds its columns (kernels.cuh)
            const int cls = boxClassOf(kind), variant = jobBoxVariant(h.z), boxX = jobBoxX(h.z), boxY = jobBoxY(h.z);
            const int width = (int)((unsigned)h.w >> kJobWidthShift);
            const uint32_t boxBytes = (uint32_t)((cls == 0 ? class0BoxW(width) : stageBoxW(K, cls)) * boxVariantRows(K, cls, variant));
            mbarExpectTx(full + st, (kind == kJobSeam ? 2 : 1) * boxBytes + recBytes);
            tmaLoadBox(groupBase + st * kStage, &maps.map[pl][boxMapIndex(K, cls, width, variant)], boxX, boxY, full + st);
            if (kind == kJobSeam)  // the part of the window beyond the right border, from the left of the plane
              tmaLoadBox(groupBase + (st + 1) * kStage, &maps.map[pl][boxMapIndex(K, 0, 0, variant)], boxX - planes[pl].srcW, boxY, full + st);
          }
          bulkCopyToShared(rec + 128, planes[pl].records + ((unsigned)h.w & kJobRecordMask), recBytes, full + st);
        }
      }
      advance();
      if (twoStages) {
        if (lane == 0) postEmptyJob(kJobNop);
        advance();
      }
      __syncwarp();
      if (kind == kJobExit) break;
      header = headerNext;  // next job; start claiming the one after
      headerNext = loadJob(dynamicBase + __shfl_sync(0xffffffffu, claimed, 0));
      if (lane == 0) claimed = atomicAdd(jobs.claimCounter, 1);
    }
    // the producer that finishes last re-arms the scheduler for the next launch (claimCounter[0] = claims, [1] = finished)
    if (lane == 0 && atomicAdd(jobs.claimCounter + 1, 1) == (int)(gridDim.x * GROUPS) - 1) {
      jobs.claimCounter[0] = 0;
      jobs.claimCounter[1] = 0;
      __threadfence();
    }
    return;
  }

  // ===================================== consumers ===================================================================
  const int group = warpId / kGroupWarps, warp = warpId % kGroupWarps;
  unsigned char* groupBase = smem + L::kWeights + group * L::kGroupBytes;
  const uint32_t boxAddr = smemAddr(groupBase), recAddr = smemAddr(groupBase + S * kStage);
  uint64_t* full = barBase + group * 2 * S;
  uint64_t* empty = full + S;
  const uint32_t wAddr = smemAddr(wsmem);
  mbarWait(weightBar, 0);
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the planes may still be in use by earlier kernels until here
  auto now = []() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; };
  unsigned long long* trace = jobs.trace && warp == 0 && lane == 0 ? jobs.trace + (size_t)(blockIdx.x * GROUPS + group) * kTraceJobsPerGroup * 4 : nullptr;
  uint32_t traced = 0;
  for (uint32_t st = 0, phase = 0;;) {
    // (the timestamps go to the trace at once: two 64-bit values held over a job cost the K = 8 kernel a spill)
    unsigned long long* const row = trace && traced < kTraceJobsPerGroup ? trace + traced * 4 : nullptr;
    if (row) row[0] = now();
    mbarWait(full + st, phase);
    if (row) row[1] = now();
    const uint32_t rec = recAddr + st * kRec;
    const uint4 h = ldsVec(rec);
    const int kind = ((int)h.y >> kJobKindShift) & kJobKindMask;
    if (kind == kJobExit) break;
    const int outX = (int)h.x & ~kJobQuadMask, outY = (int)h.y & kJobRowMask;
    const PlaneView& pv = planes[(int)h.y >> kJobPlaneShift];
    if (kind == kJobShare || kind == kJobShareStay) {
      if constexpr (K >= 4) {
        const uint32_t mine = rec + 128 + warp * shareWarpRecordBytes(K);
        uint4 r[shareRows(K) / 8];
#pragma unroll
        for (int b = 0; b < shareRows(K) / 8; ++b) r[b] = ldsVec(mine + b * 512 + lane * 16);
        const uint32_t header = ldsWord(mine + shareRows(K) / 8 * 512 + lane * 4);
        uint8_t* dst = pv.dst + (size_t)(outY + (warp >> 1) * shareRows(K)) * pv.dstPitch + (outX + (warp & 1) * 32 + (int)(header >> kRecordColumnShift));
        if (kind == kJobShare) computeShareJob<K, stageBoxW(K, 2), VS, shareRows(K), false>(dst, pv.dstPitch, boxAddr + st * kStage, r, header, wAddr);
        else computeShareJob<K, stageBoxW(K, 2), VS, shareRows(K), true>(dst, pv.dstPitch, boxAddr + st * kStage, r, header, wAddr);
      }
    } else if (kind == kJobClass0) {
      uint4 r;
      const int quad = ((int)h.x & kJobQuadMask) - 1;
      if (quad < 0) {
        r = ldsVec(rec + 128 + warp * 512 + lane * 16);
      } else {  // one 16 x 16 quadrant: records of the live warps and steps only (kernels.cuh), the others skip
        r = make_uint4(kRecordSkip, kRecordSkip, kRecordSkip, kRecordSkip);
        if ((warp >> 2) == (quad >> 1)) {
          const uint2 v = ldsVec2Imm<0>(rec + 128 + (warp & 3) * 256 + lane * 8);
          if (quad & 1) { r.z = v.x; r.w = v.y; } else { r.x = v.x; r.y = v.y; }
        }
      }
      const int width = (int)(h.w >> kJobWidthShift);  // the pitch of its box: one instantiation per width
      staticFor<class0Widths(K)>([&](auto W) {
        constexpr int w = decltype(W)::value;
        if (width == w) computeTileJob<K, class0BoxW(w), VS>(pv, boxAddr + st * kStage, outX, outY, r, wAddr, warp);
      });
    } else if (kind == kJobClass1) {
      computeTileJob<K, stageBoxW(K, 1), VS>(pv, boxAddr + st * kStage, outX, outY, ldsVec(rec + 128 + warp * 512 + lane * 16), wAddr, warp);
    } else if (kind == kJobSeam) {
      // two complementary class-0 boxes (zero-filled outside the plane) in this stage and the next: OR the second into
      // the first -- all warps of the group, then everybody waits for everybody
      {
        uint4* a = reinterpret_cast<uint4*>(groupBase + st * kStage);
        const uint4* b = reinterpret_cast<const uint4*>(groupBase + (st + 1) * kStage);
        for (int i = warp * 32 + lane; i < (int)(kBox0 / 16); i += kGroupThreads) {
          uint4 x = a[i];
          const uint4 y = b[i];
          x.x |= y.x; x.y |= y.y; x.z |= y.z; x.w |= y.w;
          a[i] = x;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // these writes precede later TMA writes to the stage
      }
      groupBarrier(group);
      computeTileJob<K, stageBoxW(K, 0), VS>(pv, boxAddr + st * kStage, outX, outY, ldsVec(rec + 128 + warp * 512 + lane * 16), wAddr, warp);
    } else if (kind == kJobCap) {
      computeCapJob<K, stageBoxW(K, 0), VS>(pv, boxAddr + st * kStage, rec + 128, (int)h.x, wAddr, warp, lane);
    } else if (kind == kJobBorder) {
      computeBorderJob<K, VS>(pv, rec + 128, (int)h.x, wsmem, warp, lane);
    }
    __syncwarp();
    if (lane == 0) mbarArrive(empty + st);  // this warp is done with the stage (its shared-memory reads are complete)
    if (row) {
      row[2] = now(); row[3] = kind;
      ++traced;
    }
    if (++st == S) { st = 0; phase ^= 1; }
  }
}

template <int K, int COPIES, int GROUPS>
cudaError_t prepareFrameK(LaunchCfg& cfg) {
  static DeviceLaunchCfg cfgs;
  constexpr int threads = GROUPS * (kGroupWarps + 1) * 32, smemBytes = FrameLayout<K, COPIES, GROUPS>::kTotal;
  return prepare<gatherFrameKernel<K, COPIES, GROUPS>>(cfgs, threads, smemBytes, cfg);
}

template <int K, int COPIES, int GROUPS>
cudaError_t launchFrameK(const FrameGatherParams& p, const StagedParams& jobs, const void* tensorMaps, int numSMs,
                         cudaStream_t stream, bool programmatic) {
  FrameTensorMaps<K> maps;
  for (int i = 0; i < kMaxFramePlanes; ++i)  // unused planes: valid descriptors that no job refers to
    std::memcpy(maps.map[i], static_cast<const CUtensorMap*>(tensorMaps) + (size_t)(i < p.numPlanes ? i : 0) * kMaxBoxMaps,
                sizeof(maps.map[i]));
  constexpr int threads = GROUPS * (kGroupWarps + 1) * 32, smemBytes = FrameLayout<K, COPIES, GROUPS>::kTotal;
  LaunchCfg cfg;
  cudaError_t err = prepareFrameK<K, COPIES, GROUPS>(cfg);
  if (err != cudaSuccess) return err;
  const int grid = std::min(numSMs * cfg.perSM, (jobs.numTiles + GROUPS * 2 - 1) / (GROUPS * 2));  // persistent: one CTA per SM
  cudaLaunchConfig_t lc{};
  lc.gridDim = dim3(grid);
  lc.blockDim = dim3(threads);
  lc.dynamicSmemBytes = smemBytes;
  lc.stream = stream;
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;  // see griddepcontrol.* in the kernel
  attr.val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = &attr;
  lc.numAttrs = programmatic ? 1 : 0;
  err = cudaLaunchKernelEx(&lc, gatherFrameKernel<K, COPIES, GROUPS>, p, jobs, maps);
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  return err;
}

}  // namespace

cudaError_t prepareGatherFrame(int kernelSize) {
  LaunchCfg cfg;
  switch (kernelSize) {
    case 2: return prepareFrameK<2, weightCopies(2), gatherGroups(2)>(cfg);
    case 4: return prepareFrameK<4, weightCopies(4), gatherGroups(4)>(cfg);
    case 8: return prepareFrameK<8, weightCopies(8), gatherGroups(8)>(cfg);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launchGatherFrame(const FrameGatherParams& p, const StagedParams& jobs, const void* tensorMaps, int numSMs,
                              cudaStream_t stream, bool programmatic) {
  if (jobs.numTiles <= 0) return cudaSuccess;
  if (p.numPlanes < 1 || p.numPlanes > kMaxFramePlanes) return cudaErrorInvalidValue;
  switch (p.kernelSize) {
    case 2: return launchFrameK<2, weightCopies(2), gatherGroups(2)>(p, jobs, tensorMaps, numSMs, stream, programmatic);
    case 4: return launchFrameK<4, weightCopies(4), gatherGroups(4)>(p, jobs, tensorMaps, numSMs, stream, programmatic);
    case 8: return launchFrameK<8, weightCopies(8), gatherGroups(8)>(p, jobs, tensorMaps, numSMs, stream, programmatic);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace t360
