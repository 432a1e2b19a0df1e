// Device-side interface of the remap hot path (sm_90a).  See kernels.cu.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "flat_view.h"
#include "oriented_view.h"

namespace t360 {

// One gather launch: dst[y][x] = interpolate(src, samples[y][x]) for a whole plane.
struct GatherParams {
  const uint8_t* src;  // (blurred) input plane
  int srcW, srcH, srcPitch;
  uint8_t* dst;
  int dstW, dstH, dstPitch;
  const int2* samples;  // sampling records {col0, (row0 << 10) | phase}, tile-major (see "sampling records" below)
  int tilesPerRow;      // 32-column tiles per row of tiles
  const int16_t* weights;  // device copy of the [1024][k][k] table (nullptr for nearest)
  int kernelSize;          // 1, 2, 4, 8
  int transparent;         // BORDER_TRANSPARENT (barrel layouts) instead of BORDER_WRAP
};

// ---- the persistent frame gather (gatherFrameKernel) -------------------------------------------------------------
// One CTA per SM: gatherGroups(k) GROUPS of 8 consumer warps + 1 producer warp each, all sharing one copy of the weight
// tables in shared memory.  A producer claims jobs from the frame's job list (an atomic counter, one job at a time: batches of 2 / 4 left groups idle at the end of a frame on the B200, where this
// was chosen; not re-measured on the H100),
// and for every job fills one stage of its group's two-stage ring: the job header (st.shared), the job's
// compact sampling records (cp.async.bulk) and its source window (ONE cp.async.bulk.tensor.2d box from the
// pitch-linear plane), all signalled through the stage's "full" mbarrier.  The consumer warps wait for "full", compute,
// and each arrives on the stage's "empty" mbarrier: no global load, no claim, no CTA-wide barrier on the consumer side.
//
// A JOB is a block of output pixels of one image plane:
struct GatherJob {
  int outX, outY;    // outY carries the job kind (kJobKindShift) and the image plane (kJobPlaneShift)
  int boxXY;         // boxX | boxY << 16 | box variant: boxX % 16 == 0, its low four bits name the tensor map (box height)
  int recordOffset;  // of the job's compact records, in 16-byte units from the plane's record buffer; in the device's
                     // list bits kJobWidthShift.. name the width of a class-0 box (class0BoxW)
};
// A job's source box is ONE TMA box, but not always the whole stage buffer: every box class has kBoxVariants tensor maps
// of decreasing height (boxVariantRows below), and a job names the lowest one that still holds the rows its windows span
// (cfg2: the share jobs span 63 of the 72 rows their stage buffer holds, the 32 x 32 tiles 47 of 64, the quadrants 36 of
// 64: 18 % fewer bytes from L2 into shared memory than with whole boxes).  Loading a box as a series of 8-row TMA boxes
// instead -- one tensor map per class, any height -- saves 21 % of the bytes but costs the producer 6 - 9 TMA instructions
// (+ as many L2 prefetches) per job, which made the frame slower than the bytes it saved (measured on the B200, where
// this was decided; not re-measured on the H100).
constexpr int kBoxVariants = 3;
__host__ __device__ constexpr int jobBoxField(int boxX, int boxY, int variant) { return boxX | (boxY << 16) | variant; }
__host__ __device__ constexpr int jobBoxX(int boxXY) { return boxXY & 0xfff0; }
__host__ __device__ constexpr int jobBoxY(int boxXY) { return (int)((unsigned)boxXY >> 16); }
__host__ __device__ constexpr int jobBoxVariant(int boxXY) { return boxXY & 15; }
using StagedTile = GatherJob;
// kJobGeneral: a 32 x 32 tile whose windows fit no box (the pole caps).  It is an entry of the plan's tile list only;
// the kernel runs its pixels as kJobCap jobs (grouped by source position into class-0 boxes) and, the few whose window
// leaves the plane (wraps), as kJobBorder jobs (one tap at a time through L1).
constexpr int kJobClass0 = 0, kJobClass1 = 1, kJobGeneral = 2, kJobShareStay = 3, kJobShare = 4, kJobNop = 5, kJobExit = 6, kJobSeam = 7,
              kJobCap = 8, kJobBorder = 9;
// A 32 x 32 job may cover one 16 x 16 quadrant of its tile only (a tile whose windows fit no box as a whole, but whose
// quadrants do: the ring around a pole cap): outX carries 1 + the quadrant in its low bits (0: the whole tile), and the
// records of the pixels outside the quadrant have kRecordSkip set.
constexpr int kJobQuadMask = 7;
constexpr uint32_t kRecordSkip = 0x8000u;
constexpr int kJobKindShift = 24, kJobRowMask = (1 << kJobKindShift) - 1;
constexpr int kJobPlaneShift = 28, kJobKindMask = (1 << (kJobPlaneShift - kJobKindShift)) - 1;

constexpr int kGroupThreads = 256, kGroupWarps = kGroupThreads / 32;
// consumer groups per CTA (+ one producer warp): as many as the rings fit beside the weight tables in 227 KB
__host__ __device__ constexpr int gatherGroups(int k) { return k == 8 ? 2 : 3; }
constexpr int kGatherTileW = 32, kFrameTileH = 32;  // generic jobs: 32 x 32, four pixels per thread
// a warp of a 32 x 32 job takes its 32 x 4 pixels in four steps of one 8 x 4 patch each
constexpr int kTilePatchW = 8, kTilePatchH = 4, kRowsPerPatchStep = 4;
constexpr int kShareW = 64;  // share jobs: 2 x 4 warps of 32 columns x shareRows(k) rows
__host__ __device__ constexpr int shareRows(int /*k*/) { return 8; }
__host__ __device__ constexpr int shareH(int k) { return 4 * shareRows(k); }
// Staging boxes (bytes x rows).  The shared-memory row pitch is the box width (TMA writes dense rows).  192 B = 48 words
// puts consecutive rows 16 banks apart: the 32 adjacent pixels of a share-job warp span <= 13 words of 1-2 source rows,
// so their window loads are conflict-free (1.10 wavefronts per load in the bank model, 1.57 at 96 B).  Polar tiles
// (a warp's pixels drift over many rows) are worst at 192 B (2.9) and want a pitch that is 4 * odd words: 208 B (2.3).
constexpr int kNumBoxClasses = 3;  // tensor map index: 0 = class 0 / seam, 1 = class 1, 2 = share
__host__ __device__ constexpr int boxClassOf(int kind) { return (kind == kJobShare || kind == kJobShareStay) ? 2 : (kind == kJobClass1 ? 1 : 0); }
__host__ __device__ constexpr int stageBoxW(int /*k*/, int cls) { return cls == 2 ? 192 : (cls == 0 ? 208 : 240); }
__host__ __device__ constexpr int stageBoxH(int k, int cls) {
  return k == 8 ? (cls == 2 ? 80 : (cls == 0 ? 72 : 128)) : (cls == 2 ? 72 : (cls == 0 ? 64 : 96));
}
// rows of variant v of a class's box (v = 0: the whole stage buffer): share H, H - 8, H - 16; class 0 H, H - 16, H - 24
// (the best three heights for the cfg2 plan, whose tiles need 40 / 48 / 56 / 64 rows in 3744 / 1852 / 1084 / 848 jobs
// and whose share jobs 56 / 64 / 72 in 624 / 2644 / 1120); class 1 has the whole box only
__host__ __device__ constexpr int boxVariantRows(int k, int cls, int v) {
  return cls == 1 || v == 0 ? stageBoxH(k, cls) : (cls == 2 ? stageBoxH(k, cls) - 8 * v : stageBoxH(k, cls) - 8 - 8 * v);
}
// the lowest variant that holds `rows` rows
__host__ __device__ constexpr int boxVariantFor(int k, int cls, int rows) {
  int v = 0;
  while (v + 1 < kBoxVariants && cls != 1 && boxVariantRows(k, cls, v + 1) >= rows) ++v;
  return v;
}
// A class-0 tile or quadrant job also loads a box of one of kClass0Widths widths, the narrowest that holds the columns its
// windows span: a polar tile's windows cover a rotated patch of the source whose columns are mostly far fewer than 208
// bytes (cfg2: 80 / 112 / 144 / 208 B hold 12 / 55 / 23 / 10 % of the tiles and quadrants; their boxes lose 39 % of their
// bytes; profiles/box_footprint.py).  The box lands in shared memory at a pitch of its width, and the device's copy of
// the job's records holds its window offsets at that pitch (gather_plan.h: deviceRecords; the plan itself keeps the stage
// buffer's 208 B).  Every width is 4 * odd words, like 208 B (bank model of the tile jobs' window loads:
// profiles/box_footprint.py).  Seam jobs (two boxes ORed together) and pole-cap jobs (cut to fill 208 B) keep the whole
// width.  The device's job list carries the width in the top bits of GatherJob::recordOffset (0: 208 B).
constexpr int kClass0Widths = 4, kJobWidthShift = 28, kJobRecordMask = (1 << kJobWidthShift) - 1;
__host__ __device__ constexpr int class0BoxW(int w) { return w == 0 ? 208 : (w == 1 ? 144 : (w == 2 ? 112 : 80)); }
// Widths a kernel size uses: Lanczos4 (K = 8) keeps the whole width (with the narrow boxes cfg4 was 6 % slower in an
// A/B on an H100 SXM at 700 W; DESIGN.md section 6)
__host__ __device__ constexpr int class0Widths(int k) { return k == 8 ? 1 : kClass0Widths; }
// the narrowest width that holds `cols` bytes of a row
__host__ __device__ constexpr int class0WidthFor(int k, int cols) {
  int w = 0;
  while (w + 1 < class0Widths(k) && class0BoxW(w + 1) >= cols) ++w;
  return w;
}
// The tensor maps of a plane for kernel size k, one per box shape it uses: class 0 (width w, height variant v) at
// w * kBoxVariants + v, class 1, then the share box's heights (16 maps for K = 2 and 4, 7 for K = 8).
__host__ __device__ constexpr int boxMaps(int k) { return class0Widths(k) * kBoxVariants + 1 + kBoxVariants; }
constexpr int kMaxBoxMaps = kClass0Widths * kBoxVariants + 1 + kBoxVariants;
__host__ __device__ constexpr int boxMapIndex(int k, int cls, int width, int variant) {
  return cls == 0 ? width * kBoxVariants + variant : (cls == 1 ? class0Widths(k) * kBoxVariants : class0Widths(k) * kBoxVariants + 1 + variant);
}
__host__ __device__ constexpr int boxMapClass(int k, int i) {
  return i < class0Widths(k) * kBoxVariants ? 0 : (i == class0Widths(k) * kBoxVariants ? 1 : 2);
}
__host__ __device__ constexpr int boxMapW(int k, int i) { return boxMapClass(k, i) == 0 ? class0BoxW(i / kBoxVariants) : stageBoxW(k, boxMapClass(k, i)); }
__host__ __device__ constexpr int boxMapRows(int k, int i) {
  return boxMapClass(k, i) == 0 ? boxVariantRows(k, 0, i % kBoxVariants)
         : boxMapClass(k, i) == 1 ? stageBoxH(k, 1)
                                  : boxVariantRows(k, 2, i - class0Widths(k) * kBoxVariants - 1);
}

// Stages of a group's ring (a stage = one box + one record buffer).  Three fit beside the cubic tables if the boxes lose
// a few rows (not measured since no job reads its windows through L1 any more; at the time the third stage left too
// little L1 for those reads and made the frame slower, measured on the B200).
__host__ __device__ constexpr int gatherStages(int /*k*/) { return 2; }
// one stage buffer (TMA destinations need 128-byte alignment; the tail absorbs the over-read of a window's last word)
__host__ __device__ constexpr int stageBytesOf(int k) {
  const int a = stageBoxW(k, 2) * stageBoxH(k, 2), b = stageBoxW(k, 0) * stageBoxH(k, 0);
  return ((a > b ? a : b) + 64 + 127) & ~127;
}

// Weight tables in shared memory.  Phase a = (fracY << 5) | fracX lives in SLOT weightSlotOf(k, a); the K*K int16
// weights of a slot are K*K/8 16-byte vectors (k >= 4), vector v of copy c at byte
//     v * weightVectorStride(k, copies) + c * 16384 + slot * 16
// A 128-bit shared load is served 8 lanes (one quarter-warp) at a time out of 8 bank groups of 16 bytes, the group
// being slot & 7 = (fracX >> 1) & 7.  With 32 pixels per warp the fullest group holds ~6-7 of them whatever the hash
// (bank model: 6.3 wavefronts per load instead of 4).  So the cubic table is kept TWICE, the second copy rotated by one
// bank group (slot s of copy 1 sits where slot (s & ~7) | ((s + 1) & 7) of copy 0 would; rotations by 2 - 5 groups
// model worse), and the host -- which already deals the pixels of a row segment to lanes -- picks the copy per pixel so
// that the groups are evenly filled (an EMPTY group costs as much as an overfull one: a quarter-warp that finds no pixel
// in one group must take two of another) and then deals the pixels to quarter-warps exactly (gather_plan.cpp:
// GroupMatcher, PassDealer): 4.4 wavefronts per load in share jobs, 4.5 in tile jobs of the cfg2 plan in the offline bank
// model (profiles/weight_sim.py); with the group taken from fracX >> 2 it is 4.3 / 4.75, with a
// group that depends on fracY a share job's column could not keep its lane.
__host__ __device__ constexpr int weightSlotOf(int k, int phase) {
  (void)k;
  return (phase & ~31) | ((phase & 1) << 4) | ((phase & 31) >> 1);
}
__host__ __device__ constexpr int weightCopies(int k) { return k == 4 ? 2 : 1; }
__host__ __device__ constexpr int weightVectorStride(int k, int copies) { return (k == 2 ? 8192 : 16384) * copies; }
__host__ __device__ constexpr int weightImageBytes(int k, int copies) { return k == 2 ? 8192 * copies : (k * k / 8) * 16384 * copies; }
// position of slot s inside copy c (the rotation by one bank group)
__host__ __device__ constexpr int weightSlotInCopy(int slot, int copy) { return copy ? ((slot & ~7) | ((slot + copy) & 7)) : slot; }
// the slot field of a compact record: (position << 4) | (copy << 14), i.e. the byte offset of the slot's first vector
__host__ __device__ constexpr int weightSlotField(int k, int phase, int copy) {
  return (weightSlotInCopy(weightSlotOf(k, phase), copy) << 4) | (copy << 14);
}
constexpr int kSlotFieldMask = 0x7FF0;
// Lanczos4 has eight vectors per slot and room for one copy only (128 KB).  Its image is XOR-DIAGONAL: vector m of slot s
// sits in plane m at position s ^ m (low three bits), i.e. at byte  slotField ^ (m * kDiagonalStep)  of the image.  A
// pixel may then fetch its vectors in any XOR-rotated order m = v ^ r (v = 0 .. 7 the step, r private to the lane) and
// lands in bank group (s ^ r ^ v) & 7; with r = (s ^ lane) & 7 that is (lane ^ v) & 7: the eight lanes of a quarter-warp
// always ask for eight different bank groups, whatever their phases -- 4.0 wavefronts per 128-bit load by construction
// (it was 8.0).  The window rows are paired with the vectors through a three-stage exchange network in registers
// (integer sums do not care about the order).
constexpr int kDiagonalStep = 0x4010;  // one plane (16384 bytes) + one bank group (16 bytes)
__host__ __device__ constexpr bool weightDiagonal(int k) { return k == 8; }
__host__ __device__ constexpr int weightVectorOffset(int k, int copies, int slotFieldValue, int vector) {
  return weightDiagonal(k) ? (slotFieldValue ^ (vector * kDiagonalStep)) : slotFieldValue + vector * weightVectorStride(k, copies);
}
__host__ __device__ constexpr int weightBankGroups(int k) { return k == 2 ? 16 : 8; }
__host__ __device__ constexpr int weightLanesPerPass(int k) { return k == 2 ? 16 : 8; }

// Compact sampling records of the staged jobs (32-bit words, one buffer per plan, GatherJob::recordOffset):
//   share job    per warp w (columns 32 * (w & 1) .., rows R * (w >> 1) .., R = shareRows(k)): R / 8 blocks of 32 x uint4,
//                then 32 x uint32, by lane.  uint32 = header of the lane's column: off | column << 27,
//                off = (row0 - boxY) * 192 + (col0 - boxX) of the column's first pixel; uint4 number b = 8 x 16-bit pixel
//                records of rows 8b .., row j in half j & 1 of word (j >> 1) & 3: slotField | (d - 1), d = 1 or 2 source
//                rows between this pixel's window and the previous one's (bit 0 is clear in a column's first record);
//                kJobShareStay: slotField | d, d = 0, 1 or 2 (0 in the first record).
//                2.25 (R = 16) or 2.5 bytes per pixel.
//   other jobs   per warp w (rows 4 * w .. 4 * w + 3): 32 x uint4 by lane, word j = one pixel of the 8 x 4 patch at columns
//                8 * j ..: off (15 bits) | position << 16 (5 bits: column in patch | row in patch << 3) | slotField << 17.
//                4 bytes per pixel.  The pixels of a patch are dealt to lanes (and copies) per patch; pixels outside the
//                plane carry a position that fails the bounds check.
//   cap job      GatherJob::outX = its warp steps S (outY: no row); step s (warp s % 8) = 32 x uint2 by lane at byte 256 s:
//                {off (15 bits) | slotField << 17, or kRecordSkip;  outX | outY << 16 of the pixel in the plane}.
//                8 bytes per pixel; the 32 pixels of a step are dealt to lanes (and copies) like a patch.
//   border job   GatherJob::outX = its pixels n; pixel i = uint4 {col0, row0 << 10 | phase, outX | outY << 16, 0} at 16 i.
// The whole-plane general kernels read the full records below.
__host__ __device__ constexpr int shareWarpRecordBytes(int k) { return shareRows(k) / 8 * 32 * 16 + 32 * 4; }
__host__ __device__ constexpr int shareJobRecordBytes(int k) { return kGroupWarps * shareWarpRecordBytes(k); }
constexpr int kTileJobRecordBytes = kGroupWarps * 32 * 16;
// a quadrant job keeps the records of its four live warps and two live steps only: warp w & 3, 32 x uint2 by lane (words
// of steps 2 * (quadrant & 1) and 2 * (quadrant & 1) + 1)
constexpr int kQuadJobRecordBytes = kGroupWarps / 2 * 32 * 8;
__host__ __device__ constexpr int tileJobRecordBytes(int outXField) { return (outXField & kJobQuadMask) ? kQuadJobRecordBytes : kTileJobRecordBytes; }
// one stage of a ring: the header (padded to 128 bytes) and the records of a job
__host__ __device__ constexpr int stageRecordBytes(int k) {
  return 128 + (shareJobRecordBytes(k) > kTileJobRecordBytes ? shareJobRecordBytes(k) : kTileJobRecordBytes);
}
constexpr int kCapStepBytes = 32 * 8, kBorderPixelBytes = 16;
__host__ __device__ constexpr int capJobMaxSteps(int k) { return (stageRecordBytes(k) - 128) / kCapStepBytes; }
__host__ __device__ constexpr int borderJobMaxPixels(int k) { return (stageRecordBytes(k) - 128) / kBorderPixelBytes; }
// bytes of compact records of a job (outXField = GatherJob::outX)
__host__ __device__ constexpr int jobRecordBytes(int k, int kind, int outXField) {
  return kind == kJobShare || kind == kJobShareStay ? shareJobRecordBytes(k)
         : kind == kJobCap                          ? outXField * kCapStepBytes
         : kind == kJobBorder                       ? outXField * kBorderPixelBytes
                                                    : tileJobRecordBytes(outXField);
}
constexpr int kRecordColumnShift = 27;

// The persistent gather kernel takes the jobs of up to three image planes (Y, U, V of one frame) in ONE launch:
// one weight-table prologue and one tail per frame instead of per plane, and the dynamic scheduler balances the
// planes against each other.  Everything that differs between the planes sits in a PlaneView (+ its tensor maps).
constexpr int kMaxFramePlanes = 3;
struct PlaneView {
  const uint8_t* src;   // (blurred) input plane
  uint8_t* dst;
  const uint4* records; // compact records of the plane's jobs
  int srcW, srcH, srcPitch;
  int dstW, dstH, dstPitch;
};
struct FrameGatherParams {
  PlaneView plane[kMaxFramePlanes];
  const uint4* weightImage;  // device copy of the shared-memory image of the tables (weightImageBytes)
  int kernelSize, numPlanes;
};

// The general (whole plane, L1) kernels use FULL records, 8 bytes per pixel:
// {col0 | column << 27, row0 << 10 | phase}, tile-major over tiles of 32 x gatherTileH(k) pixels:
//   records[((ty * tilesPerRow + tx) * gatherTileH(k) + rowInTile) * 32 + lane]
// (tiles that stick out of the plane are padded with zero records).  Inside a 32-pixel row segment the records are in
// LANE order: the host deals the pixels of a segment to lanes by weight bank group (one order per 32 x 4 block).
__host__ __device__ constexpr int gatherThreads(int k) { return k == 8 ? 512 : 256; }
__host__ __device__ constexpr int gatherTileH(int k) { return gatherThreads(k) / 32 * 4; }  // 4 rows per thread

struct StagedParams {
  const GatherJob* tiles;  // device list
  int numTiles;
  int* claimCounter;        // two device ints, zero before the first launch (the kernel re-arms them): job scheduler
  // optional timeline for tuning (T360B200_debugTrace): per consumer group and job four 64-bit words
  // {wait start, data ready, done (ns, %globaltimer), kind}, kTraceJobsPerGroup jobs per group; nullptr = off
  unsigned long long* trace;
};
constexpr int kTraceJobsPerGroup = 64;

// One tile of the segmented low-pass: output rectangle and the taps to use.
struct BlurJob {
  int x0, y0, w, h;  // output rectangle (inside one plan segment)
  int kxOffset, kxCount, kyOffset, kyCount;
};

struct BlurParams {
  const uint8_t* src;
  uint8_t* dst;
  int width, height, srcPitch, dstPitch;
  const BlurJob* jobs;
  int numJobs;
  const float* taps;
  int tileSmemBytes;  // dynamic shared memory each block needs (max over jobs)
};

// One warp-job of the register-resident low-pass: a strip of up to 256 columns (8 per lane) x h rows inside one
// plan segment.  kxOffset points at the segment's horizontal taps zero-padded to kxChunks * 4 floats (16-byte
// aligned); kyOffset at the 2*hy+1 vertical taps.
struct StripJob {
  int x0, y0, w, h;
  int kxOffset, kxChunks, kxCount, kyOffset;
  int edge;  // 1: the strip's reads would cross the plane's left/right border -> clamped byte loads
};

struct StripParams {
  const uint8_t* src;
  uint8_t* dst;
  int width, height, srcPitch, dstPitch;
  const StripJob* jobs;
  int numJobs;
  const float* taps;
};

// cv::resize(INTER_AREA) shrink, one thread per destination pixel.  cellW > 0: integer ratios (sum of a cellW x cellH
// block, (sum+2)>>2 for 2x2, else rint(sum * (1.f/area))); otherwise the per-axis tap tables ({src, alpha} pairs,
// first[] offsets) with OpenCV's accumulation order: row sums over x taps, then weighted by the y taps.
struct AreaParams {
  const uint8_t* src;
  uint8_t* dst;
  int srcW, srcH, srcPitch, dstW, dstH, dstPitch;
  int cellW, cellH;
  const int2* xTaps;  // {src index, alpha bits}
  const int* xFirst;
  const int2* yTaps;
  const int* yFirst;
  // enlarging variant (cellW < 0): per destination column / row {source index, weight0 | weight1 << 16} (11-bit weights);
  // from xMax on a column reads its first source only.  dst = (((b0 * (H0 >> 4)) >> 16) + ((b1 * (H1 >> 4)) >> 16) + 2) >> 2,
  // H = S[sx] * a0 + S[sx + 1] * a1 per row.
  const int2* xLinear;
  const int2* yLinear;
  int xMax;
};
cudaError_t launchAreaResize(const AreaParams& p, cudaStream_t stream);

// One level of the input pyramids of a frame's planes in ONE launch (T360B200_transformFrameCameraMipAsync): dst =
// cv::resize(src, (ceil(srcW / 2), ceil(srcH / 2)), INTER_AREA) for every plane listed.  xTaps == nullptr: exact 2 x 2
// cells, (sum + 2) >> 2, four output bytes per thread; else the tap tables of buildAreaResize (AreaParams' layout) in
// OpenCV's accumulation order.  A block takes 128 x 8 output pixels; blocks are numbered through the planes in order.
struct PyramidPlane {
  const uint8_t* src;
  uint8_t* dst;
  int srcW, srcH, srcPitch, dstW, dstH, dstPitch;
  const int2* xTaps;
  const int* xFirst;
  const int2* yTaps;
  const int* yFirst;
  int firstBlock, blocksX;  // filled by launchPyramidLevel
};
struct PyramidParams {
  PyramidPlane plane[kMaxFramePlanes];
  int numPlanes;
};
constexpr int kPyramidBlockW = 128, kPyramidBlockH = 8;
cudaError_t launchPyramidLevel(PyramidParams p, cudaStream_t stream);

// The register-resident low-pass (hy <= kStripMaxHy) of 1-3 planes in ONE launch (StripJob::edge carries the plane in
// bits 8-9; kxOffset / kyOffset index the tap buffer, merged for several planes: lowpass_jobs.h): a frame takes one launch
// and one tail instead of three launches on three streams; a single plane's list has plane 0 throughout.
struct FrameStripParams {
  struct Plane {
    const uint8_t* src;
    uint8_t* dst;
    int width, height, srcPitch, dstPitch;
  } plane[kMaxFramePlanes];
  int numPlanes;
  const StripJob* jobs;
  int numJobs;
  const float* taps;
};
constexpr int kStripPlaneShift = 8;
cudaError_t launchBlurFrameStrips(const FrameStripParams& p, int hy, cudaStream_t stream);

constexpr int kStripLanePx = 8, kStripW = 32 * kStripLanePx, kStripMaxHy = 3;

constexpr int kBlurTileW = 64, kBlurTileH = 32;
constexpr int kBlurMaxSmem = 96 * 1024;

// Launchers: enqueue on `stream`, return the CUDA status of the launch.  Each counts the kernels it launches.
// General path for a whole plane: taps through L1, every border mode (BORDER_WRAP, BORDER_TRANSPARENT), nearest.
cudaError_t launchGather(const GatherParams& p, int numSMs, cudaStream_t stream);
// Whole planes in one persistent kernel: `jobs` lists the jobs of every plane in launch order (gather_plan.h:
// jobLaunchRank).  tensorMaps: per plane kMaxBoxMaps CUtensorMap (128 bytes each), of which the first
// boxMaps(p.kernelSize) describe its source with the staging boxes of p.kernelSize (boxMapIndex), i.e.
// [numPlanes][kMaxBoxMaps].  BORDER_WRAP only.  The kernel takes boxMaps(k) maps per plane as a parameter: 6 KB for
// K = 2 and 4, more than 4 KB of kernel parameters, which needs CUDA 12.1 and a driver of the R530 series or newer.
// programmatic: allow the launch to overlap the tail of the previous kernel on the stream (programmatic dependent launch).
cudaError_t launchGatherFrame(const FrameGatherParams& p, const StagedParams& jobs, const void* tensorMaps, int numSMs,
                              cudaStream_t stream, bool programmatic = true);
// one-time set-up of the frame kernel for kernelSize on the current device (shared-memory opt-in, occupancy): call it
// before capturing launchGatherFrame into a CUDA graph
cudaError_t prepareGatherFrame(int kernelSize);
cudaError_t launchBlur(const BlurParams& p, cudaStream_t stream);        // shared-memory tiles
cudaError_t launchBlurDirect(const BlurParams& p, cudaStream_t stream);  // any kernel size, slow
unsigned long long kernelLaunchCount();
void countKernelLaunches(long long n);  // kernels launched through a replayed CUDA graph

// ---- the per-frame gathers (view_gather.cu) ------------------------------------------------------------------------
// Frames rendered without a sampling plan: the kernel computes every pixel's sampling record itself from per-frame
// constants passed with the launch, so nothing is re-planned when they change.  One launch gathers every plane of the
// frame.  The source names where a record comes from:
//   kView         FLAT_FIXED views (yaw, pitch, hfov, vfov: view; flat_view.h), BORDER_WRAP;
//   kSphere       every other layout with an orientation (rotation) and the plan's view-independent tables
//                 (oriented_view.h: sphereSample), BORDER_WRAP, or BORDER_TRANSPARENT for BARREL and BARREL_SPLIT;
//   kMap          the caller's CV_32FC2 map of each plane, quantised as quantizeWarpMap does (quantizeAxis), BORDER_WRAP
//                 or BORDER_TRANSPARENT (transparent);
//   kLens         a fisheye lens rig (rotation, rig; oriented_view.h: lensSample) to a sphere output, with the output
//                 layout's tables, BORDER_TRANSPARENT;
//   kLensBlend    a two-lens rig with the seam feathered across a belt (rotation, rig, seamScale; lensBlendSample): every
//                 pixel gathers the lens that carries it (lens 0 unless the weight w of lens 1 is 256), and a second time,
//                 lens 1, only where both carry weight; the two values are blended as (a (256 - w) + b w + 128) >> 8;
//   kRectilinear  perspective views posed per frame (camera; rectilinearSample): a pinhole ray per pixel, no tables, looked
//                 up in the context's input (BORDER_WRAP) or, with lens set, in the rig's lenses (BORDER_TRANSPARENT);
//   kCameraMip    anti-aliased camera views (camera, mip, mipBias; mipCameraSample): kRectilinear's chain plus the pixel's
//                 footprint, which picks a level of the plane's pyramid and the weight w (0..255) of the next one; the
//                 pixel gathers its level, and the next level only where w > 0, blended as kLensBlend blends.
//   kLensPhoto    a lens rig with photometry (rotation, rig, seamScale, photo; lensPhotoSample): the hard seam
//                 (seamScale = 0) or the feathered one; each lens's sample is corrected with its gain (photoCorrect)
//                 before the seam combines them, and with photo.stats set the overlap's sums are accumulated.
//   kCameraPhoto  a camera view of a lens rig with photometry (camera, rig, seamScale, mip, mipBias, photo;
//                 cameraPhotoSample): each lens's sample is the blend of its own two levels (kCameraMip's blend; level 0
//                 alone without a pyramid), then corrected, combined and counted as kLensPhoto's.
//   kStereoCamera a camera view of a stereo rig (kCameraPhoto's constants, no seam; cameraPhotoSample<MIP, true>): the
//                 output eye split of the context's output_stereo_format, and eye e's pixels take lens e alone.
//   kLensMotion   kLensPhoto with a rig motion over the readout (rotation, rig, seamScale, photo, motion;
//                 lensMotionSample): each lens's M follows the readout time of the point it projects.
//   kCameraMotion kCameraPhoto with a rig motion (kCameraPhoto's constants and motion; cameraMotionSample).
//   kCameraAniso  anisotropic camera views (kCameraMip's constants and cameraAniso; anisoFootprint, anisoCameraSample):
//                 the pixel's footprint once, then up to 2^cameraAniso probes along its longer axis, each gathered as
//                 kCameraMip gathers a pixel, averaged over the probes BORDER_TRANSPARENT does not skip.
enum class PerFrameSource { kView, kSphere, kMap, kLens, kLensBlend, kRectilinear, kCameraMip, kLensPhoto, kCameraPhoto, kStereoCamera,
                            kLensMotion, kCameraMotion, kCameraAniso };
struct PerFramePlane {
  const uint8_t* src;  // (blurred) input plane, geometry.inW x geometry.inH
  uint8_t* dst;        // render target, geometry.mapW x geometry.mapH
  int srcPitch, dstPitch;
  SphereGeometry geometry;  // (kMap reads the four sizes only)
  const float* colTable;    // sphere tables (buildSphereTables): column entries, then row entries (nullptr: none)
  const float* rowTable;
  int tilesX, firstTile;    // filled by launchPerFrameGather
  const float2* map;        // kMap: [mapH][mapPitch] (x, y) source positions
  int mapPitch;             // in float2
};
// The per-frame constants a source does not read stay zero.
struct PerFrameGatherParams {
  PerFramePlane plane[kMaxFramePlanes];
  int numPlanes;
  FlatView view;
  Rotation rotation;
  LensRigModel rig;
  RectilinearCamera camera;
  float seamScale;   // s = 1 / (2 seamWidth), seamWidth in radians
  bool transparent;  // kMap: BORDER_TRANSPARENT instead of BORDER_WRAP
  bool lens;         // kRectilinear: the rig's lenses instead of the context's input
  uint8_t cameraAniso;  // kCameraAniso: log2 maxProbes
  const int16_t* weights;  // device copy of the [1024][k][k] table (nullptr for nearest)
  int kernelSize;
  // the pyramid sources (kCameraMip, kCameraAniso, kCameraPhoto, kStereoCamera, kCameraMotion): per plane its footprint
  // constants and pyramid levels 1..geometry.top (level 0 is the plane's src), and round(256 lodBias)
  struct MipLevel {
    uint8_t* bytes;  // written by the level's pyramid launch, read by the gather
    int w, h, pitch;
  };
  struct MipPlane {
    MipGeometry geometry;
    MipLevel level[kMipMaxLevels];  // [l - 1]: level l
  };
  MipPlane mip[kMaxFramePlanes];
  int mipBias;
  // the photometric sources (kLensPhoto, kCameraPhoto, kStereoCamera, kLensMotion, kCameraMotion): per plane its
  // photometric constants, and the statistics buffer ([numPlanes][6] sums: n, sum a', sum b', sum a'^2, sum b'^2, sum a'b',
  // zeroed by the caller in stream order; nullptr: none)
  struct LensPhoto {
    LensPhotoPlane plane[kMaxFramePlanes];
    unsigned long long* stats;
  };
  LensPhoto photo;
  // the motion sources (kLensMotion, kCameraMotion): the rig motion (its sample table staged in device memory, numSamples
  // and the lenses' readouts)
  RigMotion motion;
};
// (the block and the launch's numTiles within the 4 KB of kernel parameters every driver accepts)
static_assert(sizeof(PerFrameGatherParams) + sizeof(int) <= 4096);
constexpr int kPhotoStats = 6;  // sums per plane of kLensPhoto's statistics
// a CTA takes tiles of 32 output columns x viewTileRows(k) rows; a thread owns one column of a tile and walks down
// kViewRowsPerThread of its rows
constexpr int kViewRowsPerThread = 8;
__host__ __device__ constexpr int viewTileRows(int k) { return gatherThreads(k) / 32 * kViewRowsPerThread; }
// (every plane of a frame has the same output layout)
cudaError_t launchPerFrameGather(PerFrameGatherParams p, PerFrameSource source, int numSMs, cudaStream_t stream);

// bytes of dynamic shared memory a blur tile of (w x h) with the given tap counts needs
inline int blurTileSmem(int w, int h, int nkx, int nky) {
  const int hx = nkx / 2, hy = nky / 2;
  const int rows = h + 2 * hy;
  const int srcStride = (w + 2 * hx + 3) & ~3;
  return rows * srcStride + rows * w * 4;
}

}  // namespace t360
