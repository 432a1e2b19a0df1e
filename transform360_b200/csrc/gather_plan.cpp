// Host side of the gather plan: job classification and record layout (see gather_plan.h, kernels.cuh).
#include "gather_plan.h"

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <thread>
#include <utility>

namespace t360 {
namespace {

// fn(begin, end) over [0, n) on up to 32 host threads (the work items are independent and write disjoint outputs)
template <class F>
void parallelRanges(int n, size_t workPerItem, F fn) {
  unsigned nt = std::thread::hardware_concurrency();
  if (nt == 0) nt = 1;
  if (nt > 32) nt = 32;
  if (static_cast<size_t>(n) * workPerItem < (1u << 16)) nt = 1;
  const int chunk = (n + static_cast<int>(nt) - 1) / static_cast<int>(nt);
  std::vector<std::thread> pool;
  for (unsigned t = 1; t < nt; ++t) {
    const int b = static_cast<int>(t) * chunk, e = std::min(n, b + chunk);
    if (b < e) pool.emplace_back(fn, b, e);
  }
  fn(0, std::min(n, chunk));
  for (auto& th : pool) th.join();
}

// ---- bank-group balancing ------------------------------------------------------------------------------------
// Pixel i may read its weights from copy c of the table, which puts it into bank group (base[i] + c) & 7.  Finds an
// assignment in which no group takes more than `cap` pixels (augmenting paths; 32 pixels, 8 groups).
struct GroupMatcher {
  int n, copies, cap;
  const int* base;
  int groupOf[32], load[8];
  bool visited[8];

  bool place(int i) {
    for (int c = 0; c < copies; ++c) {
      const int g = (base[i] + c) & 7;
      if (visited[g]) continue;
      visited[g] = true;
      if (load[g] < cap) {
        ++load[g];
        groupOf[i] = g;
        return true;
      }
      for (int j = 0; j < n; ++j) {
        if (j == i || groupOf[j] != g) continue;
        groupOf[j] = -1;  // try to move j elsewhere (its other choices; g itself is marked visited)
        if (place(j)) {   // j took a seat in another group: g keeps its load, i takes j's seat
          groupOf[i] = g;
          return true;
        }
        groupOf[j] = g;
      }
    }
    return false;
  }
  bool run() {
    std::fill(groupOf, groupOf + 32, -1);
    std::fill(load, load + 8, 0);
    for (int i = 0; i < n; ++i) {
      std::fill(visited, visited + 8, false);
      if (!place(i)) return false;
    }
    return true;
  }
  // After run(): evens the loads out below the cap as well.  A pass (quarter-warp) is full only if it finds a pixel in
  // every group it may not take two of, so an EMPTY group costs as much as an overfull one (loads 4,4,4,0,5,5,5,5 deal
  // to 2+2+2+2 = 8 wavefronts, 4,4,3,1,5,5,5,5 to 5).  Moves one pixel along a chain of groups from a group with load L
  // to one with load <= L - 2 while such a chain exists (every move lowers the sum of squared loads).
  void balance() {
    for (bool improved = true; improved;) {
      improved = false;
      for (int src = 0; src < 8 && !improved; ++src) {
        int from[8], via[8], queue[8], head = 0, tail = 0;
        std::fill(from, from + 8, -1);
        from[src] = src;
        queue[tail++] = src;
        while (head < tail && !improved) {
          const int g = queue[head++];
          for (int j = 0; j < n && !improved; ++j) {
            if (groupOf[j] != g) continue;
            for (int c = 0; c < copies; ++c) {
              const int t = (base[j] + c) & 7;
              if (from[t] >= 0) continue;
              from[t] = g;
              via[t] = j;
              queue[tail++] = t;
              if (load[t] + 2 <= load[src]) {  // shift one pixel along src -> .. -> t
                for (int cur = t; cur != src; cur = from[cur]) groupOf[via[cur]] = cur;
                ++load[t];
                --load[src];
                improved = true;
                break;
              }
            }
          }
        }
      }
    }
  }
};

// Full records: device order of the 8-byte sampling records the general kernels read.  Each row is cut into segments
// of 32 pixels (= one warp); inside a segment the pixels are dealt to LANES by weight bank group (one order per
// 32 x 4 block, so that a thread keeps one output column).  The pixel's column travels in the record's top 5 bits.
void buildFullRecords(const HostPlan& h, std::vector<int2>& out, int tilesPerRow, int tileH) {
  const int k = h.kernelSize;
  constexpr int kRows = 4;
  parallelRanges((h.mapH + kRows - 1) / kRows, static_cast<size_t>(h.mapW) * kRows, [&](int blockBegin, int blockEnd) {
  for (int yb = blockBegin * kRows; yb < blockEnd * kRows; yb += kRows) {
    for (int x0 = 0; x0 < h.mapW; x0 += 32) {
      const int n = std::min(32, h.mapW - x0);
      int laneOf[32], copyOf[32], slot[32];
      const SamplePoint* first = &h.samples[static_cast<size_t>(yb) * h.mapW];
      for (int i = 0; i < n; ++i) slot[i] = k >= 2 ? weightSlotOf(k, first[x0 + i].rowPhase & 1023) : 0;
      if (k >= 2) dealLanes(k, 1, n, slot, laneOf, copyOf);
      else for (int i = 0; i < n; ++i) laneOf[i] = i;
      for (int y = yb; y < std::min(h.mapH, yb + kRows); ++y) {
        const SamplePoint* row = &h.samples[static_cast<size_t>(y) * h.mapW];
        const size_t tile = static_cast<size_t>(y / tileH) * tilesPerRow + x0 / 32;
        int2* dst = &out[(tile * tileH + y % tileH) * 32];
        for (int c = 0; c < n; ++c) {
          const SamplePoint& sp = row[x0 + c];
          dst[laneOf[c]] = int2{static_cast<int>((static_cast<unsigned>(sp.col0) & ((1u << kRecordColumnShift) - 1)) |
                                                 (static_cast<unsigned>(c) << kRecordColumnShift)),
                                sp.rowPhase};
        }
      }
    }
  }
  });
}

struct TileClass {
  int kind = -1;  // kJob*; -1: covered by the share job that starts at the tile to its left (or at this tile)
  int boxX = 0, boxY = 0, boxRows = 0;  // boxRows: the source rows the job's windows really span (<= the class's box height)
  bool shareStart = false;
  bool quads = false;  // four class-0 jobs, one per 16 x 16 quadrant, each with its own box
  int quadBoxX[4] = {}, quadBoxY[4] = {}, quadBoxRows[4] = {};
};

// Bounding box of the source windows of a block of output pixels.
struct Extent {
  int minC = INT32_MAX, maxC = INT32_MIN, minR = INT32_MAX, maxR = INT32_MIN;
};
Extent extentOf(const HostPlan& h, int x0, int y0, int x1, int y1) {
  Extent e;
  for (int y = y0; y < y1; ++y) {
    const SamplePoint* row = &h.samples[static_cast<size_t>(y) * h.mapW];
    for (int x = x0; x < x1; ++x) {
      const int c = row[x].col0, r = row[x].rowPhase >> 10;
      e.minC = std::min(e.minC, c); e.maxC = std::max(e.maxC, c);
      e.minR = std::min(e.minR, r); e.maxR = std::max(e.maxR, r);
    }
  }
  return e;
}

// A 64 x shareH block qualifies as a share job when every column keeps its first source column down the rows, steps
// 1 or 2 source rows per output row (0 - 2: kJobShareStay), and the windows of the whole block fit one 192-byte-wide
// box inside the plane.
bool shareBlock(const HostPlan& h, int x0, int y0, TileClass& out) {
  const int k = h.kernelSize, kShareH = shareH(k);
  if (k < 4 || x0 + kShareW > h.mapW || y0 + kShareH > h.mapH) return false;
  bool stays = false;
  for (int y = y0 + 1; y < y0 + kShareH; ++y) {
    const SamplePoint* a = &h.samples[static_cast<size_t>(y - 1) * h.mapW + x0];
    const SamplePoint* b = a + h.mapW;
    for (int x = 0; x < kShareW; ++x) {
      const int d = (b[x].rowPhase >> 10) - (a[x].rowPhase >> 10);
      if (b[x].col0 != a[x].col0 || d < 0 || d > 2) return false;
      stays = stays || d == 0;
    }
  }
  const Extent e = extentOf(h, x0, y0, x0 + kShareW, y0 + kShareH);
  if (e.minC < 0 || e.minR < 0 || e.maxC + k > h.inW || e.maxR + k > h.inH) return false;
  const int boxX = e.minC & ~15;
  if (e.maxC + k - boxX > stageBoxW(k, 2) || e.maxR + k - e.minR > stageBoxH(k, 2)) return false;
  out.kind = stays ? kJobShareStay : kJobShare;
  out.boxX = boxX;
  out.boxY = e.minR;
  out.boxRows = e.maxR + k - e.minR;
  out.shareStart = true;
  return true;
}

// class of the box that holds the windows of the pixel block [x0, x1) x [y0, y1): 0, 1 or -1
int boxClassFor(const HostPlan& h, int x0, int y0, int x1, int y1, int maxClass, int* boxX, int* boxY, int* boxRows) {
  const int k = h.kernelSize;
  const Extent e = extentOf(h, x0, y0, x1, y1);
  if (e.minC < 0 || e.minR < 0 || e.maxC + k > h.inW || e.maxR + k > h.inH) return -1;
  *boxX = e.minC & ~15;
  *boxY = e.minR;
  *boxRows = e.maxR + k - e.minR;
  for (int cls = 0; cls <= maxClass; ++cls)
    if (e.maxC + k - *boxX <= stageBoxW(k, cls) && e.maxR + k - e.minR <= stageBoxH(k, cls)) return cls;
  return -1;
}

void classifyTile(const HostPlan& h, int x0, int y0, bool seamPossible, TileClass& out) {
  const int k = h.kernelSize;
  const int x1 = std::min(h.mapW, x0 + kGatherTileW), y1 = std::min(h.mapH, y0 + kFrameTileH);
  const int cls = boxClassFor(h, x0, y0, x1, y1, 1, &out.boxX, &out.boxY, &out.boxRows);
  if (cls == 0) {
    out.kind = kJobClass0;
    return;
  }
  // The ring around a pole cap: the tile's windows span hundreds of columns, those of a 16 x 16 quadrant fit a class-0
  // box.  Also preferred to a class-1 job, whose box takes both stage buffers of a group and so cannot be loaded while
  // the group computes (its group waits for every class-1 job's data; class-0 boxes arrive while the previous job runs).
  if (x1 - x0 == kGatherTileW && y1 - y0 == kFrameTileH) {
    bool all = true;
    for (int q = 0; q < 4 && all; ++q) {
      const int qx = x0 + 16 * (q & 1), qy = y0 + 16 * (q >> 1);
      all = boxClassFor(h, qx, qy, qx + 16, qy + 16, 0, &out.quadBoxX[q], &out.quadBoxY[q], &out.quadBoxRows[q]) == 0;
    }
    if (all) {
      out.kind = kJobClass0;
      out.quads = true;
      return;
    }
  }
  if (cls == 1) {
    out.kind = kJobClass1;
    return;
  }
  // windows that cross the left/right border only (BORDER_WRAP): do they fit a class-0 box that wraps around it?
  const Extent e = extentOf(h, x0, y0, x1, y1);
  if (seamPossible && e.minR >= 0 && e.maxR + k <= h.inH && e.maxR + k - e.minR <= stageBoxH(k, 0)) {
    const int W = h.inW, half = W / 2;  // columns rotated by half a plane: the border is in the middle of the range
    int lo = INT32_MAX, hi = INT32_MIN;
    for (int y = y0; y < y1; ++y)
      for (int x = x0; x < x1; ++x) {
        int cw = h.samples[static_cast<size_t>(y) * h.mapW + x].col0 % W;
        if (cw < 0) cw += W;
        const int rot = cw + half >= W ? cw + half - W : cw + half;
        lo = std::min(lo, rot); hi = std::max(hi, rot);
      }
    const int first = lo - half < 0 ? lo - half + W : lo - half;  // leftmost first column, in plane coordinates
    const int bx = first & ~15;
    if (hi - lo + (first - bx) + k <= stageBoxW(k, 0) && bx + stageBoxW(k, 0) > W) {
      out.kind = kJobSeam;
      out.boxX = bx;
      out.boxY = e.minR;
      out.boxRows = e.maxR + k - e.minR;
      return;
    }
  }
  out.kind = kJobGeneral;  // no box holds the tile: its pixels go to coverPoleCaps
  out.boxX = out.boxY = out.boxRows = 0;
}

inline uint32_t slotField(int k, int phase, int copy) { return static_cast<uint32_t>(weightSlotField(k, phase, copy)); }

// compact records of a share job (kernels.cuh)
void writeShareRecords(const HostPlan& h, const GatherJob& job, uint32_t* out) {
  const int k = h.kernelSize, copies = weightCopies(k), kShareRows = shareRows(k), kShareH = shareH(k);
  const int x0 = job.outX, y0 = job.outY & kJobRowMask, boxX = jobBoxX(job.boxXY), boxY = jobBoxY(job.boxXY);
  const int pitch = stageBoxW(k, 2);
  const bool stay = ((job.outY >> kJobKindShift) & kJobKindMask) == kJobShareStay;
  for (int wx = 0; wx < kShareW / 32; ++wx) {
    for (int wy = 0; wy < kShareH / kShareRows; ++wy) {
      // the bank group of a pixel's weights depends on fracX only, which a column keeps (up to rounding jitter of the
      // map): one lane order and one copy choice per column and warp, found on the warp's first row
      int slot[32], laneOf[32], copyOf[32];
      const SamplePoint* first = &h.samples[static_cast<size_t>(y0 + wy * kShareRows) * h.mapW + x0 + wx * 32];
      for (int i = 0; i < 32; ++i) slot[i] = weightSlotOf(k, first[i].rowPhase & 1023);
      dealLanes(k, copies, 32, slot, laneOf, copyOf);
      const int w = wy * (kShareW / 32) + wx;
      uint32_t* words = out + static_cast<size_t>(w) * (shareWarpRecordBytes(k) / 4);
      uint32_t* headers = words + kShareRows / 8 * 32 * 4;
      for (int c = 0; c < 32; ++c) {
        const int lane = laneOf[c], x = x0 + wx * 32 + c, ya = y0 + wy * kShareRows;
        const SamplePoint* col = &h.samples[static_cast<size_t>(ya) * h.mapW + x];
        const int off = ((col->rowPhase >> 10) - boxY) * pitch + (col->col0 - boxX);
        headers[lane] = static_cast<uint32_t>(off) | (static_cast<uint32_t>(c) << kRecordColumnShift);
        for (int j = 0; j < kShareRows; ++j) {
          const SamplePoint& sp = col[static_cast<size_t>(j) * h.mapW];
          const int first = stay ? 0 : 1;
          const int d = j == 0 ? first : (sp.rowPhase >> 10) - (col[static_cast<size_t>(j - 1) * h.mapW].rowPhase >> 10);
          const uint32_t rec = slotField(k, sp.rowPhase & 1023, copyOf[c]) | static_cast<uint32_t>(d - first);  // kJobShare: bit 0 = a second row
          uint32_t& word = words[(j >> 3) * 32 * 4 + lane * 4 + ((j >> 1) & 3)];
          word = (j & 1) ? (word | (rec << 16)) : rec;
        }
      }
    }
  }
}

// compact records of a 32 x 32 job (class 0, class 1): warp w takes rows 4w .. 4w+3 in four steps of one 8 x 4 patch
// each (a compact patch keeps the 32 source windows of a step close together: 1.6 shared-memory wavefronts per window
// load in the bank model where a 32 x 1 row segment costs 2.2 on the polar faces)
void writeTileRecords(const HostPlan& h, const GatherJob& job, uint32_t* out) {
  const int k = h.kernelSize, copies = weightCopies(k);
  const int kind = (job.outY >> kJobKindShift) & kJobKindMask;
  const int x0 = job.outX & ~kJobQuadMask, y0 = job.outY & kJobRowMask, boxX = jobBoxX(job.boxXY), boxY = jobBoxY(job.boxXY);
  const int pitch = stageBoxW(k, boxClassOf(kind));
  // the live rectangle: the whole tile, or one quadrant
  const int quad = (job.outX & kJobQuadMask) - 1;
  const int lx0 = quad < 0 ? x0 : x0 + 16 * (quad & 1), ly0 = quad < 0 ? y0 : y0 + 16 * (quad >> 1);
  const int lx1 = quad < 0 ? x0 + kGatherTileW : lx0 + 16, ly1 = quad < 0 ? y0 + kFrameTileH : ly0 + 16;
  for (int w = 0; w < kGroupWarps; ++w)
    for (int j = 0; j < kRowsPerPatchStep; ++j) {
      // a quadrant job: only its live warps (rows) and steps (columns) have records, 32 x uint2 per warp
      if (quad >= 0 && ((w >> 2) != (quad >> 1) || (j >> 1) != (quad & 1))) continue;
      uint32_t* words = quad < 0 ? out + static_cast<size_t>(w) * 32 * 4 : out + static_cast<size_t>(w & 3) * 32 * 2;
      const int stride = quad < 0 ? 4 : 2, word = quad < 0 ? j : (j & 1);
      // the pixels of the patch that exist, in position order; the others keep a position that fails the bounds check
      int slot[32], laneOf[32], copyOf[32], posOf[32], n = 0;
      bool present[32] = {};
      for (int pos = 0; pos < 32; ++pos) {
        const int x = x0 + kTilePatchW * j + (pos & (kTilePatchW - 1)), y = y0 + kTilePatchH * w + pos / kTilePatchW;
        if (x >= h.mapW || y >= h.mapH || x < lx0 || x >= lx1 || y < ly0 || y >= ly1) continue;
        present[pos] = true;
        posOf[n] = pos;
        slot[n++] = weightSlotOf(k, h.samples[static_cast<size_t>(y) * h.mapW + x].rowPhase & 1023);
      }
      dealLanes(k, copies, n, slot, laneOf, copyOf);  // n < 32: identity order
      int lane = n;
      for (int pos = 0; pos < 32; ++pos)
        if (!present[pos]) words[(lane++) * stride + word] = (static_cast<uint32_t>(pos) << 16) | kRecordSkip;
      for (int i = 0; i < n; ++i) {
        const int pos = posOf[i];
        const int x = x0 + kTilePatchW * j + (pos & (kTilePatchW - 1)), y = y0 + kTilePatchH * w + pos / kTilePatchW;
        const SamplePoint& sp = h.samples[static_cast<size_t>(y) * h.mapW + x];
        int col0 = sp.col0;
        if (kind == kJobSeam) {  // first column relative to the unwrapped box (boxX <= col0 < boxX + box width)
          int cw = col0 % h.inW;
          if (cw < 0) cw += h.inW;
          col0 = boxX + (cw - boxX + h.inW) % h.inW;
        }
        const int off = ((sp.rowPhase >> 10) - boxY) * pitch + (col0 - boxX);
        words[laneOf[i] * stride + word] = static_cast<uint32_t>(off) | (static_cast<uint32_t>(pos) << 16) |
                                           (slotField(k, sp.rowPhase & 1023, copyOf[i]) << 17);
      }
    }
}

// The output rectangle of a tile or share job (not clipped to the plane).
JobRect tileRect(const GatherJob& job, int k) {
  const int kind = (job.outY >> kJobKindShift) & kJobKindMask, quad = (job.outX & kJobQuadMask) - 1;
  JobRect r;
  r.x0 = job.outX & ~kJobQuadMask;
  r.y0 = job.outY & kJobRowMask;
  if (quad >= 0) { r.x0 += 16 * (quad & 1); r.y0 += 16 * (quad >> 1); }
  const bool share = kind == kJobShare || kind == kJobShareStay;
  r.x1 = r.x0 + (quad >= 0 ? 16 : (share ? kShareW : kGatherTileW));
  r.y1 = r.y0 + (quad >= 0 ? 16 : (share ? shareH(k) : kFrameTileH));
  return r;
}

// A pole-cap or border job with its records, before it has a place in the plan's record buffer.
struct PixelJob {
  GatherJob job;
  std::vector<uint32_t> words;
  JobRect rect;
  int needRows;
};

struct CapPixel {
  int x, y, col0, rowPhase;
  int row() const { return rowPhase >> 10; }
};

PixelJob capJob(const HostPlan& h, const CapPixel* px, int n) {
  const int k = h.kernelSize, copies = weightCopies(k), pitch = stageBoxW(k, 0);
  PixelJob j;
  int minC = INT32_MAX, minR = INT32_MAX, maxR = INT32_MIN;
  j.rect = JobRect{INT32_MAX, INT32_MAX, INT32_MIN, INT32_MIN};
  for (int i = 0; i < n; ++i) {
    minC = std::min(minC, px[i].col0);
    minR = std::min(minR, px[i].row());
    maxR = std::max(maxR, px[i].row());
    j.rect = JobRect{std::min(j.rect.x0, px[i].x), std::min(j.rect.y0, px[i].y), std::max(j.rect.x1, px[i].x + 1), std::max(j.rect.y1, px[i].y + 1)};
  }
  const int boxX = minC & ~15, boxY = minR, steps = (n + 31) / 32;
  j.job = GatherJob{steps, kJobCap << kJobKindShift, jobBoxField(boxX, boxY, boxVariantFor(k, 0, maxR + k - minR)), 0};
  j.needRows = maxR + k;
  j.words.assign(static_cast<size_t>(steps) * kCapStepBytes / 4, 0u);
  for (int s = 0; s < steps; ++s) {
    const CapPixel* step = px + 32 * s;
    const int m = std::min(32, n - 32 * s);
    int slot[32], laneOf[32], copyOf[32];
    for (int i = 0; i < m; ++i) slot[i] = weightSlotOf(k, step[i].rowPhase & 1023);
    dealLanes(k, copies, m, slot, laneOf, copyOf);  // m < 32: identity order
    uint32_t* words = &j.words[static_cast<size_t>(s) * kCapStepBytes / 4];
    for (int lane = m; lane < 32; ++lane) words[2 * lane] = kRecordSkip;
    for (int i = 0; i < m; ++i) {
      const int off = (step[i].row() - boxY) * pitch + (step[i].col0 - boxX);
      words[2 * laneOf[i]] = static_cast<uint32_t>(off) | (slotField(k, step[i].rowPhase & 1023, copyOf[i]) << 17);
      words[2 * laneOf[i] + 1] = static_cast<uint32_t>(step[i].x) | (static_cast<uint32_t>(step[i].y) << 16);
    }
  }
  return j;
}

PixelJob borderJob(const HostPlan& h, const CapPixel* px, int n) {
  PixelJob j;
  j.job = GatherJob{n, kJobBorder << kJobKindShift, 0, 0};
  j.needRows = 0;  // (a window that wraps vertically reads the last rows)
  j.rect = JobRect{INT32_MAX, INT32_MAX, INT32_MIN, INT32_MIN};
  j.words.assign(static_cast<size_t>(n) * kBorderPixelBytes / 4, 0u);
  for (int i = 0; i < n; ++i) {
    j.words[4 * i] = static_cast<uint32_t>(px[i].col0);
    j.words[4 * i + 1] = static_cast<uint32_t>(px[i].rowPhase);
    j.words[4 * i + 2] = static_cast<uint32_t>(px[i].x) | (static_cast<uint32_t>(px[i].y) << 16);
    j.needRows = std::max(j.needRows, px[i].row() >= 0 && px[i].row() + h.kernelSize <= h.inH ? px[i].row() + h.kernelSize : h.inH);
    j.rect = JobRect{std::min(j.rect.x0, px[i].x), std::min(j.rect.y0, px[i].y), std::max(j.rect.x1, px[i].x + 1), std::max(j.rect.y1, px[i].y + 1)};
  }
  return j;
}

// The pixels of the tiles that no box holds (the pole caps: a tile's windows span hundreds of source columns there) are
// grouped by SOURCE position instead: bands of source rows that fit a class-0 box, each cut greedily into runs of columns
// that fit one (the fewest boxes for the band), each box into jobs of at most capJobMaxSteps(k) warp steps.  Inside a
// job the pixels go in output order, so that a warp's byte stores land in as few output rows as the wedge allows.
// Pixels whose window leaves the plane (BORDER_WRAP; NaN map entries) go to border jobs, per tile: a job's output
// rectangle and source rows stay those of one tile (a plane streamed in row bands gets its output bands back early).
void coverPoleCaps(const HostPlan& h, const std::vector<TileClass>& cls, int tilesX, int tilesY, std::vector<PixelJob>& out) {
  const int k = h.kernelSize, boxW = stageBoxW(k, 0), boxH = stageBoxH(k, 0);
  std::vector<CapPixel> cap, border;
  std::vector<size_t> tileBorderStart;  // the border pixels of a tile are border[tileBorderStart[i] .. [i + 1])
  for (int ty = 0; ty < tilesY; ++ty)
    for (int tx = 0; tx < tilesX; ++tx) {
      if (cls[static_cast<size_t>(ty) * tilesX + tx].kind != kJobGeneral) continue;
      tileBorderStart.push_back(border.size());
      for (int y = ty * kFrameTileH; y < std::min(h.mapH, (ty + 1) * kFrameTileH); ++y)
        for (int x = tx * kGatherTileW; x < std::min(h.mapW, (tx + 1) * kGatherTileW); ++x) {
          const SamplePoint& sp = h.samples[static_cast<size_t>(y) * h.mapW + x];
          const CapPixel p{x, y, sp.col0, sp.rowPhase};
          const bool inside = p.col0 >= 0 && p.row() >= 0 && p.col0 + k <= h.inW && p.row() + k <= h.inH;
          (inside ? cap : border).push_back(p);
        }
    }
  if (cap.empty() && border.empty()) return;
  if (h.mapW > 65536 || h.mapH > 65536) throw std::invalid_argument("gather plan: pole-cap records hold 16-bit output positions");
  auto outputOrder = [](const CapPixel& a, const CapPixel& b) { return a.y != b.y ? a.y < b.y : a.x < b.x; };
  std::sort(cap.begin(), cap.end(), [](const CapPixel& a, const CapPixel& b) {
    return a.row() != b.row() ? a.row() < b.row() : (a.y != b.y ? a.y < b.y : a.x < b.x);
  });
  for (size_t b0 = 0; b0 < cap.size();) {
    size_t b1 = b0;
    while (b1 < cap.size() && cap[b1].row() + k - cap[b0].row() <= boxH) ++b1;
    std::sort(cap.begin() + b0, cap.begin() + b1, [](const CapPixel& a, const CapPixel& b) {
      return a.col0 != b.col0 ? a.col0 < b.col0 : (a.y != b.y ? a.y < b.y : a.x < b.x);
    });
    for (size_t c0 = b0; c0 < b1;) {
      const int boxX = cap[c0].col0 & ~15;
      size_t c1 = c0;
      while (c1 < b1 && cap[c1].col0 + k - boxX <= boxW) ++c1;
      std::sort(cap.begin() + c0, cap.begin() + c1, outputOrder);
      const int n = static_cast<int>(c1 - c0), jobs = ((n + 31) / 32 + capJobMaxSteps(k) - 1) / capJobMaxSteps(k);
      const int per = ((n + jobs - 1) / jobs + 31) / 32 * 32;
      for (int i = 0; i < n; i += per) out.push_back(capJob(h, &cap[c0 + i], std::min(per, n - i)));
      c0 = c1;
    }
    b0 = b1;
  }
  tileBorderStart.push_back(border.size());
  for (size_t t = 0; t + 1 < tileBorderStart.size(); ++t)  // (in output order already: a tile's pixels row by row)
    for (size_t i = tileBorderStart[t]; i < tileBorderStart[t + 1]; i += borderJobMaxPixels(k))
      out.push_back(borderJob(h, &border[i], static_cast<int>(std::min(tileBorderStart[t + 1] - i, static_cast<size_t>(borderJobMaxPixels(k))))));
}

}  // namespace

// Deals load[g] pixels of every group to passes of `lanes` pixels with at most h[q] pixels of one group in pass q
// (augmenting paths: a pixel that finds its admissible passes full moves a pixel of another group on).
struct PassDealer {
  int groups, passes, lanes;
  int h[4], share[16][4], fill[4];
  bool seen[4];

  bool put(int g) {
    for (int q = 0; q < passes; ++q) {
      if (seen[q] || share[g][q] >= h[q]) continue;
      seen[q] = true;
      if (fill[q] < lanes) {
        ++share[g][q];
        ++fill[q];
        return true;
      }
      for (int other = 0; other < groups; ++other) {
        if (other == g || share[other][q] == 0) continue;
        --share[other][q];
        if (put(other)) {  // `other` found a seat in a pass not visited yet: g takes the one it left
          ++share[g][q];
          return true;
        }
        ++share[other][q];
      }
    }
    return false;
  }
  bool deal(const int* load) {
    std::memset(share, 0, sizeof(share));
    std::fill(fill, fill + 4, 0);
    for (int g = 0; g < groups; ++g)
      for (int i = 0; i < load[g]; ++i) {
        std::fill(seen, seen + 4, false);
        if (!put(g)) return false;
      }
    return true;
  }
};

int dealLanes(int k, int copies, int n, const int* slot, int* laneOf, int* copyOf) {
  const int groups = weightBankGroups(k), lanesPerPass = weightLanesPerPass(k), passes = 32 / lanesPerPass;
  for (int i = 0; i < n; ++i) { laneOf[i] = i; copyOf[i] = 0; }
  if (n < 32) return 0;
  int group[32];
  if (copies > 1 && groups == 8) {
    int base[32];
    for (int i = 0; i < n; ++i) base[i] = slot[i] & 7;
    GroupMatcher m{n, copies, 0, base, {}, {}, {}};
    for (m.cap = 4; m.cap <= 32; ++m.cap)
      if (m.run()) break;
    m.balance();
    for (int i = 0; i < n; ++i) {
      group[i] = m.groupOf[i];
      copyOf[i] = (m.groupOf[i] - base[i]) & 7;
    }
  } else {
    for (int i = 0; i < n; ++i) group[i] = slot[i] & (groups - 1);
  }
  // How many pixels of each group go to each pass (quarter-warp).  A pass costs as many wavefronts as its fullest group
  // holds pixels, so the load costs H = h[0] + .. + h[passes - 1] when no group has more than h[q] pixels in pass q.
  // Exact: the smallest H (from max(passes, fullest group) upwards) and pass heights h for which the pixels can be dealt
  // -- a transportation problem of groups x passes, solved with augmenting paths.  (A greedy deal ended at 6 - 8
  // wavefronts for most warps whose fullest group holds 5 pixels; cfg2: 4.97 -> 4.5 per load in tile jobs.)
  int load[16] = {};
  for (int i = 0; i < n; ++i) ++load[group[i]];
  int share[16][4] = {}, height[4] = {};
  {
    int fullest = 0;
    for (int g = 0; g < groups; ++g) fullest = std::max(fullest, load[g]);
    PassDealer d{groups, passes, lanesPerPass, {}, {}, {}, {}};
    bool done = false;
    for (int total = std::max(passes, fullest); !done; ++total) {
      // non-increasing heights h[0] >= h[1] >= .. >= 1 with sum `total`, most balanced first
      int h[4] = {1, 1, 1, 1};
      auto tryHeights = [&]() {
        std::copy(h, h + 4, d.h);
        if (!d.deal(load)) return false;
        std::memcpy(share, d.share, sizeof(share));
        std::copy(h, h + 4, height);
        return true;
      };
      if (passes == 2) {
        for (h[1] = total / 2; h[1] >= 1 && !done; --h[1]) { h[0] = total - h[1]; done = tryHeights(); }
      } else {
        for (h[3] = total / 4; h[3] >= 1 && !done; --h[3])
          for (h[2] = (total - h[3]) / 3; h[2] >= h[3] && !done; --h[2])
            for (h[1] = (total - h[3] - h[2]) / 2; h[1] >= h[2] && !done; --h[1]) {
              h[0] = total - h[3] - h[2] - h[1];
              done = tryHeights();
            }
      }
    }
  }
  // Which pixels: neighbouring columns of a group stay in one pass -- they tend to carry the same phase (the same slot:
  // one broadcast read), in this row and in the rows below that reuse the order.
  int nextLane[4];
  for (int q = 0; q < passes; ++q) nextLane[q] = q * lanesPerPass;
  for (int g = 0; g < groups; ++g) {
    int q = 0;
    for (int i = 0; i < n; ++i) {
      if (group[i] != g) continue;
      while (share[g][q] == 0) ++q;
      --share[g][q];
      laneOf[i] = nextLane[q]++;
    }
  }
  int wavefronts = 0;
  for (int q = 0; q < passes; ++q) wavefronts += height[q];
  return wavefronts;
}

std::vector<uint8_t> buildWeightImage(int k, const int16_t* table) {
  const int copies = weightCopies(k);
  std::vector<uint8_t> img(static_cast<size_t>(weightImageBytes(k, copies)), 0);
  for (int phase = 0; phase < 1024; ++phase) {
    const int slot = weightSlotOf(k, phase);
    const int16_t* cell = table + static_cast<size_t>(phase) * k * k;
    if (k == 2) {
      std::memcpy(&img[static_cast<size_t>(slot) * 8], cell, 8);
      continue;
    }
    for (int c = 0; c < copies; ++c)
      for (int v = 0; v < k * k / 8; ++v)  // vector v = the 8 weights 8v .. 8v+7 of the row-major window
        std::memcpy(&img[static_cast<size_t>(weightVectorOffset(k, copies, (weightSlotInCopy(slot, c) << 4) | (c << 14), v))], cell + v * 8, 16);
  }
  return img;
}

void buildGatherPlan(const HostPlan& h, bool stageTiles, GatherPlan& g) {
  g = GatherPlan{};
  const int k = h.kernelSize;
  if (k <= 0) return;
  g.tileH = gatherTileH(k);
  g.tilesPerRow = (h.mapW + kGatherTileW - 1) / kGatherTileW;
  g.tileRows = (h.mapH + g.tileH - 1) / g.tileH;
  g.records.assign(static_cast<size_t>(g.tilesPerRow) * g.tileRows * g.tileH * kGatherTileW, int2{0, 0});
  buildFullRecords(h, g.records, g.tilesPerRow, g.tileH);
  if (!stageTiles) return;

  // ---- cut the plane into jobs: 64 x 32 share blocks where the geometry allows, 32 x 32 tiles elsewhere
  const int tilesX = g.tilesPerRow, tilesY = (h.mapH + kFrameTileH - 1) / kFrameTileH;
  // seam tiles need whole 16-byte columns on both sides of the border and a plane much wider than the box
  const bool seamPossible = h.inW % 16 == 0 && h.inW >= 4 * stageBoxW(k, 0);
  std::vector<TileClass> cls(static_cast<size_t>(tilesX) * tilesY);
  const int blockRows = shareH(k) / kFrameTileH;  // tile rows a share block spans
  parallelRanges((tilesY + blockRows - 1) / blockRows, static_cast<size_t>(h.mapW) * shareH(k), [&](int byBegin, int byEnd) {
    for (int by = byBegin; by < byEnd; ++by)
      for (int tx = 0; tx < tilesX; tx += 2) {
        TileClass* c = &cls[static_cast<size_t>(by) * blockRows * tilesX + tx];
        if (shareBlock(h, tx * 32, by * shareH(k), c[0])) continue;  // the other tiles of the block stay -1: covered
        for (int ty = by * blockRows; ty < std::min(tilesY, (by + 1) * blockRows); ++ty)
          for (int t = tx; t < std::min(tilesX, tx + 2); ++t)
            classifyTile(h, t * 32, ty * kFrameTileH, seamPossible, cls[static_cast<size_t>(ty) * tilesX + t]);
      }
  });

  // the tile list, sorted by rank: general tiles (no box, no records) first, then the staged kinds in launch order
  for (int ty = 0; ty < tilesY; ++ty)
    for (int tx = 0; tx < tilesX; ++tx) {
      const TileClass& c = cls[static_cast<size_t>(ty) * tilesX + tx];
      const int kind = c.kind;
      if (kind < 0) continue;
      for (int q = 0; q < (c.quads ? 4 : 1); ++q) {
        GatherJob job{tx * 32, ty * kFrameTileH | (kind << kJobKindShift),
                      kind == kJobGeneral ? 0 : jobBoxField(c.boxX, c.boxY, boxVariantFor(k, boxClassOf(kind), c.boxRows)), 0};
        if (c.quads) {
          job.outX |= q + 1;
          job.boxXY = jobBoxField(c.quadBoxX[q], c.quadBoxY[q], boxVariantFor(k, 0, c.quadBoxRows[q]));
        }
        g.jobs.push_back(job);
      }
      switch (kind) {
        case kJobGeneral: ++g.numGeneral; break;
        case kJobSeam: ++g.numSeam; break;
        case kJobShare: case kJobShareStay: ++g.numShare; break;
        default: g.numStaged[kind] += c.quads ? 4 : 1; break;
      }
    }
  std::stable_sort(g.jobs.begin(), g.jobs.end(), [](const GatherJob& a, const GatherJob& b) { return jobLaunchRank(a) < jobLaunchRank(b); });
  size_t offset = 0;  // bytes
  for (GatherJob& job : g.jobs) {
    const int kind = (job.outY >> kJobKindShift) & kJobKindMask;
    if (kind == kJobGeneral) continue;
    job.recordOffset = static_cast<int>(offset / 16);
    offset += jobRecordBytes(k, kind, job.outX);
  }
  g.compact.assign(offset / 4, 0u);
  std::vector<int> needRows(g.jobs.size(), h.inH);
  std::vector<JobRect> rects(g.jobs.size());
  std::vector<uint8_t> widths(g.jobs.size(), 0);
  parallelRanges(static_cast<int>(g.jobs.size()), 2048, [&](int begin, int end) {
    for (int i = begin; i < end; ++i) {
      const GatherJob& job = g.jobs[i];
      JobRect& r = rects[i];
      r = tileRect(job, k);
      r.x1 = std::min(r.x1, h.mapW);
      r.y1 = std::min(r.y1, h.mapH);
      const int kind = (job.outY >> kJobKindShift) & kJobKindMask;
      if (kind == kJobGeneral) continue;
      // the source rows the job reads: what a caller that streams the plane in must have delivered before it runs
      const Extent e = extentOf(h, r.x0, r.y0, r.x1, r.y1);
      if (e.minR >= 0 && e.maxR + k <= h.inH) needRows[i] = e.maxR + k;
      if (kind == kJobClass0) widths[i] = static_cast<uint8_t>(class0WidthFor(k, e.maxC + k - jobBoxX(job.boxXY)));
      uint32_t* out = g.compact.data() + static_cast<size_t>(job.recordOffset) * 4;
      if (boxClassOf(kind) == 2) writeShareRecords(h, job, out);
      else writeTileRecords(h, job, out);
    }
  });

  // the pixels of the general tiles: pole-cap and border jobs, their records after the tiles'
  std::vector<PixelJob> pixelJobs;
  coverPoleCaps(h, cls, tilesX, tilesY, pixelJobs);
  for (PixelJob& pj : pixelJobs) {
    const int kind = (pj.job.outY >> kJobKindShift) & kJobKindMask;
    pj.job.recordOffset = static_cast<int>(offset / 16);
    offset += jobRecordBytes(k, kind, pj.job.outX);
    g.capJobs.push_back(pj.job);
    g.capRecords.insert(g.capRecords.end(), pj.words.begin(), pj.words.end());
    ++(kind == kJobCap ? g.numCap : g.numBorder);
  }

  // the launch list: index into `jobs`, or -1 - index into capJobs
  std::vector<int> launch;
  for (size_t i = 0; i < g.jobs.size(); ++i)
    if (((g.jobs[i].outY >> kJobKindShift) & kJobKindMask) != kJobGeneral) launch.push_back(static_cast<int>(i));
  for (size_t i = 0; i < g.capJobs.size(); ++i) launch.push_back(-1 - static_cast<int>(i));
  auto jobOf = [&](int i) -> const GatherJob& { return i >= 0 ? g.jobs[i] : g.capJobs[-1 - i]; };
  std::stable_sort(launch.begin(), launch.end(), [&](int a, int b) { return jobLaunchRank(jobOf(a)) < jobLaunchRank(jobOf(b)); });
  for (int i : launch) {
    g.launchJobs.push_back(jobOf(i));
    g.launchNeedRows.push_back(i >= 0 ? needRows[i] : pixelJobs[-1 - i].needRows);
    g.launchRects.push_back(i >= 0 ? rects[i] : pixelJobs[-1 - i].rect);
    g.launchBoxWidths.push_back(i >= 0 ? widths[i] : 0);
  }
  if (offset / 16 > static_cast<size_t>(kJobRecordMask)) throw std::invalid_argument("gather plan: too many sampling records");
}

int pipelineChunks(int inW, int inH) {
  const long long bytes = static_cast<long long>(inW) * inH;
  return static_cast<int>(std::min<long long>(8, std::max<long long>(2, bytes / (3ll << 20))));
}

WaveSchedule scheduleWaves(const std::vector<int>& needRows, const std::vector<JobRect>& rects, int inH, int mapW, int mapH, int chunks) {
  WaveSchedule w;
  const int rowsPer = ((inH + chunks - 1) / chunks + 7) & ~7;
  w.chunkRowEnd.assign(chunks, inH);
  for (int c = 0; c < chunks; ++c) w.chunkRowEnd[c] = std::min(inH, (c + 1) * rowsPer);
  auto waveOf = [&](int rows) {
    int c = 0;
    while (c + 1 < chunks && w.chunkRowEnd[c] < rows) ++c;
    return c;
  };
  std::vector<std::vector<int>> byWave(chunks);
  const int bands = (mapH + 31) / 32;
  std::vector<int> complete(bands, 0);  // per band: the wave after which it is complete
  for (size_t i = 0; i < needRows.size(); ++i) {
    const int c = waveOf(needRows[i]);
    byWave[c].push_back(static_cast<int>(i));
    const JobRect& r = rects[i];
    for (int band = r.y0 / 32; band <= (r.y1 - 1) / 32; ++band) complete[band] = std::max(complete[band], c);
  }
  w.waveStart.assign(chunks + 1, 0);
  for (int c = 0; c < chunks; ++c) {
    w.waveStart[c] = static_cast<int>(w.order.size());
    w.order.insert(w.order.end(), byWave[c].begin(), byWave[c].end());
  }
  w.waveStart[chunks] = static_cast<int>(w.order.size());
  w.rects.assign(chunks, {});
  for (int band = 0; band < bands;) {  // adjacent bands that complete together: one copy
    const int c = complete[band];
    int end = band + 1;
    while (end < bands && complete[end] == c) ++end;
    w.rects[c].push_back(JobRect{0, band * 32, mapW, std::min(mapH, end * 32)});
    band = end;
  }
  return w;
}

std::vector<GatherJob> deviceJobs(const GatherPlan& g) {
  std::vector<GatherJob> out(g.launchJobs);
  for (size_t i = 0; i < out.size(); ++i) out[i].recordOffset |= static_cast<int>(g.launchBoxWidths[i]) << kJobWidthShift;
  return out;
}

std::vector<uint32_t> deviceRecords(const GatherPlan& g, int k) {
  std::vector<uint32_t> out(g.compact);
  out.insert(out.end(), g.capRecords.begin(), g.capRecords.end());
  const int wide = stageBoxW(k, 0);
  for (size_t i = 0; i < g.launchJobs.size(); ++i) {
    if (g.launchBoxWidths[i] == 0) continue;
    const GatherJob& job = g.launchJobs[i];
    const uint32_t narrow = static_cast<uint32_t>(class0BoxW(g.launchBoxWidths[i]));
    uint32_t* w = out.data() + static_cast<size_t>(job.recordOffset) * 4;
    for (int j = 0; j < jobRecordBytes(k, kJobClass0, job.outX) / 4; ++j) {
      if (w[j] & kRecordSkip) continue;
      const uint32_t off = w[j] & 0x7fffu;
      w[j] = (w[j] & ~0x7fffu) | (off / wide * narrow + off % wide);
    }
  }
  return out;
}

}  // namespace t360
