// The low-pass job lists (lowpass_jobs.h).
#include "lowpass_jobs.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <utility>

namespace t360 {

namespace {

// heaviest jobs first: the hardware block scheduler then balances the tail
bool heavierStrip(const StripJob& a, const StripJob& b) {
  return static_cast<long long>(a.kxChunks + 2) * a.h * (1 + 3 * (a.edge & 1)) > static_cast<long long>(b.kxChunks + 2) * b.h * (1 + 3 * (b.edge & 1));
}

void sortStrips(BlurLists& l) {
  for (std::vector<StripJob>& v : l.strips) std::stable_sort(v.begin(), v.end(), heavierStrip);
}

}  // namespace

void buildBlurLists(const std::vector<LowPassSegment>& segments, const std::vector<float>& planTaps, int planeW, int planeH,
                    int stereoFormat, BlurLists& out, bool* needsClear) {
  for (auto& v : out.strips) v.clear();
  out.tiles.clear();
  out.direct.clear();
  std::vector<float>& taps = out.taps;
  std::vector<int>& source = out.tapSource;
  taps = planTaps;  // original taps first (offsets of the plan stay valid), padded copies appended
  source.resize(taps.size());
  for (size_t i = 0; i < source.size(); ++i) source[i] = static_cast<int>(i) + 1;
  int offX[2] = {0, 0}, offY[2] = {0, 0}, passes = 1;
  if (stereoFormat == STEREO_FORMAT_LR) { passes = 2; offX[1] = static_cast<int>(0.5 * planeW); }
  else if (stereoFormat == STEREO_FORMAT_TB) { passes = 2; offY[1] = static_cast<int>(0.5 * planeH); }
  std::vector<uint8_t> covered(needsClear ? static_cast<size_t>(planeW) * planeH : 0, 0);
  int tileSmem = 0;
  // a warp-job covers 256 columns x `rows` rows; keep the grid at several thousand warps even for small planes
  const long long stripsPerRow = (planeW + kStripW - 1) / kStripW;
  // (each job recomputes 2*hy rows of horizontal sums at its top and bottom, so never fewer than 8 rows)
  const long long wanted = static_cast<long long>(planeH) * stripsPerRow / 5000;
  const int rowsBudget = wanted >= 32 ? 32 : (wanted >= 16 ? 16 : 8);

  auto sameTaps = [&](int offA, int nA, int offB, int nB) {
    return nA == nB && (offA == offB || std::memcmp(&planTaps[offA], &planTaps[offB], sizeof(float) * nA) == 0);
  };
  // horizontal taps zero-padded to whole chunks of 4 at a 16-byte aligned offset (fma(0, p, s) == s exactly)
  std::map<std::pair<int, int>, std::pair<int, int>> paddedKx;
  auto padKx = [&](int off, int n) {
    auto it = paddedKx.find({off, n});
    if (it != paddedKx.end()) return it->second;
    while (taps.size() % 4) { taps.push_back(0.f); source.push_back(0); }
    const int at = static_cast<int>(taps.size()), chunks = (n + 3) / 4;
    for (int i = 0; i < chunks * 4; ++i) {
      taps.push_back(i < n ? planTaps[off + i] : 0.f);
      source.push_back(i < n ? off + i + 1 : 0);
    }
    return paddedKx[{off, n}] = std::make_pair(at, chunks);
  };
  std::map<int, int> paddedKy1;  // a single vertical tap k becomes {0, k, 0}
  auto padKy = [&](int off, int n) {
    if (n != 1) return off;
    auto it = paddedKy1.find(off);
    if (it != paddedKy1.end()) return it->second;
    const int at = static_cast<int>(taps.size());
    taps.push_back(0.f); taps.push_back(planTaps[off]); taps.push_back(0.f);
    source.push_back(0); source.push_back(off + 1); source.push_back(0);
    return paddedKy1[off] = at;
  };

  for (int pass = 0; pass < passes; ++pass) {
    // segments of one band that are horizontally adjacent and carry bit-identical kernels (always the case when
    // the view-dependent scale is 1, e.g. no off-centre projection) are merged into one wide segment
    // a segment that does not fit the plane is dropped, like the reference's caught cv::Exception (cpp:183-203) -- each
    // one on its own, before any merging
    auto fits = [&](const LowPassSegment& g) {
      const int l = g.left + offX[pass], t = g.top + offY[pass];
      return l >= 0 && t >= 0 && g.width > 0 && g.height > 0 && l + g.width <= planeW && t + g.height <= planeH;
    };
    size_t i = 0;
    while (i < segments.size()) {
      LowPassSegment s = segments[i];
      size_t j = i + 1;
      if (!fits(s)) { i = j; continue; }
      while (j < segments.size()) {
        const LowPassSegment& n = segments[j];
        if (n.top != s.top || n.height != s.height || n.left != s.left + s.width || !fits(n) ||
            !sameTaps(n.kxOffset, n.kxCount, s.kxOffset, s.kxCount) || !sameTaps(n.kyOffset, n.kyCount, s.kyOffset, s.kyCount))
          break;
        s.width += n.width;
        ++j;
      }
      i = j;
      const int left = s.left + offX[pass], top = s.top + offY[pass];
      if (needsClear)
        for (int y = 0; y < s.height; ++y) std::memset(&covered[static_cast<size_t>(top + y) * planeW + left], 1, s.width);
      const int hy = s.kyCount / 2;
      if (hy <= kStripMaxHy && (s.kyCount & 1) && (s.kxCount & 1)) {
        const auto kx = padKx(s.kxOffset, s.kxCount);
        const int kyOff = padKy(s.kyOffset, s.kyCount), hx = s.kxCount / 2;
        const int rows = std::min(rowsBudget, kx.second <= 3 ? 32 : (kx.second <= 8 ? 16 : 8));
        for (int ty = 0; ty < s.height; ty += rows)
          for (int tx = 0; tx < s.width; tx += kStripW) {
            StripJob j{left + tx, top + ty, std::min(kStripW, s.width - tx), std::min(rows, s.height - ty), kx.first, kx.second, s.kxCount, kyOff, 0};
            // interior strips read whole aligned words: first byte - 3 and the last prefetched group must stay in the row
            const int firstByte = j.x0 - hx, lastByte = j.x0 + kStripW - kStripLanePx - hx + 4 * (kx.second + 3) + 7;
            j.edge = (firstByte - 4 < 0 || lastByte >= planeW) ? 1 : 0;
            out.strips[std::max(hy, 1) - 1].push_back(j);
          }
      } else {
        for (int ty = 0; ty < s.height; ty += kBlurTileH)
          for (int tx = 0; tx < s.width; tx += kBlurTileW) {
            BlurJob j{left + tx, top + ty, std::min(kBlurTileW, s.width - tx), std::min(kBlurTileH, s.height - ty),
                      s.kxOffset, s.kxCount, s.kyOffset, s.kyCount};
            const long long need = static_cast<long long>(blurTileSmem(j.w, j.h, j.kxCount, j.kyCount));
            if (need <= kBlurMaxSmem) {
              out.tiles.push_back(j);
              tileSmem = std::max(tileSmem, static_cast<int>(need));
            } else {
              out.direct.push_back(j);
            }
          }
      }
    }
  }
  if (needsClear) *needsClear = std::find(covered.begin(), covered.end(), 0) != covered.end();
  sortStrips(out);
  out.tileSmem = tileSmem;
}

BlurLists mergeBlurLists(const BlurLists* const* planes, int numPlanes) {
  BlurLists m;
  for (int p = 0; p < numPlanes; ++p) {
    const BlurLists& l = *planes[p];
    while (m.taps.size() % 4) { m.taps.push_back(0.f); m.tapSource.push_back(0); }  // (padded horizontal taps stay aligned)
    const int base = static_cast<int>(m.taps.size());
    m.taps.insert(m.taps.end(), l.taps.begin(), l.taps.end());
    for (int s : l.tapSource) m.tapSource.push_back(s ? (p << kTapPlaneShift) | s : 0);
    for (int c = 0; c < kStripMaxHy; ++c)
      for (StripJob j : l.strips[c]) {
        j.kxOffset += base;
        j.kyOffset += base;
        j.edge |= p << kStripPlaneShift;
        m.strips[c].push_back(j);
      }
  }
  sortStrips(m);
  return m;
}

BlurLayout packBlurLists(const BlurLists& l, std::vector<uint8_t>& jobs, std::vector<uint8_t>& taps) {
  auto append = [](std::vector<uint8_t>& blob, const void* data, size_t bytes) {
    blob.resize((blob.size() + 15) & ~size_t(15));
    const size_t at = blob.size();
    blob.insert(blob.end(), static_cast<const uint8_t*>(data), static_cast<const uint8_t*>(data) + bytes);
    return at;
  };
  BlurLayout a;
  for (int c = 0; c < kStripMaxHy; ++c) {
    a.numStrips[c] = static_cast<int>(l.strips[c].size());
    a.stripAt[c] = append(jobs, l.strips[c].data(), l.strips[c].size() * sizeof(StripJob));
  }
  a.numTiles = static_cast<int>(l.tiles.size());
  a.tileAt = append(jobs, l.tiles.data(), l.tiles.size() * sizeof(BlurJob));
  a.numDirect = static_cast<int>(l.direct.size());
  a.directAt = append(jobs, l.direct.data(), l.direct.size() * sizeof(BlurJob));
  a.numTaps = static_cast<int>(l.taps.size());
  a.tapAt = append(taps, l.taps.data(), l.taps.size() * sizeof(float));
  a.tileSmem = l.tileSmem;
  return a;
}

}  // namespace t360
