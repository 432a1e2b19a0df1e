// Device-independent part of the gather plan of one plane: how the output plane is cut into jobs for the persistent
// gather kernel and how the sampling records are laid out for it.  Pure host code (no CUDA call), so that the CPU
// test-suite can check it without a GPU (T360B200_hostPlanGather).  See kernels.cuh for the formats.
#pragma once

#include <cstdint>
#include <vector>

#include "host_plan.h"
#include "kernels.cuh"

namespace t360 {

struct JobRect {
  int x0, y0, x1, y1;
};

struct GatherPlan {
  int tilesPerRow = 0, tileRows = 0, tileH = 0;  // grid of the FULL records: tiles of 32 x tileH pixels (general kernels)
  std::vector<int2> records;                     // full records: tile-major, lane-ordered (kernels.cuh)
  // The plane cut into share blocks and 32 x 32 tiles, sorted by jobLaunchRank (empty: the plan is not staged), and the
  // compact records of its staged entries.  A general entry (a pole-cap tile) has no box and no records: its pixels are
  // in capJobs.
  std::vector<GatherJob> jobs;
  std::vector<uint32_t> compact;
  // The pixels of the general tiles as pole-cap and border jobs; their record offsets count on after `compact`, i.e. in
  // the device's record buffer  compact ++ capRecords.
  std::vector<GatherJob> capJobs;
  std::vector<uint32_t> capRecords;
  // What the frame kernel runs: `jobs` without the general tiles, and capJobs, in launch order; per job the source rows
  // [0, n) it reads (inH if a window wraps vertically) and the bounding rectangle of the output pixels it writes.
  std::vector<GatherJob> launchJobs;
  std::vector<int> launchNeedRows;
  std::vector<JobRect> launchRects;
  // per launch job the width of its class-0 box (kernels.cuh: class0BoxW; 0 for every other kind), which the device's
  // copy of the list carries in GatherJob::recordOffset (deviceJobs) and the device's records in their pitch
  // (deviceRecords)
  std::vector<uint8_t> launchBoxWidths;
  int numStaged[2] = {}, numSeam = 0, numGeneral = 0, numShare = 0, numCap = 0, numBorder = 0;
  int totalStaged() const { return numSeam + numShare + numStaged[0] + numStaged[1] + numCap; }
};

// stageTiles: cut the plane into jobs for the persistent kernel (kernel size >= 2 and BORDER_WRAP); otherwise only the
// full records are produced (nearest neighbour, barrel layouts: whole-plane general kernels).
void buildGatherPlan(const HostPlan& h, bool stageTiles, GatherPlan& g);

// The job list the frame kernel claims from: launchJobs with each class-0 box width in the top bits of recordOffset.
std::vector<GatherJob> deviceJobs(const GatherPlan& g);
// The record buffer the frame kernel reads: compact ++ capRecords, with the window offsets of a job that loads a narrow
// class-0 box at that box's pitch instead of the stage buffer's 208 bytes (kernels.cuh: class0BoxW).
std::vector<uint32_t> deviceRecords(const GatherPlan& g, int k);

// Launch order of the jobs: border (latency-bound reads through L1, few; in the tile list: the general tiles), seam and class 1 (both need the two stage
// buffers of a group), pole caps, share jobs, and finally the small class-0 tiles through the double-buffered TMA
// pipeline, which leaves a short, fine-grained tail (the cheapest jobs, the 16 x 16 quadrants, come last of all: every
// group has up to three jobs claimed ahead, so the launch ends within about three of its last jobs).  A list sorted by
// this rank (stably: a frame's list keeps the planes in order inside a rank) is in launch order.
inline int jobLaunchRank(const GatherJob& job) {
  switch ((job.outY >> kJobKindShift) & kJobKindMask) {
    case kJobBorder: case kJobGeneral: return 0;
    case kJobSeam: return 1;
    case kJobClass1: return 2;
    case kJobCap: return 3;
    case kJobShareStay: return 4;
    case kJobShare: return 5;
    default: return (job.outX & kJobQuadMask) ? 7 : 6;  // class 0: whole tiles, then quadrants
  }
}


// Streaming a large host plane through the device (the synchronous host-pointer call): the input arrives in `chunks` row
// bands of one size, rounded up to 8 rows; wave c is one frame-kernel launch of the launch jobs whose source rows
// [0, needRows) have all arrived with chunk c (launch order kept inside a wave); the output goes back in 32-row bands of
// the full width, each after the last wave that writes into it (adjacent bands that complete together: one rectangle).
// Contiguous bands, not per-job rectangles: a band split into the faces of a cube-map row would finish earlier per face,
// but strided rectangle copies are much slower than whole contiguous bands.
struct WaveSchedule {
  std::vector<int> chunkRowEnd;             // per chunk: rows [0, end) have arrived after it (trailing chunks may be empty)
  std::vector<int> order;                   // the launch jobs, wave by wave
  std::vector<int> waveStart;               // chunks + 1 entries: wave c is order[waveStart[c] .. waveStart[c + 1])
  std::vector<std::vector<JobRect>> rects;  // per wave: the output rectangles copied back after it
};
// How many row bands a plane of inW x inH bytes is streamed in: one per 3 MiB, 2 to 8.
int pipelineChunks(int inW, int inH);
// needRows, rects: per launch job (GatherPlan::launchNeedRows, launchRects).
WaveSchedule scheduleWaves(const std::vector<int>& needRows, const std::vector<JobRect>& rects, int inH, int mapW, int mapH, int chunks);

// Deals n <= 32 pixels of one warp step to lanes (and table copies) so that the lanes one shared-memory pass serves
// together ask for different bank groups of the weight table.  slot[i] = weightSlotOf(k, phase of pixel i).
// laneOf[i] = lane of pixel i, copyOf[i] = table copy it reads.  Returns the modelled wavefronts of one weight load.
int dealLanes(int k, int copies, int n, const int* slot, int* laneOf, int* copyOf);

// The shared-memory image of the interpolation weights the frame kernel copies in (layout: kernels.cuh, "Weight tables
// in shared memory"), from OpenCV's table int16 [1024][k][k].  weightImageBytes(k, weightCopies(k)) bytes.
std::vector<uint8_t> buildWeightImage(int k, const int16_t* table);

}  // namespace t360
