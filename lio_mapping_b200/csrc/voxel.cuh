// Device VoxelGrid workspace (see voxel.cu).
#pragma once
#include "primitives.cuh"

namespace lio {

struct VoxelGrid {
  int cap = 0, nstatus = 0;
  DevMem<unsigned> keys_a, vals_a, keys_b, vals_b;
  RadixSortTemp rs;
  DevMem<unsigned long long> status;
  DevMem<unsigned> bbox;
  DevMem<int> ticket;     // [0] tile ticket, [1] sticky PCL index-overflow flag, [2] clamped input count
  int init(int cap);
  // in: min(*n_dev, n_max) points (n_max <= cap).  out: centroids in ascending voxel-index order, at most out_cap of
  // them are stored; *nout_dev always receives the full count (callers compare it with out_cap after their next sync).
  // vox_key_out (optional): the voxel index of every output centroid.
  int run(const float4 *in, const int *n_dev, int n_max, float leaf, float4 *out, int out_cap, int *nout_dev,
          unsigned *vox_key_out, cudaStream_t st, int *launches);
  int *overflow_flag() const { return ticket + 1; }
};

// One cloud of a segmented VoxelGrid: n points at p, filtered in place with its own leaf; off = its start in the concatenation.
struct VgJob { float4 *p; int n, off; float leaf; };
constexpr int kVgMaxJobs = 256;   // the job id takes the top 8 bits of the 32-bit sort key
constexpr int kVgJobBits = 24;    // ... and the PCL voxel index the low 24: a job whose index range exceeds 2^24 is an error

// Many clouds filtered as separate pcl::VoxelGrid calls (each its own bounding box and PCL index arithmetic, output in ascending
// voxel order written back over its input) with a fixed number of launches: the clouds are concatenated, keyed by
// (job << 24) | voxel index and sorted once.  Bit-identical to VoxelGrid::run on each cloud.
struct SegVoxelGrid {
  int cap = 0;                     // points of the concatenation the workspace holds (grows in reserve)
  VoxelGrid ws;                    // key / value / sort / look-back buffers sized cap; ticket[0] emit tile, [1] index-bound error, [2] n
  DevMem<float4> cat, out;
  DevMem<VgJob> d_jobs;
  DevMem<unsigned> jbbox;          // [kVgMaxJobs][6] ordered-uint bounding boxes
  DevMem<int> jstart;              // [kVgMaxJobs + 1] first output of every job, then the output total
  DevMem<int> jn;                  // [kVgMaxJobs + 1] output count of every job, then the index-bound error flag
  int init();
  int reserve(int total);
  // h_jobs (pinned, njobs <= kVgMaxJobs, every n > 0, total = sum of n) is uploaded asynchronously: keep it unchanged until the
  // stream has passed this call.  h_jn (pinned) receives the njobs output counts and the error flag at [njobs] asynchronously.
  int run(const VgJob *h_jobs, int njobs, int total, int *h_jn, cudaStream_t st, int *launches);
};

}  // namespace lio
