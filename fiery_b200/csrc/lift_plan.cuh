// Geometry plan of the lift: everything the tile kernels need to know about WHERE the frustum points of a batch land, computed
// once per batch of calibrations and shared by the forward and the backward kernel (and by later calls while the rig is static).
//
// get_geometry (fiery/models/fiery.py:193-208) and the voxel indices / mask / ranks of projection_to_birds_eye_view
// (fiery.py:236-256) depend only on (intrinsics, extrinsics, frustum, BEV grid) -- not on the head tensor.  At fixed (camera,
// column, depth) the h image rows of a column fall into one BEV pillar or a handful (Z has one cell, cameras are close to
// level), so the geometry of a tile reduces to RUNS: per (depth, column) pair the rows at which the pillar changes, and the
// pillar (rank, or -1 = masked) of every run.  ~0.3 MB per frame instead of the reference's 17 MB of int64 indices.
//
// Plan buffer layout (bytes), for n_frames frames of n_cameras cameras, n_wtiles column tiles per image:
//   [ tile records : n_tiles * PLAN_TILE_BYTES ]   tile = (frame * n_cameras + camera) * n_wtiles + column tile
//   [ touched maps : n_frames * pillars bytes  ]   1 where a pillar receives at least one point (the layout pass reads it)
// Tile record:
//   mask  [192] u32   pair = depth * 4 + column; bit h (1 <= h < rows) set <=> pillar(row h) != pillar(row h-1)
//   off   [192] u16   index of the pair's first run in runs[]
//   soff  [ 64] u16   index of stream (rg, column, j)'s first entry in streams[]; stream = (rg * 4 + column) * 4 + j
//   n_runs, n_stream  u32
//   runs    [PLAN_CAP] i32   forward order: pair-major, runs of a pair in row order
//   streams [PLAN_CAP + pads] i32   backward order: the rows are cut into PLAN_RG row groups [rows*rg/4, rows*(rg+1)/4); stream
//           (rg, column, j) lists, for depth 4g + j, g = 0, 1, ..., the run that contains the group's first row followed by the
//           runs that start inside the group -- exactly the sequence of gradient rows thread (rg, column) of the backward
//           kernel gathers for its slot j -- and ends with two -1 entries (the kernel prefetches two entries ahead).
#pragma once
#include "lift_tile.cuh"

namespace fiery {

constexpr int PLAN_PAIRS = DPAD * WT;         // (depth, column) pairs of a tile
constexpr int PLAN_RG = 4;                   // row groups of the backward kernel
constexpr int PLAN_ND = 4;                   // depths per backward depth group (slots j)
constexpr int PLAN_STREAMS = PLAN_RG * WT * PLAN_ND;
constexpr int PLAN_MAX_ROWS = 32;
constexpr int PLAN_CAP = PLAN_PAIRS * PLAN_MAX_ROWS;            // worst case: every pair changes pillar at every row
constexpr int PLAN_STREAM_CAP = PLAN_CAP + 2 * PLAN_STREAMS;    // + two pad entries per stream

constexpr int PLAN_OFF_MASK = 0;
constexpr int PLAN_OFF_OFF = PLAN_OFF_MASK + PLAN_PAIRS * 4;
constexpr int PLAN_OFF_SOFF = PLAN_OFF_OFF + PLAN_PAIRS * 2;
constexpr int PLAN_OFF_COUNTS = PLAN_OFF_SOFF + PLAN_STREAMS * 2;
constexpr int PLAN_OFF_RUNS = PLAN_OFF_COUNTS + 16;
constexpr int PLAN_OFF_STREAMS = PLAN_OFF_RUNS + PLAN_CAP * 4;
constexpr int PLAN_TILE_BYTES = (PLAN_OFF_STREAMS + PLAN_STREAM_CAP * 4 + 127) & ~127;

// Rows of partial sums a tile of the deterministic forward may store: a (depth, column) pair has at most one run per image row.
__host__ __device__ inline int det_runs_per_tile(int rows) { return PLAN_PAIRS * rows; }

struct PlanView {
    const unsigned char* tiles;     // tile records of this launch's first frame onwards
    const unsigned char* touched;   // touched map of the same frame onwards (n_frames * pillars bytes)
};

__host__ __device__ inline size_t plan_bytes(long long n_frames, int n_cameras, int n_wtiles, long long pillars) {
    const size_t tiles = static_cast<size_t>(n_frames) * n_cameras * n_wtiles * PLAN_TILE_BYTES;
    const size_t touched = (static_cast<size_t>(n_frames) * pillars + 127) & ~static_cast<size_t>(127);
    return tiles + touched;
}

__host__ __device__ inline PlanView plan_view(const void* plan, long long n_frames_total, int n_cameras, int n_wtiles, long long pillars,
                                              long long frame0) {
    const unsigned char* base = static_cast<const unsigned char*>(plan);
    PlanView v;
    v.tiles = base + static_cast<size_t>(frame0) * n_cameras * n_wtiles * PLAN_TILE_BYTES;
    v.touched = base + static_cast<size_t>(n_frames_total) * n_cameras * n_wtiles * PLAN_TILE_BYTES + static_cast<size_t>(frame0) * pillars;
    return v;
}

// Event pairs around the kernel launches of one forward call (fiery_lift_forward_timed): kind 0 = plan kernel, 1 = tile kernel,
// 2 = layout pass.
struct LaunchTimer {
    static constexpr int MAX = 64;
    cudaEvent_t ev[2 * MAX];
    int kind[MAX];
    int n = 0, cap = 0;
};

// first row of row group rg (rg may be PLAN_RG: one past the last row)
__host__ __device__ __forceinline__ int plan_group_row(int rows, int rg) { return (rows * rg) / PLAN_RG; }

// ---- host side of the lift, defined in c_api.cu and next to the kernels ------------------------------------------------------------
int check_lift_geometry(const LiftParams& P);      // rows and depth bins of a plan's tile record
int encode_bev_map(CUtensorMap* map, float* bev, long long pillars, int channels, int n_frames, int box_pillars);
int launch_lift_plan(const LiftParams& P, unsigned char* tiles, unsigned char* touched, int want_streams, cudaStream_t stream);
int launch_forward_cols(const LiftParams& P, const void* head, cudaStream_t stream);
int launch_forward_cols_det(const LiftParams& P, const void* head, cudaStream_t stream);
int launch_det_reduce(const LiftParams& P, int nf, const unsigned char* tiles, const float* partials, int* start, int* cursor,
                      int* lists, float* out, int zero_empty, cudaStream_t stream);
// the two forward launchers take the same arguments: c_api.cu calls both through one pointer type
int launch_lift_forward(const LiftParams& P, const void* head, int head_dtype, float* bev_out, void* scratch, const void* plan,
                        const float* warp_theta, const unsigned char* warp_copy, cudaStream_t stream);
int launch_lift_forward_det(const LiftParams& P, const void* head, int head_dtype, float* bev_out, void* workspace, const void* plan,
                            const float* warp_theta, const unsigned char* warp_copy, cudaStream_t stream);
size_t lift_scratch_bytes(const LiftParams& P);
size_t lift_det_workspace_bytes(const LiftParams& P);
int lift_forward_launches(const LiftParams& P);
void lift_set_max_chunk_frames(int n);
void lift_set_timer(LaunchTimer* t);
int launch_point_indices(const LiftParams& P, int64_t* idx_out, uint8_t* valid_out, int32_t* pillar_out, cudaStream_t stream);
int launch_compose(int n, const float* K, const float* E, float* combined, float* translation, cudaStream_t stream);
size_t lift_backward_relayout_bytes(const LiftParams& P);
int launch_lift_backward(const LiftParams& P, const void* head, float* workspace, const void* plan, cudaStream_t stream);

}  // namespace fiery
