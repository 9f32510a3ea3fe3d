// Forward camera->BEV lift for sm_90a, host side and the passes around the tile kernel (lift_fwd_cols.cu): the NCHW layout
// pass, the integer index dump and the calibration composition used by the parity checks, and the launchers.
//
// Replaces, per call: Fiery.get_geometry (fiery/models/fiery.py:193-208), the tail of Encoder.forward
// (fiery/models/encoder.py:98-102), and Fiery.projection_to_birds_eye_view incl. VoxelsSumming
// (fiery/models/fiery.py:221-273, fiery/utils/geometry.py:283-314).
#include <atomic>
#include <mutex>

#include "lift_plan.cuh"
#include "warp_sample.cuh"

namespace fiery {

// ---------------------------------------------------------------------------------------------------------------------
// Fallback layout pass for NCHW output when X*Y is not a multiple of 4 (the TMA pass below needs a 16-byte row pitch):
// accum (B', X*Y, C) -> bev (B', C, X*Y).  One thread per pillar: a lane reads its pillar's 256-byte accumulator row as 16
// independent 16-byte loads (its own two cache lines, so the sectors are fully used through L1), and the warp then writes one
// channel of 32 consecutive pillars per store instruction -- a full 128-byte line.  Only ~1/3-1/2 of the pillars receive any
// point, and the tile kernel marks those in a byte map: unmarked pillars are written as zeros without touching the
// accumulator; marked rows (and, when the marks live in the scratch, the marks) are re-zeroed on the way (scratch invariant of
// include/fiery_b200.h).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FIN_THREADS = 256;
__global__ void __launch_bounds__(FIN_THREADS)
finalize_nchw_kernel(float* __restrict__ accum, unsigned char* __restrict__ flags, float* __restrict__ bev,
                     long long pillars, int blocks_per_frame, int clear_marks) {
    constexpr int C = 64;
    const int frame = blockIdx.x / blocks_per_frame;
    const long long pl = static_cast<long long>(blockIdx.x % blocks_per_frame) * FIN_THREADS + threadIdx.x;
    if (pl >= pillars) return;
    unsigned char* f = flags + static_cast<size_t>(frame) * pillars + pl;
    float4 v[C / 4];
    if (*f) {
        float4* row = reinterpret_cast<float4*>(accum + (static_cast<size_t>(frame) * pillars + pl) * C);
#pragma unroll
        for (int q = 0; q < C / 4; ++q) v[q] = row[q];
#pragma unroll
        for (int q = 0; q < C / 4; ++q) row[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (clear_marks) *f = 0;
    } else {
#pragma unroll
        for (int q = 0; q < C / 4; ++q) v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float* dst = bev + static_cast<size_t>(frame) * C * pillars + pl;
#pragma unroll
    for (int q = 0; q < C / 4; ++q) {
        dst[static_cast<size_t>(4 * q + 0) * pillars] = v[q].x;
        dst[static_cast<size_t>(4 * q + 1) * pillars] = v[q].y;
        dst[static_cast<size_t>(4 * q + 2) * pillars] = v[q].z;
        dst[static_cast<size_t>(4 * q + 3) * pillars] = v[q].w;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Layout pass built on the copy engine.  A CTA takes FT_P consecutive pillars of one frame:
//   1. one thread per pillar reads the pillar's touched byte and, if set, fetches the pillar's 256-byte accumulator row with
//      a 1-D bulk copy (cp.async.bulk, completion on an mbarrier) -- only rows that received points are read, each as one
//      contiguous 256-byte burst;
//   2. the (pillar, channel) block is transposed shared -> shared: 16-byte reads in an XOR-rotated chunk order (every
//      quarter-warp phase covers all 32 banks), 4-byte writes with bank = lane; rows that were not fetched read as zero;
//   3. one tiled TMA store writes the (64 channels x FT_P pillars) block into the NCHW output (256 contiguous bytes per
//      channel row), and a 256-byte bulk copy of zeros per fetched row plus a byte store per mark restore the scratch
//      invariant of include/fiery_b200.h.
// Needs X*Y to be a multiple of 4 (16-byte row pitch of the output map).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FT_P = 64;
constexpr int FT_THREADS = 256;

__device__ __forceinline__ void bulk_store_1d(void* dst, const void* src, uint32_t bytes, uint64_t policy) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                 ::"l"(dst), "r"(smem_addr(src)), "r"(bytes), "l"(policy) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, uint64_t policy) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3, %4}], [%1], %5;"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(src)), "r"(c0), "r"(c1), "r"(c2), "l"(policy) : "memory");
}

// L2 priority of the restored zeros: evict_last while another frame group of the lane reduces into the same rows next, evict_normal
// after the lane's last group so that a call leaves no raised-priority lines behind
__device__ __forceinline__ uint64_t l2_restore_policy(int last_in_lane) {
    return last_in_lane ? l2_evict_normal() : l2_evict_last();
}

__global__ void __launch_bounds__(FT_THREADS)
finalize_tma_kernel(const __grid_constant__ CUtensorMap bev_map, float* __restrict__ accum, unsigned char* __restrict__ touched,
                    long long pillars, int tiles_per_frame, int frame_out0, int clear_marks, int last_in_lane) {
    constexpr int C = 64;
    __shared__ __align__(128) float s_in[FT_P * C];      // [pillar][channel]: bulk-copy destination
    __shared__ __align__(128) float s_out[C * FT_P];     // [channel][pillar]: TMA store source
    __shared__ __align__(16) float s_zero[C];
    __shared__ __align__(8) uint64_t bar;
    __shared__ unsigned char s_flag[FT_P];
    const int tid = threadIdx.x;
    const int frame = blockIdx.x / tiles_per_frame;
    const long long p0 = static_cast<long long>(blockIdx.x % tiles_per_frame) * FT_P;
    if (tid == 0) {
        tma_prefetch_desc(&bev_map);
        mbar_init(&bar, FT_P);
        fence_mbar_init();
    }
    if (tid >= FT_THREADS - C) s_zero[tid - (FT_THREADS - C)] = 0.f;
    __syncthreads();
    float* row = nullptr;
    unsigned char* mark = nullptr;
    if (tid < FT_P) {
        const long long p = p0 + tid;
        unsigned char f = 0;
        if (p < pillars) {
            mark = touched + static_cast<size_t>(frame) * pillars + p;
            f = *mark;
        }
        s_flag[tid] = f;
        if (f) {
            row = accum + (static_cast<size_t>(frame) * pillars + p) * C;
            mbar_arrive_expect_tx(&bar, C * 4);
            bulk_load_1d(s_in + tid * C, row, C * 4, &bar, l2_evict_last());
        } else {
            mbar_arrive(&bar);
        }
    }
    __syncthreads();                                    // s_flag
    mbar_wait(&bar, 0);                                 // every fetched row has landed
    {
        // 16-byte reads: a quarter-warp (8 lanes = 8 pillars, rows 256 B apart) reads the 8 different 16-byte chunks
        // chunk0 + (i ^ (lane & 7)) of a 32-channel block, so every LDS.128 phase covers all 32 banks; the four values go to
        // channel rows 4*chunk .. 4*chunk+3 of this lane's pillar column (bank = lane)
        const int lane = tid & 31, w = tid >> 5;
        const int pl = (w & 1) * 32 + lane;             // pillar of this lane
        const int chunk0 = ((w >> 1) & 1) * 8;          // 32-channel block = 8 chunks of 4 channels
        const int i0 = (w >> 2) * 4;                    // this warp's four of the eight rotations
        const bool have = s_flag[pl] != 0;
        const float4* src = reinterpret_cast<const float4*>(s_in + pl * C);
        float* dst = s_out + pl;
        const int l7 = lane & 7;
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
            const int chunk = chunk0 + ((i0 + ii) ^ l7);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (have) v = src[chunk];
            float* d = dst + chunk * (4 * FT_P);
            d[0] = v.x; d[FT_P] = v.y; d[2 * FT_P] = v.z; d[3 * FT_P] = v.w;
        }
    }
    fence_proxy_async();                                // generic-proxy writes (s_out, s_zero) -> visible to the copy engine
    __syncthreads();
    if (tid == 0) tma_store_3d(&bev_map, s_out, static_cast<int>(p0), 0, frame_out0 + frame, l2_evict_first());   // written once
    if (row) {                                          // restore the all-zero scratch
        bulk_store_1d(row, s_zero, C * 4, l2_restore_policy(last_in_lane));
        if (clear_marks) *mark = 0;             // marks of a caller-owned plan stay: the plan is reused
    }
    if (tid == 0 || row) tma_store_commit_and_wait();   // the shared sources must outlive the copies
}

// ---------------------------------------------------------------------------------------------------------------------
// Layout pass with the warp of cumulative_warp_features folded in (SURVEY.md section 8f next-1; fiery/models/fiery.py:143-146,
// fiery/utils/geometry.py:181-253): instead of transposing the channel-last accumulator of a frame into the NCHW output and letting
// a second kernel re-read it, every OUTPUT pixel of the frame gathers its (up to) four bilinear neighbours straight from the
// accumulator -- whose 256-byte channel rows are exactly what a gather wants -- and the blended pixel goes to the NCHW output.
// Present frames (copy flag) take their own pillar with weight one: bit-identical to the plain layout pass.  Sample positions
// and the blend order are those of warp_forward_kernel (warp_sample.cuh).  A quarter-warp serves one output pixel (lane = two
// 16-byte pieces of the channel row: one full 128-byte line per quarter and load instruction), four neighbours are fetched
// before the first use; pillars that received no point (mark byte clear) are not read.  The (64 pixels x 64 channels) block is
// turned through padded shared memory (conflict-free both ways) so that every store instruction writes 128 contiguous bytes of a
// channel plane.  A source pillar is read by several CTAs, so the accumulator cannot be cleared here: clear_touched_kernel
// restores the all-zero scratch afterwards.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FW_P = 64;
constexpr int FW_THREADS = 256;
__global__ void __launch_bounds__(FW_THREADS)
finalize_warp_kernel(const float* __restrict__ accum, const unsigned char* __restrict__ touched, float* __restrict__ bev,
                     long long pillars, int H, int W, int tiles_per_frame, int frame_out0, const float* __restrict__ theta,
                     const unsigned char* __restrict__ copy_mask) {
    constexpr int C = 64;
    __shared__ float s_out[C][FW_P + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int frame = blockIdx.x / tiles_per_frame;
    const long long p0 = static_cast<long long>(blockIdx.x % tiles_per_frame) * FW_P;
    const int gframe = frame_out0 + frame;
    const float* acc_f = accum + static_cast<size_t>(frame) * pillars * C;
    const unsigned char* tch = touched + static_cast<size_t>(frame) * pillars;
    const int l = lane & 7, q = lane >> 3;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
        const int pxl = pass * 32 + warp * 4 + q;
        const long long pix = p0 + pxl;
        float4 a[4], b[4];
        float w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            a[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            b[k] = a[k];
            w[k] = 0.f;
        }
        if (pix < pillars) {
            const SamplePos s = make_sample(theta, copy_mask, gframe, static_cast<int>(pix), W, H, 0);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                w[k] = s.w[k];
                if (s.ok[k] && tch[s.off[k]]) {
                    const float4* row = reinterpret_cast<const float4*>(acc_f + static_cast<size_t>(s.off[k]) * C);
                    a[k] = __ldg(row + l);
                    b[k] = __ldg(row + 8 + l);
                }
            }
        }
        // the blend of warp_forward_kernel: w0*v0, then fma with neighbours 1..3
        float4 ra, rb;
#define FIERY_BLEND(f) \
        ra.f = fmaf(w[3], a[3].f, fmaf(w[2], a[2].f, fmaf(w[1], a[1].f, w[0] * a[0].f))); \
        rb.f = fmaf(w[3], b[3].f, fmaf(w[2], b[2].f, fmaf(w[1], b[1].f, w[0] * b[0].f)));
        FIERY_BLEND(x) FIERY_BLEND(y) FIERY_BLEND(z) FIERY_BLEND(w)
#undef FIERY_BLEND
        s_out[4 * l + 0][pxl] = ra.x; s_out[4 * l + 1][pxl] = ra.y; s_out[4 * l + 2][pxl] = ra.z; s_out[4 * l + 3][pxl] = ra.w;
        s_out[32 + 4 * l + 0][pxl] = rb.x; s_out[32 + 4 * l + 1][pxl] = rb.y; s_out[32 + 4 * l + 2][pxl] = rb.z; s_out[32 + 4 * l + 3][pxl] = rb.w;
    }
    __syncthreads();
    float* dst = bev + static_cast<size_t>(gframe) * C * pillars + p0;
    const uint64_t once = l2_evict_first();             // the output is written once
#pragma unroll
    for (int cc = 0; cc < C / (FW_THREADS / 32); ++cc) {
        const int c = warp * (C / (FW_THREADS / 32)) + cc;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int px = half * 32 + lane;
            if (p0 + px < pillars)
                asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;"
                             ::"l"(dst + static_cast<size_t>(c) * pillars + px), "f"(s_out[c][px]), "l"(once) : "memory");
        }
    }
}

// Restores the all-zero scratch after finalize_warp_kernel: a warp looks at 32 marks and zeroes the 256-byte accumulator row of
// every marked pillar with one 8-byte store per lane; marks that live in the scratch are cleared too (a caller's plan keeps its own).
__global__ void __launch_bounds__(256)
clear_touched_kernel(float* __restrict__ accum, unsigned char* __restrict__ touched, long long n_pillars, int clear_marks,
                     int last_in_lane) {
    const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const unsigned char f = p < n_pillars ? touched[p] : 0;
    unsigned m = __ballot_sync(0xffffffffu, f != 0);
    const long long base = p - lane;
    const uint64_t policy = l2_restore_policy(last_in_lane);
    while (m) {
        const int i = __ffs(m) - 1;
        m &= m - 1;
        asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %1}, %2;"
                     ::"l"(accum + static_cast<size_t>(base + i) * 64 + 2 * lane), "f"(0.f), "l"(policy) : "memory");
    }
    if (f && clear_marks) touched[p] = 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Integer index dump (fiery.py:236-256) for parity checks; one thread per (frame, camera, depth, row, column) point.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void point_indices_kernel(const LiftParams P, int64_t* __restrict__ idx_out, uint8_t* __restrict__ valid_out,
                                     int32_t* __restrict__ pillar_out, long long n_points_total) {
    const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gid >= n_points_total) return;
    const int w = static_cast<int>(gid % P.ww);
    long long r = gid / P.ww;
    const int h = static_cast<int>(r % P.hh); r /= P.hh;
    const int d = static_cast<int>(r % P.D); r /= P.D;
    const int cam_flat = static_cast<int>(r);
    CameraTransform T;
    load_camera(P.calib_mode, P.calib_a, P.calib_b, cam_flat, T);
    const float depth = P.fd[d];
    const ColumnTerms ct = column_terms(T, P.fu[w], depth);
    float p[3];
    ego_point(T, ct, P.fv[h], depth, p);
    const int pl = pillar_of(P.grid, p);
    if (pillar_out) pillar_out[gid] = pl;
    if (valid_out) valid_out[gid] = pl >= 0 ? 1 : 0;
    if (idx_out) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            // the reference's own expression: true division, then .long() (fiery.py:236-237)
            const float s = __fdiv_rn(__fsub_rn(p[a], P.grid.off[a]), P.grid.res[a]);
            idx_out[gid * 3 + a] = static_cast<int64_t>(s);
        }
    }
}

__global__ void compose_calibration_kernel(int n, const float* __restrict__ K, const float* __restrict__ E,
                                           float* __restrict__ combined, float* __restrict__ translation) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    CameraTransform T;
    compose_camera(K + i * 9, E + i * 16, T);
    for (int k = 0; k < 9; ++k) combined[i * 9 + k] = T.m[k];
    for (int k = 0; k < 3; ++k) translation[i * 3 + k] = T.t[k];
}

// ---------------------------------------------------------------------------------------------------------------------
// host launchers (called from c_api.cu)
// ---------------------------------------------------------------------------------------------------------------------
// Frames per launch.  Chunks small enough to keep the accumulator L2-resident pay for extra launches and single-wave grids, so the
// chunk only bounds the scratch footprint (1 GiB: accumulator + marks of a chunk).
static std::atomic<int> g_max_chunk_frames{0};       // fiery_lift_set_max_chunk_frames (test hook: forces the multi-pass path)
void lift_set_max_chunk_frames(int n) { g_max_chunk_frames.store(n > 0 ? n : 0); }

static int lift_chunk_frames(const LiftParams& P) {
    const long long per_frame = P.pillars * P.C * 4 + P.pillars;
    long long c = (1ll << 30) / (per_frame > 0 ? per_frame : 1);
    const int forced = g_max_chunk_frames.load();
    if (forced > 0 && forced < c) c = forced;
    if (c > P.n_frames) c = P.n_frames;
    return static_cast<int>(c < 1 ? 1 : c);
}

// Side streams and fork/join events of the forward chains: created once per host thread and device (thread_local, so concurrent
// callers never share or race on them), reused by every call -- nothing is created or destroyed on the launch path.
constexpr int MAX_CHAINS = 4;     // frame groups of a pass
constexpr int MAX_LANES = 2;      // streams (and scratch slices) they run on, see lane_layout
struct ChainResources {
    cudaStream_t side[MAX_LANES - 1] = {};
    cudaEvent_t fork = nullptr;
    cudaEvent_t done[MAX_LANES - 1] = {};
    bool ready = false;
};
static int chain_resources(ChainResources** out) {
    static thread_local ChainResources pool[16];
    int dev = 0;
    FIERY_CUDA_CHECK(cudaGetDevice(&dev));
    FIERY_REQUIRE(dev >= 0 && dev < 16, "device %d out of range for the chain resources", dev);
    ChainResources& r = pool[dev];
    if (!r.ready) {
        for (int i = 0; i < MAX_LANES - 1; ++i) {
            FIERY_CUDA_CHECK(cudaStreamCreateWithFlags(&r.side[i], cudaStreamNonBlocking));
            FIERY_CUDA_CHECK(cudaEventCreateWithFlags(&r.done[i], cudaEventDisableTiming));
        }
        FIERY_CUDA_CHECK(cudaEventCreateWithFlags(&r.fork, cudaEventDisableTiming));
        r.ready = true;
    }
    *out = &r;
    return FIERY_OK;
}

// NCHW output: the frames of a chunk are cut into groups, each a tile kernel -> layout pass chain, spread over the lanes below.
// The layout pass of one group (DRAM-bound) runs beside the tile kernel of the other lane (issue-bound); only the last pass is
// exposed.  A group whose tile kernel cannot fill the GPU once loses more than the overlap gains, so a group keeps at least one
// tile per SM of an H100 SXM (132).  The count is host logic (fiery_lift_forward_launches answers without a device), hence a
// constant rather than the device's SM count.
constexpr int CHAIN_MIN_TILES = 132;
int lift_forward_groups(const LiftParams& P, int frames_in_chunk) {
    if (P.bev_layout == FIERY_BEV_NHWC) return 1;          // no layout pass to hide
    int groups = frames_in_chunk < MAX_CHAINS ? frames_in_chunk : MAX_CHAINS;
    const long long tiles_per_frame = static_cast<long long>(P.n_cameras) * P.n_wtiles;
    while (groups > 1 && (frames_in_chunk / groups) * tiles_per_frame < CHAIN_MIN_TILES) --groups;
    return groups < 1 ? 1 : groups;
}

// Scratch lanes.  The frame groups of a pass share the scratch in (at most MAX_LANES) slices: group g runs on lane g % lanes, i.e. on
// that lane's stream and in that lane's slice, so a lane runs tile(g) -> layout(g) -> tile(g + lanes) -> ...  Stream order alone
// guarantees that the layout pass of one group has restored the zeros before the next group of the lane reduces into the slice.
// Frames of one rig touch nearly the same pillars, so the next group's reductions land on lines the layout pass has just re-zeroed
// in L2 (kept there with evict_last hints) instead of fetching zeros from DRAM, and the scratch of a pass is the largest group of
// each lane, not the whole chunk.  Fewer lanes move fewer bytes but overlap less of the layout passes with tile kernels: on an H100
// two lanes beat three and four on every bench workload (DESIGN.md section 2.3).  Host logic, like the group count.
struct LaneLayout {
    int groups, lanes;
    int frames;                               // scratch frames of the pass
    int slice0[MAX_LANES];                    // first scratch frame of each lane's slice
};
static int group_start(int nf, int groups, int g) { return static_cast<int>(static_cast<long long>(nf) * g / groups); }
static LaneLayout lane_layout(const LiftParams& P, int frames_in_chunk) {
    LaneLayout L;
    L.groups = lift_forward_groups(P, frames_in_chunk);
    L.lanes = L.groups < MAX_LANES ? L.groups : MAX_LANES;
    L.frames = 0;
    for (int l = 0; l < L.lanes; ++l) {
        int largest = 0;
        for (int g = l; g < L.groups; g += L.lanes) {
            const int n = group_start(frames_in_chunk, L.groups, g + 1) - group_start(frames_in_chunk, L.groups, g);
            largest = n > largest ? n : largest;
        }
        L.slice0[l] = L.frames;
        L.frames += largest;
    }
    return L;
}

// frames of scratch a call needs: the lanes' frames of its largest pass
static int scratch_frames(const LiftParams& P) {
    const int chunk = lift_chunk_frames(P);
    const int full = lane_layout(P, chunk).frames;
    if (P.n_frames % chunk == 0) return full;
    const int tail = lane_layout(P, P.n_frames % chunk).frames;     // the last pass is shorter and may be cut into fewer groups
    return tail > full ? tail : full;
}

// scratch (NCHW output): [accumulator (F, X*Y, C) fp32][marks (F, X*Y) bytes, padded to 128], F = scratch_frames; all zero between calls
size_t lift_scratch_bytes(const LiftParams& P) {
    if (P.bev_layout != FIERY_BEV_NCHW || P.n_frames <= 0) return 0;
    const size_t f = static_cast<size_t>(scratch_frames(P));
    return f * P.pillars * P.C * 4 + ((f * P.pillars + 127) & ~static_cast<size_t>(127));
}

// kernel launches of one forward call (include/fiery_b200.h: fiery_lift_forward_launches)
int lift_forward_launches(const LiftParams& P) {
    if (P.n_frames <= 0) return 0;
    const int per_group = 1 + (P.bev_layout == FIERY_BEV_NCHW ? 1 : 0);
    const int chunk = lift_chunk_frames(P);
    int n = 0;
    for (int f0 = 0; f0 < P.n_frames; f0 += chunk)
        n += per_group * lift_forward_groups(P, (P.n_frames - f0 < chunk) ? P.n_frames - f0 : chunk);
    return n;
}

// Per-launch timing (bench / profiling): when set, every kernel launch of the next forward call on this host thread is bracketed by
// a pair of events on its own stream; see fiery_lift_forward_timed in c_api.cu.
static thread_local LaunchTimer* g_timer = nullptr;
void lift_set_timer(LaunchTimer* t) { g_timer = t; }
static inline void timer_begin(cudaStream_t st, int kind) {
    if (g_timer && g_timer->n < g_timer->cap) {
        g_timer->kind[g_timer->n] = kind;
        cudaEventRecord(g_timer->ev[2 * g_timer->n], st);
    }
}
static inline void timer_end(cudaStream_t st) {
    if (g_timer && g_timer->n < g_timer->cap) {
        cudaEventRecord(g_timer->ev[2 * g_timer->n + 1], st);
        ++g_timer->n;
    }
}

// The NCHW layout pass of both forward paths: the warped pass when a warp is given, else the TMA pass when the output has a 16-byte
// row pitch, else the fallback pass.
struct LayoutPass {
    const float* warp_theta;
    const unsigned char* warp_copy;
    bool tma;                                       // the TMA pass's output map needs a 16-byte row pitch
    CUtensorMap bev_map;
};
static int prepare_layout_pass(LayoutPass* L, const LiftParams& P, float* bev_out, const float* warp_theta,
                               const unsigned char* warp_copy) {
    *L = LayoutPass{warp_theta, warp_copy, P.pillars % 4 == 0, {}};
    if (P.bev_layout != FIERY_BEV_NCHW || !L->tma || warp_theta) return FIERY_OK;
    return encode_bev_map(&L->bev_map, bev_out, P.pillars, P.C, P.n_frames, FT_P);
}

// output frames frame0 .. frame0 + n_frames - 1 from their accumulator rows and marks
static void launch_layout_pass(const LayoutPass& L, const LiftParams& P, float* accum, unsigned char* marks, float* bev_out, int frame0,
                               int n_frames, int clear_marks, int last_in_lane, cudaStream_t st) {
    if (L.warp_theta) {
        const int tpf = static_cast<int>((P.pillars + FW_P - 1) / FW_P);
        finalize_warp_kernel<<<static_cast<unsigned>(tpf) * n_frames, FW_THREADS, 0, st>>>(
            accum, marks, bev_out, P.pillars, P.grid.X, P.grid.Y, tpf, frame0, L.warp_theta, L.warp_copy);
    } else if (L.tma) {
        const int tpf = static_cast<int>((P.pillars + FT_P - 1) / FT_P);
        finalize_tma_kernel<<<static_cast<unsigned>(tpf) * n_frames, FT_THREADS, 0, st>>>(
            L.bev_map, accum, marks, P.pillars, tpf, frame0, clear_marks, last_in_lane);
    } else {
        const int bpf = static_cast<int>((P.pillars + FIN_THREADS - 1) / FIN_THREADS);
        finalize_nchw_kernel<<<static_cast<unsigned>(bpf) * n_frames, FIN_THREADS, 0, st>>>(
            accum, marks, bev_out + static_cast<size_t>(frame0) * P.C * P.pillars, P.pillars, bpf, clear_marks);
    }
}

// warp_theta != NULL: the layout pass samples every frame under its (2, 3) affine map (frames flagged in warp_copy pass through) --
// the lift followed by cumulative_warp_features in one chain; NCHW output only
int launch_lift_forward(const LiftParams& P, const void* head, int head_dtype, float* bev_out, void* scratch, const void* plan,
                        const float* warp_theta, const unsigned char* warp_copy, cudaStream_t stream) {
    const bool nchw = P.bev_layout == FIERY_BEV_NCHW;
    FIERY_REQUIRE(scratch != nullptr || !nchw, "NCHW output needs the zeroed scratch buffer of fiery_lift_scratch_bytes()");
    LiftParams Q = P;
    Q.head_f16 = head_dtype == FIERY_DTYPE_F16 ? head : nullptr;
    // lift into a channel-last accumulator (NHWC: the caller's zero-filled output itself), then the layout pass for NCHW; several
    // passes only to bound the scratch footprint
    const int chunk = lift_chunk_frames(P);
    float* accum = static_cast<float*>(scratch);    // [accumulator floats of the lanes][one mark byte per pillar]
    unsigned char* scratch_marks =
        nchw ? reinterpret_cast<unsigned char*>(accum + static_cast<size_t>(scratch_frames(P)) * P.pillars * P.C) : nullptr;
    LayoutPass pass;
    int rc = prepare_layout_pass(&pass, P, bev_out, warp_theta, warp_copy);
    if (rc != FIERY_OK) return rc;
    ChainResources* res = nullptr;
    for (int f0 = 0; f0 < P.n_frames; f0 += chunk) {
        const int nf = (P.n_frames - f0 < chunk) ? P.n_frames - f0 : chunk;
        const LaneLayout lanes = lane_layout(P, nf);
        cudaStream_t chain[MAX_LANES] = {stream};
        if (lanes.lanes > 1) {                      // fork: the side streams start behind everything queued on the caller's
            if (!res) {
                rc = chain_resources(&res);
                if (rc != FIERY_OK) return rc;
            }
            for (int l = 1; l < lanes.lanes; ++l) chain[l] = res->side[l - 1];
            FIERY_CUDA_CHECK(cudaEventRecord(res->fork, stream));
        }
        for (int g = 0; g < lanes.groups; ++g) {
            const int s0 = group_start(nf, lanes.groups, g), s1 = group_start(nf, lanes.groups, g + 1);
            const int lane = g % lanes.lanes;
            const bool last_in_lane = g + lanes.lanes >= lanes.groups;
            const size_t slice = static_cast<size_t>(lanes.slice0[lane]);
            cudaStream_t st = chain[lane];
            if (lane > 0 && g < lanes.lanes) FIERY_CUDA_CHECK(cudaStreamWaitEvent(st, res->fork, 0));
            Q.frame0 = f0 + s0;
            Q.n_frames = s1 - s0;
            unsigned char* marks = nullptr;         // "pillar receives a point" bytes the layout pass reads
            if (plan) {                             // caller-owned plan of the whole batch: read only, marks included
                const PlanView v = plan_view(plan, P.n_frames, P.n_cameras, P.n_wtiles, P.pillars, Q.frame0);
                Q.plan_tiles = v.tiles;
                Q.touched = nullptr;
                marks = const_cast<unsigned char*>(v.touched);
            } else {                                // the tile kernel evaluates the geometry itself and marks into the scratch
                Q.plan_tiles = nullptr;
                marks = nchw ? scratch_marks + slice * P.pillars : nullptr;
                Q.touched = marks;
            }
            Q.accum = nchw ? accum + slice * P.pillars * P.C
                           : bev_out + static_cast<size_t>(Q.frame0) * P.pillars * P.C;
            timer_begin(st, 1);
            rc = launch_forward_cols(Q, head, st);
            timer_end(st);
            if (rc != FIERY_OK) return rc;
            if (nchw) {
                timer_begin(st, 2);
                launch_layout_pass(pass, P, Q.accum, marks, bev_out, Q.frame0, Q.n_frames, plan ? 0 : 1, last_in_lane ? 1 : 0, st);
                if (warp_theta) {
                    const long long n = P.pillars * Q.n_frames;
                    clear_touched_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(Q.accum, marks, n, plan ? 0 : 1,
                                                                                                 last_in_lane ? 1 : 0);
                }
                timer_end(st);
                FIERY_CUDA_CHECK(cudaGetLastError());
            }
            if (lane > 0 && last_in_lane) {         // join the lane back into the caller's stream
                FIERY_CUDA_CHECK(cudaEventRecord(res->done[lane - 1], st));
                FIERY_CUDA_CHECK(cudaStreamWaitEvent(stream, res->done[lane - 1], 0));
            }
        }
    }
    return FIERY_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Deterministic forward (fiery_lift_forward_deterministic; kernels and summation order: lift_det.cu).  Per pass of frames, in the
// workspace: [plan of the pass (internal plan only)][partial sums: a row of 64 floats per possible run][channel-last accumulator
// (NCHW output only)][list starts][list cursors][lists].  Everything is sized for the worst case -- one run per frustum point -- so
// no count ever comes back to the host, and a pass holds as many frames as fit the cap the default path's scratch has (1 GiB).
// ---------------------------------------------------------------------------------------------------------------------
struct DetLayout {
    int frames;                                          // frames per pass
    size_t plan, partials, accum, start, cursor, lists, total;   // byte offsets into the workspace, and its size
};
static size_t det_align(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }
static DetLayout det_layout(const LiftParams& P) {
    const size_t tpf = static_cast<size_t>(P.n_cameras) * P.n_wtiles;
    const size_t rows = tpf * det_runs_per_tile(P.hh);
    const bool nchw = P.bev_layout == FIERY_BEV_NCHW;
    const size_t per_frame = tpf * PLAN_TILE_BYTES + P.pillars + rows * 64 * 4 + (nchw ? P.pillars * 64 * 4 : 0) + P.pillars * 8 + rows * 4;
    long long c = static_cast<long long>((1ull << 30) / per_frame);
    const int forced = g_max_chunk_frames.load();
    if (forced > 0 && forced < c) c = forced;
    if (c > P.n_frames) c = P.n_frames;
    DetLayout L;
    L.frames = static_cast<int>(c < 1 ? 1 : c);
    const size_t f = L.frames;
    L.plan = 0;
    L.partials = det_align(plan_bytes(L.frames, P.n_cameras, P.n_wtiles, P.pillars));
    L.accum = L.partials + det_align(f * rows * 64 * 4);
    L.start = L.accum + (nchw ? det_align(f * P.pillars * 64 * 4) : 0);
    L.cursor = L.start + det_align(f * P.pillars * 4);
    L.lists = L.cursor + det_align(f * P.pillars * 4);
    L.total = L.lists + det_align(f * rows * 4);
    return L;
}

size_t lift_det_workspace_bytes(const LiftParams& P) { return P.n_frames > 0 ? det_layout(P).total : 0; }

int launch_lift_forward_det(const LiftParams& P, const void* head, int head_dtype, float* bev_out, void* workspace, const void* plan,
                            const float* warp_theta, const unsigned char* warp_copy, cudaStream_t stream) {
    const bool nchw = P.bev_layout == FIERY_BEV_NCHW;
    FIERY_REQUIRE(workspace != nullptr, "the deterministic forward needs the workspace of fiery_lift_deterministic_workspace_bytes()");
    const DetLayout W = det_layout(P);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    float* partials = reinterpret_cast<float*>(ws + W.partials);
    float* accum = reinterpret_cast<float*>(ws + W.accum);
    int* start = reinterpret_cast<int*>(ws + W.start);
    int* cursor = reinterpret_cast<int*>(ws + W.cursor);
    int* lists = reinterpret_cast<int*>(ws + W.lists);
    LayoutPass pass;
    int rc = prepare_layout_pass(&pass, P, bev_out, warp_theta, warp_copy);
    if (rc != FIERY_OK) return rc;
    LiftParams Q = P;
    Q.head_f16 = head_dtype == FIERY_DTYPE_F16 ? head : nullptr;
    Q.touched = nullptr;
    for (int f0 = 0; f0 < P.n_frames; f0 += W.frames) {
        Q.frame0 = f0;
        Q.n_frames = (P.n_frames - f0 < W.frames) ? P.n_frames - f0 : W.frames;
        const unsigned char* marks;
        if (plan) {
            const PlanView v = plan_view(plan, P.n_frames, P.n_cameras, P.n_wtiles, P.pillars, f0);
            Q.plan_tiles = v.tiles;
            marks = v.touched;
        } else {                                     // a forward-only plan of this pass's frames (no backward streams)
            const PlanView v = plan_view(ws + W.plan, Q.n_frames, P.n_cameras, P.n_wtiles, P.pillars, 0);
            FIERY_CUDA_CHECK(cudaMemsetAsync(const_cast<unsigned char*>(v.touched), 0, static_cast<size_t>(Q.n_frames) * P.pillars, stream));
            rc = launch_lift_plan(Q, const_cast<unsigned char*>(v.tiles), const_cast<unsigned char*>(v.touched), 0, stream);
            if (rc != FIERY_OK) return rc;
            Q.plan_tiles = v.tiles;
            marks = v.touched;
        }
        Q.accum = partials;
        rc = launch_forward_cols_det(Q, head, stream);
        if (rc != FIERY_OK) return rc;
        float* out = nchw ? accum : bev_out + static_cast<size_t>(f0) * P.pillars * P.C;
        rc = launch_det_reduce(Q, Q.n_frames, Q.plan_tiles, partials, start, cursor, lists, out, nchw ? 0 : 1, stream);
        if (rc != FIERY_OK) return rc;
        if (!nchw) continue;
        // the layout passes of the default path, unchanged; they read exactly the marked rows, which the reduction has written.  The
        // workspace needs no restoring, so marks are never cleared and the accumulator's rows need not be re-zeroed after the warp.
        launch_layout_pass(pass, P, accum, const_cast<unsigned char*>(marks), bev_out, f0, Q.n_frames, 0, 1, stream);
        FIERY_CUDA_CHECK(cudaGetLastError());
    }
    return FIERY_OK;
}

int launch_point_indices(const LiftParams& P, int64_t* idx_out, uint8_t* valid_out, int32_t* pillar_out, cudaStream_t stream) {
    const long long total = static_cast<long long>(P.n_frames) * P.n_cameras * P.D * P.hh * P.ww;
    if (total == 0) return FIERY_OK;
    const int threads = 256;
    point_indices_kernel<<<static_cast<unsigned>((total + threads - 1) / threads), threads, 0, stream>>>(
        P, idx_out, valid_out, pillar_out, total);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_compose(int n, const float* K, const float* E, float* combined, float* translation, cudaStream_t stream) {
    if (n == 0) return FIERY_OK;
    compose_calibration_kernel<<<(n + 127) / 128, 128, 0, stream>>>(n, K, E, combined, translation);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
