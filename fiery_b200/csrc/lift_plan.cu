// Geometry plan kernel (layout and rationale: lift_plan.cuh).
//
// get_geometry (fiery/models/fiery.py:193-208) + voxel index / mask / rank of every frustum point (fiery.py:236-256), evaluated with
// the reference's exact fp32 operation order (geometry.cuh) and reduced on the fly to pillar runs.  One CTA per tile (camera image x
// 4 feature-map columns), one thread per (depth, column) pair walking the image rows.
#include "lift_plan.cuh"

namespace fiery {

template <bool POW2>
__global__ void __launch_bounds__(PLAN_PAIRS)
lift_plan_kernel(const LiftParams P, unsigned char* __restrict__ tiles, unsigned char* __restrict__ touched, int want_streams) {
    __shared__ float s_cam[12];
    __shared__ float s_u[WT];
    __shared__ float s_v[PLAN_MAX_ROWS];
    __shared__ float s_d[DPAD];
    __shared__ unsigned s_mask[PLAN_PAIRS];
    __shared__ int s_warp_sum[PLAN_PAIRS / 32];
    __shared__ unsigned short s_seg[PLAN_RG * PLAN_PAIRS];   // segment lengths, then offsets, in (rg, col, j, g) order
    __shared__ int s_tmp[PLAN_MAX_ROWS * PLAN_PAIRS];     // [k][pair]: pillar of the pair's k-th run

    const int tid = threadIdx.x;
    const int wtile = blockIdx.x % P.n_wtiles;
    const int img_local = blockIdx.x / P.n_wtiles;      // (frame, camera) within this launch
    const int img = P.frame0 * P.n_cameras + img_local; // absolute: indexes the calibration
    const int frame = img_local / P.n_cameras;          // launch-local: indexes the touched map
    const int w0 = wtile * WT;
    const int hh = P.hh;
    unsigned char* rec = tiles + static_cast<size_t>(blockIdx.x) * PLAN_TILE_BYTES;

    if (tid < WT) s_u[tid] = (w0 + tid < P.ww) ? P.fu[w0 + tid] : 0.f;
    if (tid >= 32 && tid < 64) s_v[tid - 32] = P.fv[min(tid - 32, hh - 1)];
    if (tid >= 64 && tid < 64 + DPAD) s_d[tid - 64] = (tid - 64 < P.D) ? P.fd[tid - 64] : 0.f;
    if (tid == PLAN_PAIRS - 1) {                        // one lane composes R @ K^-1 (fiery.py:203)
        CameraTransform T;
        load_camera(P.calib_mode, P.calib_a, P.calib_b, img, T);
#pragma unroll
        for (int i = 0; i < 9; ++i) s_cam[i] = T.m[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) s_cam[9 + i] = T.t[i];
    }
    __syncthreads();

    // ---- runs of my pair ---------------------------------------------------------------------------------------------------
    const int pair = tid, d = pair >> 2, col = pair & 3;
    const bool dead = d >= P.D || w0 + col >= P.ww;
    unsigned mask = 0;
    int n = 1;
    if (dead) {
        s_tmp[pair] = -1;
    } else {
        CameraTransform T;
#pragma unroll
        for (int i = 0; i < 9; ++i) T.m[i] = s_cam[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) T.t[i] = s_cam[9 + i];
        const PillarMap<POW2> pillar(P.grid);
        unsigned char* tmap = touched ? touched + static_cast<size_t>(frame) * P.pillars : nullptr;
        const float depth = s_d[d];
        const ColumnTerms ct = column_terms(T, s_u[col], depth);
        int prev = 0;
        n = 0;
#pragma unroll 4
        for (int h = 0; h < hh; ++h) {
            const int cur = pillar(T, ct, s_v[h], depth);
            if (h == 0 || cur != prev) {
                if (h) mask |= 1u << h;
                s_tmp[n * PLAN_PAIRS + pair] = cur;
                ++n;
                if (tmap && cur >= 0) tmap[cur] = 1;
            }
            prev = cur;
        }
    }
    s_mask[pair] = mask;

    // ---- exclusive scan of the run counts over the pairs: offsets into runs[] -------------------------------------------------
    const int lane = tid & 31, warp = tid >> 5;
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp_sum[warp] = incl;
    __syncthreads();
    int base = 0;
#pragma unroll
    for (int w = 0; w < PLAN_PAIRS / 32; ++w) base += (w < warp) ? s_warp_sum[w] : 0;
    const int off = base + incl - n;
    reinterpret_cast<unsigned*>(rec + PLAN_OFF_MASK)[pair] = mask;
    reinterpret_cast<unsigned short*>(rec + PLAN_OFF_OFF)[pair] = static_cast<unsigned short>(off);
    {
        int* runs = reinterpret_cast<int*>(rec + PLAN_OFF_RUNS) + off;
        for (int k = 0; k < n; ++k) runs[k] = s_tmp[k * PLAN_PAIRS + pair];
    }

    if (tid == PLAN_PAIRS - 1) reinterpret_cast<unsigned*>(rec + PLAN_OFF_COUNTS)[0] = static_cast<unsigned>(base + incl);   // n_runs
    if (!want_streams) {                                 // forward-only plan: the backward streams are not built
        if (tid == 0) reinterpret_cast<unsigned*>(rec + PLAN_OFF_COUNTS)[1] = 0u;
        return;
    }

    // ---- backward streams: per (row group, column, slot j) the runs of depths j, 4 + j, 8 + j, ... clipped to the row group --------
    // A segment = the runs of one pair inside one row group: the run that contains the group's first row + the runs that start
    // inside the group.  Stream (rg, col, j) = segments of depth groups g = 0..11 in order + two pad entries; the streams follow each
    // other in streams[].  Offsets: exclusive scan over the 768 segment lengths in (rg, col, j, g) order, + 2 per preceding stream.
    constexpr int NG = DPAD / PLAN_ND;
    const int g_of = d / PLAN_ND, j_of = d % PLAN_ND;
    unsigned in_group[PLAN_RG], upto[PLAN_RG];
#pragma unroll
    for (int rg = 0; rg < PLAN_RG; ++rg) {
        const int r_lo = plan_group_row(hh, rg), r_hi = plan_group_row(hh, rg + 1);
        upto[rg] = (2u << r_lo) - 1u;                                                   // rows 0 .. r_lo
        in_group[rg] = (r_hi >= 32 ? 0xffffffffu : ((1u << r_hi) - 1u)) & ~upto[rg];    // rows r_lo + 1 .. r_hi - 1
        s_seg[((rg * WT + col) * PLAN_ND + j_of) * NG + g_of] = static_cast<unsigned short>(1 + __popc(mask & in_group[rg]));
    }
    __syncthreads();
    {   // thread t scans the ordered entries 4t .. 4t+3 (one third of a stream), then warp / block prefix
        const int e0 = tid * 4;
        const int l0 = s_seg[e0], l1 = s_seg[e0 + 1], l2 = s_seg[e0 + 2], l3 = s_seg[e0 + 3];
        int tot = l0 + l1 + l2 + l3, inc = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_warp_sum[warp] = inc;       // (the run-count sums in s_warp_sum were consumed before the barrier above)
        __syncthreads();
        int sbase = 0;
#pragma unroll
        for (int w = 0; w < PLAN_PAIRS / 32; ++w) sbase += (w < warp) ? s_warp_sum[w] : 0;
        const int ex = sbase + inc - tot + 2 * (e0 / NG);                               // + the pads of the streams before mine
        s_seg[e0] = static_cast<unsigned short>(ex);
        s_seg[e0 + 1] = static_cast<unsigned short>(ex + l0);
        s_seg[e0 + 2] = static_cast<unsigned short>(ex + l0 + l1);
        s_seg[e0 + 3] = static_cast<unsigned short>(ex + l0 + l1 + l2);
        if (tid == PLAN_PAIRS - 1) reinterpret_cast<unsigned*>(rec + PLAN_OFF_COUNTS)[1] = static_cast<unsigned>(ex + tot + 2);   // n_stream
    }
    __syncthreads();
    int* streams = reinterpret_cast<int*>(rec + PLAN_OFF_STREAMS);
#pragma unroll
    for (int rg = 0; rg < PLAN_RG; ++rg) {
        int pos = s_seg[((rg * WT + col) * PLAN_ND + j_of) * NG + g_of];
        const int k0 = __popc(mask & upto[rg]);                                         // the run that contains row r_lo
        const int c = __popc(mask & in_group[rg]);                                      // runs that start inside the group
        for (int k = k0; k <= k0 + c; ++k) streams[pos++] = s_tmp[k * PLAN_PAIRS + pair];
        if (g_of == NG - 1) {                                                           // last segment of its stream: the pads
            streams[pos] = -1;
            streams[pos + 1] = -1;
        }
    }
    if (tid < PLAN_STREAMS) reinterpret_cast<unsigned short*>(rec + PLAN_OFF_SOFF)[tid] = s_seg[tid * NG];
}

int launch_lift_plan(const LiftParams& P, unsigned char* tiles, unsigned char* touched, int want_streams, cudaStream_t stream) {
    int rc = check_lift_geometry(P);
    if (rc != FIERY_OK) return rc;
    const long long n_tiles = static_cast<long long>(P.n_frames) * P.n_cameras * P.n_wtiles;
    if (n_tiles == 0) return FIERY_OK;
    if (P.grid.pow2[0] && P.grid.pow2[1])
        lift_plan_kernel<true><<<static_cast<unsigned>(n_tiles), PLAN_PAIRS, 0, stream>>>(P, tiles, touched, want_streams);
    else
        lift_plan_kernel<false><<<static_cast<unsigned>(n_tiles), PLAN_PAIRS, 0, stream>>>(P, tiles, touched, want_streams);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
