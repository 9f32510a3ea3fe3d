// BEV feature warping: the step right after the lift (SURVEY.md section 8f, next-1).
//
// Replaces the heavy part of warp_features / cumulative_warp_features (fiery/utils/geometry.py:181-253, call site
// fiery/models/fiery.py:143-146): torch.nn.functional.affine_grid + grid_sample (bilinear or nearest, zero padding,
// align_corners=False) of a (C, H, W) feature map under a 2x3 affine map theta.  The 6-DoF pose algebra that produces theta
// (pose_vec2mat, cumulative products, mat2pose_vec: a few 4x4 matrices per sequence) runs in warp_theta_kernel, one thread per
// sequence, so a whole cumulative_warp_features call is two launches.
//
// HBM-bound gather: algorithmic bytes per map = read C*H*W*4 + write C*H*W*4.  One thread per output pixel and group of 8
// channels; the sample position and the four weights are computed once per pixel, a warp covers 32 consecutive columns so
// the stores are full 128-byte lines and the four gathered rows are near-contiguous for the small rotations of ego motion.
// All 32 gathers of a thread are issued before the first use (memory-level parallelism is what bounds a gather), and the
// plane stride is a template constant for the reference's grids so that every load/store uses an immediate offset from one
// of four neighbour pointers instead of 64-bit address arithmetic per access.
#include "common.cuh"
#include "warp_sample.cuh"

namespace fiery {

constexpr int WARP_THREADS = 256;
constexpr int WARP_CH = 8;        // channels per thread

// PLANE > 0: H*W known at compile time (200x200 and 400x200 grids); PLANE == 0: generic
template <int PLANE>
__global__ void __launch_bounds__(WARP_THREADS)
warp_forward_kernel(int C, int H, int W, const float* __restrict__ x, long long x_stride, const float* __restrict__ theta,
                    const unsigned char* __restrict__ copy_mask, float* __restrict__ out, long long out_stride, int nearest) {
    const int plane = PLANE ? PLANE : H * W;
    const int pix = blockIdx.x * WARP_THREADS + threadIdx.x;
    if (pix >= plane) return;
    const int map = blockIdx.z, c0 = blockIdx.y * WARP_CH;
    const SamplePos s = make_sample(theta, copy_mask, map, pix, W, H, nearest);
    const float* src = x + map * x_stride + static_cast<long long>(c0) * plane;
    float* dst = out + map * out_stride + static_cast<long long>(c0) * plane + pix;
    const float* p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = src + s.off[k];
    const int nc = C - c0;                                   // >= 1
    float v[WARP_CH][4];
#pragma unroll
    for (int c = 0; c < WARP_CH; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k)
            v[c][k] = (s.ok[k] && c < nc) ? __ldg(p[k] + c * plane) : 0.f;
#pragma unroll
    for (int c = 0; c < WARP_CH; ++c) {
        float r = s.w[0] * v[c][0];
        r = fmaf(s.w[1], v[c][1], r);
        r = fmaf(s.w[2], v[c][2], r);
        r = fmaf(s.w[3], v[c][3], r);
        if (c < nc) __stcs(dst + c * plane, r);
    }
}

// Adjoint as a gather, one thread per SOURCE pixel and 32 channels: grad_x[p] = sum over the output pixels q whose sample touches p
// of w(q, p) * grad_out[q].  The candidates q come from the resumable window scan of warp_sample.cuh (3x3..4x4 candidates for the
// rotations warp_features builds, at most a handful of hits); the hits of a round are collected first, then all their loads are
// issued together -- a load inside the search loop would serialise on its latency.  No atomics, no zero-fill of grad_x,
// deterministic; consecutive source pixels have consecutive candidates, so the loads coalesce like the forward's.
constexpr int WB_CH = 32;
constexpr int WB_M = 6;
template <int PLANE>
__global__ void __launch_bounds__(WARP_THREADS, 2)
warp_backward_gather_kernel(int C, int H, int W, const float* __restrict__ gout, long long gout_stride, const float* __restrict__ theta,
                            const unsigned char* __restrict__ copy_mask, float* __restrict__ gx, long long gx_stride, int nearest) {
    const int plane = PLANE ? PLANE : H * W;
    // channel stride in 64 bits: 31 * plane passes 2^31 once H * W > 69.3 M, well inside the accepted H * W < 2^27
    const long long cstride = plane;
    const int pix = blockIdx.x * WARP_THREADS + threadIdx.x;
    if (pix >= plane) return;
    const int map = blockIdx.z, c0 = blockIdx.y * WB_CH;
    const int nc = C - c0;
    const float* g = gout + map * gout_stride + c0 * cstride;
    float* dst = gx + map * gx_stride + c0 * cstride + pix;
    if (copy_mask && copy_mask[map]) {                       // the present frame passed through: so does its gradient
        float v[WB_CH];                                      // all loads first: a store between them would order them
#pragma unroll
        for (int c = 0; c < WB_CH; ++c) v[c] = c < nc ? __ldcs(g + c * cstride + pix) : 0.f;
#pragma unroll
        for (int c = 0; c < WB_CH; ++c)
            if (c < nc) __stcs(dst + c * cstride, v[c]);
        return;
    }
    const float* th = theta + map * 6;
    float acc[WB_CH];
#pragma unroll
    for (int c = 0; c < WB_CH; ++c) acc[c] = 0.f;
    AdjointScan scan = adjoint_scan_begin(inverse_map(th, W, H), pix, W, H, nearest);
    int m_off[WB_M];
    float m_w[WB_M];
    int n_match;
    while ((n_match = adjoint_scan_next<WB_M>(scan, th, W, H, nearest, m_off, m_w)) > 0) {
#pragma unroll
        for (int cb = 0; cb < WB_CH; cb += 8) {            // 8 channels x WB_M candidates: up to 48 loads in flight per thread
            float v[8][WB_M];
#pragma unroll
            for (int c = 0; c < 8; ++c)
#pragma unroll
                for (int k = 0; k < WB_M; ++k) v[c][k] = (k < n_match && cb + c < nc) ? __ldg(g + m_off[k] + (cb + c) * cstride) : 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c)
#pragma unroll
                for (int k = 0; k < WB_M; ++k) acc[cb + c] = fmaf(m_w[k], v[c][k], acc[cb + c]);
        }
    }
#pragma unroll
    for (int c = 0; c < WB_CH; ++c)
        if (c < nc) __stcs(dst + c * cstride, acc[c]);
}

// ---- pose algebra: flow (b, T, 6) -> theta (b*T, 2, 3) -------------------------------------------------------------------
struct Mat4 { float m[4][4]; };

// pose_vec2mat (geometry.py:145-160) with euler2mat (geometry.py:110-142): R = Rx @ Ry @ Rz, last column = translation
__device__ Mat4 pose_to_mat(const float* __restrict__ v) {
    float sx, cx, sy, cy, sz, cz;
    sincosf(v[3], &sx, &cx); sincosf(v[4], &sy, &cy); sincosf(v[5], &sz, &cz);
    const float X[3][3] = {{1.f, 0.f, 0.f}, {0.f, cx, -sx}, {0.f, sx, cx}};
    const float Y[3][3] = {{cy, 0.f, sy}, {0.f, 1.f, 0.f}, {-sy, 0.f, cy}};
    const float Z[3][3] = {{cz, -sz, 0.f}, {sz, cz, 0.f}, {0.f, 0.f, 1.f}};
    float XY[3][3];
    Mat4 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            float a = 0.f;
            for (int k = 0; k < 3; ++k) a += X[i][k] * Y[k][j];
            XY[i][j] = a;
        }
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            float a = 0.f;
            for (int k = 0; k < 3; ++k) a += XY[i][k] * Z[k][j];
            r.m[i][j] = a;
        }
        r.m[i][3] = v[i];
    }
    r.m[3][0] = r.m[3][1] = r.m[3][2] = 0.f; r.m[3][3] = 1.f;
    return r;
}

// the (2, 3) map of warp_features (geometry.py:197-219) from a z angle and an xy translation
__device__ void write_theta(float* __restrict__ th, float angle, float tx, float ty, float ex, float ey) {
    float sn, cs;
    sincosf(angle, &sn, &cs);
    th[0] = cs; th[1] = -sn; th[2] = ty / ey;
    th[3] = sn; th[4] = cs;  th[5] = -(tx / ex);
}

// cumulative != 0: the loop of cumulative_warp_features (geometry.py:241-251), one thread per sequence: frame T-1 is the
// present (copy flag set, theta zero), frame t < T-1 gets mat2pose_vec(flow[t] @ ... @ flow[T-2]).  cumulative == 0: every row
// of flow is used directly (warp_features), T is ignored.
__global__ void warp_theta_kernel(int n_seq, int T, int cumulative, const float* __restrict__ flow, float ex, float ey,
                                  float* __restrict__ theta, unsigned char* __restrict__ copy_mask) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_seq) return;
    if (!cumulative) {
        const float* v = flow + static_cast<long long>(b) * 6;
        write_theta(theta + static_cast<long long>(b) * 6, v[5], v[0], v[1], ex, ey);
        if (copy_mask) copy_mask[b] = 0;
        return;
    }
    const float* f = flow + static_cast<long long>(b) * T * 6;
    float* th = theta + static_cast<long long>(b) * T * 6;
    for (int k = 0; k < 6; ++k) th[(T - 1) * 6 + k] = 0.f;
    copy_mask[b * T + T - 1] = 1;
    if (T < 2) return;
    Mat4 cum = pose_to_mat(f + (T - 2) * 6);
    for (int t = T - 2; t >= 0; --t) {
        // mat2pose_vec (geometry.py:82-107): only the z angle and the xy translation reach warp_features
        write_theta(th + t * 6, atan2f(-cum.m[0][1], cum.m[0][0]), cum.m[0][3], cum.m[1][3], ex, ey);
        copy_mask[b * T + t] = 0;
        if (t == 0) break;
        const Mat4 left = pose_to_mat(f + (t - 1) * 6);
        Mat4 next;
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) {
                float a = 0.f;
                for (int k = 0; k < 4; ++k) a += left.m[i][k] * cum.m[k][j];
                next.m[i][j] = a;
            }
        cum = next;
    }
}

template <int PLANE>
static void launch_warp_plane(int forward, dim3 grid, int C, int H, int W, const float* a, long long a_stride, const float* theta,
                              const unsigned char* copy_mask, float* b, long long b_stride, int nearest, cudaStream_t stream) {
    if (forward) {
        warp_forward_kernel<PLANE><<<grid, WARP_THREADS, 0, stream>>>(C, H, W, a, a_stride, theta, copy_mask, b, b_stride, nearest);
    } else {
        const dim3 ggrid(grid.x, (C + WB_CH - 1) / WB_CH, grid.z);
        warp_backward_gather_kernel<PLANE><<<ggrid, WARP_THREADS, 0, stream>>>(C, H, W, a, a_stride, theta, copy_mask, b, b_stride, nearest);
    }
}

int launch_warp(int forward, int n_maps, int C, int H, int W, const float* a, long long a_stride, const float* theta,
                const unsigned char* copy_mask, float* b, long long b_stride, int nearest, cudaStream_t stream) {
    if (n_maps == 0) return FIERY_OK;
    FIERY_REQUIRE(static_cast<long long>(H) * W < (1ll << 27) && n_maps <= 65535, "warp: map too large / too many maps");
    const int plane = H * W;
    const dim3 grid((plane + WARP_THREADS - 1) / WARP_THREADS, (C + WARP_CH - 1) / WARP_CH, n_maps);
    FIERY_REQUIRE(grid.y <= 65535, "warp: too many channels");
    if (plane == 40000) launch_warp_plane<40000>(forward, grid, C, H, W, a, a_stride, theta, copy_mask, b, b_stride, nearest, stream);
    else if (plane == 80000) launch_warp_plane<80000>(forward, grid, C, H, W, a, a_stride, theta, copy_mask, b, b_stride, nearest, stream);
    else launch_warp_plane<0>(forward, grid, C, H, W, a, a_stride, theta, copy_mask, b, b_stride, nearest, stream);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_warp_theta(int n_seq, int T, int cumulative, const float* flow, float ex, float ey, float* theta,
                      unsigned char* copy_mask, cudaStream_t stream) {
    if (n_seq == 0) return FIERY_OK;
    warp_theta_kernel<<<(n_seq + 63) / 64, 64, 0, stream>>>(n_seq, T, cumulative, flow, ex, ey, theta, copy_mask);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
