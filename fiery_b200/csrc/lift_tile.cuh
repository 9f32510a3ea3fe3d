// What the lift's tile kernels share: the forward (lift_fwd_cols.cu), the backward (lift_bwd.cu) and the geometry plan
// (lift_plan.cu).
//
// Work unit ("tile"): one camera image of one frame, WT = 4 adjacent feature-map columns, all h rows, all D depth bins, all C
// channels.  The forward and the backward fetch the tile from the NCHW head tensor (fiery/models/encoder.py:96 output) with two
// TMA loads that deliver it as prob[row][depth][col4] and ctx[row][k][cl][col4]: the tensor maps do the permutation, nothing is
// transposed in shared memory.
#pragma once
#include "geometry.cuh"

namespace fiery {

constexpr int WT = 4;        // feature-map columns per tile (16 B: the minimum TMA inner box)
constexpr int DPAD = 48;     // depth slots of a tile (D <= 48)

struct LiftParams {
    int n_frames, n_cameras;
    int frame0;              // first frame of this launch (frames are processed in chunks)
    int D, C, hh, ww;
    int n_wtiles;            // ceil(ww / WT)
    int head_channels;       // D + C, or C without the depth distribution
    int use_depth;
    int calib_mode;
    const float* calib_a;
    const float* calib_b;
    const float* fu;         // (w) frustum pixel column coordinate   fiery.py:120
    const float* fv;         // (h) frustum pixel row coordinate      fiery.py:122
    const float* fd;         // (D) frustum depth                     fiery.py:115
    const void* head_f16;    // forward, half-precision head tensor (fetched with cp.async; fp32 heads come through the tensor maps)
    float* accum;            // forward: (B', X*Y, C) channel-last accumulation target
    unsigned char* touched;  // forward without a plan, NCHW output: (B', X*Y) byte map of pillars that receive a point
    const unsigned char* plan_tiles;    // geometry plan (lift_plan.cuh): tile records of this launch's first frame onwards, or NULL
    const float* grad_bev;   // backward: (B', X*Y, C) or (B', C, X*Y)
    float* grad_head;        // backward output
    int bev_layout;
    long long pillars;       // X*Y
    GridParams grid;
};

// Tensor maps of a head tensor (or of its gradient) in the tile layouts: depth is 4-D (w, d, h, image) with box (4, 48, h, 1);
// ctx is 5-D (w, cl, k, h, image) with box (4, C / channels_per_lane, channels_per_lane, h, 1), channel = channels_per_lane*cl + k.
// The dimension order of the maps is the shared-memory order; the strides do the permutation.  Defined in c_api.cu.
struct HeadMapsCols {
    CUtensorMap depth;
    CUtensorMap ctx;
};
int encode_head_maps_cols(HeadMapsCols* maps, const void* head, const LiftParams& P, int channels_per_lane);

// FMA on a pair of adjacent values held in one 64-bit register pair: acc.lo += a.lo * b.lo, acc.hi += a.hi * b.hi (two FFMA)
__device__ __forceinline__ void ffma2(unsigned long long& acc, unsigned long long a, unsigned long long b) {
    asm("{\n\t.reg .f32 a0, a1, b0, b1, c0, c1;\n\t"
        "mov.b64 {a0, a1}, %1;\n\tmov.b64 {b0, b1}, %2;\n\tmov.b64 {c0, c1}, %0;\n\t"
        "fma.rn.f32 c0, a0, b0, c0;\n\tfma.rn.f32 c1, a1, b1, c1;\n\t"
        "mov.b64 %0, {c0, c1};\n\t}" : "+l"(acc) : "l"(a), "l"(b));
}

// softmax over depth (encoder.py:99) in place on prob[row][d][col] of a block of NT threads; lane = (d mod 8, col): conflict free,
// reductions by shuffle
template <int NT>
__device__ __forceinline__ void softmax_depth(const LiftParams& P, float* s_prob, int hh) {
    constexpr float L2E = 1.4426950408889634f;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c8 = lane >> 2, col = lane & 3;
    for (int row = warp; row < hh; row += NT / 32) {
        float* base = s_prob + (row * DPAD + c8) * WT + col;
        float x[DPAD / 8];
        if (P.use_depth) {
            float m = -INFINITY;
#pragma unroll
            for (int k = 0; k < DPAD / 8; ++k) {
                x[k] = (c8 + 8 * k < P.D) ? base[k * 8 * WT] : -INFINITY;
                m = fmaxf(m, x[k]);
            }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
            const float m2 = m * L2E;
            float sum = 0.f;
#pragma unroll
            for (int k = 0; k < DPAD / 8; ++k) {
                x[k] = exp2f(fmaf(x[k], L2E, -m2));         // exp(x - max); padding (-inf) gives 0
                sum += x[k];
            }
            sum += __shfl_xor_sync(0xffffffffu, sum, 4);
            sum += __shfl_xor_sync(0xffffffffu, sum, 8);
            sum += __shfl_xor_sync(0xffffffffu, sum, 16);
            const float inv = __fdiv_rn(1.0f, sum);
#pragma unroll
            for (int k = 0; k < DPAD / 8; ++k) base[k * 8 * WT] = x[k] * inv;
        } else {
#pragma unroll
            for (int k = 0; k < DPAD / 8; ++k) base[k * 8 * WT] = (c8 + 8 * k < P.D) ? 1.0f : 0.f;   // encoder.py:102
        }
    }
}

}  // namespace fiery
