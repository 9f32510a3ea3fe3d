// Frustum -> ego -> voxel arithmetic shared by every kernel (geometry plan, forward tile kernel, index dump).
//
// The reference computes, per frustum point (u, v, d) of camera i (fiery/models/fiery.py:199-205, 236-247):
//     q   = (u*d, v*d, d)
//     p   = (R @ inverse(K)) @ q + t                       batched 3x3 @ 3x1 on the CPU/GPU BLAS
//     s   = (p - (bev_start - bev_res/2)) / bev_res        fp32
//     idx = s.long()                                       truncation toward zero
//     keep = 0 <= idx < bev_dimension on all three axes
// Bit-exact integer parity needs the exact fp32 operation order.  oracle/gen_golden.py establishes that torch-CPU's
// result equals individually rounded mul/add in k = 0,1,2 order with no FMA contraction; all arithmetic here is
// therefore written with __fmul_rn/__fadd_rn/__fsub_rn/__fdiv_rn, which nvcc never fuses.
#pragma once
#include "common.cuh"

namespace fiery {

struct CameraTransform {
    float m[9];  // combined = R @ K^-1, row-major
    float t[3];  // translation
};

// combined = R @ inverse(K) (fiery.py:203).  inverse(K) follows LAPACK's solve-with-identity route that
// torch.linalg.inv takes on CPU: getrf with partial pivoting (column scaled by the reciprocal pivot, sgetf2), then
// getrs: forward/back substitution per identity column with true division by the diagonal (strsm).  For pinhole intrinsics (upper-triangular K) this reproduces torch-CPU
// bit-for-bit (tests/test_oracle_golden.py); for a general 3x3 it agrees to a few ulp.
__device__ inline void compose_camera(const float* __restrict__ K, const float* __restrict__ E, CameraTransform& out) {
    float a[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) a[i][j] = K[i * 3 + j];
    float b[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};

#pragma unroll
    for (int j = 0; j < 3; ++j) {
        int p = j;
        float best = fabsf(a[j][j]);
#pragma unroll
        for (int i = j + 1; i < 3; ++i) {
            const float v = fabsf(a[i][j]);
            if (v > best) { best = v; p = i; }          // first maximum, like isamax
        }
        // row swap with compile-time row numbers after unrolling, so a[][] and b[][] stay in registers
#pragma unroll
        for (int i = j + 1; i < 3; ++i) {
            if (p == i) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const float x = a[j][k]; a[j][k] = a[i][k]; a[i][k] = x;
                    const float y = b[j][k]; b[j][k] = b[i][k]; b[i][k] = y;
                }
            }
        }
        const float rcp = __fdiv_rn(1.0f, a[j][j]);      // sgetf2 scales the column by the reciprocal pivot
#pragma unroll
        for (int i = j + 1; i < 3; ++i) a[i][j] = __fmul_rn(a[i][j], rcp);
#pragma unroll
        for (int i = j + 1; i < 3; ++i)
#pragma unroll
            for (int k = j + 1; k < 3; ++k) a[i][k] = __fsub_rn(a[i][k], __fmul_rn(a[i][j], a[j][k]));
    }
    // b currently holds P (row-permuted identity).  Solve L y = P, then U x = y, column by column.
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int i = k + 1; i < 3; ++i) b[i][c] = __fsub_rn(b[i][c], __fmul_rn(a[i][k], b[k][c]));
#pragma unroll
        for (int k = 2; k >= 0; --k) {
            b[k][c] = __fdiv_rn(b[k][c], a[k][k]);
#pragma unroll
            for (int i = 0; i < k; ++i) b[i][c] = __fsub_rn(b[i][c], __fmul_rn(a[i][k], b[k][c]));
        }
    }
    // combined = R @ Kinv, accumulate k = 0,1,2, no FMA
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float r0 = E[i * 4 + 0], r1 = E[i * 4 + 1], r2 = E[i * 4 + 2];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float acc = __fmul_rn(r0, b[0][j]);
            acc = __fadd_rn(acc, __fmul_rn(r1, b[1][j]));
            acc = __fadd_rn(acc, __fmul_rn(r2, b[2][j]));
            out.m[i * 3 + j] = acc;
        }
        out.t[i] = E[i * 4 + 3];
    }
}

// Loads the transform of camera `cam` (flat index frame*n + camera) in either calibration mode.
__device__ inline void load_camera(int calib_mode, const float* __restrict__ calib_a, const float* __restrict__ calib_b,
                                   int cam, CameraTransform& out) {
    if (calib_mode == FIERY_CALIB_COMPOSED) {
#pragma unroll
        for (int i = 0; i < 9; ++i) out.m[i] = calib_a[cam * 9 + i];
#pragma unroll
        for (int i = 0; i < 3; ++i) out.t[i] = calib_b[cam * 3 + i];
    } else {
        compose_camera(calib_a + cam * 9, calib_b + cam * 16, out);
    }
}

// BEV grid constants in the form the kernels consume.
struct GridParams {
    float off[3];       // bev_start - bev_res/2 (fp32)
    float res[3];
    float inv_res[2];   // exact reciprocal when res is a power of two (then s = a * inv_res is exact == a / res)
    int pow2[2];
    float z_lo, z_hi;   // closed interval of (z - off_z) that maps to 0 <= iz < Z
    int X, Y;
    float x_lim, y_lim; // smallest float >= X (>= Y): for every float s, trunc(s) < X  <=>  s < x_lim
};

__host__ inline bool is_pow2_float(float r) {
    int e;
    return r > 0.f && frexpf(r, &e) == 0.5f;
}

// float(n) rounds to nearest, so above 2^24 it can fall below n (2^24 + 1 -> 2^24), and s < float(n) would drop s = n - 1
__host__ inline float float_at_or_above(int n) {
    const float f = static_cast<float>(n);
    return static_cast<double>(f) < n ? nextafterf(f, INFINITY) : f;
}

__host__ inline GridParams make_grid_params(const fiery_lift_desc_t& d) {
    GridParams g;
    for (int a = 0; a < 3; ++a) { g.off[a] = d.bev_offset[a]; g.res[a] = d.bev_resolution[a]; }
    for (int a = 0; a < 2; ++a) { g.pow2[a] = is_pow2_float(g.res[a]) ? 1 : 0; g.inv_res[a] = 1.0f / g.res[a]; }
    g.z_lo = d.z_valid_lo; g.z_hi = d.z_valid_hi;
    g.X = d.bev_x; g.Y = d.bev_y;
    g.x_lim = float_at_or_above(d.bev_x); g.y_lim = float_at_or_above(d.bev_y);
    return g;
}

// Per-(camera, column, depth) partial products that do not depend on the image row.
struct ColumnTerms {
    float a[3];   // M[r][0] * (u*d)
    float c[3];   // M[r][2] * d
};

__device__ __forceinline__ ColumnTerms column_terms(const CameraTransform& T, float u, float d) {
    ColumnTerms ct;
    const float ud = __fmul_rn(u, d);                                   // fiery.py:202
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        ct.a[r] = __fmul_rn(T.m[r * 3 + 0], ud);
        ct.c[r] = __fmul_rn(T.m[r * 3 + 2], d);
    }
    return ct;
}

// Ego-frame position of the point: p_r = ((M[r][0]*(u*d) + M[r][1]*(v*d)) + M[r][2]*d) + t_r   (fiery.py:204-205)
__device__ __forceinline__ void ego_point(const CameraTransform& T, const ColumnTerms& ct, float v, float d, float p[3]) {
    const float vd = __fmul_rn(v, d);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        float acc = __fadd_rn(ct.a[r], __fmul_rn(T.m[r * 3 + 1], vd));
        acc = __fadd_rn(acc, ct.c[r]);
        p[r] = __fadd_rn(acc, T.t[r]);
    }
}

// Scaled coordinate s = (p - off) / res on axis `axis` in {0,1} (fiery.py:236).
__device__ __forceinline__ float scaled_xy(const GridParams& g, int axis, float p) {
    const float a = __fsub_rn(p, g.off[axis]);
    return g.pow2[axis] ? __fmul_rn(a, g.inv_res[axis]) : __fdiv_rn(a, g.res[axis]);
}

// Pillar (= rank, fiery.py:252-256 with Z == 1) of an ego-frame point, or -1 if it is masked out
// (fiery.py:240-247).  trunc(s) >= 0  <=>  s > -1 ;  trunc(s) < X  <=>  s < x_lim ; NaN fails both.
__device__ __forceinline__ int pillar_of(const GridParams& g, const float p[3]) {
    const float sx = scaled_xy(g, 0, p[0]);
    const float sy = scaled_xy(g, 1, p[1]);
    const float az = __fsub_rn(p[2], g.off[2]);
    const bool ok = (sx > -1.0f) && (sx < g.x_lim) && (sy > -1.0f) && (sy < g.y_lim) &&
                    (az >= g.z_lo) && (az <= g.z_hi);
    const int ix = static_cast<int>(sx);   // cvt.rzi: truncation toward zero, like .long()
    const int iy = static_cast<int>(sy);
    return ok ? ix * g.Y + iy : -1;
}

// Same mask-and-rank as pillar_of, as one predicate chain (6 setp + selp): ordered comparisons are false for NaN.
__device__ __forceinline__ int select_pillar(float sx, float sy, float az, float Xf, float Yf, float z_lo, float z_hi, int rank) {
    int r;
    asm("{\n\t.reg .pred p;\n\t"
        "setp.gt.f32 p, %1, 0fBF800000;\n\t"
        "setp.lt.and.f32 p, %1, %4, p;\n\t"
        "setp.gt.and.f32 p, %2, 0fBF800000, p;\n\t"
        "setp.lt.and.f32 p, %2, %5, p;\n\t"
        "setp.ge.and.f32 p, %3, %6, p;\n\t"
        "setp.le.and.f32 p, %3, %7, p;\n\t"
        "selp.s32 %0, %8, -1, p;\n\t}"
        : "=r"(r)
        : "f"(sx), "f"(sy), "f"(az), "f"(Xf), "f"(Yf), "f"(z_lo), "f"(z_hi), "r"(rank));
    return r;
}

// Point -> pillar evaluation of the plan and the forward tile kernel: pillar_of after ego_point, with the grid constants hoisted
// out of the point loop into plain floats.  POW2: both horizontal resolutions are powers of two, so the scale is an exact multiply.
template <bool POW2>
struct PillarMap {
    float offx, offy, offz, kx, ky, Xf, Yf, z_lo, z_hi;
    int Y;

    __device__ __forceinline__ explicit PillarMap(const GridParams& g)
        : offx(g.off[0]), offy(g.off[1]), offz(g.off[2]), kx(POW2 ? g.inv_res[0] : g.res[0]), ky(POW2 ? g.inv_res[1] : g.res[1]),
          Xf(g.x_lim), Yf(g.y_lim), z_lo(g.z_lo), z_hi(g.z_hi), Y(g.Y) {}

    // pillar (rank) of the point at frustum row coordinate v and depth d of the column `ct`, or -1 if it is masked out
    __device__ __forceinline__ int operator()(const CameraTransform& T, const ColumnTerms& ct, float v, float d) const {
        float p[3];
        ego_point(T, ct, v, d, p);                                        // fiery.py:199-205
        const float ax = __fsub_rn(p[0], offx), ay = __fsub_rn(p[1], offy), az = __fsub_rn(p[2], offz);
        const float sx = POW2 ? __fmul_rn(ax, kx) : __fdiv_rn(ax, kx);    // fiery.py:236 (the scale is exact when res is 2^k)
        const float sy = POW2 ? __fmul_rn(ay, ky) : __fdiv_rn(ay, ky);
        const int rank = static_cast<int>(sx) * Y + static_cast<int>(sy); // truncation, fiery.py:237,252-256
        return select_pillar(sx, sy, az, Xf, Yf, z_lo, z_hi, rank);       // mask, fiery.py:240-247
    }
};

}  // namespace fiery
