// Sample positions of warp_features (fiery/utils/geometry.py:181-222): torch.nn.functional.affine_grid + grid_sample (bilinear or
// nearest, zero padding, align_corners=False) of one output pixel under a 2x3 affine map.  Shared by the standalone warp kernels
// (warp.cu) and the warp epilogue of the lift (lift_fwd.cu: finalize_warp_kernel), so both sample with the same arithmetic.
#pragma once
#include "common.cuh"

namespace fiery {

struct SamplePos {
    int off[4];      // element offsets of the 4 neighbours inside one channel plane (0 for out-of-range ones)
    float w[4];      // bilinear weights
    bool ok[4];      // neighbour inside the map (zero padding otherwise: never loaded)
};

// affine_grid (align_corners=False): normalised pixel centres x_i = (2i+1)/W - 1; grid = theta @ (x, y, 1)
// grid_sample unnormalise (align_corners=False): ix = ((gx + 1) * W - 1) / 2
__device__ __forceinline__ float norm_centre(int i, int n) { return (2.0f * i + 1.0f) / n - 1.0f; }
__device__ __forceinline__ void sample_coords_norm(const float* __restrict__ th, float xs, float ys, int W, int H, float& ix, float& iy) {
    const float gx = fmaf(th[0], xs, fmaf(th[1], ys, th[2]));
    const float gy = fmaf(th[3], xs, fmaf(th[4], ys, th[5]));
    ix = ((gx + 1.0f) * W - 1.0f) * 0.5f;
    iy = ((gy + 1.0f) * H - 1.0f) * 0.5f;
}
__device__ __forceinline__ void sample_coords(const float* __restrict__ th, int i, int j, int W, int H, float& ix, float& iy) {
    sample_coords_norm(th, norm_centre(i, W), norm_centre(j, H), W, H, ix, iy);
}

// The adjoint as a gather (warp_backward_gather_kernel): the output pixels that sample a given source
// pixel lie in a small window around the inverse image of that pixel.  InverseMap: inverse of the linear part of (i, j) -> (ix, iy)
// in pixel units, and whether that window is small enough to enumerate -- every map warp_features builds is a rotation
// (determinant 1); for anything else (strong scaling, singular or non-finite maps) the scan covers the whole image: slow, but any
// theta gives the exact adjoint.
struct InverseMap {
    float ia, ib, ic, id;    // (i, j) = inv * ((ix, iy) - (ix0, iy0))
    float ix0, iy0;
    bool windowed;
};
__device__ __forceinline__ InverseMap inverse_map(const float* __restrict__ th, int W, int H) {
    InverseMap m;
    const float a = th[0], b = th[1] * W / H, c = th[3] * H / W, d = th[4];
    sample_coords(th, 0, 0, W, H, m.ix0, m.iy0);
    const float det = a * d - b * c;
    m.ia = d / det; m.ib = -b / det; m.ic = -c / det; m.id = a / det;
    const float ei = fabsf(m.ia) + fabsf(m.ib), ej = fabsf(m.ic) + fabsf(m.id);
    m.windowed = fabsf(det) >= 0.25f && ei <= 4.f && ej <= 4.f && fabsf(m.ix0) < 1e6f && fabsf(m.iy0) < 1e6f;   // false for NaN / inf too
    return m;
}

// Resumable scan over the candidate output pixels of one source pixel: adjoint_scan_next() returns the next (at most M) candidates
// whose sample used the pixel -- element offset in the output plane and the weight the forward gave the pixel, computed with the
// forward's own arithmetic -- so that the caller can issue their loads together.
struct AdjointScan {
    int i, j, i_lo, i_hi, j_hi;      // next candidate; exhausted when j > j_hi
    int j_step;                      // several threads can share one pixel's window: thread `part` of `parts` takes every parts-th row
    float sx, sy;
};
__device__ __forceinline__ AdjointScan adjoint_scan_begin(const InverseMap& m, int pix, int W, int H, int nearest, int part = 0,
                                                          int parts = 1) {
    AdjointScan s;
    s.j_step = parts;
    s.sx = static_cast<float>(pix % W);
    s.sy = static_cast<float>(pix / W);
    int j_lo = 0;
    s.i_lo = 0; s.i_hi = W - 1; s.j_hi = H - 1;
    if (m.windowed) {
        const float dx = s.sx - m.ix0, dy = s.sy - m.iy0;
        const float ci = m.ia * dx + m.ib * dy, cj = m.ic * dx + m.id * dy;
        const float r = nearest ? 0.5f : 1.0f;
        const float slack = 0.05f + 1e-4f * (fabsf(ci) + fabsf(cj));            // rounding of the forward's coordinates and of this inverse
        const float ei = r * (fabsf(m.ia) + fabsf(m.ib)) + slack, ej = r * (fabsf(m.ic) + fabsf(m.id)) + slack;
        s.i_lo = static_cast<int>(fmaxf(ceilf(ci - ei), 0.f));
        s.i_hi = static_cast<int>(fminf(floorf(ci + ei), W - 1.f));
        j_lo = static_cast<int>(fmaxf(ceilf(cj - ej), 0.f));
        s.j_hi = static_cast<int>(fminf(floorf(cj + ej), H - 1.f));
    }
    s.i = s.i_lo;
    s.j = s.i_lo <= s.i_hi ? j_lo + part : s.j_hi + 1;
    return s;
}
template <int M>
__device__ __forceinline__ int adjoint_scan_next(AdjointScan& s, const float* __restrict__ th, int W, int H, int nearest,
                                                 int (&off)[M], float (&wgt)[M]) {
    int n = 0;
#pragma unroll
    for (int k = 0; k < M; ++k) { off[k] = 0; wgt[k] = 0.f; }
    while (s.j <= s.j_hi && n < M) {
        float ix, iy;
        sample_coords_norm(th, norm_centre(s.i, W), norm_centre(s.j, H), W, H, ix, iy);
        float w = 0.f;
        if (nearest) {
            if (nearbyintf(ix) == s.sx && nearbyintf(iy) == s.sy) w = 1.f;
        } else {
            const float x0f = floorf(ix), y0f = floorf(iy);
            const float kx = s.sx - x0f, ky = s.sy - y0f;                       // which of the candidate's four neighbours this pixel is
            if ((kx == 0.f || kx == 1.f) && (ky == 0.f || ky == 1.f)) {
                const float fx = ix - x0f, fy = iy - y0f;
                w = (kx == 0.f ? 1.f - fx : fx) * (ky == 0.f ? 1.f - fy : fy);
            }
        }
        if (w != 0.f) {                                                          // also false for NaN coordinates
            const int o = s.j * W + s.i;
#pragma unroll
            for (int k = 0; k < M; ++k)
                if (k == n) { off[k] = o; wgt[k] = w; }
            ++n;
        }
        if (++s.i > s.i_hi) { s.i = s.i_lo; s.j += s.j_step; }
    }
    return n;
}

__device__ __forceinline__ SamplePos make_sample(const float* __restrict__ theta, const unsigned char* __restrict__ copy_mask,
                                                 int map, int pix, int W, int H, int nearest) {
    SamplePos s;
#pragma unroll
    for (int k = 0; k < 4; ++k) { s.off[k] = 0; s.w[k] = 0.f; s.ok[k] = false; }
    if (copy_mask && copy_mask[map]) {          // the present frame of a sequence passes through unchanged (geometry.py:243)
        s.off[0] = pix; s.w[0] = 1.f; s.ok[0] = true;
        return s;
    }
    float ix, iy;
    sample_coords(theta + map * 6, pix % W, pix / W, W, H, ix, iy);
    if (nearest) {
        const float rx = nearbyintf(ix), ry = nearbyintf(iy);          // round half to even, like grid_sample 'nearest'
        const bool ok = rx >= 0.f && rx < W && ry >= 0.f && ry < H;
        s.off[0] = ok ? static_cast<int>(ry) * W + static_cast<int>(rx) : 0;
        s.w[0] = 1.f; s.ok[0] = ok;
        return s;
    }
    const float x0f = floorf(ix), y0f = floorf(iy);
    const float fx = ix - x0f, fy = iy - y0f;
    const float wx[2] = {1.f - fx, fx}, wy[2] = {1.f - fy, fy};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float xf = x0f + (k & 1), yf = y0f + (k >> 1);
        const bool ok = xf >= 0.f && xf < W && yf >= 0.f && yf < H;        // also false for NaN / huge coordinates
        s.off[k] = ok ? static_cast<int>(yf) * W + static_cast<int>(xf) : 0;
        s.w[k] = wx[k & 1] * wy[k >> 1];
        s.ok[k] = ok;
    }
    return s;
}

}  // namespace fiery
