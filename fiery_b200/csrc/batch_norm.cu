// BatchNorm3d over a (b, C, s, X, Y) fp32 tensor with an optional fused ReLU and residual add, forward and backward, train and eval
// (include/fiery_b200.h, fiery_batch_norm_*).  Every pass is bandwidth-bound; none uses atomics, and every summation order depends on
// the shape only, so results are bit-reproducible and do not depend on where a plane lies in memory.
//
// Each (b, c, t) pixel plane is cut into pieces of BN_PIECE pixels (the last one shorter), so the partial pass has enough CTAs to
// fill the GPU even when the planes are few and large.  One CTA takes one piece: thread i holds chunks i, i + 256, i + 512, i + 768
// (4 pixels each) in registers.
//   forward partial:  the piece's mean (block sum / count) and M2 = sum (x - piece mean)^2, both from the registers (two passes
//                     over values read once);
//   backward partial: sum g' and sum g' (x - mu), g' = dy masked by the forward's ReLU when it is fused.
// A thread adds its chunks in ascending order, each chunk as (p0 + p1) + (p2 + p3); the warps reduce by an xor butterfly and the 8
// warp sums are added in ascending order.  The per-channel finalize (one thread per channel) merges the channel's pieces in
// ascending (b, t, piece) order in fp64: Chan's formula for (count, mean, M2), plain sums for the backward.  The apply passes use
// the same pieces.
#include "bn_coef.cuh"
#include "plane_chunks.cuh"

namespace fiery {

constexpr int BN_THREADS = 256;
constexpr int BN_CHUNKS = 4;                                   // chunks per thread: the whole piece sits in registers
constexpr int BN_PIECE = BN_THREADS * BN_CHUNKS * 4;           // 4096 pixels
constexpr long long BN_MAX_GRID = 1ll << 30;
constexpr int BN_MIN_CTAS = 4;                                 // resident CTAs per SM the register budget allows

struct BnShape {
    long long pieces;                                          // batch * channels * frames * per_plane
    long long per_channel;                                     // pieces of one channel: batch * frames * per_plane
    long long sb, sc, st;                                      // x's strides, elements
    int channels, frames, pixels, per_plane;
};

struct BnPiece {
    long long x_off, out_off, part;                            // x offset, offset in the contiguous tensors, partial index
    int c, n;                                                  // channel, pixels in the piece
};

__device__ __forceinline__ BnPiece bn_piece(const BnShape& s, long long g) {
    const long long plane = g / s.per_plane;
    const int j = static_cast<int>(g - plane * s.per_plane);
    const long long t = plane % s.frames, c = (plane / s.frames) % s.channels, b = plane / (static_cast<long long>(s.frames) * s.channels);
    BnPiece p;
    p.c = static_cast<int>(c);
    p.n = min(BN_PIECE, s.pixels - j * BN_PIECE);
    p.x_off = b * s.sb + c * s.sc + t * s.st + static_cast<long long>(j) * BN_PIECE;
    p.out_off = plane * s.pixels + static_cast<long long>(j) * BN_PIECE;
    p.part = c * s.per_channel + (b * s.frames + t) * s.per_plane + j;
    return p;
}

// scale = gamma / sqrt(var + eps), shift = beta - mean * scale, in fp64 from the fp32 statistics and rounded once.  The forward's
// finalize and both backward passes call it, so the backward's ReLU mask sees exactly the forward's scale and shift.
__device__ __forceinline__ void bn_scale_shift(const float* __restrict__ w, const float* __restrict__ bias, float mean, float var,
                                               double eps, int c, float& scale, float& shift) {
    const double s = (w ? static_cast<double>(w[c]) : 1.0) / sqrt(static_cast<double>(var) + eps);
    scale = static_cast<float>(s);
    shift = static_cast<float>((bias ? static_cast<double>(bias[c]) : 0.0) - static_cast<double>(mean) * s);
}

// sum over the CTA in the order above; every thread gets the total.  sh: BN_THREADS / 32 floats.
__device__ __forceinline__ float bn_block_sum(float v, float* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float total = sh[0];
#pragma unroll
    for (int w = 1; w < BN_THREADS / 32; ++w) total += sh[w];
    __syncthreads();                                           // sh is rewritten by the next call
    return total;
}

__device__ __forceinline__ float bn_chunk_sum(float4 v) { return (v.x + v.y) + (v.z + v.w); }

__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) bn_stats_kernel(const BnShape s, const float* __restrict__ x, float2* __restrict__ part) {
    __shared__ float sh[BN_THREADS / 32];
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const float* xp = x + p.x_off;
        const bool vec = aligned16_ptr(xp);
        const int n_chunks = (p.n + 3) / 4;
        float4 v[BN_CHUNKS];
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            v[u] = q < n_chunks ? load_chunk4(xp, q, p.n, vec) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float a = 0.f;
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) a += bn_chunk_sum(v[u]);
        const float mean = bn_block_sum(a, sh) / static_cast<float>(p.n);
        float m2 = 0.f;
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int i = 4 * (threadIdx.x + u * BN_THREADS);
            const float d0 = i < p.n ? v[u].x - mean : 0.f, d1 = i + 1 < p.n ? v[u].y - mean : 0.f;
            const float d2 = i + 2 < p.n ? v[u].z - mean : 0.f, d3 = i + 3 < p.n ? v[u].w - mean : 0.f;
            m2 += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        }
        m2 = bn_block_sum(m2, sh);
        if (threadIdx.x == 0) part[p.part] = make_float2(mean, m2);
    }
}

// Chan's formula in fp64: (n, m, m2) merged with a part of nb values, mean mb and M2 m2b (fp32 for a piece, fp64 for a rank)
template <typename T>
__device__ __forceinline__ void bn_chan_step(double& n, double& m, double& m2, double nb, T mb, T m2b) {
    const double delta = static_cast<double>(mb) - m, nn = n + nb;
    m += delta * (nb / nn);
    m2 += static_cast<double>(m2b) + delta * delta * (n * nb / nn);
    n = nn;
}

// Chan's merge of channel c's pieces' (count, mean, M2) in ascending (b, t, piece) order, in fp64
__device__ __forceinline__ void bn_merge_pieces(const BnShape& s, const float2* __restrict__ part, int c, double& n, double& m, double& m2) {
    n = m = m2 = 0.0;
    const float2* pc = part + c * s.per_channel;
    for (long long k = 0; k < s.per_channel; ++k) {
        const int j = static_cast<int>(k % s.per_plane);
        const double nb = static_cast<double>(min(BN_PIECE, s.pixels - j * BN_PIECE));
        const float2 pk = pc[k];
        bn_chan_step(n, m, m2, nb, pk.x, pk.y);
    }
}

// The forward finalizes' output for channel c: the statistics, the group's count n (by channel 0, if count_out) and the coefficients
__device__ __forceinline__ void bn_forward_out(const float* w, const float* bias, float mean, float var, double n, double eps, int c,
                                               float* mean_out, float* var_out, double* count_out, BnCoef* coef) {
    mean_out[c] = mean;
    var_out[c] = var;
    if (c == 0 && count_out) *count_out = n;
    BnCoef k;
    bn_scale_shift(w, bias, mean, var, eps, c, k.scale, k.shift);
    k.mean = mean;
    k.k1 = k.k0 = 0.f;
    coef[c] = k;
}

// One thread per channel.  training: Chan's merge of the pieces' (count, mean, M2) in fp64 -> mean and biased variance; eval: the
// running statistics.  Writes the fp32 statistics and the forward's coefficients.
__global__ void bn_finalize_forward_kernel(const BnShape s, const float2* __restrict__ part, const float* __restrict__ w,
                                           const float* __restrict__ bias, const float* __restrict__ running_mean,
                                           const float* __restrict__ running_var, int training, double eps, float* __restrict__ mean_out,
                                           float* __restrict__ var_out, BnCoef* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= s.channels) return;
    float mean, var;
    if (training) {
        double n, m, m2;
        bn_merge_pieces(s, part, c, n, m, m2);
        mean = static_cast<float>(m);
        var = static_cast<float>(m2 / n);
    } else {
        mean = running_mean[c];
        var = running_var[c];
    }
    bn_forward_out(w, bias, mean, var, 0.0, eps, c, mean_out, var_out, nullptr, coef);
}

template <bool RELU, bool RESIDUAL>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) bn_apply_kernel(const BnShape s, const float* __restrict__ x, const BnCoef* __restrict__ coef,
                                                              const float* __restrict__ residual, float* __restrict__ y) {
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const float* xp = x + p.x_off;
        float* yp = y + p.out_off;
        const float* rp = RESIDUAL ? residual + p.out_off : nullptr;
        const bool vx = aligned16_ptr(xp), vy = aligned16_ptr(yp), vr = RESIDUAL && aligned16_ptr(rp);
        const float scale = coef[p.c].scale, shift = coef[p.c].shift;
        const int n_chunks = (p.n + 3) / 4;
        float4 v[BN_CHUNKS], r[BN_CHUNKS];
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            if (q < n_chunks) {
                v[u] = load_chunk4(xp, q, p.n, vx);
                if (RESIDUAL) r[u] = load_chunk4(rp, q, p.n, vr);
            }
        }
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            if (q >= n_chunks) continue;
            float o[4] = {fmaf(scale, v[u].x, shift), fmaf(scale, v[u].y, shift), fmaf(scale, v[u].z, shift), fmaf(scale, v[u].w, shift)};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (RELU) o[e] = o[e] < 0.f ? 0.f : o[e];      // a NaN passes, as torch's ReLU lets it
            }
            if (RESIDUAL) {
                o[0] += r[u].x;
                o[1] += r[u].y;
                o[2] += r[u].z;
                o[3] += r[u].w;
            }
            store_chunk4(yp, q, p.n, vy, make_float4(o[0], o[1], o[2], o[3]));
        }
    }
}

// g' = dy where the forward's fmaf(scale, x, shift) was not <= 0 (ReLU fused; a NaN passes, as torch's threshold_backward lets it),
// dy otherwise
template <bool RELU>
__device__ __forceinline__ float bn_masked(float dy, float x, float scale, float shift) {
    return RELU ? (fmaf(scale, x, shift) <= 0.f ? 0.f : dy) : dy;
}

template <bool RELU>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) bn_grad_sums_kernel(const BnShape s, const float* __restrict__ x, const float* __restrict__ dy,
                                                                  const float* __restrict__ w, const float* __restrict__ bias,
                                                                  const float* __restrict__ mean, const float* __restrict__ var,
                                                                  double eps, float2* __restrict__ part) {
    __shared__ float sh[BN_THREADS / 32];
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const float* xp = x + p.x_off;
        const float* gp = dy + p.out_off;
        const bool vx = aligned16_ptr(xp), vg = aligned16_ptr(gp);
        const float mu = mean[p.c];
        float scale = 0.f, shift = 0.f;
        if (RELU) bn_scale_shift(w, bias, mu, var[p.c], eps, p.c, scale, shift);
        const int n_chunks = (p.n + 3) / 4;
        float4 v[BN_CHUNKS], d[BN_CHUNKS];
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            const bool in = q < n_chunks;                       // pixels past the piece read as x = 0, dy = 0: they add zero
            v[u] = in ? load_chunk4(xp, q, p.n, vx) : make_float4(0.f, 0.f, 0.f, 0.f);
            d[u] = in ? load_chunk4(gp, q, p.n, vg) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const float4 gm = make_float4(bn_masked<RELU>(d[u].x, v[u].x, scale, shift), bn_masked<RELU>(d[u].y, v[u].y, scale, shift),
                                          bn_masked<RELU>(d[u].z, v[u].z, scale, shift), bn_masked<RELU>(d[u].w, v[u].w, scale, shift));
            s1 += bn_chunk_sum(gm);
            s2 += bn_chunk_sum(make_float4(gm.x * (v[u].x - mu), gm.y * (v[u].y - mu), gm.z * (v[u].z - mu), gm.w * (v[u].w - mu)));
        }
        s1 = bn_block_sum(s1, sh);
        s2 = bn_block_sum(s2, sh);
        if (threadIdx.x == 0) part[p.part] = make_float2(s1, s2);
    }
}

// The fp64 sums (S1, S2) of channel c's pieces' (sum g', sum g' (x - mu)) in ascending (b, t, piece) order, and from them the weight
// and bias gradients S2 / sqrt(var + eps) and S1, each when asked for
__device__ __forceinline__ void bn_sum_pieces(const BnShape& s, const float2* part, const float* var, double eps, int c, float* grad_w,
                                              float* grad_b, double& s1, double& s2) {
    s1 = s2 = 0.0;
    const float2* pc = part + c * s.per_channel;
    for (long long k = 0; k < s.per_channel; ++k) {
        const float2 pk = pc[k];
        s1 += static_cast<double>(pk.x);
        s2 += static_cast<double>(pk.y);
    }
    const double ve = static_cast<double>(var[c]) + eps;
    if (grad_w) grad_w[c] = static_cast<float>(s2 / sqrt(ve));
    if (grad_b) grad_b[c] = static_cast<float>(s1);
}

// The training backward's coefficients of channel c from its n values' sums: the forward's scale and shift (so its ReLU mask), k1, k0
__device__ __forceinline__ BnCoef bn_backward_coef(const float* w, const float* bias, float mean, float var, double eps, int c, double n,
                                                   double s1, double s2) {
    BnCoef k;
    k.mean = mean;
    bn_scale_shift(w, bias, mean, var, eps, c, k.scale, k.shift);
    const double ve = static_cast<double>(var) + eps;
    k.k1 = static_cast<float>(-static_cast<double>(k.scale) * s2 / (n * ve));
    k.k0 = static_cast<float>(-static_cast<double>(k.scale) * s1 / n);
    return k;
}

// One thread per channel: the pieces' sums (when reduced), the weight and bias gradients, and the coefficients of dx.
__global__ void bn_finalize_backward_kernel(const BnShape s, const float2* __restrict__ part, int reduced, const float* __restrict__ w,
                                            const float* __restrict__ bias, const float* __restrict__ mean, const float* __restrict__ var,
                                            int training, double eps, float* __restrict__ grad_w, float* __restrict__ grad_b,
                                            BnCoef* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= s.channels) return;
    double s1 = 0.0, s2 = 0.0;                                 // the gradients asked for imply reduced
    if (reduced) bn_sum_pieces(s, part, var, eps, c, grad_w, grad_b, s1, s2);
    BnCoef k = bn_backward_coef(w, bias, mean[c], var[c], eps, c, static_cast<double>(s.per_channel / s.per_plane) * s.pixels, s1, s2);
    if (!training) k.k1 = k.k0 = 0.f;
    coef[c] = k;
}

template <bool RELU, bool TRAINING>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) bn_grad_apply_kernel(const BnShape s, const float* __restrict__ x, const float* __restrict__ dy,
                                                                   const BnCoef* __restrict__ coef, float* __restrict__ dx) {
    constexpr bool READ_X = RELU || TRAINING;
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const float* xp = x + p.x_off;
        const float* gp = dy + p.out_off;
        float* op = dx + p.out_off;
        const bool vx = aligned16_ptr(xp), vg = aligned16_ptr(gp), vo = aligned16_ptr(op);
        const BnCoef k = coef[p.c];
        const int n_chunks = (p.n + 3) / 4;
        float4 v[BN_CHUNKS], d[BN_CHUNKS];
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            if (q < n_chunks) {
                d[u] = load_chunk4(gp, q, p.n, vg);
                if (READ_X) v[u] = load_chunk4(xp, q, p.n, vx);
            }
        }
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            if (q >= n_chunks) continue;
            const float xs[4] = {READ_X ? v[u].x : 0.f, READ_X ? v[u].y : 0.f, READ_X ? v[u].z : 0.f, READ_X ? v[u].w : 0.f};
            const float ds[4] = {d[u].x, d[u].y, d[u].z, d[u].w};
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float gm = bn_masked<RELU>(ds[e], xs[e], k.scale, k.shift);
                o[e] = TRAINING ? fmaf(k.scale, gm, fmaf(k.k1, xs[e] - k.mean, k.k0)) : k.scale * gm;
            }
            store_chunk4(op, q, p.n, vo, make_float4(o[0], o[1], o[2], o[3]));
        }
    }
}

static BnShape bn_shape(const fiery_batch_norm_desc_t* d) {
    BnShape s;
    s.channels = d->channels;
    s.frames = d->frames;
    s.pixels = d->pixels;
    s.per_plane = (d->pixels + BN_PIECE - 1) / BN_PIECE;
    s.per_channel = static_cast<long long>(d->batch) * d->frames * s.per_plane;
    s.pieces = s.per_channel * d->channels;
    s.sb = d->stride_b;
    s.sc = d->stride_c;
    s.st = d->stride_t;
    return s;
}

static size_t bn_coef_bytes(int channels) { return (static_cast<size_t>(channels) * sizeof(BnCoef) + 255) / 256 * 256; }

size_t batch_norm_workspace_bytes(const fiery_batch_norm_desc_t* d) {
    const BnShape s = bn_shape(d);
    return bn_coef_bytes(d->channels) + static_cast<size_t>(s.pieces) * sizeof(float2);
}

static unsigned bn_grid(const BnShape& s) { return static_cast<unsigned>(s.pieces < BN_MAX_GRID ? s.pieces : BN_MAX_GRID); }

// The workspace: the per-channel coefficients, then one partial per piece
struct BnWork { BnCoef* coef; float2* part; };
static BnWork bn_work(const fiery_batch_norm_desc_t* d, void* workspace) {
    return {static_cast<BnCoef*>(workspace), reinterpret_cast<float2*>(static_cast<char*>(workspace) + bn_coef_bytes(d->channels))};
}

// The forward's statistics and coefficients: the batch's (the stats pass and the merge) in training, the running ones in eval
static void bn_batch_coef(const fiery_batch_norm_desc_t* d, const BnShape& s, const float* x, const float* w, const float* bias,
                          const float* running_mean, const float* running_var, float* mean_out, float* var_out, BnCoef* coef, float2* part,
                          cudaStream_t stream) {
    if (d->training) bn_stats_kernel<<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, part);
    bn_finalize_forward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(s, part, w, bias, running_mean, running_var, d->training, d->eps,
                                                                              mean_out, var_out, coef);
}

// The passes over the pieces below launch nothing for a rank of a group with no values (no pieces).
static void bn_apply(const fiery_batch_norm_desc_t* d, const BnShape& s, const float* x, const BnCoef* coef, const float* residual, float* y,
                     cudaStream_t stream) {
    if (!s.pieces) return;
    if (d->relu && residual) bn_apply_kernel<true, true><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, coef, residual, y);
    else if (d->relu) bn_apply_kernel<true, false><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, coef, nullptr, y);
    else if (residual) bn_apply_kernel<false, true><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, coef, residual, y);
    else bn_apply_kernel<false, false><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, coef, nullptr, y);
}

static void bn_grad_sums(const fiery_batch_norm_desc_t* d, const BnShape& s, const float* x, const float* dy, const float* w, const float* bias,
                         const float* mean, const float* var, float2* part, cudaStream_t stream) {
    if (!s.pieces) return;
    if (d->relu) bn_grad_sums_kernel<true><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, dy, w, bias, mean, var, d->eps, part);
    else bn_grad_sums_kernel<false><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, dy, w, bias, mean, var, d->eps, part);
}

static void bn_grad_apply(const fiery_batch_norm_desc_t* d, const BnShape& s, const float* x, const float* dy, const BnCoef* coef, float* dx,
                          cudaStream_t stream) {
    if (!s.pieces) return;
    if (d->relu && d->training) bn_grad_apply_kernel<true, true><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, dy, coef, dx);
    else if (d->relu) bn_grad_apply_kernel<true, false><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, dy, coef, dx);
    else if (d->training) bn_grad_apply_kernel<false, true><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, dy, coef, dx);
    else bn_grad_apply_kernel<false, false><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, dy, coef, dx);
}

int launch_batch_norm_forward(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* running_mean,
                              const float* running_var, const float* residual, float* y, float* mean_out, float* var_out,
                              void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    const auto [coef, part] = bn_work(d, workspace);
    bn_batch_coef(d, s, x, w, bias, running_mean, running_var, mean_out, var_out, coef, part, stream);
    bn_apply(d, s, x, coef, residual, y, stream);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_batch_norm_coef(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* running_mean,
                           const float* running_var, float* mean_out, float* var_out, void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    const auto [coef, part] = bn_work(d, workspace);
    bn_batch_coef(d, s, x, w, bias, running_mean, running_var, mean_out, var_out, coef, part, stream);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_batch_norm_backward(const fiery_batch_norm_desc_t* d, const float* x, const float* dy, const float* w, const float* bias,
                               const float* mean, const float* var, float* dx, float* grad_w, float* grad_b, void* workspace,
                               cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    const auto [coef, part] = bn_work(d, workspace);
    // the sums are needed for the weight and bias gradients, and for dx in training
    const bool reduce = grad_w || grad_b || (dx && d->training);
    if (reduce) bn_grad_sums(d, s, x, dy, w, bias, mean, var, part, stream);
    bn_finalize_backward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(s, part, reduce, w, bias, mean, var, d->training, d->eps,
                                                                               grad_w, grad_b, coef);
    if (dx) bn_grad_apply(d, s, x, dy, coef, dx, stream);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// The spatial GRU's state update (spatial_gru.cu) on one step's s (batch, channels, 1, X, Y): the statistics and finalize above, then
//   h' = (1 - u) h + u max(fmaf(scale, s, shift), 0)
// written straight to the output frame; its backward from dh' = grad_out + carry gives
//   da = u dh' (then the BN + ReLU backward above on (s, da)), dG_u = dh' (a - h) u (1 - u), carry = (1 - u) dh'.
// u and carry lie like s; h and the output frame have contiguous planes X*Y apart and their own batch strides.
// ------------------------------------------------------------------------------------------------------------------------------
struct GruPieceAt {
    long long b, pix;                                          // batch element, first pixel of the piece
};
__device__ __forceinline__ GruPieceAt gru_piece_at(const BnShape& s, long long g) {
    const long long plane = g / s.per_plane;
    GruPieceAt r;
    r.b = plane / s.channels;
    r.pix = (g - plane * s.per_plane) * BN_PIECE;
    return r;
}

__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) gru_blend_kernel(const BnShape s, const float* __restrict__ x, const BnCoef* __restrict__ coef,
                                                               const float* __restrict__ u, const float* __restrict__ h, long long hsb,
                                                               float* __restrict__ out, long long osb) {
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const GruPieceAt at = gru_piece_at(s, g);
        const long long hw = static_cast<long long>(p.c) * s.pixels + at.pix;
        const float* xp = x + p.x_off;
        const float* up = u + p.x_off;
        const float* hp = h + at.b * hsb + hw;
        float* op = out + at.b * osb + hw;
        const bool vx = aligned16_ptr(xp), vu = aligned16_ptr(up), vh = aligned16_ptr(hp), vo = aligned16_ptr(op);
        const float scale = coef[p.c].scale, shift = coef[p.c].shift;
        const int n_chunks = (p.n + 3) / 4;
#pragma unroll
        for (int k = 0; k < BN_CHUNKS; ++k) {
            const int q = threadIdx.x + k * BN_THREADS;
            if (q >= n_chunks) continue;
            const float4 v = load_chunk4(xp, q, p.n, vx), uu = load_chunk4(up, q, p.n, vu), hh = load_chunk4(hp, q, p.n, vh);
            const float vs[4] = {v.x, v.y, v.z, v.w}, us[4] = {uu.x, uu.y, uu.z, uu.w}, hs[4] = {hh.x, hh.y, hh.z, hh.w};
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float a = fmaf(scale, vs[e], shift);
                a = a < 0.f ? 0.f : a;                         // a NaN passes, as torch's ReLU lets it
                o[e] = (1.f - us[e]) * hs[e] + us[e] * a;
            }
            store_chunk4(op, q, p.n, vo, make_float4(o[0], o[1], o[2], o[3]));
        }
    }
}

__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) gru_blend_grad_kernel(const BnShape s, const float* __restrict__ x, const float* __restrict__ w,
                                                                    const float* __restrict__ bias, const float* __restrict__ mean,
                                                                    const float* __restrict__ var, double eps, const float* __restrict__ u,
                                                                    const float* __restrict__ h, long long hsb, const float* __restrict__ go,
                                                                    long long gsb, float* __restrict__ carry, float* __restrict__ da,
                                                                    float* __restrict__ dgu, long long dsb) {
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const GruPieceAt at = gru_piece_at(s, g);
        const long long hw = static_cast<long long>(p.c) * s.pixels + at.pix;
        float scale, shift;
        bn_scale_shift(w, bias, mean[p.c], var[p.c], eps, p.c, scale, shift);
        const float* xp = x + p.x_off;
        const float* up = u + p.x_off;
        float* cp = carry + p.x_off;
        float* ap = da + p.x_off;
        const float* hp = h + at.b * hsb + hw;
        const float* gp = go + at.b * gsb + hw;
        float* dp = dgu + at.b * dsb + hw;
        const bool vx = aligned16_ptr(xp), vu = aligned16_ptr(up), vc = aligned16_ptr(cp), va = aligned16_ptr(ap);
        const bool vh = aligned16_ptr(hp), vg = aligned16_ptr(gp), vd = aligned16_ptr(dp);
        const int n_chunks = (p.n + 3) / 4;
#pragma unroll
        for (int k = 0; k < BN_CHUNKS; ++k) {
            const int q = threadIdx.x + k * BN_THREADS;
            if (q >= n_chunks) continue;
            const float4 v = load_chunk4(xp, q, p.n, vx), uu = load_chunk4(up, q, p.n, vu), hh = load_chunk4(hp, q, p.n, vh);
            const float4 gg = load_chunk4(gp, q, p.n, vg), cc = load_chunk4(cp, q, p.n, vc);
            const float vs[4] = {v.x, v.y, v.z, v.w}, us[4] = {uu.x, uu.y, uu.z, uu.w}, hs[4] = {hh.x, hh.y, hh.z, hh.w};
            const float gs[4] = {gg.x, gg.y, gg.z, gg.w}, cs[4] = {cc.x, cc.y, cc.z, cc.w};
            float oa[4], od[4], oc[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float a = fmaf(scale, vs[e], shift);
                a = a < 0.f ? 0.f : a;
                const float dh = gs[e] + cs[e];
                oa[e] = us[e] * dh;
                od[e] = dh * (a - hs[e]) * (us[e] * (1.f - us[e]));
                oc[e] = (1.f - us[e]) * dh;
            }
            store_chunk4(ap, q, p.n, va, make_float4(oa[0], oa[1], oa[2], oa[3]));
            store_chunk4(dp, q, p.n, vd, make_float4(od[0], od[1], od[2], od[3]));
            store_chunk4(cp, q, p.n, vc, make_float4(oc[0], oc[1], oc[2], oc[3]));
        }
    }
}

int launch_gru_blend_forward(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* running_mean,
                             const float* running_var, const float* u, const float* h, long long hsb, float* out, long long osb,
                             float* mean_out, float* var_out, void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    const auto [coef, part] = bn_work(d, workspace);
    bn_batch_coef(d, s, x, w, bias, running_mean, running_var, mean_out, var_out, coef, part, stream);
    gru_blend_kernel<<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, coef, u, h, hsb, out, osb);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_gru_blend_backward(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* mean,
                              const float* var, const float* u, const float* h, long long hsb, const float* go, long long gsb, float* carry,
                              float* da, float* dgu, long long dsb, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    gru_blend_grad_kernel<<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, w, bias, mean, var, d->eps, u, h, hsb, go, gsb, carry, da, dgu, dsb);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// The decoder's output heads' backward (output_head.cu): out = W1 relu(bn(y)) + b1 on y (maps, C, 1, X, Y) contiguous, with n <= 8
// outputs.  The 1x1's input gradient da[c, p] = sum_{j < n} W1[j, c] g[j, p] (fp32, fmaf in ascending j) is never stored: both passes below recompute it from the piece's n rows of g, which every channel's pieces read again
// (from L2: g is n / C of y's size).  Over the pieces above:
//   sums pass:  bn_grad_sums_kernel<RELU = true>'s (S1, S2) on (y, da), bit for bit; and each piece's 1x1 weight-gradient partials
//               sum g[j, p] a[c, p] (a = relu(fmaf(scale, y, shift))) and, in channel 0's pieces, its bias-gradient partials
//               sum g[j, p], each summed in the pieces' order (thread chunks ascending, a chunk as (p0 + p1) + (p2 + p3), the block sum);
//   finalize:   bn_finalize_backward_kernel; dW1 and db1 the fp64 sums of their partials in ascending (map, piece) order;
//   apply pass: bn_grad_apply_kernel<RELU = true, TRAINING>'s dx on (y, da), bit for bit.
// g is (maps, n, X*Y) contiguous; W1[j][c] is at w1[j * ld + c].
// ------------------------------------------------------------------------------------------------------------------------------
struct HeadGrad {
    const float* g;
    const float* w1;
    int n, ld;
};

// the piece's chunk q of da (g read at gp, the piece's first pixel in row 0 of its map's g)
__device__ __forceinline__ float4 head_da(const HeadGrad& h, const float* gp, long long pixels, int c, int q, int n_px, bool vec) {
    float4 da = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < h.n; ++j) {
        const float w = __ldg(h.w1 + static_cast<long long>(j) * h.ld + c);
        const float4 gj = load_chunk4(gp + j * pixels, q, n_px, vec);
        da = make_float4(fmaf(w, gj.x, da.x), fmaf(w, gj.y, da.y), fmaf(w, gj.z, da.z), fmaf(w, gj.w, da.w));
    }
    return da;
}

__device__ __forceinline__ float4 head_relu(float4 v, float scale, float shift) {
    const BnCoef k{scale, shift, 0.f, 0.f, 0.f};
    return make_float4(bn_relu_apply(k, v.x), bn_relu_apply(k, v.y), bn_relu_apply(k, v.z), bn_relu_apply(k, v.w));
}

__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) head_grad_sums_kernel(const BnShape s, const float* __restrict__ y, const HeadGrad h,
                                                                    const float* __restrict__ w, const float* __restrict__ bias,
                                                                    const float* __restrict__ mean, const float* __restrict__ var,
                                                                    double eps, float2* __restrict__ part, float* __restrict__ wpart,
                                                                    float* __restrict__ bpart) {
    __shared__ float sh[BN_THREADS / 32];
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const GruPieceAt at = gru_piece_at(s, g);
        const float* xp = y + p.x_off;
        const float* gp = h.g + at.b * h.n * s.pixels + at.pix;
        const bool vx = aligned16_ptr(xp), vg = aligned16_ptr(gp);
        const float mu = mean[p.c];
        float scale, shift;
        bn_scale_shift(w, bias, mu, var[p.c], eps, p.c, scale, shift);
        const int n_chunks = (p.n + 3) / 4;
        float4 v[BN_CHUNKS];
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            v[u] = q < n_chunks ? load_chunk4(xp, q, p.n, vx) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // the 1x1's partials, row j at a time: sum g a over the piece, and (channel 0) sum g
        const bool w_part = wpart != nullptr, b_part = bpart != nullptr && p.c == 0;
        for (int j = 0; j < h.n && (w_part || b_part); ++j) {
            float sw = 0.f, sb = 0.f;
#pragma unroll
            for (int u = 0; u < BN_CHUNKS; ++u) {
                const int q = threadIdx.x + u * BN_THREADS;
                if (q >= n_chunks) continue;
                const float4 gj = load_chunk4(gp + static_cast<long long>(j) * s.pixels, q, p.n, vg);
                const float4 a = head_relu(v[u], scale, shift);
                sw += bn_chunk_sum(make_float4(gj.x * a.x, gj.y * a.y, gj.z * a.z, gj.w * a.w));
                sb += bn_chunk_sum(gj);
            }
            if (w_part) {
                sw = bn_block_sum(sw, sh);
                if (threadIdx.x == 0) wpart[p.part * h.n + j] = sw;
            }
            if (b_part) {
                sb = bn_block_sum(sb, sh);
                if (threadIdx.x == 0) bpart[p.part * h.n + j] = sb;
            }
        }
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            const float4 d = q < n_chunks ? head_da(h, gp, s.pixels, p.c, q, p.n, vg) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 gm = make_float4(bn_masked<true>(d.x, v[u].x, scale, shift), bn_masked<true>(d.y, v[u].y, scale, shift),
                                          bn_masked<true>(d.z, v[u].z, scale, shift), bn_masked<true>(d.w, v[u].w, scale, shift));
            s1 += bn_chunk_sum(gm);
            s2 += bn_chunk_sum(make_float4(gm.x * (v[u].x - mu), gm.y * (v[u].y - mu), gm.z * (v[u].z - mu), gm.w * (v[u].w - mu)));
        }
        s1 = bn_block_sum(s1, sh);
        s2 = bn_block_sum(s2, sh);
        if (threadIdx.x == 0) part[p.part] = make_float2(s1, s2);
    }
}

// One thread per output: i < n * C -> grad_w[i] (j = i / C, c = i % C) from channel c's pieces; else grad_b[i - n * C] from channel 0's
__global__ void head_wgrad_finalize_kernel(const BnShape s, int n, const float* __restrict__ wpart, const float* __restrict__ bpart,
                                           float* __restrict__ grad_w, float* __restrict__ grad_b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int nw = n * s.channels;
    if (i >= nw + n || (i < nw && !grad_w) || (i >= nw && !grad_b)) return;
    const int j = i < nw ? i / s.channels : i - nw, c = i < nw ? i % s.channels : 0;
    const float* pp = (i < nw ? wpart : bpart) + c * s.per_channel * n + j;
    double acc = 0.0;
    for (long long k = 0; k < s.per_channel; ++k) acc += static_cast<double>(pp[k * n]);
    if (i < nw) grad_w[i] = static_cast<float>(acc);
    else grad_b[j] = static_cast<float>(acc);
}

template <bool TRAINING>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) head_grad_apply_kernel(const BnShape s, const float* __restrict__ y, const HeadGrad h,
                                                                     const BnCoef* __restrict__ coef, float* __restrict__ dx) {
    for (long long g = blockIdx.x; g < s.pieces; g += gridDim.x) {
        const BnPiece p = bn_piece(s, g);
        const GruPieceAt at = gru_piece_at(s, g);
        const float* xp = y + p.x_off;
        const float* gp = h.g + at.b * h.n * s.pixels + at.pix;
        float* op = dx + p.out_off;
        const bool vx = aligned16_ptr(xp), vg = aligned16_ptr(gp), vo = aligned16_ptr(op);
        const BnCoef k = coef[p.c];
        const int n_chunks = (p.n + 3) / 4;
        float4 v[BN_CHUNKS];
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            if (q < n_chunks) v[u] = load_chunk4(xp, q, p.n, vx);
        }
#pragma unroll
        for (int u = 0; u < BN_CHUNKS; ++u) {
            const int q = threadIdx.x + u * BN_THREADS;
            if (q >= n_chunks) continue;
            const float4 d = head_da(h, gp, s.pixels, p.c, q, p.n, vg);
            const float xs[4] = {v[u].x, v[u].y, v[u].z, v[u].w}, ds[4] = {d.x, d.y, d.z, d.w};
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float gm = bn_masked<true>(ds[e], xs[e], k.scale, k.shift);
                o[e] = TRAINING ? fmaf(k.scale, gm, fmaf(k.k1, xs[e] - k.mean, k.k0)) : k.scale * gm;
            }
            store_chunk4(op, q, p.n, vo, make_float4(o[0], o[1], o[2], o[3]));
        }
    }
}

// the backward's workspace: batch_norm_workspace_bytes(d) (coefficients, then the (S1, S2) partials), then n weight-gradient partials
// per piece, then n bias-gradient partials per piece of channel 0
struct HeadWork { BnCoef* coef; float2* part; float* wpart; float* bpart; };
static size_t head_wpart_bytes(const BnShape& s, int n) { return (static_cast<size_t>(s.pieces) * n * sizeof(float) + 255) / 256 * 256; }

size_t output_head_backward_workspace_bytes(const fiery_batch_norm_desc_t* d, int n) {
    const BnShape s = bn_shape(d);
    return (batch_norm_workspace_bytes(d) + 255) / 256 * 256 + head_wpart_bytes(s, n) + static_cast<size_t>(s.per_channel) * n * sizeof(float);
}

static HeadWork head_work(const fiery_batch_norm_desc_t* d, const BnShape& s, int n, void* workspace) {
    const BnWork b = bn_work(d, workspace);
    char* wp = static_cast<char*>(workspace) + (batch_norm_workspace_bytes(d) + 255) / 256 * 256;
    return {b.coef, b.part, reinterpret_cast<float*>(wp), reinterpret_cast<float*>(wp + head_wpart_bytes(s, n))};
}

// d: the head's norm over y (relu 1); grad_y, grad_bn_w / grad_bn_b, grad_w (n, C) and grad_b (n) may each be NULL
int launch_output_head_backward(const fiery_batch_norm_desc_t* d, const float* y, const float* g, const float* w1, int ld, int n,
                                const float* w, const float* bias, const float* mean, const float* var, float* grad_y, float* grad_bn_w,
                                float* grad_bn_b, float* grad_w, float* grad_b, void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    const HeadWork k = head_work(d, s, n, workspace);
    const HeadGrad h{g, w1, n, ld};
    // the sums are needed for the norm's and the 1x1's weight and bias gradients, and for grad_y in training
    const bool reduce = grad_bn_w || grad_bn_b || grad_w || grad_b || (grad_y && d->training);
    if (reduce)
        head_grad_sums_kernel<<<bn_grid(s), BN_THREADS, 0, stream>>>(s, y, h, w, bias, mean, var, d->eps, k.part, grad_w ? k.wpart : nullptr,
                                                                     grad_b ? k.bpart : nullptr);
    if (grad_y || grad_bn_w || grad_bn_b)
        bn_finalize_backward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(s, k.part, reduce, w, bias, mean, var, d->training,
                                                                                   d->eps, grad_bn_w, grad_bn_b, k.coef);
    if (grad_w || grad_b)
        head_wgrad_finalize_kernel<<<(n * (d->channels + 1) + 127) / 128, 128, 0, stream>>>(s, n, k.wpart, k.bpart, grad_w, grad_b);
    if (grad_y && d->training) head_grad_apply_kernel<true><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, y, h, k.coef, grad_y);
    else if (grad_y) head_grad_apply_kernel<false><<<bn_grid(s), BN_THREADS, 0, stream>>>(s, y, h, k.coef, grad_y);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// Statistics over several ranks (fiery_batch_norm_*_gathered, fiery_spatial_gru_*_step_*).  Each rank reduces its own pieces as
// above into one fp64 triplet per channel -- (n, mean, M2) forward, (n, S1, S2) backward -- the caller gathers the ranks' triplets
// into (world, channels, 3), and the gathered finalize merges them in ascending rank order with the same formulas, starting from
// rank 0's triplet (so one rank gives exactly the single-rank finalize's numbers).  A rank with no values has n = 0 and adds nothing.
// ------------------------------------------------------------------------------------------------------------------------------
__global__ void bn_local_forward_kernel(const BnShape s, const float2* __restrict__ part, double* __restrict__ stats) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= s.channels) return;
    double n, m, m2;
    bn_merge_pieces(s, part, c, n, m, m2);
    stats[3 * c] = n;
    stats[3 * c + 1] = m;
    stats[3 * c + 2] = m2;
}

__global__ void bn_gathered_forward_kernel(int world, int channels, const double* __restrict__ gathered, const float* __restrict__ w,
                                           const float* __restrict__ bias, double eps, float* __restrict__ mean_out,
                                           float* __restrict__ var_out, double* __restrict__ count_out, BnCoef* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= channels) return;
    double n = gathered[3 * c], m = gathered[3 * c + 1], m2 = gathered[3 * c + 2];
    for (int r = 1; r < world; ++r) {
        const double* g = gathered + (static_cast<long long>(r) * channels + c) * 3;
        if (g[0] != 0.0) bn_chan_step(n, m, m2, g[0], g[1], g[2]);           // a rank with no values adds nothing
    }
    bn_forward_out(w, bias, static_cast<float>(m), static_cast<float>(m2 / n), n, eps, c, mean_out, var_out, count_out, coef);
}

// the rank's (n, S1, S2) and its own weight and bias gradients (the local sums, as torch's SyncBatchNorm)
__global__ void bn_local_backward_kernel(const BnShape s, const float2* __restrict__ part, const float* __restrict__ var, double eps,
                                         float* __restrict__ grad_w, float* __restrict__ grad_b, double* __restrict__ sums) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= s.channels) return;
    double s1, s2;
    bn_sum_pieces(s, part, var, eps, c, grad_w, grad_b, s1, s2);
    sums[3 * c] = static_cast<double>(s.per_channel / s.per_plane) * s.pixels;
    sums[3 * c + 1] = s1;
    sums[3 * c + 2] = s2;
}

__global__ void bn_gathered_backward_kernel(int world, int channels, const double* __restrict__ gathered, const float* __restrict__ w,
                                            const float* __restrict__ bias, const float* __restrict__ mean, const float* __restrict__ var,
                                            double eps, BnCoef* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= channels) return;
    double n = gathered[3 * c], s1 = gathered[3 * c + 1], s2 = gathered[3 * c + 2];
    for (int r = 1; r < world; ++r) {
        const double* g = gathered + (static_cast<long long>(r) * channels + c) * 3;
        n += g[0];
        s1 += g[1];
        s2 += g[2];
    }
    coef[c] = bn_backward_coef(w, bias, mean[c], var[c], eps, c, n, s1, s2);
}

int launch_batch_norm_local_stats(const fiery_batch_norm_desc_t* d, const float* x, double* stats, void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    float2* part = bn_work(d, workspace).part;
    if (s.pieces) bn_stats_kernel<<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, part);
    bn_local_forward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(s, part, stats);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_batch_norm_coef_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* w, const float* bias,
                                    float* mean_out, float* var_out, double* count_out, void* workspace, cudaStream_t stream) {
    bn_gathered_forward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(world, d->channels, gathered, w, bias, d->eps, mean_out,
                                                                              var_out, count_out, bn_work(d, workspace).coef);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_batch_norm_forward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* w,
                                       const float* bias, const float* residual, float* y, float* mean_out, float* var_out,
                                       double* count_out, void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    launch_batch_norm_coef_gathered(d, world, gathered, w, bias, mean_out, var_out, count_out, workspace, stream);
    bn_apply(d, s, x, bn_work(d, workspace).coef, residual, y, stream);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_batch_norm_local_grad_sums(const fiery_batch_norm_desc_t* d, const float* x, const float* dy, const float* w, const float* bias,
                                      const float* mean, const float* var, double* sums, float* grad_w, float* grad_b, void* workspace,
                                      cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    float2* part = bn_work(d, workspace).part;
    bn_grad_sums(d, s, x, dy, w, bias, mean, var, part, stream);
    bn_local_backward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(s, part, var, d->eps, grad_w, grad_b, sums);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_batch_norm_backward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* dy,
                                        const float* w, const float* bias, const float* mean, const float* var, float* dx, void* workspace,
                                        cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    BnCoef* coef = bn_work(d, workspace).coef;
    bn_gathered_backward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(world, d->channels, gathered, w, bias, mean, var, d->eps, coef);
    bn_grad_apply(d, s, x, dy, coef, dx, stream);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// the spatial GRU's step under gathered statistics: the finalize above, then the blend into the output frame
int launch_gru_blend_forward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* w,
                                      const float* bias, const float* u, const float* h, long long hsb, float* out, long long osb,
                                      float* mean_out, float* var_out, double* count_out, void* workspace, cudaStream_t stream) {
    const BnShape s = bn_shape(d);
    BnCoef* coef = bn_work(d, workspace).coef;
    bn_gathered_forward_kernel<<<(d->channels + 127) / 128, 128, 0, stream>>>(world, d->channels, gathered, w, bias, d->eps, mean_out,
                                                                              var_out, count_out, coef);
    gru_blend_kernel<<<bn_grid(s), BN_THREADS, 0, stream>>>(s, x, coef, u, h, hsb, out, osb);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
