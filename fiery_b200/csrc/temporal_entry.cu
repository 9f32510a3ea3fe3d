// The temporal block's 1x1x1 input projections as one GEMM (TemporalBlock, fiery/layers/temporal.py:218-281): the three paths'
// conv_1x1x1_norm_activated convolutions and the projection's Conv3d all read the block input x (b, K, s, X, Y), so
//
//   y[o][f][p] = sum_k W[o][k] * x[f][k][p]  (+ sum_j W[o][K + j] * e[f][j])        f = frame (b, t), p = pixel of X*Y
//
// with W the four weights stacked along o (N_out = 35 + 35 + 35 + 64 = 169 in the first block, 32 x 3 = 96 in the second).  The
// optional e (E <= 8 channels per frame, constant over the map: the egopose) enters as a per-(frame, o) bias computed in fp32, so the
// concatenated 70-channel input never has to exist.  All three kernels run on the tensor cores: wgmma, TF32 operands, fp32
// accumulation.  Weights are rounded to TF32 (cvt.rna) when packed; activations and output gradients are read from fp32 by the
// tensor core, which truncates them.
//
// Output channels are numbered "padded": segment q (one conv, C_q channels) occupies rows [off_q, off_q + C_q) with off_q the sum of
// the earlier segments' channel counts rounded up to 8, so every segment's gradient tile starts on an 8-row swizzle group in shared
// memory.  Npad = off_{n_seg}.
//
// Forward: one CTA per SM, persistent over 128-pixel tiles of one frame.  The input tile (Kpad channels x 128 pixels) is TMA-loaded as
// it lies -- pixel planes contiguous, arbitrary frame / channel strides, so both the permuted concat (frame-major) and an NCDHW tensor
// (channel-major) are read without a copy; channels K .. Kpad and pixels past X*Y are the TMA's zero fill.  D (128 pixels x Npad) =
// x^T W^T with the pixel tile as the register A operand (as in depth_layer.cu) and the packed weights as the K-major B operand.  The
// epilogue goes through shared memory, 32 output channels at a time, so each output row is stored as 256 contiguous bytes into its
// segment's contiguous (b, C_q, s, X, Y) tensor.
// Input gradient: dx (pixels x K) = dy^T W over the 64-pixel tiles; the four segments' gradient tiles are TMA-loaded into one padded
// tile and read as the register A operand, the transposed pack is the B operand; dx is written with the input's strides.
// Weight gradient: dW (Npad x K + E) = sum over pixels of dy x^T; both tiles are pixel-contiguous, so both are K-major shared-memory
// operands.  With E > 0 the egopose is written into the input tile's rows K .. K + E - 1 (TF32-rounded) so its columns come out of the
// same MMAs.  The 64-pixel tiles are cut into chunks whose boundaries depend on (frames, X*Y) only; each chunk stores its partial and a
// reduce kernel adds the partials in ascending chunk order: bit-reproducible, no atomics.
#include "bn_coef.cuh"
#include "wgmma.cuh"
#include "wgrad_chunks.cuh"

namespace fiery {

constexpr int TE_MAX_E = 8, TE_MAX_SEG = 4;
constexpr int TE_FWD_PX = 128;                     // pixels per forward tile (two consumer warpgroups)
constexpr int TE_BWD_PX = 64;                      // pixels per backward tile
constexpr int TE_STG_PITCH = 66;                   // staging row pitch (floats): conflict-free fragment writes
constexpr int TE_STG_FLOATS = 32 * TE_STG_PITCH;   // 32 channels x 64 pixels
constexpr int TE_SMEM_MAX = 232448;                // sm_90 opt-in shared memory per block
constexpr int TE_SMEM_SLACK = 1024 + 256;          // alignment + barriers
constexpr int TE_ROW_TABLE_BYTES = 2 * 256 * (8 + 4);   // forward: per warpgroup and padded output row, destination + bias

static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

struct TeShape {
    int batch, frames, pixels, K, Kpad, E, n_seg, n_out, Npad, Npad32;
    int seg_ch[TE_MAX_SEG], seg_off[TE_MAX_SEG + 1], nat_off[TE_MAX_SEG + 1];
    long long sb, st, sc;                          // input strides, elements
};

static TeShape te_shape(const fiery_temporal_entry_desc_t* d) {
    TeShape s{};
    s.batch = d->batch;
    s.frames = d->frames;
    s.pixels = d->pixels;
    s.K = d->in_channels;
    s.Kpad = round_up(d->in_channels, 32);
    s.E = d->extra_channels;
    s.n_seg = d->n_segments;
    s.sb = d->in_stride_b;
    s.st = d->in_stride_t;
    s.sc = d->in_stride_c;
    for (int q = 0; q < s.n_seg; ++q) {
        s.seg_ch[q] = d->seg_channels[q];
        s.seg_off[q + 1] = s.seg_off[q] + round_up(d->seg_channels[q], 8);
        s.nat_off[q + 1] = s.nat_off[q] + d->seg_channels[q];
    }
    s.Npad = s.seg_off[s.n_seg];
    s.Npad32 = round_up(s.Npad, 32);
    s.n_out = s.nat_off[s.n_seg];
    return s;
}

// Packed weights (floats): F = forward B operand (NCH*64 rows o, K32 columns k), then T = input-gradient B operand (NCHK*64 rows k,
// Npad32 columns o), both TF32-rounded; then the egopose columns (Npad rows x 8) in fp32.
struct TePack {
    int nch, k32, nchk, npad32;
    size_t f_floats, t_floats, e_floats;
};
static TePack te_pack_layout(const TeShape& s) {
    TePack p;
    p.nch = (s.Npad + 63) / 64;
    p.k32 = s.Kpad;
    p.nchk = (s.Kpad + 63) / 64;
    p.npad32 = s.Npad32;
    p.f_floats = static_cast<size_t>(p.nch) * 64 * p.k32;
    p.t_floats = static_cast<size_t>(p.nchk) * 64 * p.npad32;
    p.e_floats = static_cast<size_t>(s.Npad) * TE_MAX_E;
    return p;
}

size_t temporal_entry_packed_bytes(const fiery_temporal_entry_desc_t* d) {
    const TeShape s = te_shape(d);
    const TePack p = te_pack_layout(s);
    return (p.f_floats + p.t_floats + p.e_floats) * sizeof(float);
}

// padded output row -> natural row (o of the stacked weight), or -1 for a padding row
__host__ __device__ __forceinline__ int te_natural_row(const TeShape& s, int o) {
    for (int q = 0; q < s.n_seg; ++q)
        if (o >= s.seg_off[q] && o < s.seg_off[q] + s.seg_ch[q]) return s.nat_off[q] + o - s.seg_off[q];
    return -1;
}

__global__ void te_pack_kernel(TeShape s, TePack p, const float* __restrict__ w, float* __restrict__ packed) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int ld = s.K + s.E;                      // row length of the stacked weight (N_out, K + E)
    float v = 0.f;
    if (i < p.f_floats) {
        const int o = static_cast<int>(i / p.k32), k = static_cast<int>(i % p.k32);
        const int on = o < s.Npad ? te_natural_row(s, o) : -1;
        if (on >= 0 && k < s.K) v = __uint_as_float(to_tf32(w[static_cast<size_t>(on) * ld + k]));
    } else if (i < p.f_floats + p.t_floats) {
        const size_t j = i - p.f_floats;
        const int k = static_cast<int>(j / p.npad32), o = static_cast<int>(j % p.npad32);
        const int on = o < s.Npad ? te_natural_row(s, o) : -1;
        if (on >= 0 && k < s.K) v = __uint_as_float(to_tf32(w[static_cast<size_t>(on) * ld + k]));
    } else if (i < p.f_floats + p.t_floats + p.e_floats) {
        const size_t j = i - p.f_floats - p.t_floats;
        const int o = static_cast<int>(j / TE_MAX_E), e = static_cast<int>(j % TE_MAX_E);
        const int on = te_natural_row(s, o);
        if (on >= 0 && e < s.E) v = w[static_cast<size_t>(on) * ld + s.K + e];
    } else {
        return;
    }
    packed[i] = v;
}

int launch_temporal_entry_pack(const fiery_temporal_entry_desc_t* d, const float* w, float* packed, cudaStream_t stream) {
    const TeShape s = te_shape(d);
    const TePack p = te_pack_layout(s);
    const size_t n = p.f_floats + p.t_floats + p.e_floats;
    te_pack_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(s, p, w, packed);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// shared device helpers
// ------------------------------------------------------------------------------------------------------------------------------
// acc[c] (64 pixel rows x 64 columns of n-chunk c) += tile rows 32 kg .. 32 kg + 31 (as the register A operand, pixel rows pa / pb)
// x the B atom at b_atom (NC*64 K-major rows of 32 fp32 k); 4 k-steps, drained before returning.  BN: each fragment value v of
// channel row ch becomes bn_relu_apply(coef[ch], v) (coef: one entry per tile row, zero past the input's channels) before the
// tensor core truncates it, as it truncates the plain input.
template <int NC, bool BN = false>
__device__ __forceinline__ void te_mma_group(float (&acc)[NC][32], const unsigned char* tile, int rows, int kg, int pa, int pb,
                                             uint32_t b_atom, const BnCoef* coef = nullptr) {
    uint32_t a[4][4];
    load_pixel_frags<4>(a, tile, rows, 32 * kg, pa, pb);
    if constexpr (BN) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int ch = 32 * kg + 8 * k + (threadIdx.x & 3);
            const BnCoef lo = coef[ch], hi = coef[ch + 4];
            a[k][0] = __float_as_uint(bn_relu_apply(lo, __uint_as_float(a[k][0])));
            a[k][1] = __float_as_uint(bn_relu_apply(lo, __uint_as_float(a[k][1])));
            a[k][2] = __float_as_uint(bn_relu_apply(hi, __uint_as_float(a[k][2])));
            a[k][3] = __float_as_uint(bn_relu_apply(hi, __uint_as_float(a[k][3])));
        }
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int c = 0; c < NC; ++c) wgmma_tf32_rs<64>(acc[c], a[k], gmma_desc_sw128(b_atom + c * 64 * 128 + k * 32, 16, 1024));
    wgmma_commit();
    wgmma_wait<0>();
}

// One warpgroup's epilogue for 32 accumulator columns (n-chunk c, half h) of its 64 pixel rows: fragments -> staging (channel rows
// of 64 pixels) -> one 256-byte row store per channel.  row_ptr(col) gives the destination of column col's 64 pixels (nullptr: skip)
// and its bias; with RES also the row of 64 pixels added after the bias (row_ptr(col, bias, res)).  bar_id: the warpgroup's named
// barrier.
template <bool RES = false, typename RowFn>
__device__ __forceinline__ void te_store_cols(const float (&acc)[32], int h, float* stg, int bar_id, int n_valid_px, RowFn row_ptr) {
    const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int r0 = 16 * wq + (lane >> 2);
    const int pa = tile_pixel(r0), pb = tile_pixel(r0 + 8);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + cq + e;
            stg[col * TE_STG_PITCH + pa] = acc[4 * (4 * h + j) + e];
            stg[col * TE_STG_PITCH + pb] = acc[4 * (4 * h + j) + 2 + e];
        }
    named_barrier(bar_id, 128);
#pragma unroll
    for (int col = 8 * wq; col < 8 * wq + 8; ++col) {
        float bias = 0.f;
        if constexpr (RES) {
            const float* res = nullptr;
            float* dst = row_ptr(col, bias, res);
            if (dst != nullptr && 2 * lane < n_valid_px) {
                const float2 v = *reinterpret_cast<const float2*>(stg + col * TE_STG_PITCH + 2 * lane);
                const float2 r = *reinterpret_cast<const float2*>(res + 2 * lane);
                *reinterpret_cast<float2*>(dst + 2 * lane) = make_float2((v.x + bias) + r.x, (v.y + bias) + r.y);
            }
        } else {
            float* dst = row_ptr(col, bias);
            if (dst != nullptr && 2 * lane < n_valid_px) {
                const float2 v = *reinterpret_cast<const float2*>(stg + col * TE_STG_PITCH + 2 * lane);
                *reinterpret_cast<float2*>(dst + 2 * lane) = make_float2(v.x + bias, v.y + bias);
            }
        }
    }
    named_barrier(bar_id, 128);
}

// the four segments' output-gradient tiles (round8(C_q) rows x 32 pixels per block, 2 blocks) of frame (b, t), pixels p0 ..
struct TeGradMaps {
    CUtensorMap gy[TE_MAX_SEG];                    // segment q: (X*Y, s, C_q, b), box (32, 1, rows q, 1), swizzle 128B; rows q =
                                                   // round8(C_q), the last segment's up to Npad32 (zero fill to a 32-row group)
};
__device__ __forceinline__ void te_load_grad_tile(const TeGradMaps& maps, const TeShape& s, unsigned char* dst, int rows, uint64_t* bar,
                                                  int b, int t, int p0) {
    for (int q = 0; q < s.n_seg; ++q)
#pragma unroll
        for (int blk = 0; blk < TE_BWD_PX / 32; ++blk)
            tma_load_4d(dst + blk * rows * 128 + s.seg_off[q] * 128, &maps.gy[q], bar, p0 + 32 * blk, t, 0, b);
}

// ------------------------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------------------------
struct TeFwdMaps {
    CUtensorMap w;                                 // F region: (K32, NCH*64), box (32, NCH*64), swizzle 128B
    CUtensorMap x;                                 // input: (X*Y, K, s, b), box (32, Kpad, 1, 1), swizzle 128B
};
struct TeOut {
    float* p[TE_MAX_SEG];
};

constexpr int TE_FWD_THREADS = 2 * 128 + 32;

// BN: the Bottleneck's up projection -- every input value goes through bn_relu_apply with its channel's coefficients (coef, K
// entries, copied to s_coef with zeros up to Kpad) as the consumers read it; the instantiation without it is the entry's forward.
template <int NCH, bool BN>
__device__ __forceinline__ void te_fwd_body(const TeFwdMaps& maps, const TeShape& s, const float* __restrict__ extra,
                                            const float* __restrict__ w_extra, const TeOut& out, int stages, int tiles_per_frame, int n_tiles,
                                            const BnCoef* __restrict__ coef, BnCoef* s_coef) {
    const int k32 = (s.Kpad + 31) & ~31;
    const int w_atom = NCH * 64 * 128;
    const int x_bytes = 4 * s.Kpad * 128;
    unsigned char* s_w = dynamic_smem_1024();
    unsigned char* s_x = s_w + (k32 / 32) * w_atom;
    float* s_stg = reinterpret_cast<float*>(s_x + stages * x_bytes);
    float** s_rowptr = reinterpret_cast<float**>(s_stg + 2 * TE_STG_FLOATS);        // [2][256]
    float* s_rowbias = reinterpret_cast<float*>(s_rowptr + 2 * 256);                // [2][256]
    uint64_t* w_full = reinterpret_cast<uint64_t*>(s_rowbias + 2 * 256);
    const MbarRing ring(w_full + 1, stages);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&maps.w);
        tma_prefetch_desc(&maps.x);
        mbar_init(w_full, 1);                          // published to the async proxy by the fence in ring.init
        ring.init(8);
    }
    if constexpr (BN)
        for (int c = threadIdx.x; c < s.Kpad; c += blockDim.x) s_coef[c] = c < s.K ? coef[c] : BnCoef{};
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {                               // ===== TMA producer: weights once, then this CTA's input tiles =====
            mbar_arrive_expect_tx(w_full, (k32 / 32) * w_atom);
            for (int a = 0; a < k32 / 32; ++a) tma_load_3d(s_w + a * w_atom, &maps.w, w_full, 32 * a, 0, 0);
            int it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
                const int st = ring.produce(it, x_bytes);
                const int f = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TE_FWD_PX;
                unsigned char* dst = s_x + st * x_bytes;
#pragma unroll
                for (int blk = 0; blk < TE_FWD_PX / 32; ++blk)
                    tma_load_4d(dst + blk * s.Kpad * 128, &maps.x, ring.full + st, p0 + 32 * blk, 0, f % s.frames, f / s.frames);
            }
        }
        return;
    }

    // ===== consumers: warpgroup g owns pixel rows 64g .. 64g + 63 =====
    const int g = warp >> 2;
    const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
    const int pa = tile_pixel(r0), pb = tile_pixel(r0 + 8);
    const uint32_t w_addr = smem_addr(s_w);
    float* stg = s_stg + g * TE_STG_FLOATS;
    mbar_wait(w_full, 0);
    int it = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
        const int f = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TE_FWD_PX;
        const int b = f / s.frames, tt = f % s.frames;
        const unsigned char* tile = s_x + ring.consume(it) * x_bytes;
        float acc[NCH][32];
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
#pragma unroll 1
        for (int kg = 0; kg < k32 / 32; ++kg)          // 32 channels (4 k-steps, 16 fragment registers) at a time
            te_mma_group<NCH, BN>(acc, tile, s.Kpad, kg, pa, pb, w_addr + kg * w_atom, s_coef);
#pragma unroll
        for (int c = 0; c < NCH; ++c) wgmma_fence_operands(acc[c]);
        ring.release(it);                              // this warp's part of the tile has been read

        const int pbase = p0 + 64 * g;
        const int n_valid = s.pixels - pbase;
        // this tile's row table, one entry per padded output row: where the row's 64 pixels go (nullptr: a padding row) and its
        // egopose bias.  te_store_cols reads 32 rows at a time, so every row below Npad32 needs an entry.  The previous tile's last
        // te_store_cols ended on the warpgroup's barrier, so nothing reads the table any more; the first barrier inside
        // te_store_cols publishes it.
        float** rowptr = s_rowptr + 256 * g;
        float* rowbias = s_rowbias + 256 * g;
        for (int o = threadIdx.x & 127; o < s.Npad32; o += 128) {
            float* dst = nullptr;
            float bias = 0.f;
            for (int q = 0; q < s.n_seg; ++q) {
                if (o >= s.seg_off[q] && o < s.seg_off[q] + s.seg_ch[q]) {
                    dst = out.p[q] + ((static_cast<size_t>(b) * s.seg_ch[q] + (o - s.seg_off[q])) * s.frames + tt) * s.pixels + pbase;
                    if (extra) {
                        const float* e_f = extra + static_cast<size_t>(f) * s.E;
                        for (int j = 0; j < s.E; ++j) bias = fmaf(__ldg(w_extra + o * TE_MAX_E + j), __ldg(e_f + j), bias);
                    }
                }
            }
            rowptr[o] = dst;
            rowbias[o] = bias;
        }
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (64 * c + 32 * h >= s.Npad) continue;
                te_store_cols(acc[c], h, stg, 1 + g, n_valid, [&](int col, float& bias) -> float* {
                    const int o = 64 * c + 32 * h + col;
                    bias = rowbias[o];
                    return rowptr[o];
                });
            }
    }
}

template <int NCH>
__global__ void __launch_bounds__(TE_FWD_THREADS, 1)
temporal_entry_fwd_kernel(const __grid_constant__ TeFwdMaps maps, const TeShape s, const float* __restrict__ extra,
                          const float* __restrict__ w_extra, const TeOut out, int stages, int tiles_per_frame, int n_tiles) {
    te_fwd_body<NCH, false>(maps, s, extra, w_extra, out, stages, tiles_per_frame, n_tiles, nullptr, nullptr);
}

template <int NCH>
__global__ void __launch_bounds__(TE_FWD_THREADS, 1)
bottleneck_entry_fwd_kernel(const __grid_constant__ TeFwdMaps maps, const TeShape s, const TeOut out, int stages, int tiles_per_frame,
                            int n_tiles, const BnCoef* __restrict__ coef) {
    __shared__ BnCoef s_coef[128];
    te_fwd_body<NCH, true>(maps, s, nullptr, nullptr, out, stages, tiles_per_frame, n_tiles, coef, s_coef);
}

// The decoder's output heads' 1x1 (output_head.cu): the Bottleneck's BN + ReLU prologue, and the head's bias folded in as the one
// extra channel (E = 1) whose value `ones[f]` is 1 in every map f, so the epilogue adds fmaf(b1[o], 1, 0) = b1[o] exactly.  N <= 8.
__global__ void __launch_bounds__(TE_FWD_THREADS, 1)
output_head_fwd_kernel(const __grid_constant__ TeFwdMaps maps, const TeShape s, const float* __restrict__ ones,
                       const float* __restrict__ w_extra, const TeOut out, int stages, int tiles_per_frame, int n_tiles,
                       const BnCoef* __restrict__ coef) {
    __shared__ BnCoef s_coef[128];
    te_fwd_body<1, true>(maps, s, ones, w_extra, out, stages, tiles_per_frame, n_tiles, coef, s_coef);
}

// ------------------------------------------------------------------------------------------------------------------------------
// input gradient
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int TE_DG_THREADS = 128 + 32;

struct TeDgradMaps {
    TeGradMaps g;
    CUtensorMap w;                                 // T region: (Npad32, NCHK*64), box (32, NCHK*64), swizzle 128B
};

// BIAS: every output row k of frame f = (b, t) gets bias[f * K + k] added in the epilogue (the temporal aggregation's pooled-vector
// term); RES: every output value gets the value of res at its place (res has gx's strides) added after that (the Bottleneck's skip
// connection); the instantiation with neither is the entry's input gradient.
template <int NCHK, bool BIAS, bool RES = false>
__device__ __forceinline__ void te_dgrad_body(const TeDgradMaps& maps, const TeShape& s, float* __restrict__ gx,
                                              const float* __restrict__ bias, int stages, int tiles_per_frame, int n_tiles,
                                              const float* __restrict__ res = nullptr) {
    const int npad32 = (s.Npad + 31) & ~31;
    const int rows = (s.Npad + 63) & ~63;          // grad tile rows per 32-pixel block
    const int w_atom = NCHK * 64 * 128;
    const int g_bytes = 2 * rows * 128;
    unsigned char* s_w = dynamic_smem_1024();
    unsigned char* s_g = s_w + (npad32 / 32) * w_atom;
    float* stg = reinterpret_cast<float*>(s_g + stages * g_bytes);
    uint64_t* w_full = reinterpret_cast<uint64_t*>(stg + TE_STG_FLOATS);
    const MbarRing ring(w_full + 1, stages);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 4 && lane == 0) {
        tma_prefetch_desc(&maps.w);
        for (int q = 0; q < s.n_seg; ++q) tma_prefetch_desc(&maps.g.gy[q]);
        mbar_init(w_full, 1);                          // published to the async proxy by the fence in ring.init
        ring.init(4);
    }
    __syncthreads();

    if (warp == 4) {
        if (lane == 0) {
            mbar_arrive_expect_tx(w_full, (npad32 / 32) * w_atom);
            for (int a = 0; a < npad32 / 32; ++a) tma_load_3d(s_w + a * w_atom, &maps.w, w_full, 32 * a, 0, 0);
            int it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
                const int st = ring.produce(it, 2 * s.Npad32 * 128);
                const int f = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TE_BWD_PX;
                te_load_grad_tile(maps.g, s, s_g + st * g_bytes, rows, ring.full + st, f / s.frames, f % s.frames, p0);
            }
        }
        return;
    }

    const int r0 = 16 * warp + (lane >> 2);
    const int pa = tile_pixel(r0), pb = tile_pixel(r0 + 8);
    const uint32_t w_addr = smem_addr(s_w);
    mbar_wait(w_full, 0);
    int it = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
        const int f = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TE_BWD_PX;
        const int b = f / s.frames, tt = f % s.frames;
        const unsigned char* tile = s_g + ring.consume(it) * g_bytes;
        float acc[NCHK][32];
#pragma unroll
        for (int c = 0; c < NCHK; ++c)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
#pragma unroll 1
        for (int kg = 0; kg < npad32 / 32; ++kg)       // 32 output channels at a time
            te_mma_group<NCHK>(acc, tile, rows, kg, pa, pb, w_addr + kg * w_atom);
#pragma unroll
        for (int c = 0; c < NCHK; ++c) wgmma_fence_operands(acc[c]);
        ring.release(it);

        const size_t off = static_cast<size_t>(b) * s.sb + static_cast<size_t>(tt) * s.st + p0;
        float* base = gx + off;
#pragma unroll
        for (int c = 0; c < NCHK; ++c)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (64 * c + 32 * h >= s.K) continue;
                if constexpr (RES) {
                    te_store_cols<true>(acc[c], h, stg, 1, s.pixels - p0, [&](int col, float&, const float*& r) -> float* {
                        const int k = 64 * c + 32 * h + col;
                        r = res + off + static_cast<size_t>(k) * s.sc;
                        return k < s.K ? base + static_cast<size_t>(k) * s.sc : nullptr;
                    });
                } else {
                    te_store_cols(acc[c], h, stg, 1, s.pixels - p0, [&](int col, float& b_k) -> float* {
                        const int k = 64 * c + 32 * h + col;
                        if (BIAS && k < s.K) b_k = __ldg(bias + static_cast<size_t>(f) * s.K + k);
                        return k < s.K ? base + static_cast<size_t>(k) * s.sc : nullptr;
                    });
                }
            }
    }
}

template <int NCHK>
__global__ void __launch_bounds__(TE_DG_THREADS, 1)
temporal_entry_dgrad_kernel(const __grid_constant__ TeDgradMaps maps, const TeShape s, float* __restrict__ gx, int stages,
                            int tiles_per_frame, int n_tiles) {
    te_dgrad_body<NCHK, false>(maps, s, gx, nullptr, stages, tiles_per_frame, n_tiles);
}

template <int NCHK>
__global__ void __launch_bounds__(TE_DG_THREADS, 1)
temporal_aggregation_kernel(const __grid_constant__ TeDgradMaps maps, const TeShape s, float* __restrict__ out,
                            const float* __restrict__ bias, int stages, int tiles_per_frame, int n_tiles) {
    te_dgrad_body<NCHK, true>(maps, s, out, bias, stages, tiles_per_frame, n_tiles);
}

template <int NCHK>
__global__ void __launch_bounds__(TE_DG_THREADS, 1)
bottleneck_entry_dgrad_kernel(const __grid_constant__ TeDgradMaps maps, const TeShape s, float* __restrict__ gx,
                              const float* __restrict__ res, int stages, int tiles_per_frame, int n_tiles) {
    te_dgrad_body<NCHK, false, true>(maps, s, gx, nullptr, stages, tiles_per_frame, n_tiles, res);
}

// ------------------------------------------------------------------------------------------------------------------------------
// weight gradient
// ------------------------------------------------------------------------------------------------------------------------------
struct TeWgradMaps {
    TeGradMaps g;
    CUtensorMap x;                                 // as TeFwdMaps::x but box (32, Kpad, 1, 1) into 64-pixel tiles
};

static long long te_bwd_tiles(int n_frames, int pixels) {
    return static_cast<long long>(n_frames) * ((pixels + TE_BWD_PX - 1) / TE_BWD_PX);
}
static int te_wgrad_chunks(int n_frames, int pixels) { return wgrad_chunks(te_bwd_tiles(n_frames, pixels), WG_MAX_CHUNKS); }
// partial: (Nrows = round64(Npad)) x (Kx = round64(K + E)) floats per chunk
static size_t te_partial_floats(const TeShape& s) {
    return static_cast<size_t>(round_up(s.Npad, 64)) * round_up(s.K + s.E, 64);
}

size_t temporal_entry_wgrad_workspace_bytes(const fiery_temporal_entry_desc_t* d) {
    const TeShape s = te_shape(d);
    return static_cast<size_t>(te_wgrad_chunks(s.batch * s.frames, s.pixels)) * te_partial_floats(s) * sizeof(float);
}

// grid: one CTA per chunk; warpgroup mb (of Nrows / 64) accumulates output rows 64 mb .. 64 mb + 63 against all NC column chunks.
// Thread 0 issues the loads: at iteration it, after the barrier that ends every warpgroup's MMAs on tile it - 1, tile it + stages - 1.
// BN: the Bottleneck's up projection -- before the MMAs read a landed input tile, its values of channels k < K at pixels inside the
// frame become bn_relu_apply(s_coef[k], v) in shared memory (the zero fill past the frame's pixels stays 0); the tensor core then
// truncates them as it truncates the plain input.  The instantiation without it is the entry's weight gradient.
template <int NC, bool BN>
__device__ __forceinline__ void te_wgrad_body(const TeWgradMaps& maps, const TeShape& s, const float* __restrict__ extra,
                                              float* __restrict__ partial, int stages, int tiles_per_frame, int n_tiles,
                                              const BnCoef* __restrict__ coef, BnCoef* s_coef) {
    unsigned char* smem = dynamic_smem_1024();
    const int rows = (s.Npad + 63) & ~63, xrows = 64 * NC;
    const int g_bytes = 2 * rows * 128, stage_bytes = g_bytes + 2 * xrows * 128;
    const MbarRing ring(reinterpret_cast<uint64_t*>(smem + stages * stage_bytes), stages);
    const int nthreads = blockDim.x;
    const int t0 = static_cast<int>(static_cast<long long>(blockIdx.x) * n_tiles / gridDim.x);
    const int t1 = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * n_tiles / gridDim.x);
    const int tx_bytes = 2 * (s.Npad32 + s.Kpad) * 128;

    auto load = [&](int i) {                       // tile t0 + i into stage i % stages
        const int t = t0 + i, f = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TE_BWD_PX;
        const int b = f / s.frames, tt = f % s.frames;
        const int st = ring.arm(i, tx_bytes);
        unsigned char* dst = smem + st * stage_bytes;
        te_load_grad_tile(maps.g, s, dst, rows, ring.full + st, b, tt, p0);
#pragma unroll
        for (int blk = 0; blk < TE_BWD_PX / 32; ++blk)
            tma_load_4d(dst + g_bytes + blk * xrows * 128, &maps.x, ring.full + st, p0 + 32 * blk, 0, tt, b);
    };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&maps.x);
        for (int q = 0; q < s.n_seg; ++q) tma_prefetch_desc(&maps.g.gy[q]);
        ring.init(0);
        for (int i = 0; i < stages - 1 && t0 + i < t1; ++i) load(i);
    }
    if constexpr (BN)
        for (int c = threadIdx.x; c < s.K; c += nthreads) s_coef[c] = coef[c];
    __syncthreads();

    const int mb = threadIdx.x >> 7;
    float acc[NC][32];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;

    for (int i = 0; t0 + i < t1; ++i) {
        named_barrier(1, nthreads);                // every warpgroup is done with tile i - 1: its stage may be refilled
        if (threadIdx.x == 0 && t0 + i + stages - 1 < t1) load(i + stages - 1);
        unsigned char* tile = smem + ring.consume(i) * stage_bytes;
        if (s.E > 0) {                             // egopose rows K .. K + E - 1 of the input tile (zero past the frame's pixels)
            const int t = t0 + i, f = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TE_BWD_PX;
            for (int idx = threadIdx.x; idx < s.E * TE_BWD_PX; idx += nthreads) {
                const int j = idx / TE_BWD_PX, px = idx % TE_BWD_PX;
                const float v = p0 + px < s.pixels ? __ldg(extra + static_cast<size_t>(f) * s.E + j) : 0.f;
                *reinterpret_cast<uint32_t*>(tile + g_bytes + tile_offset(xrows, s.K + j, px)) = to_tf32(v);
            }
            fence_proxy_async();
            named_barrier(2, nthreads);
        }
        if constexpr (BN) {                        // generic writes, then the async proxy's MMAs read them: fence, then barrier
            const int t = t0 + i, n_px = min(TE_BWD_PX, s.pixels - (t % tiles_per_frame) * TE_BWD_PX);
            for (int idx = threadIdx.x; idx < s.K * TE_BWD_PX; idx += nthreads) {
                const int k = idx / TE_BWD_PX, px = idx % TE_BWD_PX;
                if (px < n_px) {
                    float* v = reinterpret_cast<float*>(tile + g_bytes + tile_offset(xrows, k, px));
                    *v = bn_relu_apply(s_coef[k], *v);
                }
            }
            fence_proxy_async();
            named_barrier(2, nthreads);
        }
        const uint32_t g_addr = smem_addr(tile) + mb * 64 * 128, x_addr = smem_addr(tile + g_bytes);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TE_BWD_PX / 8; ++ks) {
            const int blk = ks >> 2, kk = ks & 3;
            const uint64_t da = gmma_desc_sw128(g_addr + blk * rows * 128 + 32 * kk, 16, 1024);
#pragma unroll
            for (int c = 0; c < NC; ++c)
                wgmma_tf32_ss<64>(acc[c], da, gmma_desc_sw128(x_addr + blk * xrows * 128 + c * 64 * 128 + 32 * kk, 16, 1024));
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int c = 0; c < NC; ++c) wgmma_fence_operands(acc[c]);
    }

    // this chunk's partial: accumulator (row o, column k) -> partial[chunk][o][k]
    const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, cq = 2 * (lane & 3);
    float* dst = partial + static_cast<size_t>(blockIdx.x) * rows * xrows;
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int o = 64 * mb + 16 * wq + (lane >> 2) + 8 * half;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<float2*>(dst + static_cast<size_t>(o) * xrows + 64 * c + 8 * j + cq) =
                    make_float2(acc[c][4 * j + 2 * half], acc[c][4 * j + 2 * half + 1]);
        }
}

template <int NC>
__global__ void __launch_bounds__(512, 1)
temporal_entry_wgrad_kernel(const __grid_constant__ TeWgradMaps maps, const TeShape s, const float* __restrict__ extra,
                            float* __restrict__ partial, int stages, int tiles_per_frame, int n_tiles) {
    te_wgrad_body<NC, false>(maps, s, extra, partial, stages, tiles_per_frame, n_tiles, nullptr, nullptr);
}

template <int NC>
__global__ void __launch_bounds__(512, 1)
bottleneck_entry_wgrad_kernel(const __grid_constant__ TeWgradMaps maps, const TeShape s, float* __restrict__ partial, int stages,
                              int tiles_per_frame, int n_tiles, const BnCoef* __restrict__ coef) {
    __shared__ BnCoef s_coef[128];
    te_wgrad_body<NC, true>(maps, s, nullptr, partial, stages, tiles_per_frame, n_tiles, coef, s_coef);
}

// grad_w (N_out, K + E) index -> its place in a chunk's partial (padded row o, column k)
struct TeWgradOffset {
    TeShape s;
    __device__ size_t operator()(int i) const {
        const int ld = s.K + s.E;
        const int on = i / ld, k = i % ld;
        int o = 0;
        for (int q = 0; q < s.n_seg; ++q)
            if (on >= s.nat_off[q] && on < s.nat_off[q + 1]) o = s.seg_off[q] + on - s.nat_off[q];
        return static_cast<size_t>(o) * ((ld + 63) & ~63) + k;
    }
};

// ------------------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------------------
// the block input (b, t, channel, X*Y) with its strides; box (32 pixels, Kpad channels)
static int te_encode_input(CUtensorMap* map, const TeShape& s, const float* x) {
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(s.pixels), static_cast<cuuint64_t>(s.K), static_cast<cuuint64_t>(s.frames),
                          static_cast<cuuint64_t>(s.batch)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(s.sc) * 4, static_cast<cuuint64_t>(s.st) * 4, static_cast<cuuint64_t>(s.sb) * 4};
    cuuint32_t box[4] = {32, static_cast<cuuint32_t>(s.Kpad), 1, 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "temporal entry input");
}

static int te_encode_grads(TeGradMaps* maps, const TeShape& s, const float* const* gy) {
    for (int q = 0; q < s.n_seg; ++q) {
        const cuuint64_t C = static_cast<cuuint64_t>(s.seg_ch[q]), P = static_cast<cuuint64_t>(s.pixels), S = static_cast<cuuint64_t>(s.frames);
        cuuint64_t dims[4] = {P, S, C, static_cast<cuuint64_t>(s.batch)};
        cuuint64_t strides[3] = {P * 4, S * P * 4, C * S * P * 4};
        const int box_rows = q + 1 < s.n_seg ? round_up(s.seg_ch[q], 8) : s.Npad32 - s.seg_off[q];
        cuuint32_t box[4] = {32, 1, static_cast<cuuint32_t>(box_rows), 1};
        const int rc = encode_tensor_map(&maps->gy[q], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, gy[q], dims, strides, box, nullptr,
                                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "temporal entry output gradient");
        if (rc != FIERY_OK) return rc;
    }
    return FIERY_OK;
}

static int te_encode_pack(CUtensorMap* map, const float* base, int cols, int rows, const char* what) {
    cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), 1};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(cols) * 4, static_cast<cuuint64_t>(cols) * rows * 4};
    cuuint32_t box[3] = {32, static_cast<cuuint32_t>(rows), 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, what);
}

static int te_stages(int fixed_bytes, int stage_bytes) {
    const int n = (TE_SMEM_MAX - TE_SMEM_SLACK - fixed_bytes) / stage_bytes;
    return n < 4 ? n : 4;
}

constexpr int TE_COEF_BYTES = 128 * sizeof(BnCoef);  // the BN instantiations' static shared memory

// coef: nullptr (the entry's forward) or the Bottleneck's BN + ReLU prologue coefficients (K entries); coef with extra: the output
// head's forward (extra the ones that carry the bias)
static int te_launch_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* packed,
                             float* const* out, const BnCoef* coef, cudaStream_t stream) {
    const TeShape s = te_shape(d);
    const TePack p = te_pack_layout(s);
    TeFwdMaps maps;
    int rc = te_encode_pack(&maps.w, packed, p.k32, p.nch * 64, "temporal entry forward weights");
    if (rc == FIERY_OK) rc = te_encode_input(&maps.x, s, x);
    if (rc != FIERY_OK) return rc;
    TeOut o{};
    for (int q = 0; q < s.n_seg; ++q) o.p[q] = out[q];
    const int fixed = static_cast<int>(p.f_floats * 4) + 2 * TE_STG_FLOATS * 4 + TE_ROW_TABLE_BYTES;
    const int stages = te_stages(fixed + (coef ? TE_COEF_BYTES : 0), 4 * s.Kpad * 128);
    const int smem = fixed + stages * 4 * s.Kpad * 128 + TE_SMEM_SLACK;
    const int tiles_per_frame = (s.pixels + TE_FWD_PX - 1) / TE_FWD_PX;
    const long long n_tiles = static_cast<long long>(s.batch) * s.frames * tiles_per_frame;
    FIERY_REQUIRE(n_tiles < (1ll << 31), "temporal entry: too many pixel tiles");
    unsigned grid = 0;
    if ((rc = persistent_grid(n_tiles, &grid)) != FIERY_OK) return rc;
    const float* we = packed + p.f_floats + p.t_floats;
    if (coef && extra) {
        FIERY_REQUIRE(s.E == 1 && p.nch == 1 && s.Kpad <= 128, "output head: one extra channel, n <= 8 outputs and C <= 128");
        if ((rc = set_dynamic_smem(output_head_fwd_kernel, smem)) != FIERY_OK) return rc;
        output_head_fwd_kernel<<<grid, TE_FWD_THREADS, smem, stream>>>(maps, s, extra, we, o, stages, tiles_per_frame,
                                                                       static_cast<int>(n_tiles), coef);
        FIERY_CUDA_CHECK(cudaGetLastError());
        return FIERY_OK;
    }
    if (coef) {
        FIERY_REQUIRE(s.E == 0 && s.Kpad <= 128, "bottleneck: the up projection takes no extra channels and K <= 128");
        switch (p.nch) {
#define TE_BN_FWD_CASE(N)                                                                                                           \
    case N:                                                                                                                         \
        if ((rc = set_dynamic_smem(bottleneck_entry_fwd_kernel<N>, smem)) != FIERY_OK) return rc;                                   \
        bottleneck_entry_fwd_kernel<N><<<grid, TE_FWD_THREADS, smem, stream>>>(maps, s, o, stages, tiles_per_frame,                 \
                                                                               static_cast<int>(n_tiles), coef);                    \
        break;
            TE_BN_FWD_CASE(1) TE_BN_FWD_CASE(2)
#undef TE_BN_FWD_CASE
            default: return set_error(FIERY_E_INVALID, "bottleneck: up projection N_out padded to %d rows", s.Npad);
        }
        FIERY_CUDA_CHECK(cudaGetLastError());
        return FIERY_OK;
    }
    switch (p.nch) {
#define TE_FWD_CASE(N)                                                                                                              \
    case N:                                                                                                                         \
        if ((rc = set_dynamic_smem(temporal_entry_fwd_kernel<N>, smem)) != FIERY_OK) return rc;                                     \
        temporal_entry_fwd_kernel<N><<<grid, TE_FWD_THREADS, smem, stream>>>(maps, s, extra, we, o, stages, tiles_per_frame,       \
                                                                             static_cast<int>(n_tiles));                           \
        break;
        TE_FWD_CASE(1) TE_FWD_CASE(2) TE_FWD_CASE(3) TE_FWD_CASE(4)
#undef TE_FWD_CASE
        default: return set_error(FIERY_E_INVALID, "temporal entry: N_out padded to %d rows", s.Npad);
    }
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_temporal_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* packed,
                                  float* const* out, cudaStream_t stream) {
    return te_launch_forward(d, x, extra, packed, out, nullptr, stream);
}

int launch_bottleneck_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* packed, const BnCoef* coef, float* out,
                                    cudaStream_t stream) {
    return te_launch_forward(d, x, nullptr, packed, &out, coef, stream);
}

// ones: batch * frames floats of value 1, the extra channel that carries the bias
int launch_output_head_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* ones, const float* packed,
                                     const BnCoef* coef, float* out, cudaStream_t stream) {
    return te_launch_forward(d, x, ones, packed, &out, coef, stream);
}

// bias: nullptr (the entry's input gradient) or (batch * frames, K) fp32 added to every pixel of its frame's row k (the temporal
// aggregation's forward); res: nullptr or a tensor laid out as gx, added to it (the Bottleneck's input gradient plus its skip)
static int te_launch_dgrad(const fiery_temporal_entry_desc_t* d, const float* const* gy, const float* packed, const float* bias,
                           const float* res, float* gx, cudaStream_t stream) {
    const TeShape s = te_shape(d);
    const TePack p = te_pack_layout(s);
    TeDgradMaps maps;
    int rc = te_encode_pack(&maps.w, packed + p.f_floats, p.npad32, p.nchk * 64, "temporal entry transposed weights");
    if (rc == FIERY_OK) rc = te_encode_grads(&maps.g, s, gy);
    if (rc != FIERY_OK) return rc;
    const int rows = round_up(s.Npad, 64);
    const int fixed = static_cast<int>(p.t_floats * 4) + TE_STG_FLOATS * 4;
    const int stages = te_stages(fixed, 2 * rows * 128);
    const int smem = fixed + stages * 2 * rows * 128 + TE_SMEM_SLACK;
    const int tiles_per_frame = (s.pixels + TE_BWD_PX - 1) / TE_BWD_PX;
    const long long n_tiles = te_bwd_tiles(s.batch * s.frames, s.pixels);
    FIERY_REQUIRE(n_tiles < (1ll << 31), "temporal entry: too many pixel tiles");
    unsigned grid = 0;
    if ((rc = persistent_grid(n_tiles, &grid)) != FIERY_OK) return rc;
    const int nt = static_cast<int>(n_tiles);
    if (res != nullptr) {
        if (p.nchk == 1) {
            if ((rc = set_dynamic_smem(bottleneck_entry_dgrad_kernel<1>, smem)) != FIERY_OK) return rc;
            bottleneck_entry_dgrad_kernel<1><<<grid, TE_DG_THREADS, smem, stream>>>(maps, s, gx, res, stages, tiles_per_frame, nt);
        } else {
            if ((rc = set_dynamic_smem(bottleneck_entry_dgrad_kernel<2>, smem)) != FIERY_OK) return rc;
            bottleneck_entry_dgrad_kernel<2><<<grid, TE_DG_THREADS, smem, stream>>>(maps, s, gx, res, stages, tiles_per_frame, nt);
        }
    } else if (p.nchk == 1 && bias == nullptr) {
        if ((rc = set_dynamic_smem(temporal_entry_dgrad_kernel<1>, smem)) != FIERY_OK) return rc;
        temporal_entry_dgrad_kernel<1><<<grid, TE_DG_THREADS, smem, stream>>>(maps, s, gx, stages, tiles_per_frame, nt);
    } else if (bias == nullptr) {
        if ((rc = set_dynamic_smem(temporal_entry_dgrad_kernel<2>, smem)) != FIERY_OK) return rc;
        temporal_entry_dgrad_kernel<2><<<grid, TE_DG_THREADS, smem, stream>>>(maps, s, gx, stages, tiles_per_frame, nt);
    } else if (p.nchk == 1) {
        if ((rc = set_dynamic_smem(temporal_aggregation_kernel<1>, smem)) != FIERY_OK) return rc;
        temporal_aggregation_kernel<1><<<grid, TE_DG_THREADS, smem, stream>>>(maps, s, gx, bias, stages, tiles_per_frame, nt);
    } else {
        if ((rc = set_dynamic_smem(temporal_aggregation_kernel<2>, smem)) != FIERY_OK) return rc;
        temporal_aggregation_kernel<2><<<grid, TE_DG_THREADS, smem, stream>>>(maps, s, gx, bias, stages, tiles_per_frame, nt);
    }
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_temporal_entry_dgrad(const fiery_temporal_entry_desc_t* d, const float* const* gy, const float* packed, const float* bias,
                                float* gx, cudaStream_t stream) {
    return te_launch_dgrad(d, gy, packed, bias, nullptr, gx, stream);
}

int launch_bottleneck_entry_dgrad(const fiery_temporal_entry_desc_t* d, const float* gy, const float* packed, const float* res, float* gx,
                                  cudaStream_t stream) {
    return te_launch_dgrad(d, &gy, packed, nullptr, res, gx, stream);
}

// coef: nullptr (the entry's weight gradient) or the Bottleneck's BN + ReLU prologue coefficients of x (K entries)
static int te_launch_wgrad(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* const* gy,
                           const BnCoef* coef, float* gw, void* workspace, cudaStream_t stream) {
    const TeShape s = te_shape(d);
    const int n_frames = s.batch * s.frames;
    const int n_chunks = te_wgrad_chunks(n_frames, s.pixels);
    float* partial = static_cast<float*>(workspace);
    if (n_chunks > 0) {
        TeWgradMaps maps;
        int rc = te_encode_input(&maps.x, s, x);
        if (rc == FIERY_OK) rc = te_encode_grads(&maps.g, s, gy);
        if (rc != FIERY_OK) return rc;
        const int rows = round_up(s.Npad, 64), nc = round_up(s.K + s.E, 64) / 64;
        const int stage_bytes = 2 * (rows + 64 * nc) * 128;
        const int stages = te_stages(64 + (coef ? TE_COEF_BYTES : 0), stage_bytes);
        const int smem = stages * stage_bytes + TE_SMEM_SLACK;
        const int tiles_per_frame = (s.pixels + TE_BWD_PX - 1) / TE_BWD_PX;
        FIERY_REQUIRE(te_bwd_tiles(n_frames, s.pixels) < (1ll << 31), "temporal entry: too many pixel tiles");
        const int n_tiles = static_cast<int>(te_bwd_tiles(n_frames, s.pixels));
        const unsigned threads = static_cast<unsigned>(2 * rows);          // one warpgroup per 64 output rows
        if (coef) {
            FIERY_REQUIRE(nc == 1 && s.E == 0, "bottleneck: the up projection's weight gradient takes K <= 64 and no extra channels");
            if ((rc = set_dynamic_smem(bottleneck_entry_wgrad_kernel<1>, smem)) != FIERY_OK) return rc;
            bottleneck_entry_wgrad_kernel<1><<<n_chunks, threads, smem, stream>>>(maps, s, partial, stages, tiles_per_frame, n_tiles, coef);
            FIERY_CUDA_CHECK(cudaGetLastError());
            return launch_wgrad_reduce(partial, n_chunks, te_partial_floats(s), s.n_out * (s.K + s.E), TeWgradOffset{s}, gw, stream);
        }
        switch (nc) {
#define TE_WG_CASE(N)                                                                                                              \
    case N:                                                                                                                        \
        if ((rc = set_dynamic_smem(temporal_entry_wgrad_kernel<N>, smem)) != FIERY_OK) return rc;                                  \
        temporal_entry_wgrad_kernel<N><<<n_chunks, threads, smem, stream>>>(maps, s, extra, partial, stages, tiles_per_frame, n_tiles); \
        break;
            TE_WG_CASE(1) TE_WG_CASE(2) TE_WG_CASE(3)
#undef TE_WG_CASE
            default: return set_error(FIERY_E_INVALID, "temporal entry: K + E = %d", s.K + s.E);
        }
        FIERY_CUDA_CHECK(cudaGetLastError());
    }
    return launch_wgrad_reduce(partial, n_chunks, te_partial_floats(s), s.n_out * (s.K + s.E), TeWgradOffset{s}, gw, stream);
}

int launch_temporal_entry_wgrad(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* const* gy,
                                float* gw, void* workspace, cudaStream_t stream) {
    return te_launch_wgrad(d, x, extra, gy, nullptr, gw, workspace, stream);
}

int launch_bottleneck_entry_wgrad(const fiery_temporal_entry_desc_t* d, const float* x, const BnCoef* coef, const float* gy, float* gw,
                                  void* workspace, cudaStream_t stream) {
    return te_launch_wgrad(d, x, nullptr, &gy, coef, gw, workspace, stream);
}

}  // namespace fiery
