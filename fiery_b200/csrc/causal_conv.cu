// The temporal model's causal convolutions (CausalConv3d, fiery/layers/temporal.py:65-85): a zero pad of (kt - 1) frames in front and
// one pixel around the map, then a bias-free Conv3d with kernel (kt, 3, 3), kt in {1, 2}, on a contiguous fp32 (b, C, s, X, Y) tensor:
//
//   y[o, t, p]  = sum_{tau, dy, dx, i} W[o, i, tau, dy, dx] * x[i, t + tau - (kt - 1), p + (dy - 1, dx - 1)]
//   gx[i, t, p] = sum_{tau, dy, dx, o} W[o, i, tau, dy, dx] * gy[o, t + (kt - 1) - tau, p - (dy - 1, dx - 1)]
//   gW[o, i, tau, dy, dx] = sum_{b, t, p} gy[o, t, p] * x[i, t + tau - (kt - 1), p + (dy - 1, dx - 1)]
//
// All three run on the tensor cores: wgmma, TF32 operands, fp32 accumulation.  Weights are rounded to TF32 (cvt.rna) when packed, and
// every register A operand (the forward's x, the input gradient's gy, the weight gradient's x) is rounded the same way as it is read
// out of shared memory: nearest rounding halves the error of the tensor core's own truncation, which the weight gradient's
// shared-memory gy operand still gets.  No padded copy of the input exists:
// every load is a TMA box at shifted coordinates, and the TMA's zero fill for coordinates outside the tensor is the padding -- the
// spatial ring, frame -1 in the forward and frame s in the input gradient.
//
// Forward and input gradient: one kernel.  The input gradient is the forward's convolution on gy with the weights transposed in
// (o, i), the spatial taps mirrored and the time taps reading forward (frames t .. t + kt - 1) instead of back, so the two differ only
// in the pack they read and a frame offset.  One CTA per output tile of 8 rows x 16 columns (128 pixels, two consumer warpgroups of
// 4 x 16 pixels).  The producer warp loads the kt halo tiles (Kpad channels x 10 x 28 pixels, no swizzle) once and streams the 9 kt
// taps' weight slices (N x Kpad, K-major, 128-byte swizzle) through a ring.  Each tap's MMAs read the pixel tile out of the halo tile
// at the tap's shift as the register A operand: the halo's 28-column rows make a channel plane 280 floats = 24 banks apart, so the
// 4 channels x 8 consecutive pixels of a fragment load hit 32 different banks.  N = the output channels rounded up to 8
// (wgmma_tf32_rs<N>, wgmma.cuh).  Each accumulator row of a warp is 8 consecutive pixels of one map row, so the fragments are stored
// straight to the (b, C, s, X, Y) output: every warp store fills whole 32-byte sectors.
//
// Weight gradient: D (input channels, one m64 block) x (output channels rounded up to 8) = sum over pixels of x_tap gy^T.  Tiles are
// 32-pixel runs of one map row; CTA (chunk, (tau, dy)) owns the three taps dx = 0, 1, 2.  The gy run is the K-major shared-memory B
// operand; the x run of the tap's frame and row is loaded once, 4 columns early and 44 wide, and read as the register A operand at
// each dx's shift (im2col from shared memory; 44-float rows put a fragment's 8 channels x 4 pixels on 32 banks).  The summation order
// is wgrad_chunks.cuh's: bit-reproducible, no atomics.
//
// Both kernels are written over halo tiles and segments (causal_conv.cuh), so the spatial GRU (spatial_gru.cu) runs its 3x3
// convolutions on them too: its inputs [x_t, h] are two halo tiles from two tensors, its outputs up to two segments of the accumulator
// with their own epilogues.  A causal convolution is one map read at kt frame offsets and one stored segment.
#include "bn_coef.cuh"
#include "causal_conv.cuh"
#include "wgmma.cuh"
#include "wgrad_chunks.cuh"

namespace fiery {

constexpr int CC_HY_OFF = 3;                       // halo column of input column y0 + c + dx - 1 is c + dx + CC_HY_OFF
constexpr int CC_FWD_THREADS = 2 * 128 + 32;
constexpr int CC_WG_STAGES = 4;
constexpr int CC_WG_X_BYTES = 64 * CC_WG_XP * 4;   // 64 input-channel rows (zero past C_in): 11 KB, a multiple of 1024

static CcShape cc_shape(const fiery_causal_conv3d_desc_t* d) {
    return CcShape{d->batch, d->frames, d->grid_x, d->grid_y, d->in_channels, d->out_channels, d->kt, 9 * d->kt};
}

// One direction's pack: (taps, ka, n, 32) floats -- tap j's B operand is ka 128-byte-swizzle atoms of n K-major rows x 32 k.
struct CcPackDir {
    int n, kpad, ka;
    size_t floats;
};
static CcPackDir cc_pack_dir(int n_channels, int k_channels, int taps) {
    CcPackDir p;
    p.n = cc_round8(n_channels);
    p.kpad = cc_round8(k_channels);
    p.ka = (p.kpad + 31) / 32;
    p.floats = static_cast<size_t>(taps) * p.ka * p.n * 32;
    return p;
}

// the forward pack F (rows o, k = i), then the input gradient's T (rows i, k = o; time taps reversed, spatial taps mirrored)
size_t causal_conv_packed_bytes(const fiery_causal_conv3d_desc_t* d) {
    const CcShape s = cc_shape(d);
    return (cc_pack_dir(s.cout, s.cin, s.taps).floats + cc_pack_dir(s.cin, s.cout, s.taps).floats) * sizeof(float);
}

__global__ void causal_conv_pack_kernel(CcShape s, CcPackDir f, CcPackDir t, const float* __restrict__ w, float* __restrict__ packed) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool fwd = i < f.floats;
    if (!fwd && i >= f.floats + t.floats) return;
    const CcPackDir& p = fwd ? f : t;
    const size_t j = fwd ? i : i - f.floats;
    const int k = static_cast<int>(j % 32), n = static_cast<int>(j / 32 % p.n), a = static_cast<int>(j / 32 / p.n % p.ka);
    const int tap = static_cast<int>(j / 32 / p.n / p.ka);
    const int c = 32 * a + k;
    const int jt = tap / 9, ay = tap / 3 % 3, ax = tap % 3;
    float v = 0.f;
    if (fwd) {
        if (n < s.cout && c < s.cin) v = __uint_as_float(to_tf32(w[((static_cast<size_t>(n) * s.cin + c) * s.kt + jt) * 9 + ay * 3 + ax]));
    } else if (n < s.cin && c < s.cout) {
        v = __uint_as_float(to_tf32(w[((static_cast<size_t>(c) * s.cin + n) * s.kt + (s.kt - 1 - jt)) * 9 + (2 - ay) * 3 + (2 - ax)]));
    }
    packed[i] = v;
}

int launch_causal_conv_pack(const fiery_causal_conv3d_desc_t* d, const float* w, float* packed, cudaStream_t stream) {
    const CcShape s = cc_shape(d);
    const CcPackDir f = cc_pack_dir(s.cout, s.cin, s.taps), t = cc_pack_dir(s.cin, s.cout, s.taps);
    const size_t n = f.floats + t.floats;
    causal_conv_pack_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(s, f, t, w, packed);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// forward and input gradient
// ------------------------------------------------------------------------------------------------------------------------------
// one accumulator value of output segment o, channel ch, at (b, t, pixel pix)
__device__ __forceinline__ void cc_epilogue(const CcOutSeg& o, float bias_init, size_t plane, int b, int ch, int t, size_t pix, float v) {
    const size_t cp = static_cast<size_t>(ch) * plane + pix;
    float* dst = o.p + b * o.sb + ch * o.sc + t * o.st + pix;
    switch (o.mode) {
        case CC_STORE: *dst = v; break;
        case CC_ADD: *dst += v; break;
        case CC_GATE_U: *dst = 1.f / (1.f + expf(-(v + o.bias[ch] + bias_init))); break;
        case CC_GATE_R: {
            const float r = 1.f / (1.f + expf(-(v + o.bias[ch] + bias_init)));
            o.r[b * o.rsb + cp] = r;
            *dst = (1.f - r) * o.h[b * o.hsb + cp];
            break;
        }
        case CC_RESET_GRAD: {
            const float r = o.r[b * o.rsb + cp], h = o.h[b * o.hsb + cp];
            o.aux[b * o.asb + cp] = -v * h * (r * (1.f - r));
            *dst += (1.f - r) * v;
            break;
        }
        default: break;
    }
}

// SEG = false: the causal convolution -- kt halo tiles of map 0 with one channel count, a CC_WSTAGES ring, one stored segment; every
// per-halo quantity is the uniform one, so its instantiations compile to the single-input kernel.  SEG = true: the per-halo maps,
// channel counts and ring depth of CcFwdLaunch, and the segment epilogues.  BN (with SEG = false, one halo): the Bottleneck's 3x3
// convolution -- once the halo tile has landed, each of its values of channel c < cin at a map position becomes
// bn_relu_apply(coef[c], v) in shared memory; the zero fill outside the map (the padding of the normalized map) stays 0.
template <int N, bool SEG, bool BN>
__device__ __forceinline__ void cc_fwd_body(const CcFwdMaps& maps, const CcFwdLaunch& L, const BnCoef* __restrict__ coef, int cin) {
    const int taps = 9 * L.halos;
    const int stages = SEG ? L.stages : CC_WSTAGES;
    const int w_bytes = SEG ? L.stage_bytes : L.ka[0] * N * 128;
    const int x_floats = L.kpad[0] * CC_PLANE;                    // SEG = false: every halo tile
    auto kpad_of = [&](int h) { return SEG ? L.kpad[h] : L.kpad[0]; };
    auto ka_of = [&](int h) { return SEG ? L.ka[h] : L.ka[0]; };
    auto x_off_of = [&](int h) { return SEG ? L.x_off[h] : h * x_floats; };
    unsigned char* s_w = dynamic_smem_1024();
    const float* s_x = reinterpret_cast<const float*>(s_w + stages * w_bytes);
    uint64_t* x_full = reinterpret_cast<uint64_t*>(const_cast<float*>(s_x) + x_off_of(L.halos - 1) + kpad_of(L.halos - 1) * CC_PLANE);
    const MbarRing ring(x_full + 1, stages);

    int tile = blockIdx.x;
    const int ty = tile % L.tiles_y;
    tile /= L.tiles_y;
    const int tx = tile % L.tiles_x;
    const int f = tile / L.tiles_x, b = f / L.frames, t = f % L.frames;
    const int x0 = tx * CC_TX, y0 = ty * CC_TY;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&maps.x[0]);
        if (SEG && L.halos > 1 && L.map[1] != 0) tma_prefetch_desc(&maps.x[1]);
        tma_prefetch_desc(&maps.w);
        mbar_init(x_full, 1);                          // published to the async proxy by the fence in ring.init
        ring.init(8);
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {                               // ===== TMA producer: the halo tiles, then the taps' weight slices =====
            int x_bytes = 0;
            for (int h = 0; h < L.halos; ++h) x_bytes += kpad_of(h) * CC_PLANE * 4;
            mbar_arrive_expect_tx(x_full, x_bytes);
            for (int h = 0; h < L.halos; ++h)
                tma_load_5d(const_cast<float*>(s_x) + x_off_of(h), &maps.x[SEG ? L.map[h] : 0], x_full, y0 - 4, x0 - 1, t + L.t_off[h], 0,
                            b);
            for (int j = 0; j < taps; ++j) {
                const int h = j / 9, ka = ka_of(h);
                const int st = ring.produce(j, ka * N * 128);
                const int atom = SEG ? L.atom0[h] + (j % 9) * ka : j * ka;
                for (int a = 0; a < ka; ++a) tma_load_3d(s_w + st * w_bytes + a * N * 128, &maps.w, ring.full + st, 0, 0, atom + a);
            }
        }
        return;
    }

    // ===== consumers: warp w of warpgroup g owns tile row 4g + w; accumulator rows 16w + lane/4 (+ 8) = columns lane/4 (+ 8) =====
    const int row = 4 * (warp >> 2) + (warp & 3);
    const int col = lane >> 2, kq = lane & 3;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    mbar_wait(x_full, 0);
    if constexpr (BN) {                                // the halo tile is read by generic loads only: a barrier suffices
        float* hx = const_cast<float*>(s_x);
        for (int idx = threadIdx.x; idx < cin * CC_PLANE; idx += 256) {
            const int c = idx / CC_PLANE, r = idx % CC_PLANE;
            const int gx = x0 - 1 + r / CC_HY, gy = y0 - 4 + r % CC_HY;
            if (gx >= 0 && gx < L.X && gy >= 0 && gy < L.Y) hx[idx] = bn_relu_apply(coef[c], hx[idx]);
        }
        named_barrier(1, 256);
    }
#pragma unroll 1
    for (int j = 0; j < taps; ++j) {
        const int jt = j / 9, ay = j / 3 % 3, ax = j % 3;
        const int nks = kpad_of(jt) / 8, ka = ka_of(jt);
        const float* h = s_x + x_off_of(jt) + (row + ay) * CC_HY + col + ax + CC_HY_OFF + kq * CC_PLANE;
        const uint32_t wb = smem_addr(s_w + ring.consume(j) * w_bytes);
#pragma unroll 1
        for (int a = 0; a < ka; ++a) {                 // 32 channels (4 k-steps) at a time
            uint32_t fr[4][4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float* hk = h + (32 * a + 8 * k) * CC_PLANE;
                const bool on = 4 * a + k < nks;
                fr[k][0] = on ? to_tf32(hk[0]) : 0u;
                fr[k][1] = on ? to_tf32(hk[8]) : 0u;
                fr[k][2] = on ? to_tf32(hk[4 * CC_PLANE]) : 0u;
                fr[k][3] = on ? to_tf32(hk[4 * CC_PLANE + 8]) : 0u;
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (4 * a + k < nks) wgmma_tf32_rs<N>(acc, fr[k], gmma_desc_sw128(wb + a * N * 128 + k * 32, 16, 1024));
            wgmma_commit();
            wgmma_wait<0>();
        }
        wgmma_fence_operands(acc);
        ring.release(j);                               // this warp is done with the slice
    }

    const int gx = x0 + row;
    if (gx >= L.X) return;
    const size_t plane = static_cast<size_t>(L.X) * L.Y;
    if constexpr (!SEG) {
        const CcOutSeg& o = L.seg[0];
#pragma unroll
        for (int jn = 0; jn < N / 8; ++jn)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = 8 * jn + 2 * kq + e;
                if (c >= o.n) continue;
                float* dst = o.p + b * o.sb + c * o.sc + t * o.st + static_cast<size_t>(gx) * L.Y + y0 + col;
                if (y0 + col < L.Y) dst[0] = acc[4 * jn + e];
                if (y0 + col + 8 < L.Y) dst[8] = acc[4 * jn + 2 + e];
            }
    } else {
        const size_t pix = static_cast<size_t>(gx) * L.Y + y0 + col;
#pragma unroll
        for (int jn = 0; jn < N / 8; ++jn)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = 8 * jn + 2 * kq + e;
                for (int sg = 0; sg < L.nseg; ++sg) {
                    const CcOutSeg& o = L.seg[sg];
                    const int ch = c - o.c0;
                    if (ch < 0 || ch >= o.n) continue;
                    if (y0 + col < L.Y) cc_epilogue(o, L.bias_init, plane, b, ch, t, pix, acc[4 * jn + e]);
                    if (y0 + col + 8 < L.Y) cc_epilogue(o, L.bias_init, plane, b, ch, t, pix + 8, acc[4 * jn + 2 + e]);
                }
            }
    }
}

template <int N, bool SEG>
__global__ void __launch_bounds__(CC_FWD_THREADS, 1)
causal_conv_fwd_kernel(const __grid_constant__ CcFwdMaps maps, const __grid_constant__ CcFwdLaunch L) {
    cc_fwd_body<N, SEG, false>(maps, L, nullptr, 0);
}

template <int N>
__global__ void __launch_bounds__(CC_FWD_THREADS, 1)
bottleneck_conv_fwd_kernel(const __grid_constant__ CcFwdMaps maps, const __grid_constant__ CcFwdLaunch L, const BnCoef* __restrict__ coef,
                           int cin) {
    cc_fwd_body<N, false, true>(maps, L, coef, cin);
}

int cc_launch_fwd(int N, bool segments, const CcFwdMaps& maps, const CcFwdLaunch& L, long long n_tiles, cudaStream_t stream) {
    FIERY_REQUIRE(n_tiles < (1ll << 31), "3x3 conv: too many pixel tiles");
    if (n_tiles == 0) return FIERY_OK;
    const int smem = cc_fwd_smem(L);
    FIERY_REQUIRE(smem <= CC_MAX_SMEM, "3x3 conv: %d bytes of shared memory", smem);
    FIERY_REQUIRE(segments || (N <= 64 && L.stages == CC_WSTAGES), "3x3 conv: the single-input kernel takes N <= 64");
    int rc;
    switch (N) {
#define CC_FWD_CASE(NN)                                                                                                            \
    case NN:                                                                                                                       \
        if (segments) {                                                                                                            \
            if ((rc = set_dynamic_smem(causal_conv_fwd_kernel<NN, true>, smem)) != FIERY_OK) return rc;                            \
            causal_conv_fwd_kernel<NN, true><<<static_cast<unsigned>(n_tiles), CC_FWD_THREADS, smem, stream>>>(maps, L);           \
        } else {                                                                                                                   \
            if ((rc = set_dynamic_smem(causal_conv_fwd_kernel<NN, false>, smem)) != FIERY_OK) return rc;                           \
            causal_conv_fwd_kernel<NN, false><<<static_cast<unsigned>(n_tiles), CC_FWD_THREADS, smem, stream>>>(maps, L);          \
        }                                                                                                                          \
        break;
        CC_FWD_CASE(8) CC_FWD_CASE(16) CC_FWD_CASE(24) CC_FWD_CASE(32) CC_FWD_CASE(40) CC_FWD_CASE(48) CC_FWD_CASE(56) CC_FWD_CASE(64)
#undef CC_FWD_CASE
        case 96:
            if ((rc = set_dynamic_smem(causal_conv_fwd_kernel<96, true>, smem)) != FIERY_OK) return rc;
            causal_conv_fwd_kernel<96, true><<<static_cast<unsigned>(n_tiles), CC_FWD_THREADS, smem, stream>>>(maps, L);
            break;
        case 128:
            if ((rc = set_dynamic_smem(causal_conv_fwd_kernel<128, true>, smem)) != FIERY_OK) return rc;
            causal_conv_fwd_kernel<128, true><<<static_cast<unsigned>(n_tiles), CC_FWD_THREADS, smem, stream>>>(maps, L);
            break;
        default: return set_error(FIERY_E_INVALID, "3x3 conv: %d accumulator columns", N);
    }
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// weight gradient
// ------------------------------------------------------------------------------------------------------------------------------
long long cc_wgrad_tiles(const CcShape& s) {
    return static_cast<long long>(s.batch) * s.frames * s.X * ((s.Y + CC_WG_PX - 1) / CC_WG_PX);
}
static size_t cc_partial_floats(const CcShape& s) { return static_cast<size_t>(s.taps) * s.cout * s.cin; }

size_t causal_conv_wgrad_workspace_bytes(const fiery_causal_conv3d_desc_t* d) {
    const CcShape s = cc_shape(d);
    return static_cast<size_t>(wgrad_chunks(cc_wgrad_tiles(s), WG_MAX_CHUNKS)) * cc_partial_floats(s) * sizeof(float);
}

// grid (chunks, 3 kt): CTA (chunk, tau * 3 + dy) accumulates the taps (tau, dy, 0..2) over its chunk's tiles as D (input channels x
// NO output channels) = x_tap gy^T.  Per tile the stage holds the x row run of frame t * fmul + foff + tau - (kt - 1), row x + dy - 1
// (64 channel rows of 44 columns, read as the register A operand at column offset dx + 3) and the gy run (NO K-major rows of 32 pixels
// from channel o0, the B operand).  Thread 0 issues the loads: at iteration i, after the barrier that ends the MMAs on tile i - 1, tile
// i + stages - 1 into that tile's stage.  BN (kt = 1): the Bottleneck's 3x3 convolution -- once a tile's x run has landed, each of
// its values of channel c < cin at a map position becomes bn_relu_apply(coef[c], v) in shared memory; the zero fill outside the map
// (the padding of the normalized map) stays 0.
template <int NO, bool BN>
__device__ __forceinline__ void cc_wgrad_body(const CcWgradMaps& maps, const CcShape& s, const CcWgradSeg& seg, float* __restrict__ partial,
                                              int n_tiles, const BnCoef* __restrict__ coef) {
    unsigned char* smem = dynamic_smem_1024();
    constexpr int STAGE_BYTES = CC_WG_X_BYTES + NO * 128;
    const MbarRing ring(reinterpret_cast<uint64_t*>(smem + CC_WG_STAGES * STAGE_BYTES), CC_WG_STAGES);
    const int tau = blockIdx.y / 3, dy = blockIdx.y % 3;
    const int t0 = static_cast<int>(static_cast<long long>(blockIdx.x) * n_tiles / gridDim.x);
    const int t1 = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * n_tiles / gridDim.x);
    const int runs = (s.Y + CC_WG_PX - 1) / CC_WG_PX;

    auto load = [&](int i) {                       // tile t0 + i = ((b * s + t) * X + x) * runs + run, into stage i % stages
        int t = t0 + i;
        const int run = t % runs;
        t /= runs;
        const int x = t % s.X, f = t / s.X, b = f / s.frames, tt = f % s.frames;
        const int st = ring.arm(i, STAGE_BYTES);
        unsigned char* dst = smem + st * STAGE_BYTES;
        uint64_t* bar = ring.full + st;
        const int fx = tt * seg.fmul + seg.foff + tau - (s.kt - 1);
        if (seg.first && fx < 0) tma_load_5d(dst, &maps.x_first, bar, CC_WG_PX * run - 4, x + dy - 1, 0, 0, b);
        else tma_load_5d(dst, &maps.x, bar, CC_WG_PX * run - 4, x + dy - 1, fx, 0, b);
        tma_load_5d(dst + CC_WG_X_BYTES, &maps.gy, bar, CC_WG_PX * run, x, tt, seg.o0, b);
    };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&maps.gy);
        tma_prefetch_desc(&maps.x);
        ring.init(0);
        for (int i = 0; i < CC_WG_STAGES - 1 && t0 + i < t1; ++i) load(i);
    }
    __syncthreads();

    const int w4 = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ra = 16 * w4 + (lane >> 2), kq = lane & 3;   // A fragment: channel rows ra, ra + 8; pixel columns kq, kq + 4
    float acc[3][NO / 2];
#pragma unroll
    for (int dx = 0; dx < 3; ++dx)
#pragma unroll
        for (int i = 0; i < NO / 2; ++i) acc[dx][i] = 0.f;

    for (int i = 0; t0 + i < t1; ++i) {
        __syncthreads();                           // every warp is done with tile i - 1: its stage may be refilled
        if (threadIdx.x == 0 && t0 + i + CC_WG_STAGES - 1 < t1) load(i + CC_WG_STAGES - 1);
        const int st = ring.consume(i);
        if constexpr (BN) {                        // generic writes the TMA later overwrites: fence, then barrier
            float* xr = reinterpret_cast<float*>(smem + st * STAGE_BYTES);
            const int t = t0 + i, run = t % runs, gx = (t / runs) % s.X + dy - 1;
            if (gx >= 0 && gx < s.X) {
                for (int idx = threadIdx.x; idx < seg.cin * CC_WG_XP; idx += 128) {
                    const int c = idx / CC_WG_XP, gy = CC_WG_PX * run - 4 + idx % CC_WG_XP;
                    if (gy >= 0 && gy < s.Y) xr[idx] = bn_relu_apply(coef[c], xr[idx]);
                }
            }
            fence_proxy_async();
            __syncthreads();
        }
        const float* xs = reinterpret_cast<const float*>(smem + st * STAGE_BYTES) + ra * CC_WG_XP + kq + 3;
        const uint32_t g_addr = smem_addr(smem + st * STAGE_BYTES + CC_WG_X_BYTES);
        uint32_t a[CC_WG_PX / 8][3][4];
#pragma unroll
        for (int ks = 0; ks < CC_WG_PX / 8; ++ks)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const float* p = xs + 8 * ks + dx;
                a[ks][dx][0] = to_tf32(p[0]);
                a[ks][dx][1] = to_tf32(p[8 * CC_WG_XP]);
                a[ks][dx][2] = to_tf32(p[4]);
                a[ks][dx][3] = to_tf32(p[8 * CC_WG_XP + 4]);
            }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < CC_WG_PX / 8; ++ks) {
            const uint64_t db = gmma_desc_sw128(g_addr + 32 * ks, 16, 1024);
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) wgmma_tf32_rs<NO>(acc[dx], a[ks][dx], db);
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) wgmma_fence_operands(acc[dx]);
    }

    // this chunk's partial: accumulator (row = input channel ci, column = output channel o) of tap (tau, dy, dx) ->
    // partial[chunk][tap][o0 + o][ci0 + ci]
    const size_t n_oi = static_cast<size_t>(s.cout) * s.cin;
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
        float* dst = partial + (static_cast<size_t>(blockIdx.x) * s.taps + 9 * tau + 3 * dy + dx) * n_oi;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int ci = ra + 8 * half;
            if (ci >= seg.cin) continue;
#pragma unroll
            for (int jn = 0; jn < NO / 8; ++jn)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int o = 8 * jn + 2 * kq + e;
                    if (o < seg.n_o) dst[static_cast<size_t>(seg.o0 + o) * s.cin + seg.ci0 + ci] = acc[dx][4 * jn + 2 * half + e];
                }
        }
    }
}

template <int NO>
__global__ void __launch_bounds__(128, 1)
causal_conv_wgrad_kernel(const __grid_constant__ CcWgradMaps maps, const CcShape s, const CcWgradSeg seg, float* __restrict__ partial,
                         int n_tiles) {
    cc_wgrad_body<NO, false>(maps, s, seg, partial, n_tiles, nullptr);
}

template <int NO>
__global__ void __launch_bounds__(128, 1)
bottleneck_conv_wgrad_kernel(const __grid_constant__ CcWgradMaps maps, const CcShape s, const CcWgradSeg seg, float* __restrict__ partial,
                             int n_tiles, const BnCoef* __restrict__ coef) {
    cc_wgrad_body<NO, true>(maps, s, seg, partial, n_tiles, coef);
}

// grad_w (C_out, C_in, kt, 3, 3) index -> its place in a chunk's partial (tap, o, ci)
struct CcWgradOffset {
    CcShape s;
    __device__ size_t operator()(int i) const {
        const int tap = i % s.taps, oi = i / s.taps;     // oi = o * cin + ci
        return static_cast<size_t>(tap) * s.cout * s.cin + oi;
    }
};

int cc_launch_wgrad(const CcWgradMaps& maps, const CcShape& s, const CcWgradSeg& seg, float* partial, int n_chunks, cudaStream_t stream) {
    const long long tiles = cc_wgrad_tiles(s);
    FIERY_REQUIRE(tiles < (1ll << 31), "3x3 conv: too many pixel tiles");
    if (n_chunks == 0) return FIERY_OK;
    const int no = cc_round8(seg.n_o);
    const int smem = CC_WG_STAGES * (CC_WG_X_BYTES + no * 128) + CC_SMEM_SLACK;
    const dim3 grid(static_cast<unsigned>(n_chunks), static_cast<unsigned>(3 * s.kt));
    int rc;
    switch (no) {
#define CC_WG_CASE(N)                                                                                                              \
    case N:                                                                                                                        \
        if ((rc = set_dynamic_smem(causal_conv_wgrad_kernel<N>, smem)) != FIERY_OK) return rc;                                     \
        causal_conv_wgrad_kernel<N><<<grid, 128, smem, stream>>>(maps, s, seg, partial, static_cast<int>(tiles));                   \
        break;
        CC_WG_CASE(8) CC_WG_CASE(16) CC_WG_CASE(24) CC_WG_CASE(32) CC_WG_CASE(40) CC_WG_CASE(48) CC_WG_CASE(56) CC_WG_CASE(64)
#undef CC_WG_CASE
        default: return set_error(FIERY_E_INVALID, "3x3 conv: %d output channels in one weight-gradient block", seg.n_o);
    }
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int cc_wgrad_reduce(const CcShape& s, const float* partial, int n_chunks, float* gw, cudaStream_t stream) {
    return launch_wgrad_reduce(partial, n_chunks, cc_partial_floats(s), s.cout * s.cin * s.taps, CcWgradOffset{s}, gw, stream);
}

// ------------------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------------------
int cc_encode_map(CUtensorMap* map, const float* t, int Y, int X, int S, int C, int B, const long long (&strides)[4], cuuint32_t box_y,
                  cuuint32_t box_x, cuuint32_t box_c, CUtensorMapSwizzle swizzle, const char* what) {
    cuuint64_t dims[5] = {static_cast<cuuint64_t>(Y), static_cast<cuuint64_t>(X), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(C),
                          static_cast<cuuint64_t>(B)};
    cuuint64_t st[4];
    for (int i = 0; i < 4; ++i) st[i] = static_cast<cuuint64_t>(strides[i]) * 4;
    cuuint32_t box[5] = {box_y, box_x, 1, box_c, 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, t, dims, st, box, nullptr, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             what);
}

// a contiguous (b, C, s, X, Y) activation as the 5-D map (Y, X, s, C, b)
static int cc_encode_activation(CUtensorMap* map, const CcShape& s, const float* t, int channels, cuuint32_t box_y, cuuint32_t box_x,
                                cuuint32_t box_c, CUtensorMapSwizzle swizzle, const char* what) {
    const long long XY = static_cast<long long>(s.X) * s.Y;
    const long long strides[4] = {s.Y, XY, s.frames * XY, static_cast<long long>(channels) * s.frames * XY};
    return cc_encode_map(map, t, s.Y, s.X, s.frames, channels, s.batch, strides, box_y, box_x, box_c, swizzle, what);
}

// The Bottleneck's forward: bottleneck_conv_fwd_kernel<N>, N = the output channels rounded up to 8 (8 .. 64)
static int cc_launch_bn_fwd(int N, const CcFwdMaps& maps, const CcFwdLaunch& L, long long n_tiles, const BnCoef* coef, int cin,
                            cudaStream_t stream) {
    if (n_tiles == 0) return FIERY_OK;
    const int smem = cc_fwd_smem(L);
    FIERY_REQUIRE(smem <= CC_MAX_SMEM, "3x3 conv: %d bytes of shared memory", smem);
    int rc;
    switch (N) {
#define CC_BN_FWD_CASE(NN)                                                                                                         \
    case NN:                                                                                                                       \
        if ((rc = set_dynamic_smem(bottleneck_conv_fwd_kernel<NN>, smem)) != FIERY_OK) return rc;                                 \
        bottleneck_conv_fwd_kernel<NN><<<static_cast<unsigned>(n_tiles), CC_FWD_THREADS, smem, stream>>>(maps, L, coef, cin);      \
        break;
        CC_BN_FWD_CASE(8) CC_BN_FWD_CASE(16) CC_BN_FWD_CASE(24) CC_BN_FWD_CASE(32) CC_BN_FWD_CASE(40) CC_BN_FWD_CASE(48)
        CC_BN_FWD_CASE(56) CC_BN_FWD_CASE(64)
#undef CC_BN_FWD_CASE
        default: return set_error(FIERY_E_INVALID, "bottleneck: %d accumulator columns in the 3x3 conv", N);
    }
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// forward (dgrad = 0): x (C_in channels) -> y (C_out) with pack F; input gradient (dgrad = 1): gy (C_out) -> gx (C_in) with pack T.
// coef (forward, kt = 1 only): the Bottleneck's BN + ReLU prologue on x, or nullptr.
static int cc_launch_conv(const fiery_causal_conv3d_desc_t* d, int dgrad, const float* in, const float* packed, float* out,
                          cudaStream_t stream, const BnCoef* coef = nullptr) {
    const CcShape s = cc_shape(d);
    const CcPackDir f = cc_pack_dir(s.cout, s.cin, s.taps);
    const CcPackDir p = dgrad ? cc_pack_dir(s.cin, s.cout, s.taps) : f;
    const float* w = dgrad ? packed + f.floats : packed;
    CcFwdMaps maps;
    int rc = cc_encode_activation(&maps.x[0], s, in, dgrad ? s.cout : s.cin, CC_HY, CC_HX, static_cast<cuuint32_t>(p.kpad),
                                  CU_TENSOR_MAP_SWIZZLE_NONE, dgrad ? "causal conv output gradient" : "causal conv input");
    if (rc != FIERY_OK) return rc;
    {
        cuuint64_t dims[3] = {32, static_cast<cuuint64_t>(p.n), static_cast<cuuint64_t>(s.taps) * p.ka};
        cuuint64_t strides[2] = {128, static_cast<cuuint64_t>(p.n) * 128};
        cuuint32_t box[3] = {32, static_cast<cuuint32_t>(p.n), 1};
        if ((rc = encode_tensor_map(&maps.w, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, w, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "causal conv weights")) != FIERY_OK)
            return rc;
    }
    CcFwdLaunch L{};
    L.frames = s.frames;
    L.X = s.X;
    L.Y = s.Y;
    L.tiles_x = (s.X + CC_TX - 1) / CC_TX;
    L.tiles_y = (s.Y + CC_TY - 1) / CC_TY;
    L.halos = s.kt;                                // halo jt: frame t + jt - (kt - 1) (forward) or t + jt (input gradient)
    L.stages = CC_WSTAGES;
    L.stage_bytes = p.ka * p.n * 128;
    for (int jt = 0; jt < s.kt; ++jt) {
        L.map[jt] = 0;
        L.t_off[jt] = jt - (dgrad ? 0 : s.kt - 1);
        L.kpad[jt] = p.kpad;
        L.ka[jt] = p.ka;
        L.x_off[jt] = jt * p.kpad * CC_PLANE;
        L.atom0[jt] = jt * 9 * p.ka;
    }
    const int n_out = dgrad ? s.cin : s.cout;
    const long long plane = static_cast<long long>(s.X) * s.Y;
    L.nseg = 1;
    L.seg[0].p = out;
    L.seg[0].st = plane;
    L.seg[0].sc = s.frames * plane;
    L.seg[0].sb = n_out * L.seg[0].sc;
    L.seg[0].c0 = 0;
    L.seg[0].n = n_out;
    L.seg[0].mode = CC_STORE;
    const long long n_tiles = static_cast<long long>(s.batch) * s.frames * L.tiles_x * L.tiles_y;
    FIERY_REQUIRE(n_tiles < (1ll << 31), "causal conv: too many pixel tiles");
    if (p.n > 64) return set_error(FIERY_E_INVALID, "causal conv: %d channels padded to %d", n_out, p.n);
    if (coef) {
        FIERY_REQUIRE(!dgrad && s.kt == 1, "bottleneck: the BN prologue runs in the forward of a (1, 3, 3) conv only");
        return cc_launch_bn_fwd(p.n, maps, L, n_tiles, coef, s.cin, stream);
    }
    return cc_launch_fwd(p.n, false, maps, L, n_tiles, stream);
}

int launch_causal_conv_forward(const fiery_causal_conv3d_desc_t* d, const float* x, const float* packed, float* y, cudaStream_t stream) {
    return cc_launch_conv(d, 0, x, packed, y, stream);
}

int launch_causal_conv_dgrad(const fiery_causal_conv3d_desc_t* d, const float* gy, const float* packed, float* gx, cudaStream_t stream) {
    return cc_launch_conv(d, 1, gy, packed, gx, stream);
}

int launch_bottleneck_conv_forward(const fiery_causal_conv3d_desc_t* d, const float* x, const float* packed, const BnCoef* coef, float* y,
                                   cudaStream_t stream) {
    return cc_launch_conv(d, 0, x, packed, y, stream, coef);
}

// coef: nullptr (the causal convolution's weight gradient) or the Bottleneck's BN + ReLU prologue on x (kt = 1)
static int cc_launch_conv_wgrad(const fiery_causal_conv3d_desc_t* d, const float* x, const float* gy, const BnCoef* coef, float* gw,
                                void* workspace, cudaStream_t stream) {
    const CcShape s = cc_shape(d);
    const long long tiles = cc_wgrad_tiles(s);
    const int n_chunks = wgrad_chunks(tiles, WG_MAX_CHUNKS);
    float* partial = static_cast<float*>(workspace);
    if (n_chunks > 0) {
        FIERY_REQUIRE(tiles < (1ll << 31), "causal conv: too many pixel tiles");
        const int no = cc_round8(s.cout);
        CcWgradMaps maps;
        int rc = cc_encode_activation(&maps.gy, s, gy, s.cout, CC_WG_PX, 1, static_cast<cuuint32_t>(no), CU_TENSOR_MAP_SWIZZLE_128B,
                                      "causal conv output gradient");
        if (rc == FIERY_OK)
            rc = cc_encode_activation(&maps.x, s, x, s.cin, CC_WG_XP, 1, 64, CU_TENSOR_MAP_SWIZZLE_NONE, "causal conv input");
        if (rc != FIERY_OK) return rc;
        maps.x_first = maps.x;
        const CcWgradSeg seg{0, s.cin, 0, s.cout, 1, 0, 0};
        if (coef) {
            FIERY_REQUIRE(s.kt == 1, "bottleneck: the BN prologue runs in the weight gradient of a (1, 3, 3) conv only");
            const int smem = CC_WG_STAGES * (CC_WG_X_BYTES + no * 128) + CC_SMEM_SLACK;
            const dim3 grid(static_cast<unsigned>(n_chunks), 3u);
            switch (no) {
#define CC_BN_WG_CASE(N)                                                                                                           \
    case N:                                                                                                                        \
        if ((rc = set_dynamic_smem(bottleneck_conv_wgrad_kernel<N>, smem)) != FIERY_OK) return rc;                                 \
        bottleneck_conv_wgrad_kernel<N><<<grid, 128, smem, stream>>>(maps, s, seg, partial, static_cast<int>(tiles), coef);         \
        break;
                CC_BN_WG_CASE(8) CC_BN_WG_CASE(16) CC_BN_WG_CASE(24) CC_BN_WG_CASE(32) CC_BN_WG_CASE(40) CC_BN_WG_CASE(48)
                CC_BN_WG_CASE(56) CC_BN_WG_CASE(64)
#undef CC_BN_WG_CASE
                default: return set_error(FIERY_E_INVALID, "bottleneck: %d output channels in the 3x3 weight gradient", s.cout);
            }
            FIERY_CUDA_CHECK(cudaGetLastError());
        } else if ((rc = cc_launch_wgrad(maps, s, seg, partial, n_chunks, stream)) != FIERY_OK) {
            return rc;
        }
    }
    return cc_wgrad_reduce(s, partial, n_chunks, gw, stream);
}

int launch_causal_conv_wgrad(const fiery_causal_conv3d_desc_t* d, const float* x, const float* gy, float* gw, void* workspace,
                             cudaStream_t stream) {
    return cc_launch_conv_wgrad(d, x, gy, nullptr, gw, workspace, stream);
}

int launch_bottleneck_conv_wgrad(const fiery_causal_conv3d_desc_t* d, const float* x, const BnCoef* coef, const float* gy, float* gw,
                                 void* workspace, cudaStream_t stream) {
    return cc_launch_conv_wgrad(d, x, gy, coef, gw, workspace, stream);
}

}  // namespace fiery
