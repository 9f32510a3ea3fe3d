// Backward of the first BEV convolution (bev_conv.cu): Conv2d(64, 64, 7, stride 2, padding 3, no bias) on channel-last fp32
// tensors, both gradients on the tensor cores (wgmma, TF32 operands, fp32 accumulation).
//
// Input gradient (dgrad), grad_x (B, H, W, 64) = conv_transpose(grad_y (B, Ho, Wo, 64), w).  The stride-2 transposed convolution
// splits into four stride-1 convolutions, one per output parity (p_y, p_x).  For an input row y = 2q + p:
//   grad_x[y] = sum over taps r = p + 1 (mod 2) of grad_y[q + (p + 3 - r) / 2] . w[r]      (p = 0: r in {1, 3, 5}; p = 1: {0, 2, 4, 6})
// so the four phases hold 9 + 12 + 12 + 16 = 49 taps.  One CTA per 16 x 8 patch of q walks the phases one after the other: each
// phase is the forward's implicit GEMM with element stride 1 (A = the grad_y window, K-major as it lies, TMA with zero fill outside
// the tensor; B = the tap's weight slice as (in, out), from a second, transposed pack), and its epilogue stores pixel
// (2 q_y + p_y, 2 q_x + p_x) where it lies inside (H, W).
//
// Weight gradient (wgrad), dw[o][i][r][s] = sum over pixels (b, oy, ox) of grad_y[b, oy, ox, o] . x[b, 2 oy + r - 3, 2 ox + s - 3, i]:
// a GEMM over K = B Ho Wo pixels per tap.  TF32 wgmma reads shared-memory operands K-major only, and in the channel-last layout
// both operands are pixel-major, so one is turned on chip: each 16 x 8 pixel tile of grad_y is transposed once into a K-major B
// operand (o rows, pixels along K), shared by all taps; each tap's stride-2 x window is read from a TMA tile as the register A
// operand (M = input channel).  A CTA owns one tap row r: warpgroup 0 accumulates taps s = 0..3, warpgroup 1 taps s = 4..6, each a
// 64 x 64 fp32 accumulator.  One TMA load per pixel tile brings the union of the seven taps' windows (8 rows at stride 2 x 40
// columns) so the horizontal taps share it.
// Deterministic, no atomics: the pixel tiles are cut into chunks whose boundaries depend on (n_frames, H, W) only; each chunk
// writes its partial dw to a workspace and a second kernel adds the partials in ascending chunk order.
//
// Operand rounding: the packed weights (both packs) and, in wgrad, both operands are rounded to TF32 (cvt.rna) on their way to
// the tensor core; dgrad's grad_y operand is read from fp32 by the tensor core, which truncates it -- as the forward does with x.
#include "bev_conv.cuh"
#include "wgrad_chunks.cuh"

namespace fiery {

// ------------------------------------------------------------------------------------------------------------------------------
// dgrad
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int DG_PHASE_END0 = 9, DG_PHASE_END1 = 21, DG_PHASE_END2 = 33;     // items [0, 9) phase (0,0), ... [33, 49) phase (1,1)

// item `it` of a CTA's 49 -> phase (p_y = ph >> 1, p_x = ph & 1) and tap (r, s); taps ascend in r, then s, inside a phase
__device__ __forceinline__ void dgrad_item(int it, int& ph, int& r, int& s) {
    ph = it < DG_PHASE_END0 ? 0 : it < DG_PHASE_END1 ? 1 : it < DG_PHASE_END2 ? 2 : 3;
    const int base = ph == 0 ? 0 : ph == 1 ? DG_PHASE_END0 : ph == 2 ? DG_PHASE_END1 : DG_PHASE_END2;
    const int py = ph >> 1, px = ph & 1, nx = px ? 4 : 3, l = it - base;
    r = 2 * (l / nx) + (py ? 0 : 1);
    s = 2 * (l % nx) + (px ? 0 : 1);
}

// maps.x: grad_y (64, Wo, Ho, B), box (32, 16, 8, 1), element strides 1;  maps.w: the transposed pack (tap, in, out)
__global__ void __launch_bounds__(CV_THREADS, 1)
bev_conv7x7s2_dgrad_kernel(const __grid_constant__ ConvMaps maps, float* __restrict__ gx, int H, int W, int tiles_x, int tiles_y) {
    unsigned char* smem = dynamic_smem_1024();
    const MbarRing ring(reinterpret_cast<uint64_t*>(smem + CV_STAGES * CV_STAGE_BYTES), CV_STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const int b = tile / (tiles_x * tiles_y);
    const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
    const int qy0 = ty * CV_TH, qx0 = tx * CV_TW;

    if (warp == CV_PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&maps.x);
        tma_prefetch_desc(&maps.w);
        ring.init(4 * CV_CONSUMERS);
    }
    __syncthreads();

    if (warp == CV_PRODUCER_WARP) {
        if (lane == 0) {                              // ===== TMA producer =====
            for (int it = 0; it < CV_TAPS; ++it) {
                const int st = ring.produce(it, CV_STAGE_BYTES);
                uint64_t* full = ring.full + st;
                unsigned char* a = smem + st * CV_STAGE_BYTES;
                unsigned char* bw = a + 2 * CV_A_ATOM;
                int ph, r, s;
                dgrad_item(it, ph, r, s);
                const int dy = ((ph >> 1) + 3 - r) / 2, dx = ((ph & 1) + 3 - s) / 2;     // -1 .. 2
                tma_load_4d(a, &maps.x, full, 0, qx0 + dx, qy0 + dy, b);
                tma_load_4d(a + CV_A_ATOM, &maps.x, full, 32, qx0 + dx, qy0 + dy, b);
                tma_load_3d(bw, &maps.w, full, 0, 0, r * 7 + s);
                tma_load_3d(bw + CV_B_ATOM, &maps.w, full, 32, 0, r * 7 + s);
            }
        }
        return;
    }

    // ===== consumers: warpgroup g takes accumulator rows 64g .. 64g + 63 (patch rows 4g .. 4g + 3) =====
    const int g = warp >> 2, wq = warp & 3;
    float acc[CV_C / 2];
#pragma unroll
    for (int i = 0; i < CV_C / 2; ++i) acc[i] = 0.f;
    wgmma_fence();
    int it = 0;
    for (int ph = 0; ph < 4; ++ph) {
        const int n = ph == 0 ? DG_PHASE_END0 : ph == 1 ? DG_PHASE_END1 - DG_PHASE_END0 : ph == 2 ? DG_PHASE_END2 - DG_PHASE_END1
                                                                                              : CV_TAPS - DG_PHASE_END2;
        for (int k = 0; k < n; ++k, ++it) {
            const int st = ring.consume(it);
            const uint32_t a_addr = smem_addr(smem + st * CV_STAGE_BYTES) + g * 64 * 128;
            const uint32_t b_addr = smem_addr(smem + st * CV_STAGE_BYTES) + 2 * CV_A_ATOM;
#pragma unroll
            for (int atom = 0; atom < 2; ++atom) {
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wgmma_tf32_ss<64>(acc, gmma_desc_sw128(a_addr + atom * CV_A_ATOM + 32 * kk, 16, 1024),
                                      gmma_desc_sw128(b_addr + atom * CV_B_ATOM + 32 * kk, 16, 1024));
            }
            wgmma_commit();
            // the previous tap's MMAs are complete: its stage may be refilled (a phase's first tap waits for nothing)
            wgmma_wait<1>();
            // open-coded release: a phase's first tap has no stage to release, and `if (k > 0) ring.release(it - 1)` would put the
            // warp sync under a branch in this loop (0.4% slower on an H100); here every tap syncs and only the arrival is conditional
            __syncwarp();
            if (lane == 0 && k > 0) mbar_arrive(ring.empty + (it - 1) % CV_STAGES);
        }
        // the phase's last tap: drain, store the phase's pixels (2 q_y + p_y, 2 q_x + p_x), restart the accumulator
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        ring.release(it - 1);
        const int cq = 2 * (lane & 3);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int m = 64 * g + 16 * wq + (lane >> 2) + 8 * half;
            const int y = 2 * (qy0 + m / CV_TW) + (ph >> 1), x = 2 * (qx0 + m % CV_TW) + (ph & 1);
            if (y < H && x < W) {
                float* dst = gx + ((static_cast<size_t>(b) * H + y) * W + x) * CV_C;
#pragma unroll
                for (int j = 0; j < CV_C / 8; ++j)
                    *reinterpret_cast<float2*>(dst + 8 * j + cq) = make_float2(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
            }
        }
#pragma unroll
        for (int i = 0; i < CV_C / 2; ++i) acc[i] = 0.f;
        wgmma_fence();
    }
}

// weights (O, I, 7, 7) -> (tap = r*7 + s, I, O), rounded to TF32: the K-major B operand of every dgrad tap
__global__ void pack_conv_weights_transposed_kernel(const float* __restrict__ w, float* __restrict__ packed) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= CV_TAPS * CV_C * CV_C) return;
    const int out = i % CV_C, in = (i / CV_C) % CV_C, tap = i / (CV_C * CV_C);
    packed[i] = __uint_as_float(to_tf32(w[(static_cast<size_t>(out) * CV_C + in) * CV_TAPS + tap]));
}

int launch_pack_conv_weights_transposed(const float* w_oihw, float* packed, cudaStream_t stream) {
    const int n = CV_TAPS * CV_C * CV_C;
    pack_conv_weights_transposed_kernel<<<(n + 255) / 256, 256, 0, stream>>>(w_oihw, packed);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_bev_conv_dgrad(int n_frames, int H, int W, const float* gy_nhwc, const float* w_packed_t, float* gx_nhwc, cudaStream_t stream) {
    const int Ho = conv_out_size(H), Wo = conv_out_size(W);
    ConvMaps maps;
    int rc = encode_conv_activation_map(&maps.x, gy_nhwc, n_frames, Ho, Wo, CV_TW, CV_TH, 1, 1, "conv output gradient");
    if (rc == FIERY_OK) rc = encode_conv_weight_map(&maps.w, w_packed_t, "transposed conv weights");
    if (rc != FIERY_OK) return rc;
    const int smem = CV_STAGES * CV_STAGE_BYTES + 1024 /* alignment slack */ + 256 /* barriers */;
    static OncePerDevice once;
    rc = once.run([smem]() { return set_dynamic_smem(bev_conv7x7s2_dgrad_kernel, smem); });
    if (rc != FIERY_OK) return rc;
    const int tiles_x = (Wo + CV_TW - 1) / CV_TW, tiles_y = (Ho + CV_TH - 1) / CV_TH;     // tiles of q: q < ceil(H / 2) = Ho
    bev_conv7x7s2_dgrad_kernel<<<static_cast<unsigned>(n_frames * tiles_x * tiles_y), CV_THREADS, smem, stream>>>(maps, gx_nhwc, H, W,
                                                                                                               tiles_x, tiles_y);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// wgrad
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int WG_WIN_W = 40;                          // window columns 2 ox0 - 3 .. 2 ox0 + 36 (37 used) of the seven taps s
constexpr int WG_WIN_ATOM = WG_WIN_W * CV_TH * 128;   // 8 rows x 40 columns x 32 channels, swizzle 128B: 40 KB
constexpr int WG_X_STAGE = 2 * WG_WIN_ATOM;           // both channel halves
constexpr int WG_STAGES = 2;
constexpr int WG_B_ATOM = CV_C * 128;                 // 64 output channels x 32 pixels (K-major, swizzle 128B)
constexpr int WG_B_BYTES = 4 * WG_B_ATOM;             // the tile's 128 pixels
constexpr int WG_KSTEPS = CV_TW * CV_TH / 8;          // 16 MMAs of k = 8 pixels per tile and tap
constexpr int CV_WG_MAX_CHUNKS = 18;                  // pixel chunks (x 7 tap rows = 126 CTAs); workspace <= 18 x 784 KB
constexpr int WG_THREADS = 128 * CV_CONSUMERS;         // two warpgroups, no producer warp
constexpr size_t WG_PARTIAL_FLOATS = static_cast<size_t>(CV_TAPS) * CV_C * CV_C;

static long long wgrad_tiles(int n_frames, int H, int W) {
    const int Ho = conv_out_size(H), Wo = conv_out_size(W);
    return static_cast<long long>(n_frames) * ((Wo + CV_TW - 1) / CV_TW) * ((Ho + CV_TH - 1) / CV_TH);
}

size_t bev_conv_wgrad_workspace_bytes(int n_frames, int H, int W) {
    if (n_frames < 0 || H < 1 || W < 1) return 0;
    return static_cast<size_t>(wgrad_chunks(wgrad_tiles(n_frames, H, W), CV_WG_MAX_CHUNKS)) * WG_PARTIAL_FLOATS * sizeof(float);
}

// the x window of pixel tile `tile` (both channel halves) into the stage of iteration it
__device__ __forceinline__ void wgrad_load_window(const CUtensorMap* xmap, unsigned char* xs, const MbarRing& ring, int r, int tile, int it,
                                                  int tiles_x, int tiles_y) {
    const int b = tile / (tiles_x * tiles_y), ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
    const int st = ring.arm(it, WG_X_STAGE);
    unsigned char* a = xs + st * WG_X_STAGE;
    tma_load_4d(a, xmap, ring.full + st, 0, 2 * tx * CV_TW - 3, 2 * ty * CV_TH + r - 3, b);
    tma_load_4d(a + WG_WIN_ATOM, xmap, ring.full + st, 32, 2 * tx * CV_TW - 3, 2 * ty * CV_TH + r - 3, b);
}

// One warpgroup's NS taps (s0 .. s0 + NS - 1 of row r) over the chunk's pixel tiles
template <int NS>
__device__ __forceinline__ void wgrad_consume(const CUtensorMap* xmap, unsigned char* xs, unsigned char* bs, const MbarRing& ring,
                                              const float* __restrict__ gy, float* __restrict__ partial, int r, int s0, int t0, int t1,
                                              int Ho, int Wo, int tiles_x, int tiles_y) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wq = warp & 3;
    float acc[NS][32];
#pragma unroll
    for (int t = 0; t < NS; ++t)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[t][i] = 0.f;

    for (int tile = t0; tile < t1; ++tile) {
        const int it = tile - t0;
        const int b = tile / (tiles_x * tiles_y), ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
        const int oy0 = ty * CV_TH, ox0 = tx * CV_TW;
        unsigned char* bt = bs + (it & 1) * WG_B_BYTES;
        // grad_y tile -> B operand (o rows, pixel p along K), TF32-rounded; pixels outside the output read as zero.  Lane = pixel
        // within a 32-pixel group, so the loads are 16-byte pieces of 32 pixel rows and the transposed stores hit 32 banks.
        float4 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int combo = warp * 8 + j, pg = combo >> 4, c4 = combo & 15;
            const int p = pg * 32 + lane, oy = oy0 + (p >> 4), ox = ox0 + (p & 15);
            v[j] = (oy < Ho && ox < Wo) ? __ldg(reinterpret_cast<const float4*>(gy + ((static_cast<size_t>(b) * Ho + oy) * Wo + ox) * CV_C) + c4)
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int combo = warp * 8 + j, pg = combo >> 4, c4 = combo & 15;
            unsigned char* atom = bt + pg * WG_B_ATOM + (lane & 3) * 4;
            const float e[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int o = 4 * c4 + q;
                *reinterpret_cast<uint32_t*>(atom + o * 128 + (((lane >> 2) ^ (o & 7)) << 4)) = to_tf32(e[q]);
            }
        }
        fence_proxy_async();                          // generic-proxy stores -> visible to the tensor core's async proxy
        named_barrier(1, WG_THREADS);                 // both warpgroups (their code paths differ: named barrier)
        // every warp has finished tile it - 1: its x stage may be refilled with the next tile's window
        if (threadIdx.x == 0 && tile + 1 < t1) wgrad_load_window(xmap, xs, ring, r, tile + 1, it + 1, tiles_x, tiles_y);

        const int st = ring.consume(it);
        const unsigned char* xw = xs + st * WG_X_STAGE;
        const uint32_t b_addr = smem_addr(bt);
#pragma unroll 1
        for (int kg = 0; kg < WG_KSTEPS / 2; ++kg) { // 16 pixels per group: two k-steps of 8
            uint32_t a[NS][2][4];
#pragma unroll
            for (int t = 0; t < NS; ++t)
#pragma unroll
                for (int ks = 0; ks < 2; ++ks)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int i = 16 * wq + (lane >> 2) + 8 * (e & 1);              // A row = input channel
                        const int p = 16 * kg + 8 * ks + (lane & 3) + 4 * (e >> 1);     // A column = pixel of the tile
                        const int row = (p >> 4) * WG_WIN_W + 2 * (p & 15) + s0 + t;    // window row of 128 bytes
                        const int ch = i & 31;
                        a[t][ks][e] = to_tf32(*reinterpret_cast<const float*>(xw + (i >> 5) * WG_WIN_ATOM + row * 128 +
                                                                               (((ch >> 2) ^ (row & 7)) << 4) + (ch & 3) * 4));
                    }
            wgmma_fence();
#pragma unroll
            for (int t = 0; t < NS; ++t)
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) {
                    const int k = 2 * kg + ks;
                    wgmma_tf32_rs<64>(acc[t], a[t][ks], gmma_desc_sw128(b_addr + (k >> 2) * WG_B_ATOM + 32 * (k & 3), 16, 1024));
                }
            wgmma_commit();
            wgmma_wait<0>();
        }
#pragma unroll
        for (int t = 0; t < NS; ++t) wgmma_fence_operands(acc[t]);
    }

    // partial dw of this chunk, OIHW: accumulator (row i, column o) of tap (r, s0 + t)
    float* dst = partial + static_cast<size_t>(blockIdx.y) * WG_PARTIAL_FLOATS;
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int t = 0; t < NS; ++t)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int i = 16 * wq + (lane >> 2) + 8 * half;
#pragma unroll
            for (int j = 0; j < CV_C / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int o = 8 * j + cq + e;
                    dst[(static_cast<size_t>(o) * CV_C + i) * CV_TAPS + r * 7 + s0 + t] = acc[t][4 * j + 2 * half + e];
                }
        }
}

// grid (7 tap rows r, chunks), two warpgroups and no producer warp (all 256 threads take part in the transpose); xmap: x (64, W, H, B),
// box (32, 40, 16, 1), element strides (1, 1, 2, 1)
__global__ void __launch_bounds__(WG_THREADS, 1)
bev_conv7x7s2_wgrad_kernel(const __grid_constant__ CUtensorMap xmap, const float* __restrict__ gy, float* __restrict__ partial, int Ho,
                           int Wo, int tiles_x, int tiles_y, int n_tiles) {
    unsigned char* xs = dynamic_smem_1024();
    unsigned char* bs = xs + WG_STAGES * WG_X_STAGE;
    const MbarRing ring(reinterpret_cast<uint64_t*>(bs + 2 * WG_B_BYTES), WG_STAGES);

    const int r = blockIdx.x;
    const int t0 = static_cast<int>(static_cast<long long>(blockIdx.y) * n_tiles / gridDim.y);
    const int t1 = static_cast<int>(static_cast<long long>(blockIdx.y + 1) * n_tiles / gridDim.y);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&xmap);
        ring.init(0);
        wgrad_load_window(&xmap, xs, ring, r, t0, 0, tiles_x, tiles_y);
    }
    __syncthreads();
    if (threadIdx.x < 128) wgrad_consume<4>(&xmap, xs, bs, ring, gy, partial, r, 0, t0, t1, Ho, Wo, tiles_x, tiles_y);
    else wgrad_consume<3>(&xmap, xs, bs, ring, gy, partial, r, 4, t0, t1, Ho, Wo, tiles_x, tiles_y);
}

// a chunk's partial is laid out as dw (OIHW)
struct CvWgradOffset {
    __device__ size_t operator()(int i) const { return i; }
};

int launch_bev_conv_wgrad(int n_frames, int H, int W, const float* x_nhwc, const float* gy_nhwc, float* dw_oihw, void* workspace,
                          cudaStream_t stream) {
    const long long tiles = wgrad_tiles(n_frames, H, W);
    const int n_chunks = wgrad_chunks(tiles, CV_WG_MAX_CHUNKS);
    float* partial = static_cast<float*>(workspace);
    if (n_chunks > 0) {
        FIERY_REQUIRE(tiles < (1ll << 31), "bev conv backward: too many pixels");
        CUtensorMap xmap;
        int rc = encode_conv_activation_map(&xmap, x_nhwc, n_frames, H, W, WG_WIN_W, 2 * CV_TH, 1, 2, "conv input window");
        if (rc != FIERY_OK) return rc;
        const int smem = WG_STAGES * WG_X_STAGE + 2 * WG_B_BYTES + 1024 /* alignment slack */ + 64 /* barriers */;
        static OncePerDevice once;
        rc = once.run([smem]() { return set_dynamic_smem(bev_conv7x7s2_wgrad_kernel, smem); });
        if (rc != FIERY_OK) return rc;
        const int Ho = conv_out_size(H), Wo = conv_out_size(W);
        const int tiles_x = (Wo + CV_TW - 1) / CV_TW, tiles_y = (Ho + CV_TH - 1) / CV_TH;
        bev_conv7x7s2_wgrad_kernel<<<dim3(7, n_chunks), WG_THREADS, smem, stream>>>(xmap, gy_nhwc, partial, Ho, Wo, tiles_x, tiles_y,
                                                                                   static_cast<int>(tiles));
        FIERY_CUDA_CHECK(cudaGetLastError());
    }
    return launch_wgrad_reduce(partial, n_chunks, WG_PARTIAL_FLOATS, static_cast<int>(WG_PARTIAL_FLOATS), CvWgradOffset{}, dw_oihw,
                               stream);
}

}  // namespace fiery
