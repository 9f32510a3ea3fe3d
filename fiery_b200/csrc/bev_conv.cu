// First BEV convolution on the tensor cores (SURVEY.md section 8f, next-2): Decoder.first_conv, 7x7 stride 2 padding 3,
// 64 -> 64 channels, no bias (fiery/models/decoder.py:11,59), with the folded bn1 + relu of decoder.py:60-61 as an optional epilogue.
//
// It is the first dense contraction after the lift and it consumes the lift's CHANNEL-LAST result directly: (B', X, Y, C) fp32 is
// exactly the K-major A operand of an implicit GEMM, so the NCHW layout pass of the lift disappears from this path.
//
//   D[m][o] = sum over taps (r, s) and input channels i of  x[b][2*oy + r - 3][2*ox + s - 3][i] * w[o][i][r][s]
//   M = 128 output pixels (a 16 wide x 8 tall patch), N = 64 output channels, K = 49 taps x 64 channels = 3136
//
// One CTA per output patch, warp-specialised:
//   warp 8     TMA producer: per tap, two 4-D tiled loads (box 32 ch x 16 px x 8 rows, ELEMENT STRIDE 2 along X and Y: the copy
//              engine does the stride-2 im2col; out-of-range coordinates are zero-filled = the padding) and two loads of the tap's
//              (64 out x 32 in) weight slices, all with the 128-byte swizzle the MMA expects; 4-stage ring, mbarrier full/empty
//   warps 0-7  two consumer warpgroups, warpgroup g owns output pixels 64g .. 64g + 63 (patch rows 4g .. 4g + 3): wgmma m64n64k8
//              TF32, 8 per tap, fp32 accumulator in registers; one tap's MMAs stay in flight while the next tap's are issued, a
//              stage is released once its MMAs have completed.  Epilogue: per-channel scale/shift (+ relu), 8-byte stores into the
//              channel-last output
// Operands are TF32 (10-bit mantissa: weights rounded when they are packed, activations read from fp32 by truncation), accumulation
// fp32 -- the precision cuDNN uses for this layer under torch's default allow_tf32; the parity bar (tests/test_bev_conv_gpu.py) is
// stated against an fp64 convolution: normwise < 1e-3.
#include "bev_conv.cuh"

namespace fiery {

__global__ void __launch_bounds__(CV_THREADS, 1)
bev_conv7x7s2_kernel(const __grid_constant__ ConvMaps maps, const float* __restrict__ scale, const float* __restrict__ shift,
                     int relu, float* __restrict__ y, int Ho, int Wo, int tiles_x, int tiles_y) {
    unsigned char* smem = dynamic_smem_1024();
    const MbarRing ring(reinterpret_cast<uint64_t*>(smem + CV_STAGES * CV_STAGE_BYTES), CV_STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const int b = tile / (tiles_x * tiles_y);
    const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
    const int oy0 = ty * CV_TH, ox0 = tx * CV_TW;

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
                const int r = it / 7, s = it % 7;
                // input patch of this tap: pixels (2*oy + r - 3, 2*ox + s - 3); negative / too large coordinates read as zero
                tma_load_4d(a, &maps.x, full, 0, 2 * ox0 + s - 3, 2 * oy0 + r - 3, b);
                tma_load_4d(a + CV_A_ATOM, &maps.x, full, 32, 2 * ox0 + s - 3, 2 * oy0 + r - 3, b);
                tma_load_3d(bw, &maps.w, full, 0, 0, it);
                tma_load_3d(bw + CV_B_ATOM, &maps.w, full, 32, 0, it);
            }
        }
        return;
    }

    // ===== consumers: warpgroup g takes accumulator rows 64g .. 64g + 63 =====
    const int g = warp >> 2, wq = warp & 3;
    float acc[CV_C / 2];
#pragma unroll
    for (int i = 0; i < CV_C / 2; ++i) acc[i] = 0.f;
    wgmma_fence();
    for (int it = 0; it < CV_TAPS; ++it) {
        const int st = ring.consume(it);
        const uint32_t a_addr = smem_addr(smem + st * CV_STAGE_BYTES) + g * 64 * 128;
        const uint32_t b_addr = smem_addr(smem + st * CV_STAGE_BYTES) + 2 * CV_A_ATOM;
#pragma unroll
        for (int atom = 0; atom < 2; ++atom) {
#pragma unroll
            for (int k = 0; k < 4; ++k)               // 8 TF32 values (32 bytes) per MMA along K
                wgmma_tf32_ss<64>(acc, gmma_desc_sw128(a_addr + atom * CV_A_ATOM + 32 * k, 16, 1024),
                                  gmma_desc_sw128(b_addr + atom * CV_B_ATOM + 32 * k, 16, 1024));
        }
        wgmma_commit();
        if (it > 0) {                                 // the previous tap's MMAs are complete: its stage may be refilled
            wgmma_wait<1>();
            ring.release(it - 1);
        }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int m = 64 * g + 16 * wq + (lane >> 2) + 8 * half;   // accumulator row = output pixel of the patch
        const int oy = oy0 + m / CV_TW, ox = ox0 + m % CV_TW;
        if (oy < Ho && ox < Wo) {
            float* dst = y + ((static_cast<size_t>(b) * Ho + oy) * Wo + ox) * CV_C;
#pragma unroll
            for (int j = 0; j < CV_C / 8; ++j) {
                const int c = 8 * j + cq;
                float o[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float t = acc[4 * j + 2 * half + e];
                    if (scale) t = fmaf(t, __ldg(scale + c + e), __ldg(shift + c + e));
                    o[e] = relu ? fmaxf(t, 0.f) : t;
                }
                *reinterpret_cast<float2*>(dst + c) = make_float2(o[0], o[1]);
            }
        }
    }
}

// weights (O, I, 7, 7) as PyTorch stores them -> (tap = r*7 + s, O, I): the K-major B operand of every tap
__global__ void pack_conv_weights_kernel(const float* __restrict__ w, float* __restrict__ packed) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= CV_TAPS * CV_C * CV_C) return;
    const int in = i % CV_C, out = (i / CV_C) % CV_C, tap = i / (CV_C * CV_C);
    // rounded to TF32 (nearest, ties away) here, once per weight update: the tensor core would otherwise TRUNCATE the low mantissa
    // bits of an fp32 operand.  (The activations stay as the lift wrote them -- a rounding pass over 82 MB is not worth 1.5e-4.)
    packed[i] = __uint_as_float(to_tf32(w[(static_cast<size_t>(out) * CV_C + in) * CV_TAPS + tap]));
}

int launch_pack_conv_weights(const float* w_oihw, float* packed, cudaStream_t stream) {
    const int n = CV_TAPS * CV_C * CV_C;
    pack_conv_weights_kernel<<<(n + 255) / 256, 256, 0, stream>>>(w_oihw, packed);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int launch_bev_conv(int n_frames, int H, int W, const float* x_nhwc, const float* w_packed, const float* scale, const float* shift,
                    int relu, float* y_nhwc, cudaStream_t stream) {
    const int Ho = (H + 2 * 3 - 7) / 2 + 1, Wo = (W + 2 * 3 - 7) / 2 + 1;
    ConvMaps maps;
    int rc = encode_conv_activation_map(&maps.x, x_nhwc, n_frames, H, W, 2 * CV_TW, 2 * CV_TH, 2, 2, "conv input");
    if (rc == FIERY_OK) rc = encode_conv_weight_map(&maps.w, w_packed, "conv weights");
    if (rc != FIERY_OK) return rc;
    const int smem = CV_STAGES * CV_STAGE_BYTES + 1024 /* alignment slack */ + 256 /* barriers */;
    static OncePerDevice once;
    rc = once.run([smem]() { return set_dynamic_smem(bev_conv7x7s2_kernel, smem); });
    if (rc != FIERY_OK) return rc;
    const int tiles_x = (Wo + CV_TW - 1) / CV_TW, tiles_y = (Ho + CV_TH - 1) / CV_TH;
    bev_conv7x7s2_kernel<<<static_cast<unsigned>(n_frames * tiles_x * tiles_y), CV_THREADS, smem, stream>>>(maps, scale, shift, relu, y_nhwc,
                                                                                                         Ho, Wo, tiles_x, tiles_y);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
