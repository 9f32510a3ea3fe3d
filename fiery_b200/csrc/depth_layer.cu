// Encoder.depth_layer on the tensor cores (SURVEY.md section 8f, next-3): the 1x1 convolution 128 -> D + C that produces the head
// tensor the lift consumes (fiery/models/encoder.py:36,96), as a wgmma GEMM that reads the feature map in the dtype the backbone
// emits it (fp16 / bf16 under AMP, fp32 otherwise) and writes the fp32 NCHW head tensor directly -- so an AMP step has no separate
// widening pass between the 1x1 convolution and the lift (the reference's softmax / outer product run in fp32 under autocast,
// encoder.py:99-100, and so do the tile kernels).
//
//   head[img][o][p] = bias[o] + sum_i W[o][i] * feat[img][i][p]          o < D + C <= 128,  i < 128,  p < h*w
//
// Per CTA one tile of 128 pixels of one image at a time (persistent: CTA b takes tiles b, b + grid, ...).  The padded weight matrix
// (128 x 128, K-major, 128-byte swizzle) is loaded once per CTA; feature tiles (K = 128 channels x 128 pixels, taken as they lie in
// the NCHW feature map: pixels contiguous) run through a STAGES-deep TMA ring.  Warp roles: warps 0-7 are two consumer warpgroups,
// warp 8 the TMA producer.
//   fp16 / bf16: D (128 output channels x 128 pixels) = W x feat, both operands from shared memory, the feature tile as the
//                MN-major ("transposed") B operand; warpgroup g owns output channels 64g .. 64g + 63.  An accumulator row is an output
//                channel, so a thread's float2 stores go to consecutive pixels of one plane of the head tensor.
//   fp32 (TF32): wgmma has no MN-major TF32 operand, so the product is taken transposed, D (128 pixels x 128 output channels) =
//                feat^T x W^T: the weight matrix is the K-major B operand as it lies, the feature tile is the A operand, read from
//                shared memory into registers.  Warpgroup g owns pixel rows 64g .. 64g + 63, in the order tile_pixel() gives them
//                (conflict-free fragment loads from the swizzled tile, wgmma.cuh).
#include "wgmma.cuh"

namespace fiery {

constexpr int DL_K = 128;                 // input channels (upsampling_out_channels, encoder.py:33)
constexpr int DL_M = 128;                 // padded output channels
constexpr int DL_N = 128;                 // pixels per tile
constexpr int DL_CONSUMERS = 2;           // warpgroups
constexpr int DL_PRODUCER_WARP = 4 * DL_CONSUMERS;
constexpr int DL_THREADS = 128 * DL_CONSUMERS + 32;

struct DepthLayerMaps {
    CUtensorMap w;        // (K, M) padded weights, box (128 bytes of K, 128 rows), swizzle 128B
    CUtensorMap feat;     // (pixels, K, images), box (128 bytes of pixels, 128 channels, 1), swizzle 128B
};

template <int ES>
struct DlShape {
    static constexpr int EPR = 128 / ES;                      // elements per 128-byte row
    static constexpr int ATOMS = DL_K / EPR;                  // weights: atoms of (128 rows x 128 B) along K
    static constexpr int NBLK = DL_N / EPR;                   // feature tile: blocks of (128 channels x 128 B) along the pixels
    static constexpr int MMA_K = 32 / ES;                     // K of one MMA: 16 (fp16 / bf16), 8 (TF32)
    static constexpr int W_ATOM = DL_M * 128, B_BLK = DL_K * 128;
    static constexpr int W_BYTES = ATOMS * W_ATOM, B_BYTES = NBLK * B_BLK;
    static constexpr int STAGES = ES == 2 ? 4 : 2;            // feature tiles in flight (32 KB / 64 KB each)
    static constexpr int SMEM = W_BYTES + STAGES * B_BYTES + 1024 + 256;
};

// ES: element size of the operands (2: fp16 / bf16; 4: fp32 read as TF32).  BF16 selects the 16-bit type.
template <int ES, bool BF16>
__global__ void __launch_bounds__(DL_THREADS, 1)
depth_layer_kernel(const __grid_constant__ DepthLayerMaps maps, const float* __restrict__ bias, float* __restrict__ head, int n_out,
                   int pixels, int tiles_per_image, int n_tiles) {
    using S = DlShape<ES>;
    unsigned char* s_w = dynamic_smem_1024();
    unsigned char* s_b = s_w + S::W_BYTES;
    uint64_t* w_full = reinterpret_cast<uint64_t*>(s_b + S::STAGES * S::B_BYTES);
    const MbarRing ring(w_full + 1, S::STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == DL_PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&maps.w);
        tma_prefetch_desc(&maps.feat);
        mbar_init(w_full, 1);                          // published to the async proxy by the fence in ring.init
        ring.init(4 * DL_CONSUMERS);
    }
    __syncthreads();

    if (warp == DL_PRODUCER_WARP) {
        if (lane == 0) {                               // ===== TMA producer: weights once, then this CTA's feature tiles =====
            mbar_arrive_expect_tx(w_full, S::W_BYTES);
#pragma unroll
            for (int a = 0; a < S::ATOMS; ++a) tma_load_2d(s_w + a * S::W_ATOM, &maps.w, w_full, a * S::EPR, 0);
            int it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
                const int st = ring.produce(it, S::B_BYTES);
                const int img = t / tiles_per_image, p0 = (t % tiles_per_image) * DL_N;
                unsigned char* dst = s_b + st * S::B_BYTES;
#pragma unroll
                for (int b = 0; b < S::NBLK; ++b) tma_load_3d(dst + b * S::B_BLK, &maps.feat, ring.full + st, p0 + b * S::EPR, 0, img);   // pixels past the image: zeros
            }
        }
        return;
    }

    // ===== consumers: warpgroup g, warp wq of it =====
    const int g = warp >> 2, wq = warp & 3;
    const int r0 = 64 * g + 16 * wq + (lane >> 2);     // accumulator rows r0 and r0 + 8 of this thread
    const int cq = 2 * (lane & 3);                     // accumulator columns 8j + cq, 8j + cq + 1
    const uint32_t w_addr = smem_addr(s_w);
    mbar_wait(w_full, 0);
    int it = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
        const int img = t / tiles_per_image, p0 = (t % tiles_per_image) * DL_N;
        const unsigned char* tile = s_b + ring.consume(it) * S::B_BYTES;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        if constexpr (ES == 2) {
            wgmma_fence();
            const uint32_t b_addr = smem_addr(tile);
#pragma unroll
            for (int k = 0; k < DL_K / S::MMA_K; ++k) {
                const int k0 = k * S::MMA_K;
                // A: atom k0 / EPR, rows 64g.., 32 bytes per K step inside the atom.  B: k0 rows of 128 bytes down the block (8-row
                // groups 1024 B apart), blocks of 64 pixels B_BLK apart.
                const uint64_t da = gmma_desc_sw128(w_addr + (k0 / S::EPR) * S::W_ATOM + g * 64 * 128 + (k0 % S::EPR) * ES, 16, 1024);
                const uint64_t db = gmma_desc_sw128(b_addr + k0 * 128, S::B_BLK, 1024);
                if (BF16) wgmma_m64n128k16_bf16_ss_tb(acc, da, db);
                else wgmma_m64n128k16_f16_ss_tb(acc, da, db);
            }
        } else {
            uint32_t a[DL_K / 8][4];
            load_pixel_frags<DL_K / 8>(a, tile, DL_K, 0, tile_pixel(r0), tile_pixel(r0 + 8));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < DL_K / 8; ++k) {
                const int k0 = 8 * k;
                wgmma_m64n128k8_tf32_rs(acc, a[k], gmma_desc_sw128(w_addr + (k0 / 32) * S::W_ATOM + (k0 % 32) * 4, 16, 1024));
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        ring.release(it);                              // this warp's part of the tile has been read
        if constexpr (ES == 2) {                       // rows = output channels r0, r0 + 8; columns = pixels
            float* out = head + (static_cast<size_t>(img) * n_out + r0) * pixels + p0;
            const float b0 = (bias && r0 < n_out) ? __ldg(bias + r0) : 0.f;
            const float b1 = (bias && r0 + 8 < n_out) ? __ldg(bias + r0 + 8) : 0.f;
#pragma unroll
            for (int j = 0; j < DL_N / 8; ++j) {
                const int p = 8 * j + cq;
                if (p0 + p < pixels) {                 // pixels is a multiple of 4: p + 1 is inside too
                    if (r0 < n_out) *reinterpret_cast<float2*>(out + p) = make_float2(acc[4 * j] + b0, acc[4 * j + 1] + b0);
                    if (r0 + 8 < n_out)
                        *reinterpret_cast<float2*>(out + 8 * static_cast<size_t>(pixels) + p) = make_float2(acc[4 * j + 2] + b1, acc[4 * j + 3] + b1);
                }
            }
        } else {                                       // rows = pixels tile_pixel(r0), tile_pixel(r0 + 8); columns = output channels
            const int pa = p0 + tile_pixel(r0), pb = p0 + tile_pixel(r0 + 8);
            float* out = head + static_cast<size_t>(img) * n_out * pixels;
#pragma unroll
            for (int j = 0; j < DL_M / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int o = 8 * j + cq + e;
                    if (o < n_out) {
                        const float bo = bias ? __ldg(bias + o) : 0.f;
                        if (pa < pixels) out[static_cast<size_t>(o) * pixels + pa] = acc[4 * j + e] + bo;
                        if (pb < pixels) out[static_cast<size_t>(o) * pixels + pb] = acc[4 * j + 2 + e] + bo;
                    }
                }
            }
        }
    }
}

// dtype: 0 fp32 (TF32 math), 1 fp16, 2 bf16 -- of BOTH the feature map and the padded weight matrix
int launch_depth_layer(int n_images, int pixels, int n_out, const void* feat, int dtype, const void* weight_padded, const float* bias,
                       float* head, cudaStream_t stream) {
    const int es = dtype == 0 ? 4 : 2;
    const CUtensorMapDataType dt = dtype == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : (dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    const cuuint32_t epr = 128 / es;
    DepthLayerMaps maps;
    {
        cuuint64_t dims[2] = {DL_K, DL_M};
        cuuint64_t strides[1] = {static_cast<cuuint64_t>(DL_K) * es};
        cuuint32_t box[2] = {epr, DL_M};
        const int rc = encode_tensor_map(&maps.w, dt, 2, weight_padded, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "depth layer weights");
        if (rc != FIERY_OK) return rc;
    }
    {
        cuuint64_t dims[3] = {static_cast<cuuint64_t>(pixels), DL_K, static_cast<cuuint64_t>(n_images)};
        cuuint64_t strides[2] = {static_cast<cuuint64_t>(pixels) * es, static_cast<cuuint64_t>(pixels) * DL_K * es};
        cuuint32_t box[3] = {epr, DL_K, 1};
        const int rc = encode_tensor_map(&maps.feat, dt, 3, feat, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "feature map");
        if (rc != FIERY_OK) return rc;
    }
    static OncePerDevice once;
    int rc = once.run([]() -> int {
        FIERY_CUDA_CHECK(cudaFuncSetAttribute(depth_layer_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DlShape<2>::SMEM));
        FIERY_CUDA_CHECK(cudaFuncSetAttribute(depth_layer_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DlShape<2>::SMEM));
        FIERY_CUDA_CHECK(cudaFuncSetAttribute(depth_layer_kernel<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DlShape<4>::SMEM));
        return FIERY_OK;
    });
    if (rc != FIERY_OK) return rc;
    const int tiles_per_image = (pixels + DL_N - 1) / DL_N;
    const int n_tiles = n_images * tiles_per_image;
    unsigned grid = 0;
    if ((rc = persistent_grid(n_tiles, &grid)) != FIERY_OK) return rc;
    if (dtype == 0)
        depth_layer_kernel<4, false><<<grid, DL_THREADS, DlShape<4>::SMEM, stream>>>(maps, bias, head, n_out, pixels, tiles_per_image, n_tiles);
    else if (dtype == 1)
        depth_layer_kernel<2, false><<<grid, DL_THREADS, DlShape<2>::SMEM, stream>>>(maps, bias, head, n_out, pixels, tiles_per_image, n_tiles);
    else
        depth_layer_kernel<2, true><<<grid, DL_THREADS, DlShape<2>::SMEM, stream>>>(maps, bias, head, n_out, pixels, tiles_per_image, n_tiles);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
