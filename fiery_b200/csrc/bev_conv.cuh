// Constants and host helpers shared by the first BEV convolution's forward (bev_conv.cu) and backward (bev_conv_bwd.cu):
// Conv2d(64, 64, kernel_size=7, stride=2, padding=3, bias=False) on channel-last fp32 tensors, wgmma TF32.
#pragma once
#include "wgmma.cuh"

namespace fiery {

constexpr int CV_C = 64;                      // input = output channels
constexpr int CV_TAPS = 49;
constexpr int CV_TW = 16, CV_TH = 8;          // output patch: 16 x 8 = 128 rows of the accumulator
constexpr int CV_STAGES = 4;
constexpr int CV_A_ATOM = 128 * 128;          // 128 rows x 128 bytes (32 fp32 channels), swizzle-128B atom rows
constexpr int CV_B_ATOM = 64 * 128;           // 64 output channels x 32 input channels
constexpr int CV_STAGE_BYTES = 2 * CV_A_ATOM + 2 * CV_B_ATOM;      // 48 KB
constexpr int CV_CONSUMERS = 2;               // warpgroups
constexpr int CV_PRODUCER_WARP = 4 * CV_CONSUMERS;
constexpr int CV_THREADS = 128 * CV_CONSUMERS + 32;

struct ConvMaps {
    CUtensorMap x;       // (C, W, H, B) fp32, box (32, 32, 16, 1), element strides (1, 2, 2, 1), swizzle 128B
    CUtensorMap w;       // (I, O, tap) fp32, box (32, 64, 1), swizzle 128B
};

// A channel-last fp32 activation (n_frames, H, W, 64) as a 4-D map (C, W, H, B): box (32, box_w, box_h, 1) traversed with element
// strides (1, stride_w, stride_h, 1), 128-byte swizzle; coordinates outside the tensor read as zero (the convolution's padding)
inline int encode_conv_activation_map(CUtensorMap* map, const float* t, int n_frames, int H, int W, int box_w, int box_h, int stride_w,
                                      int stride_h, const char* what) {
    cuuint64_t dims[4] = {CV_C, static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(n_frames)};
    cuuint64_t strides[3] = {CV_C * 4ull, static_cast<cuuint64_t>(W) * CV_C * 4ull, static_cast<cuuint64_t>(H) * W * CV_C * 4ull};
    cuuint32_t box[4] = {32, static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(box_h), 1};
    cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride_w), static_cast<cuuint32_t>(stride_h), 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, t, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, what);
}

// A packed weight (tap, N rows, 64 K) fp32 as a 3-D map, box (32, 64, 1): one tap's K-major B operand, half the K range per load
inline int encode_conv_weight_map(CUtensorMap* map, const float* packed, const char* what) {
    cuuint64_t dims[3] = {CV_C, CV_C, CV_TAPS};
    cuuint64_t strides[2] = {CV_C * 4ull, CV_C * CV_C * 4ull};
    cuuint32_t box[3] = {32, CV_C, 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, packed, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, what);
}

inline int conv_out_size(int n) { return (n + 2 * 3 - 7) / 2 + 1; }

}  // namespace fiery
