// The 3x3 convolution kernels of causal_conv.cu as building blocks: the forward / input-gradient kernel over up to two halo tiles
// (the causal convolution's kt time taps of one input, or the spatial GRU's two input segments, each its own tensor) with a per-output-
// segment epilogue, and the weight-gradient kernel over one (input segment, 64-output-channel block).  causal_conv.cu launches them
// for the CausalConv3d, spatial_gru.cu for the SpatialGRU.
#pragma once
#include "common.cuh"

namespace fiery {

constexpr int CC_TX = 8, CC_TY = 16;               // output tile: rows x columns of the map
// Every TMA box starts on a 16-byte boundary of the contiguous map row: the column padding comes from a box that starts 4 columns
// early (zero fill at column -4 .. -1), and the MMA operands are read from it at the tap's shift.
constexpr int CC_HX = CC_TX + 2, CC_HY = 28;       // halo box: rows x0 - 1 .. x0 + 8, columns y0 - 4 .. y0 + 23 (y0 - 1 .. y0 + 16 used)
constexpr int CC_PLANE = CC_HX * CC_HY;            // floats per channel of a halo tile: 280 = 24 banks apart
constexpr int CC_WSTAGES = 4;                      // weight-slice ring, at most
constexpr int CC_MAX_SMEM = 227 * 1024;
constexpr int CC_SMEM_SLACK = 1024 + 256;
constexpr int CC_WG_PX = 32;                       // weight gradient: pixels per tile
constexpr int CC_WG_XP = 44;                       // weight gradient x tile: columns 32 run - 4 .. 32 run + 39, 44 = 12 banks apart

__host__ __device__ __forceinline__ int cc_round8(int v) { return (v + 7) / 8 * 8; }

// How an output segment's accumulator columns c0 .. c0 + n - 1 are written (channel ch = column - c0, pixel p of frame t):
enum CcOutMode : int {
    CC_STORE = 0,        // p[b, ch, t, p] = v
    CC_ADD = 1,          // p[b, ch, t, p] += v
    CC_GATE_U = 2,       // p[b, ch, p] = u = sigmoid(v + bias[ch] + bias_init)
    CC_GATE_R = 3,       // r = sigmoid(v + bias[ch] + bias_init): r_out[b, ch, p] = r, p[b, ch, p] = (1 - r) * h[b, ch, p]
    CC_RESET_GRAD = 4,   // v = dq: aux[b, ch, p] = -v * h * r (1 - r) (the reset gate's pre-activation gradient), p[b, ch, p] += (1 - r) v
    CC_SKIP = 5,         // not written
};

// Strides in elements; pixel planes are contiguous (X*Y floats).  h, r, aux: planes X*Y apart within a batch element.
struct CcOutSeg {
    float* p;
    long long sb, sc, st;
    int c0, n, mode;
    const float* bias;
    const float* h;
    long long hsb;
    float* r;
    long long rsb;
    float* aux;
    long long asb;
};

struct CcFwdMaps {
    CUtensorMap x[2];                              // input (Y, X, s, C, b), box (28, 10, 1, kpad, 1) = CC_HY x CC_HX, no swizzle
    CUtensorMap w;                                 // pack (32, n, atoms), box (32, n, 1), swizzle 128B
};

// Halo h: kpad[h] channels of map x[map[h]] at frame t + t_off[h], its 9 taps' weight slices the pack atoms atom0[h] + tap * ka[h] + a.
struct CcFwdLaunch {
    int frames, X, Y, tiles_x, tiles_y;
    int halos, stages, stage_bytes;
    int map[2], t_off[2], kpad[2], ka[2], x_off[2], atom0[2];
    int nseg;
    float bias_init;
    CcOutSeg seg[2];
};

// The forward kernel with N accumulator columns (N = 8 .. 64 in steps of 8; with segments also 96 or 128), n_tiles = batch * frames *
// tiles_x * tiles_y.  segments = false: the causal convolution's instantiation -- L.halos tiles of map 0 at one channel count, halo h
// at float offset h * kpad[0] * CC_PLANE, pack atoms j * ka[0], a CC_WSTAGES ring and seg[0] stored; the per-halo fields, the ring
// depth and the other epilogues need segments = true.
int cc_launch_fwd(int N, bool segments, const CcFwdMaps& maps, const CcFwdLaunch& L, long long n_tiles, cudaStream_t stream);
// dynamic shared memory the forward kernel needs for these halos and this ring
inline int cc_fwd_smem(const CcFwdLaunch& L) {
    int halo = 0;
    for (int h = 0; h < L.halos; ++h) halo += L.kpad[h] * CC_PLANE * 4;
    return L.stages * L.stage_bytes + halo + CC_SMEM_SLACK;
}

// a (b, C, s, X, Y)-indexed activation with contiguous rows as the 5-D map (Y, X, s, C, b); strides in elements (X, s, C, b)
int cc_encode_map(CUtensorMap* map, const float* t, int Y, int X, int S, int C, int B, const long long (&strides)[4], cuuint32_t box_y,
                  cuuint32_t box_x, cuuint32_t box_c, CUtensorMapSwizzle swizzle, const char* what);

struct CcWgradMaps {
    CUtensorMap gy;                                // (Y, X, s, C_out, b), box (32, 1, 1, NO, 1), swizzle 128B
    CUtensorMap x;                                 // (Y, X, s, C_in, b), box (44, 1, 1, 64, 1), no swizzle
    CUtensorMap x_first;                           // read instead of x where the frame is -1 and `first` is set
};
// Totals of the weight gradient: frames counted by gy; partial (chunk, tap, o, ci) over all cout x cin.
struct CcShape {
    int batch, frames, X, Y, cin, cout, kt, taps;
};
// One launch's block: input channels ci0 .. ci0 + cin - 1 of the weight (x's channels 0 .. cin - 1, its frame t * fmul + foff + tau -
// (kt - 1)), output channels o0 .. o0 + n_o - 1 (gy's channels o0 ..).
struct CcWgradSeg {
    int ci0, cin, o0, n_o, fmul, foff, first;
};
long long cc_wgrad_tiles(const CcShape& s);
int cc_launch_wgrad(const CcWgradMaps& maps, const CcShape& s, const CcWgradSeg& seg, float* partial, int n_chunks, cudaStream_t stream);
// grad_w (cout, cin, kt, 3, 3) from the chunks' partials
int cc_wgrad_reduce(const CcShape& s, const float* partial, int n_chunks, float* gw, cudaStream_t stream);

}  // namespace fiery
