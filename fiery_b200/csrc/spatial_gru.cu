// The future prediction's SpatialGRU (fiery/layers/temporal.py:10-62) over T steps, forward and backward through time
// (include/fiery_b200.h, fiery_spatial_gru_*).  Per step t, with h the previous state (h0 at t = 0):
//
//   u = sigmoid(conv3x3([x_t, h], W_u) + b_u + g),  r = sigmoid(conv3x3([x_t, h], W_r) + b_r + g)
//   q = (1 - r) h,  s = conv3x3([x_t, q], W_s),  a = relu(BatchNorm2d(s)),  h' = (1 - u) h + u a  -> out[:, t]
//
// The convolutions are causal_conv.cu's kernels (causal_conv.cuh): each input segment ([x_t, h], [x_t, q]) is its own halo tile read
// from its own tensor, so no concat exists, and conv_update and conv_reset are one convolution with two output segments whose
// epilogue writes u, r and q.  The batch norm is batch_norm.cu's statistics and finalize on s, and its apply pass computes h' into
// the output frame.  The forward keeps u, r, q and s of every step (the backward needs u (1 - u), r (1 - r), the input q of the
// state convolution, and s for the norm); the states are the output itself.
//
// Backward, t = T-1 .. 0, with the state gradient `carry` (zero at T):
//   batch_norm.cu:  dh' = grad_out[:, t] + carry -> da = u dh', dG_u = dh' (a - h) u (1 - u), carry = (1 - u) dh';
//                   the BN + ReLU backward on (s, da) -> ds and the step's dgamma, dbeta;
//   state dgrad:    ds -> [dx_t, dq]; its epilogue turns dq into dG_r = -dq h r (1 - r) and carry += (1 - r) dq;
//   gate dgrad:     [dG_u, dG_r] -> [dx_t, dh]: added to dx_t and carry.
// Then one weight-gradient launch per (input segment, 64-output block) over all T steps in wgrad_chunks.cuh's order, the gates' bias
// gradient as per-channel sums of dG, and dgamma, dbeta summed over the steps in ascending order.  No atomics anywhere: the results
// are bit-reproducible.
#include "causal_conv.cuh"
#include "wgmma.cuh"
#include "wgrad_chunks.cuh"

namespace fiery {

int launch_gru_blend_forward(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* running_mean,
                             const float* running_var, const float* u, const float* h, long long hsb, float* out, long long osb,
                             float* mean_out, float* var_out, void* workspace, cudaStream_t stream);
int launch_gru_blend_backward(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* mean,
                              const float* var, const float* u, const float* h, long long hsb, const float* go, long long gsb, float* carry,
                              float* da, float* dgu, long long dsb, cudaStream_t stream);
size_t batch_norm_workspace_bytes(const fiery_batch_norm_desc_t* d);
int launch_batch_norm_backward(const fiery_batch_norm_desc_t* d, const float* x, const float* dy, const float* w, const float* bias,
                               const float* mean, const float* var, float* dx, float* grad_w, float* grad_b, void* workspace,
                               cudaStream_t stream);
int launch_batch_norm_local_stats(const fiery_batch_norm_desc_t* d, const float* x, double* stats, void* workspace, cudaStream_t stream);
int launch_gru_blend_forward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* w,
                                      const float* bias, const float* u, const float* h, long long hsb, float* out, long long osb,
                                      float* mean_out, float* var_out, double* count_out, void* workspace, cudaStream_t stream);
int launch_batch_norm_local_grad_sums(const fiery_batch_norm_desc_t* d, const float* x, const float* dy, const float* w, const float* bias,
                                      const float* mean, const float* var, double* sums, float* grad_w, float* grad_b, void* workspace,
                                      cudaStream_t stream);
int launch_batch_norm_backward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* dy,
                                        const float* w, const float* bias, const float* mean, const float* var, float* dx, void* workspace,
                                        cudaStream_t stream);

// accumulator columns of an output width: the instantiated N
static int gru_n(int n) { return n <= 64 ? cc_round8(n) : (n <= 96 ? 96 : 128); }

// One pack direction: rows (the MMA's N) in up to two segments, K in up to two halos; slice (halo h, tap) = ka[h] atoms of
// n rows x 32 k, 128-byte swizzle.  Forward packs read W[row, k]; transposed (input-gradient) packs W[k, row] with mirrored taps.
struct GruPack {
    int n, rseg, r0[2], rn[2], rbase[2];
    int halos, kn[2], kbase[2], kpad[2], ka[2], atom0[2];
    int transposed, cin_w;
    size_t floats;
};

static GruPack gru_pack(int rseg, const int (&rn)[2], const int (&rbase)[2], int halos, const int (&kn)[2], const int (&kbase)[2],
                        int transposed, int cin_w) {
    GruPack p{};
    p.rseg = rseg;
    int rows = 0;
    for (int i = 0; i < rseg; ++i) {
        p.r0[i] = rows;
        p.rn[i] = rn[i];
        p.rbase[i] = rbase[i];
        rows += cc_round8(rn[i]);
    }
    p.n = gru_n(rows);
    p.halos = halos;
    int atoms = 0;
    for (int h = 0; h < halos; ++h) {
        p.kn[h] = kn[h];
        p.kbase[h] = kbase[h];
        p.kpad[h] = cc_round8(kn[h]);
        p.ka[h] = (p.kpad[h] + 31) / 32;
        p.atom0[h] = atoms;
        atoms += 9 * p.ka[h];
    }
    p.transposed = transposed;
    p.cin_w = cin_w;
    p.floats = static_cast<size_t>(atoms) * p.n * 32;
    return p;
}

// the four packs: the gates' forward and input gradient, the state convolution's forward and input gradient
struct GruPacks {
    GruPack gate_f, gate_t, state_f, state_t;
    size_t off[4];
    size_t floats;
};

static GruPacks gru_packs(const fiery_spatial_gru_desc_t* d) {
    const int cx = d->x_channels, ch = d->h_channels;
    GruPacks P;
    P.gate_f = gru_pack(2, {ch, ch}, {0, ch}, 2, {cx, ch}, {0, cx}, 0, cx + ch);
    P.gate_t = gru_pack(2, {cx, ch}, {0, cx}, 2, {ch, ch}, {0, ch}, 1, cx + ch);
    P.state_f = gru_pack(1, {ch, 0}, {0, 0}, 2, {cx, ch}, {0, cx}, 0, cx + ch);
    P.state_t = gru_pack(2, {cx, ch}, {0, cx}, 1, {ch, 0}, {0, 0}, 1, cx + ch);
    const GruPack* all[4] = {&P.gate_f, &P.gate_t, &P.state_f, &P.state_t};
    size_t off = 0;
    for (int i = 0; i < 4; ++i) {
        P.off[i] = off;
        off += (all[i]->floats + 255) / 256 * 256;     // every pack 1024-byte aligned
    }
    P.floats = off;
    return P;
}

size_t spatial_gru_packed_bytes(const fiery_spatial_gru_desc_t* d) { return gru_packs(d).floats * sizeof(float); }

__global__ void gru_pack_kernel(GruPack p, const float* __restrict__ w, float* __restrict__ out) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= p.floats) return;
    const int k = static_cast<int>(i % 32), row = static_cast<int>(i / 32 % p.n);
    const int atom = static_cast<int>(i / 32 / p.n);
    const int h = (p.halos > 1 && atom >= p.atom0[1]) ? 1 : 0;
    const int tap = (atom - p.atom0[h]) / p.ka[h], a = (atom - p.atom0[h]) % p.ka[h];
    const int c = 32 * a + k;
    float v = 0.f;
    int wr = -1;
    for (int sg = 0; sg < p.rseg; ++sg)
        if (row >= p.r0[sg] && row < p.r0[sg] + p.rn[sg]) wr = p.rbase[sg] + row - p.r0[sg];
    if (wr >= 0 && c < p.kn[h]) {
        const int wk = p.kbase[h] + c;
        v = p.transposed ? w[(static_cast<size_t>(wk) * p.cin_w + wr) * 9 + 8 - tap] : w[(static_cast<size_t>(wr) * p.cin_w + wk) * 9 + tap];
        v = __uint_as_float(to_tf32(v));
    }
    out[i] = v;
}

int launch_spatial_gru_pack(const fiery_spatial_gru_desc_t* d, const float* w_gates, const float* w_state, float* packed, cudaStream_t stream) {
    const GruPacks P = gru_packs(d);
    const GruPack* all[4] = {&P.gate_f, &P.gate_t, &P.state_f, &P.state_t};
    for (int i = 0; i < 4; ++i) {
        gru_pack_kernel<<<static_cast<unsigned>((all[i]->floats + 255) / 256), 256, 0, stream>>>(*all[i], i < 2 ? w_gates : w_state,
                                                                                                 packed + P.off[i]);
        FIERY_CUDA_CHECK(cudaGetLastError());
    }
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------------------
struct GruGeom {
    int b, T, Tx, X, Y, cx, ch;
    long long XY, map_ch;                          // pixels; elements of one (b, ch) step buffer
};
static GruGeom gru_geom(const fiery_spatial_gru_desc_t* d) {
    GruGeom g;
    g.b = d->batch;
    g.T = d->frames;
    g.Tx = d->x_frames;
    g.X = d->grid_x;
    g.Y = d->grid_y;
    g.cx = d->x_channels;
    g.ch = d->h_channels;
    g.XY = static_cast<long long>(g.X) * g.Y;
    g.map_ch = static_cast<long long>(g.b) * g.ch * g.XY;
    return g;
}

// the maps of one conv: halos from tensors indexed (b, C, t, X, Y) with the given element strides (X, t, C, b)
static int gru_halo_map(CUtensorMap* m, const float* p, const GruGeom& g, int frames, int C, long long st, long long sc, long long sb,
                        int kpad, const char* what) {
    const long long strides[4] = {g.Y, st, sc, sb};
    return cc_encode_map(m, p, g.Y, g.X, frames, C, g.b, strides, CC_HY, CC_HX, static_cast<cuuint32_t>(kpad), CU_TENSOR_MAP_SWIZZLE_NONE,
                         what);
}

static int gru_weight_map(CUtensorMap* m, const float* w, const GruPack& p) {
    cuuint64_t dims[3] = {32, static_cast<cuuint64_t>(p.n), static_cast<cuuint64_t>(p.floats / 32 / p.n)};
    cuuint64_t strides[2] = {128, static_cast<cuuint64_t>(p.n) * 128};
    cuuint32_t box[3] = {32, static_cast<cuuint32_t>(p.n), 1};
    return encode_tensor_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, w, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "spatial GRU weights");
}

// the launch of one step's convolution with pack p: halos h at frames t_off[h] of maps map[h]; the ring as deep as shared memory allows
static CcFwdLaunch gru_launch(const GruGeom& g, const GruPack& p) {
    CcFwdLaunch L{};
    L.frames = 1;
    L.X = g.X;
    L.Y = g.Y;
    L.tiles_x = (g.X + CC_TX - 1) / CC_TX;
    L.tiles_y = (g.Y + CC_TY - 1) / CC_TY;
    L.halos = p.halos;
    int off = 0, stage = 0;
    for (int h = 0; h < p.halos; ++h) {
        L.map[h] = h;
        L.kpad[h] = p.kpad[h];
        L.ka[h] = p.ka[h];
        L.atom0[h] = p.atom0[h];
        L.x_off[h] = off;
        off += p.kpad[h] * CC_PLANE;
        stage = stage > p.ka[h] * p.n * 128 ? stage : p.ka[h] * p.n * 128;
    }
    L.stage_bytes = stage;
    L.stages = 1;
    L.stages = (CC_MAX_SMEM - cc_fwd_smem(L) + stage) / stage;
    if (L.stages > CC_WSTAGES) L.stages = CC_WSTAGES;
    return L;
}

static CcOutSeg gru_seg(float* p, long long sb, long long XY, int c0, int n, int mode) {
    CcOutSeg o{};
    o.p = p;
    o.sb = sb;
    o.sc = XY;
    o.st = 0;
    o.c0 = c0;
    o.n = n;
    o.mode = mode;
    return o;
}

// the saved tensors: u, r, q, s, each (T, b, ch, X, Y)
struct GruSaved {
    float *u, *r, *q, *s;
};
static GruSaved gru_saved(float* saved, const GruGeom& g) {
    const size_t n = static_cast<size_t>(g.T) * g.map_ch;
    return GruSaved{saved, saved + n, saved + 2 * n, saved + 3 * n};
}

static fiery_batch_norm_desc_t gru_bn_desc(const fiery_spatial_gru_desc_t* d, const GruGeom& g) {
    fiery_batch_norm_desc_t bn{};
    bn.batch = g.b;
    bn.channels = g.ch;
    bn.frames = 1;
    bn.pixels = static_cast<int>(g.XY);
    bn.stride_b = g.ch * g.XY;
    bn.stride_c = g.XY;
    bn.stride_t = 0;
    bn.training = d->training;
    bn.relu = 1;
    bn.eps = d->eps;
    return bn;
}

size_t spatial_gru_forward_workspace_bytes(const fiery_spatial_gru_desc_t* d) {
    const GruGeom g = gru_geom(d);
    const fiery_batch_norm_desc_t bn = gru_bn_desc(d, g);
    return batch_norm_workspace_bytes(&bn);
}

// The forward's maps and launches, set up once per call; gru_fwd_convs then runs step t's two convolutions.
struct GruFwd {
    GruGeom g;
    GruPacks P;
    GruSaved S;
    long long osb, ssb;
    CUtensorMap m_h0, m_out;
    CcFwdMaps gate, state;
    CcFwdLaunch Lg, Ls;
    long long n_tiles;
    fiery_batch_norm_desc_t bn;
};

static int gru_fwd_setup(const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* packed, const float* out,
                         float* saved, GruFwd& F) {
    const GruGeom& g = F.g = gru_geom(d);
    const GruPacks& P = F.P = gru_packs(d);
    F.S = gru_saved(saved, g);
    F.osb = static_cast<long long>(g.T) * g.ch * g.XY;
    F.ssb = g.ch * g.XY;
    const long long xst = g.Tx > 1 ? d->x_stride_t : 0;
    int rc;
    CUtensorMap m_x, m_q;
    if ((rc = gru_halo_map(&m_x, x, g, g.Tx, g.cx, g.Tx > 1 ? xst : g.XY, d->x_stride_c, d->x_stride_b, P.gate_f.kpad[0], "spatial GRU x")) ||
        (rc = gru_halo_map(&F.m_h0, h0, g, 1, g.ch, g.XY, g.XY, F.ssb, P.gate_f.kpad[1], "spatial GRU h0")) ||
        (rc = gru_halo_map(&F.m_out, out, g, g.T, g.ch, F.ssb, g.XY, F.osb, P.gate_f.kpad[1], "spatial GRU output")) ||
        (rc = gru_halo_map(&m_q, F.S.q, g, g.T, g.ch, g.map_ch, g.XY, F.ssb, P.state_f.kpad[1], "spatial GRU q")))
        return rc;
    if ((rc = gru_weight_map(&F.gate.w, packed + P.off[0], P.gate_f)) || (rc = gru_weight_map(&F.state.w, packed + P.off[2], P.state_f)))
        return rc;
    F.Lg = gru_launch(g, P.gate_f);
    F.Ls = gru_launch(g, P.state_f);
    F.Lg.nseg = 2;
    F.Lg.bias_init = d->bias_init;
    F.Ls.nseg = 1;
    F.n_tiles = static_cast<long long>(g.b) * F.Lg.tiles_x * F.Lg.tiles_y;
    F.bn = gru_bn_desc(d, g);
    F.gate.x[0] = m_x;
    F.state.x[0] = m_x;
    F.state.x[1] = m_q;
    return FIERY_OK;
}

// step t's input state: h0 at t = 0, else out[:, t - 1], and its batch stride
static const float* gru_h(const GruGeom& g, int t, const float* h0, const float* out, long long& hsb) {
    hsb = t == 0 ? g.ch * g.XY : static_cast<long long>(g.T) * g.ch * g.XY;
    return t == 0 ? h0 : out + static_cast<size_t>(t - 1) * g.ch * g.XY;
}

// step t's gates ([x_t, h] -> u, and r with q = (1 - r) h) and state convolution ([x_t, q] -> s)
static int gru_fwd_convs(GruFwd& F, int t, const float* h0, const float* out, const float* b_gates, cudaStream_t stream) {
    const GruGeom& g = F.g;
    const size_t so = static_cast<size_t>(t) * g.map_ch;
    long long hsb;
    const float* h = gru_h(g, t, h0, out, hsb);
    const int tx = g.Tx > 1 ? t : 0;
    int rc;
    F.gate.x[1] = t == 0 ? F.m_h0 : F.m_out;
    F.Lg.t_off[0] = tx;
    F.Lg.t_off[1] = t == 0 ? 0 : t - 1;
    F.Lg.seg[0] = gru_seg(F.S.u + so, F.ssb, g.XY, 0, g.ch, CC_GATE_U);
    F.Lg.seg[0].bias = b_gates;
    F.Lg.seg[1] = gru_seg(F.S.q + so, F.ssb, g.XY, cc_round8(g.ch), g.ch, CC_GATE_R);
    F.Lg.seg[1].bias = b_gates + g.ch;
    F.Lg.seg[1].h = h;
    F.Lg.seg[1].hsb = hsb;
    F.Lg.seg[1].r = F.S.r + so;
    F.Lg.seg[1].rsb = F.ssb;
    if ((rc = cc_launch_fwd(F.P.gate_f.n, true, F.gate, F.Lg, F.n_tiles, stream)) != FIERY_OK) return rc;
    F.Ls.t_off[0] = tx;
    F.Ls.t_off[1] = t;
    F.Ls.seg[0] = gru_seg(F.S.s + so, F.ssb, g.XY, 0, g.ch, CC_STORE);
    return cc_launch_fwd(F.P.state_f.n, true, F.state, F.Ls, F.n_tiles, stream);
}

int launch_spatial_gru_forward(const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* packed, const float* b_gates,
                               const float* bn_w, const float* bn_b, const float* running_mean, const float* running_var, float* out,
                               float* saved, float* means, float* vars, void* workspace, cudaStream_t stream) {
    GruFwd F;
    int rc;
    if ((rc = gru_fwd_setup(d, x, h0, packed, out, saved, F)) != FIERY_OK) return rc;
    const GruGeom& g = F.g;
    for (int t = 0; t < g.T; ++t) {
        const size_t so = static_cast<size_t>(t) * g.map_ch;
        long long hsb;
        const float* h = gru_h(g, t, h0, out, hsb);
        if ((rc = gru_fwd_convs(F, t, h0, out, b_gates, stream)) != FIERY_OK) return rc;
        // norm, ReLU and the blend into out[:, t]
        if ((rc = launch_gru_blend_forward(&F.bn, F.S.s + so, bn_w, bn_b, running_mean, running_var, F.S.u + so, h, hsb,
                                           out + static_cast<size_t>(t) * g.ch * g.XY, F.osb, means + static_cast<size_t>(t) * g.ch,
                                           vars + static_cast<size_t>(t) * g.ch, workspace, stream)) != FIERY_OK)
            return rc;
    }
    return FIERY_OK;
}

// The forward one step at a time, for statistics gathered over several ranks between the two calls: begin runs step t's
// convolutions and writes the rank's (n, mean, M2) of s; end merges the gathered triplets and blends into out[:, t].
int launch_spatial_gru_forward_step_begin(const fiery_spatial_gru_desc_t* d, int t, const float* x, const float* h0, const float* packed,
                                          const float* b_gates, const float* out, float* saved, double* stats, void* workspace,
                                          cudaStream_t stream) {
    GruFwd F;
    int rc;
    if ((rc = gru_fwd_setup(d, x, h0, packed, out, saved, F)) != FIERY_OK) return rc;
    if ((rc = gru_fwd_convs(F, t, h0, out, b_gates, stream)) != FIERY_OK) return rc;
    return launch_batch_norm_local_stats(&F.bn, F.S.s + static_cast<size_t>(t) * F.g.map_ch, stats, workspace, stream);
}

int launch_spatial_gru_forward_step_end(const fiery_spatial_gru_desc_t* d, int t, int world, const double* gathered, const float* h0,
                                        const float* bn_w, const float* bn_b, float* out, const float* saved_c, float* means, float* vars,
                                        double* count_out, void* workspace, cudaStream_t stream) {
    const GruGeom g = gru_geom(d);
    const GruSaved S = gru_saved(const_cast<float*>(saved_c), g);
    const fiery_batch_norm_desc_t bn = gru_bn_desc(d, g);
    const size_t so = static_cast<size_t>(t) * g.map_ch;
    long long hsb;
    const float* h = gru_h(g, t, h0, out, hsb);
    return launch_gru_blend_forward_gathered(&bn, world, gathered, S.s + so, bn_w, bn_b, S.u + so, h, hsb,
                                             out + static_cast<size_t>(t) * g.ch * g.XY, static_cast<long long>(g.T) * g.ch * g.XY,
                                             means + static_cast<size_t>(t) * g.ch, vars + static_cast<size_t>(t) * g.ch, count_out,
                                             workspace, stream);
}

// ------------------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------------------
// per-channel sums over (T * b) planes of X*Y: one CTA per channel, thread i adds elements i, i + 256, ... of each plane in
// ascending plane order, then a fixed tree; out[c] (= the gates' bias gradient)
__global__ void gru_channel_sums_kernel(const float* __restrict__ g, long long planes, int channels, long long XY, float* __restrict__ out) {
    __shared__ float sh[256];
    const int c = blockIdx.x;
    float acc = 0.f;
    for (long long pl = 0; pl < planes; ++pl) {
        const float* p = g + (pl * channels + c) * XY;
        for (long long i = threadIdx.x; i < XY; i += 256) acc += p[i];
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[c] = sh[0];
}

// out[c] = sum over t ascending of steps[t * n + c]
__global__ void gru_step_sums_kernel(const float* __restrict__ steps, int T, int n, float* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    float acc = 0.f;
    for (int t = 0; t < T; ++t) acc += steps[static_cast<size_t>(t) * n + c];
    out[c] = acc;
}

struct GruBwdWs {
    float *dg, *ds, *da, *carry, *dgam, *dbet, *partial;
    void* bn;
    size_t bytes;
};
static size_t gru_align(size_t b) { return (b + 255) / 256 * 256; }
static GruBwdWs gru_bwd_ws(const fiery_spatial_gru_desc_t* d, void* base) {
    const GruGeom g = gru_geom(d);
    const fiery_batch_norm_desc_t bn = gru_bn_desc(d, g);
    const CcShape sg{g.b, g.T, g.X, g.Y, g.cx + g.ch, 2 * g.ch, 1, 9};
    const int chunks = wgrad_chunks(cc_wgrad_tiles(sg), WG_MAX_CHUNKS);
    const size_t sizes[8] = {2 * static_cast<size_t>(g.T) * g.map_ch * 4, static_cast<size_t>(g.T) * g.map_ch * 4,
                             static_cast<size_t>(g.map_ch) * 4, static_cast<size_t>(g.map_ch) * 4,
                             static_cast<size_t>(g.T) * g.ch * 4, static_cast<size_t>(g.T) * g.ch * 4,
                             static_cast<size_t>(chunks) * 9 * 2 * g.ch * (g.cx + g.ch) * 4, batch_norm_workspace_bytes(&bn)};
    char* p = static_cast<char*>(base);
    size_t off[8], o = 0;
    for (int i = 0; i < 8; ++i) {
        off[i] = o;
        o += gru_align(sizes[i]);
    }
    GruBwdWs w;
    w.bytes = o;
    w.dg = reinterpret_cast<float*>(p + off[0]);
    w.ds = reinterpret_cast<float*>(p + off[1]);
    w.da = reinterpret_cast<float*>(p + off[2]);
    w.carry = reinterpret_cast<float*>(p + off[3]);
    w.dgam = reinterpret_cast<float*>(p + off[4]);
    w.dbet = reinterpret_cast<float*>(p + off[5]);
    w.partial = reinterpret_cast<float*>(p + off[6]);
    w.bn = p + off[7];
    return w;
}

size_t spatial_gru_backward_workspace_bytes(const fiery_spatial_gru_desc_t* d) { return gru_bwd_ws(d, nullptr).bytes; }

// a weight gradient over all T steps: input segments x (channels 0 .. cx - 1 of the weight) and the second segment (h-prev or q),
// output blocks of 64 channels of gy
static int gru_wgrad(const GruGeom& g, const fiery_spatial_gru_desc_t* d, const float* x, const CUtensorMap& m2, const CUtensorMap* m2_first,
                     int foff2, const float* gy, int cout, float* partial, float* gw, cudaStream_t stream) {
    const CcShape s{g.b, g.T, g.X, g.Y, g.cx + g.ch, cout, 1, 9};
    const int chunks = wgrad_chunks(cc_wgrad_tiles(s), WG_MAX_CHUNKS);
    int rc;
    CcWgradMaps maps;
    const long long gst[4] = {g.Y, static_cast<long long>(g.b) * cout * g.XY, g.XY, static_cast<long long>(cout) * g.XY};
    for (int seg = 0; seg < (g.ch > 0 ? 2 : 1); ++seg) {
        if (seg == 0) {
            const long long st[4] = {g.Y, g.Tx > 1 ? d->x_stride_t : g.XY, d->x_stride_c, d->x_stride_b};
            if ((rc = cc_encode_map(&maps.x, x, g.Y, g.X, g.Tx, g.cx, g.b, st, CC_WG_XP, 1, 64, CU_TENSOR_MAP_SWIZZLE_NONE,
                                    "spatial GRU x")) != FIERY_OK)
                return rc;
            maps.x_first = maps.x;
        } else {
            maps.x = m2;
            maps.x_first = m2_first ? *m2_first : m2;
        }
        for (int o0 = 0; o0 < cout; o0 += 64) {
            CcWgradSeg w;
            w.ci0 = seg == 0 ? 0 : g.cx;
            w.cin = seg == 0 ? g.cx : g.ch;
            w.o0 = o0;
            w.n_o = cout - o0 < 64 ? cout - o0 : 64;
            w.fmul = seg == 0 ? (g.Tx > 1 ? 1 : 0) : 1;
            w.foff = seg == 0 ? 0 : foff2;
            w.first = seg == 1 && m2_first != nullptr;
            // the block's gy box is exactly the NO = round8(n_o) rows its kernel's stage holds
            if ((rc = cc_encode_map(&maps.gy, gy, g.Y, g.X, g.T, cout, g.b, gst, CC_WG_PX, 1, static_cast<cuuint32_t>(cc_round8(w.n_o)),
                                    CU_TENSOR_MAP_SWIZZLE_128B, "spatial GRU gradient")) != FIERY_OK)
                return rc;
            if ((rc = cc_launch_wgrad(maps, s, w, partial, chunks, stream)) != FIERY_OK) return rc;
        }
    }
    return cc_wgrad_reduce(s, partial, chunks, gw, stream);
}

// The backward's maps and launches, set up once per call over the workspace W; gru_bwd_blend and gru_bwd_dgrads then run step t's
// parts, gru_bwd_weights the gradients over all steps.  The state gradient `carry` is grad_h0 when it is asked for, else W.carry.
struct GruBwd {
    GruGeom g;
    GruPacks P;
    GruSaved S;
    GruBwdWs W;
    long long osb, ssb, gsb, xsb;
    CcFwdMaps gate, state;
    CcFwdLaunch Lg, Ls;
    long long n_tiles;
    fiery_batch_norm_desc_t bn;
};

static int gru_bwd_setup(const fiery_spatial_gru_desc_t* d, const float* saved_c, const float* packed, void* workspace, GruBwd& B) {
    const GruGeom& g = B.g = gru_geom(d);
    const GruPacks& P = B.P = gru_packs(d);
    B.S = gru_saved(const_cast<float*>(saved_c), g);
    B.W = gru_bwd_ws(d, workspace);
    B.osb = static_cast<long long>(g.T) * g.ch * g.XY;
    B.ssb = g.ch * g.XY;
    B.gsb = 2 * B.ssb;
    B.xsb = static_cast<long long>(g.Tx) * g.cx * g.XY;     // grad_x: contiguous (b, Tx, cx, X, Y)
    B.bn = gru_bn_desc(d, g);
    int rc;
    CUtensorMap m_ds, m_dgu, m_dgr;
    if ((rc = gru_halo_map(&m_ds, B.W.ds, g, g.T, g.ch, g.map_ch, g.XY, B.ssb, P.state_t.kpad[0], "spatial GRU ds")) ||
        (rc = gru_halo_map(&m_dgu, B.W.dg, g, g.T, g.ch, 2 * g.map_ch, g.XY, B.gsb, P.gate_t.kpad[0], "spatial GRU dG_u")) ||
        (rc = gru_halo_map(&m_dgr, B.W.dg + g.ch * g.XY, g, g.T, g.ch, 2 * g.map_ch, g.XY, B.gsb, P.gate_t.kpad[1], "spatial GRU dG_r")))
        return rc;
    if ((rc = gru_weight_map(&B.gate.w, packed + P.off[1], P.gate_t)) || (rc = gru_weight_map(&B.state.w, packed + P.off[3], P.state_t)))
        return rc;
    B.gate.x[0] = m_dgu;
    B.gate.x[1] = m_dgr;
    B.state.x[0] = m_ds;
    B.state.x[1] = m_ds;
    B.Lg = gru_launch(g, P.gate_t);
    B.Ls = gru_launch(g, P.state_t);
    B.Lg.nseg = 2;
    B.Ls.nseg = 2;
    B.n_tiles = static_cast<long long>(g.b) * B.Lg.tiles_x * B.Lg.tiles_y;
    return FIERY_OK;
}

// step t's dh' = grad_out[:, t] + carry -> W.da, dG_u and the new carry
static int gru_bwd_blend(GruBwd& B, int t, const float* grad_out, const float* h0, const float* out, const float* means, const float* vars,
                         const float* bn_w, const float* bn_b, float* carry, cudaStream_t stream) {
    const GruGeom& g = B.g;
    const size_t so = static_cast<size_t>(t) * g.map_ch;
    long long hsb;
    const float* h = gru_h(g, t, h0, out, hsb);
    return launch_gru_blend_backward(&B.bn, B.S.s + so, bn_w, bn_b, means + static_cast<size_t>(t) * g.ch, vars + static_cast<size_t>(t) * g.ch,
                                     B.S.u + so, h, hsb, grad_out + static_cast<size_t>(t) * g.ch * g.XY, B.osb, carry, B.W.da,
                                     B.W.dg + 2 * so, B.gsb, stream);
}

// step t's input gradients from its ds: the state dgrad (ds -> [dx_t, dq]; dq -> dG_r, carry), then the gates' ([dG_u, dG_r] ->
// [dx_t, dh], both added)
static int gru_bwd_dgrads(GruBwd& B, int t, const float* h0, const float* out, float* grad_x, float* carry, cudaStream_t stream) {
    const GruGeom& g = B.g;
    const size_t so = static_cast<size_t>(t) * g.map_ch;
    long long hsb;
    const float* h = gru_h(g, t, h0, out, hsb);
    float* dg_t = B.W.dg + 2 * so;
    const int tx = g.Tx > 1 ? t : 0;
    float* dx_t = grad_x ? grad_x + static_cast<size_t>(tx) * g.cx * g.XY : nullptr;
    const bool first_dx = g.Tx > 1 || t == g.T - 1;       // the state dgrad is the first write of this dx frame
    int rc;
    B.Ls.t_off[0] = t;
    B.Ls.seg[0] = gru_seg(dx_t, B.xsb, g.XY, 0, g.cx, grad_x ? (first_dx ? CC_STORE : CC_ADD) : CC_SKIP);
    B.Ls.seg[1] = gru_seg(carry, B.ssb, g.XY, cc_round8(g.cx), g.ch, CC_RESET_GRAD);
    B.Ls.seg[1].h = h;
    B.Ls.seg[1].hsb = hsb;
    B.Ls.seg[1].r = B.S.r + so;
    B.Ls.seg[1].rsb = B.ssb;
    B.Ls.seg[1].aux = dg_t + g.ch * g.XY;
    B.Ls.seg[1].asb = B.gsb;
    if ((rc = cc_launch_fwd(B.P.state_t.n, true, B.state, B.Ls, B.n_tiles, stream)) != FIERY_OK) return rc;
    B.Lg.t_off[0] = t;
    B.Lg.t_off[1] = t;
    B.Lg.seg[0] = gru_seg(dx_t, B.xsb, g.XY, 0, g.cx, grad_x ? CC_ADD : CC_SKIP);
    B.Lg.seg[1] = gru_seg(carry, B.ssb, g.XY, cc_round8(g.cx), g.ch, CC_ADD);
    return cc_launch_fwd(B.P.gate_t.n, true, B.gate, B.Lg, B.n_tiles, stream);
}

static int gru_bwd_weights(GruBwd& B, const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* out,
                           float* grad_w_gates, float* grad_b_gates, float* grad_w_state, float* grad_bn_w, float* grad_bn_b,
                           cudaStream_t stream);

int launch_spatial_gru_backward(const fiery_spatial_gru_desc_t* d, const float* grad_out, const float* x, const float* h0, const float* out,
                                const float* saved_c, const float* means, const float* vars, const float* packed, const float* bn_w,
                                const float* bn_b, float* grad_x, float* grad_h0, float* grad_w_gates, float* grad_b_gates,
                                float* grad_w_state, float* grad_bn_w, float* grad_bn_b, void* workspace, cudaStream_t stream) {
    GruBwd B;
    int rc;
    if ((rc = gru_bwd_setup(d, saved_c, packed, workspace, B)) != FIERY_OK) return rc;
    const GruGeom& g = B.g;
    float* carry = grad_h0 ? grad_h0 : B.W.carry;
    FIERY_CUDA_CHECK(cudaMemsetAsync(carry, 0, static_cast<size_t>(g.map_ch) * 4, stream));
    for (int t = g.T - 1; t >= 0; --t) {
        const size_t so = static_cast<size_t>(t) * g.map_ch;
        // dh' -> da, dG_u, carry; then the norm's backward -> ds
        if ((rc = gru_bwd_blend(B, t, grad_out, h0, out, means, vars, bn_w, bn_b, carry, stream)) != FIERY_OK) return rc;
        if ((rc = launch_batch_norm_backward(&B.bn, B.S.s + so, B.W.da, bn_w, bn_b, means + static_cast<size_t>(t) * g.ch,
                                             vars + static_cast<size_t>(t) * g.ch, B.W.ds + so, B.W.dgam + static_cast<size_t>(t) * g.ch,
                                             B.W.dbet + static_cast<size_t>(t) * g.ch, B.W.bn, stream)) != FIERY_OK)
            return rc;
        if ((rc = gru_bwd_dgrads(B, t, h0, out, grad_x, carry, stream)) != FIERY_OK) return rc;
    }
    return gru_bwd_weights(B, d, x, h0, out, grad_w_gates, grad_b_gates, grad_w_state, grad_bn_w, grad_bn_b, stream);
}

// The backward one step at a time (t = T-1 .. 0), for statistics gathered over several ranks between the two calls: begin runs the
// blend's gradient and writes the rank's (n, S1, S2) of the norm's backward (and the step's local dgamma, dbeta); end merges the
// gathered triplets into ds and runs the step's input gradients.  The workspace and grad_h0 (or NULL) are the same in every call.
int launch_spatial_gru_backward_step_begin(const fiery_spatial_gru_desc_t* d, int t, const float* grad_out, const float* h0, const float* out,
                                           const float* saved_c, const float* means, const float* vars, const float* packed,
                                           const float* bn_w, const float* bn_b, float* grad_h0, double* sums, void* workspace,
                                           cudaStream_t stream) {
    GruBwd B;
    int rc;
    if ((rc = gru_bwd_setup(d, saved_c, packed, workspace, B)) != FIERY_OK) return rc;
    const GruGeom& g = B.g;
    float* carry = grad_h0 ? grad_h0 : B.W.carry;
    if (t == g.T - 1) FIERY_CUDA_CHECK(cudaMemsetAsync(carry, 0, static_cast<size_t>(g.map_ch) * 4, stream));
    if ((rc = gru_bwd_blend(B, t, grad_out, h0, out, means, vars, bn_w, bn_b, carry, stream)) != FIERY_OK) return rc;
    return launch_batch_norm_local_grad_sums(&B.bn, B.S.s + static_cast<size_t>(t) * g.map_ch, B.W.da, bn_w, bn_b,
                                             means + static_cast<size_t>(t) * g.ch, vars + static_cast<size_t>(t) * g.ch, sums,
                                             B.W.dgam + static_cast<size_t>(t) * g.ch, B.W.dbet + static_cast<size_t>(t) * g.ch, B.W.bn, stream);
}

int launch_spatial_gru_backward_step_end(const fiery_spatial_gru_desc_t* d, int t, int world, const double* gathered, const float* h0,
                                         const float* out, const float* saved_c, const float* means, const float* vars, const float* packed,
                                         const float* bn_w, const float* bn_b, float* grad_x, float* grad_h0, void* workspace,
                                         cudaStream_t stream) {
    GruBwd B;
    int rc;
    if ((rc = gru_bwd_setup(d, saved_c, packed, workspace, B)) != FIERY_OK) return rc;
    const GruGeom& g = B.g;
    const size_t so = static_cast<size_t>(t) * g.map_ch;
    if ((rc = launch_batch_norm_backward_gathered(&B.bn, world, gathered, B.S.s + so, B.W.da, bn_w, bn_b, means + static_cast<size_t>(t) * g.ch,
                                                  vars + static_cast<size_t>(t) * g.ch, B.W.ds + so, B.W.bn, stream)) != FIERY_OK)
        return rc;
    return gru_bwd_dgrads(B, t, h0, out, grad_x, grad_h0 ? grad_h0 : B.W.carry, stream);
}

int launch_spatial_gru_backward_weights(const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* out, const float* saved_c,
                                        const float* packed, float* grad_w_gates, float* grad_b_gates, float* grad_w_state, float* grad_bn_w,
                                        float* grad_bn_b, void* workspace, cudaStream_t stream) {
    GruBwd B;
    int rc;
    if ((rc = gru_bwd_setup(d, saved_c, packed, workspace, B)) != FIERY_OK) return rc;
    return gru_bwd_weights(B, d, x, h0, out, grad_w_gates, grad_b_gates, grad_w_state, grad_bn_w, grad_bn_b, stream);
}

// the weight gradients over all steps, the gates' bias gradient, and dgamma, dbeta summed over the steps in ascending order
static int gru_bwd_weights(GruBwd& B, const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* out,
                           float* grad_w_gates, float* grad_b_gates, float* grad_w_state, float* grad_bn_w, float* grad_bn_b,
                           cudaStream_t stream) {
    const GruGeom& g = B.g;
    const GruBwdWs& W = B.W;
    const long long osb = B.osb, ssb = B.ssb;
    const GruSaved& S = B.S;
    int rc;
    CUtensorMap m_out, m_h0, m_q;
    if (grad_w_gates || grad_w_state) {
        const long long bst[4] = {g.Y, ssb, g.XY, osb};
        const long long hst[4] = {g.Y, ssb, g.XY, ssb};
        const long long qst[4] = {g.Y, g.map_ch, g.XY, ssb};
        if ((rc = cc_encode_map(&m_out, out, g.Y, g.X, g.T, g.ch, g.b, bst, CC_WG_XP, 1, 64, CU_TENSOR_MAP_SWIZZLE_NONE, "spatial GRU output")) ||
            (rc = cc_encode_map(&m_h0, h0, g.Y, g.X, 1, g.ch, g.b, hst, CC_WG_XP, 1, 64, CU_TENSOR_MAP_SWIZZLE_NONE, "spatial GRU h0")) ||
            (rc = cc_encode_map(&m_q, S.q, g.Y, g.X, g.T, g.ch, g.b, qst, CC_WG_XP, 1, 64, CU_TENSOR_MAP_SWIZZLE_NONE, "spatial GRU q")))
            return rc;
        if (grad_w_gates && (rc = gru_wgrad(g, d, x, m_out, &m_h0, -1, W.dg, 2 * g.ch, W.partial, grad_w_gates, stream)) != FIERY_OK)
            return rc;
        if (grad_w_state && (rc = gru_wgrad(g, d, x, m_q, nullptr, 0, W.ds, g.ch, W.partial, grad_w_state, stream)) != FIERY_OK) return rc;
    }
    if (grad_b_gates) {
        gru_channel_sums_kernel<<<2 * g.ch, 256, 0, stream>>>(W.dg, static_cast<long long>(g.T) * g.b, 2 * g.ch, g.XY, grad_b_gates);
        FIERY_CUDA_CHECK(cudaGetLastError());
    }
    if (grad_bn_w) gru_step_sums_kernel<<<(g.ch + 127) / 128, 128, 0, stream>>>(W.dgam, g.T, g.ch, grad_bn_w);
    if (grad_bn_b) gru_step_sums_kernel<<<(g.ch + 127) / 128, 128, 0, stream>>>(W.dbet, g.T, g.ch, grad_bn_b);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------
// The 3x3 convolution of two input segments into two output segments on its own (fiery_conv3x3_*): the same packs, launches and
// weight-gradient blocks as the GRU's, with plain stores, so the kernels can be checked on their own.
// ------------------------------------------------------------------------------------------------------------------------------
static GruGeom conv3x3_geom(const fiery_conv3x3_desc_t* d) {
    GruGeom g;
    g.b = d->maps;
    g.T = g.Tx = 1;
    g.X = d->grid_x;
    g.Y = d->grid_y;
    g.cx = d->in_channels[0];
    g.ch = d->in_channels[1];
    g.XY = static_cast<long long>(g.X) * g.Y;
    g.map_ch = g.b * g.ch * g.XY;
    return g;
}
static GruPack conv3x3_pack(const fiery_conv3x3_desc_t* d, int transposed) {
    const int i0 = d->in_channels[0], i1 = d->in_channels[1], o0 = d->out_channels[0], o1 = d->out_channels[1];
    return transposed ? gru_pack(i1 ? 2 : 1, {i0, i1}, {0, i0}, o1 ? 2 : 1, {o0, o1}, {0, o0}, 1, i0 + i1)
                      : gru_pack(o1 ? 2 : 1, {o0, o1}, {0, o0}, i1 ? 2 : 1, {i0, i1}, {0, i0}, 0, i0 + i1);
}
static size_t conv3x3_t_offset(const fiery_conv3x3_desc_t* d) { return (conv3x3_pack(d, 0).floats + 255) / 256 * 256; }

size_t conv3x3_packed_bytes(const fiery_conv3x3_desc_t* d) { return (conv3x3_t_offset(d) + conv3x3_pack(d, 1).floats) * sizeof(float); }

int launch_conv3x3_pack(const fiery_conv3x3_desc_t* d, const float* w, float* packed, cudaStream_t stream) {
    for (int tr = 0; tr < 2; ++tr) {
        const GruPack p = conv3x3_pack(d, tr);
        gru_pack_kernel<<<static_cast<unsigned>((p.floats + 255) / 256), 256, 0, stream>>>(p, w, packed + (tr ? conv3x3_t_offset(d) : 0));
        FIERY_CUDA_CHECK(cudaGetLastError());
    }
    return FIERY_OK;
}

// dgrad = 0: (x0, x1) -> (y0, y1) with the forward pack; 1: (gy0, gy1) -> (gx0, gx1) with the transposed one
int launch_conv3x3(const fiery_conv3x3_desc_t* d, int dgrad, const float* in0, const float* in1, const float* packed, float* out0,
                   float* out1, cudaStream_t stream) {
    const GruGeom g = conv3x3_geom(d);
    const GruPack p = conv3x3_pack(d, dgrad);
    const int* kin = dgrad ? d->out_channels : d->in_channels;
    const int* kout = dgrad ? d->in_channels : d->out_channels;
    CcFwdMaps maps;
    int rc;
    const float* ins[2] = {in0, in1};
    for (int h = 0; h < p.halos; ++h)
        if ((rc = gru_halo_map(&maps.x[h], ins[h], g, 1, kin[h], g.XY, g.XY, kin[h] * g.XY, p.kpad[h], "3x3 conv input")) != FIERY_OK) return rc;
    if (p.halos == 1) maps.x[1] = maps.x[0];
    if ((rc = gru_weight_map(&maps.w, packed + (dgrad ? conv3x3_t_offset(d) : 0), p)) != FIERY_OK) return rc;
    CcFwdLaunch L = gru_launch(g, p);
    L.nseg = p.rseg;
    L.seg[0] = gru_seg(out0, kout[0] * g.XY, g.XY, 0, kout[0], CC_STORE);
    if (p.rseg > 1) L.seg[1] = gru_seg(out1, kout[1] * g.XY, g.XY, cc_round8(kout[0]), kout[1], CC_STORE);
    return cc_launch_fwd(p.n, true, maps, L, static_cast<long long>(g.b) * L.tiles_x * L.tiles_y, stream);
}

static fiery_spatial_gru_desc_t conv3x3_x_desc(const GruGeom& g) {
    fiery_spatial_gru_desc_t x{};
    x.x_stride_b = g.cx * g.XY;
    x.x_stride_t = g.cx * g.XY;
    x.x_stride_c = g.XY;
    return x;
}

size_t conv3x3_wgrad_workspace_bytes(const fiery_conv3x3_desc_t* d) {
    const GruGeom g = conv3x3_geom(d);
    const CcShape s{g.b, 1, g.X, g.Y, g.cx + g.ch, d->out_channels[0] + d->out_channels[1], 1, 9};
    return static_cast<size_t>(wgrad_chunks(cc_wgrad_tiles(s), WG_MAX_CHUNKS)) * 9 * s.cout * s.cin * sizeof(float);
}

int launch_conv3x3_wgrad(const fiery_conv3x3_desc_t* d, const float* x0, const float* x1, const float* gy, float* gw, void* workspace,
                         cudaStream_t stream) {
    const GruGeom g = conv3x3_geom(d);
    const fiery_spatial_gru_desc_t xd = conv3x3_x_desc(g);
    CUtensorMap m1;
    int rc;
    if (g.ch > 0) {
        const long long st[4] = {g.Y, g.XY, g.XY, g.ch * g.XY};
        if ((rc = cc_encode_map(&m1, x1, g.Y, g.X, 1, g.ch, g.b, st, CC_WG_XP, 1, 64, CU_TENSOR_MAP_SWIZZLE_NONE, "3x3 conv x1")) != FIERY_OK)
            return rc;
    }
    return gru_wgrad(g, &xd, x0, m1, nullptr, 0, gy, d->out_channels[0] + d->out_channels[1], static_cast<float*>(workspace), gw, stream);
}

}  // namespace fiery
