// Backward of the camera->BEV lift for sm_90a: gradient of the BEV features w.r.t. the head tensor (depth logits + context), i.e.
// autograd through fiery/models/encoder.py:99-100 (softmax, outer product) and fiery/utils/geometry.py:305-314
// (VoxelsSumming.backward = "send the voxel's gradient to every point summed into it") without ever materialising the (N, C) point
// gradient the reference builds.
//
// Per point (pixel p = (camera, row, column), depth d) with pillar pi(p, d) and G = grad_bev[:, pi]:
//     g_ctx[p][c]   = sum_d prob[p][d] * G[pi(p,d)][c]
//     g_prob[p][d]  = sum_c ctx[p][c]  * G[pi(p,d)][c]
//     g_logit[p][d] = prob[p][d] * (g_prob[p][d] - sum_d' prob[p][d'] g_prob[p][d'])          (softmax backward)
//
// Built like the forward tile kernel (lift_fwd_cols.cu):
//   * the tile (one camera image x 4 feature columns) arrives by TMA in the layouts prob[row][depth][col4] and
//     ctx[row][k][cl][col4] (channel 8*cl + k): the tensor maps do the permutation, nothing is transposed in shared memory, and the
//     results leave through the same maps (TMA stores);
//   * WHERE the points land comes from the geometry plan (lift_plan.cu), shared with the forward: per (row group, column, slot)
//     the plan lists the pillars of the runs in exactly the order this kernel consumes them ("streams");
//   * thread = (row group, column, 8 channels): pixels are independent in the backward, so a warp (4 columns x 8 channel lanes)
//     walks its <= 8 rows for one group of 4 depths at a time with the 4 x 8 gradient values G of the current pillars in
//     registers.  g_ctx accumulates in registers over the depth loop (no cross-thread reduction); g_prob is reduced over the 8
//     channel lanes with a transposing shuffle butterfly (4 SHFL per row and depth group);
//   * G gathers are software-pipelined two runs deep: registers hold the current run's gradient row, the next run's row
//     (already in flight) and the pillar of the run after that, so neither the pillar lookup nor the 256-byte gather is waited for.
#include "lift_plan.cuh"

namespace fiery {

constexpr int BW_CH = 8;                     // channels per lane: 8 lanes cover C = 64
constexpr int BW_ND = PLAN_ND;               // depths per depth group
constexpr int BW_NG = DPAD / BW_ND;          // depth groups
constexpr int BW_NT = 32 * PLAN_RG;          // threads: one warp per row group
constexpr int BW_MAXR = PLAN_MAX_ROWS / PLAN_RG;   // rows per thread

struct BwdLayout {
    int hh;
    int off_bar, off_mask, off_soff, off_prob, off_gprob, off_ctx, total;
    __host__ __device__ explicit BwdLayout(int hh_) : hh(hh_) {
        int o = 0;
        off_bar = o;    o += 16;
        off_mask = o;   o += PLAN_PAIRS * 4;
        off_soff = o;   o += PLAN_STREAMS * 2;
        o = (o + 127) & ~127;
        off_prob = o;   o += hh * DPAD * WT * 4;        // prob[row][depth][col4]
        o = (o + 127) & ~127;
        off_gprob = o;  o += hh * DPAD * WT * 4;        // g_prob, then g_logit, same layout
        o = (o + 127) & ~127;
        off_ctx = o;    o += hh * 64 * WT * 4;          // ctx[row][k][cl][col4], overwritten by g_ctx at the end
        total = o;
    }
};

// helpers on pairs of fp32 values held in one 64-bit register pair (two FFMA / FMUL each)
__device__ __forceinline__ unsigned long long pack2(float lo, float hi) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void unpack2(unsigned long long v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ unsigned long long mul2(unsigned long long a, unsigned long long b) {
    unsigned long long r;
    asm("{\n\t.reg .f32 a0, a1, b0, b1;\n\t"
        "mov.b64 {a0, a1}, %1;\n\tmov.b64 {b0, b1}, %2;\n\t"
        "mul.rn.f32 a0, a0, b0;\n\tmul.rn.f32 a1, a1, b1;\n\t"
        "mov.b64 %0, {a0, a1};\n\t}" : "=l"(r) : "l"(a), "l"(b));
    return r;
}

// One step of a slot's gather pipeline, for the lanes where `pred` != 0, as one block of straight-line predicated code (a
// conditional C++ assignment inside the unrolled row loop makes ptxas shuffle the whole register set):
//   G   <- Gn                        the run that was "next" becomes current
//   Gn  <- gradient row of `pnn`     (zeros for a masked run, pnn < 0): 2 x 16-byte loads of this lane's 8 channels
//   pnn <- streams[sp], sp += 1      the pillar of the run after that
// gbev: this lane's 8 channels of pillar 0 of the frame (channel-last rows of 64 floats = 256 bytes).
__device__ __forceinline__ void advance_slot(unsigned long long (&G)[4], unsigned long long (&Gn)[4], int& pnn, int& sp,
                                             const float* gbev, const int* streams, unsigned pred) {
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t.reg .b64 a;\n\t.reg .b32 c;\n\t"
        "setp.ne.u32 p, %12, 0;\n\t"
        "setp.ge.and.s32 q, %8, 0, p;\n\t"
        "max.s32 c, %8, 0;\n\t"
        "mad.wide.u32 a, c, 256, %10;\n\t"
        "@p mov.b64 %0, %4;\n\t@p mov.b64 %1, %5;\n\t@p mov.b64 %2, %6;\n\t@p mov.b64 %3, %7;\n\t"
        "@p mov.b64 %4, 0;\n\t@p mov.b64 %5, 0;\n\t@p mov.b64 %6, 0;\n\t@p mov.b64 %7, 0;\n\t"
        "@q ld.global.nc.v2.b64 {%4, %5}, [a];\n\t"
        "@q ld.global.nc.v2.b64 {%6, %7}, [a + 16];\n\t"
        "mad.wide.s32 a, %9, 4, %11;\n\t"
        "@p ld.global.nc.b32 %8, [a];\n\t"
        "@p add.s32 %9, %9, 1;\n\t}"
        : "+l"(G[0]), "+l"(G[1]), "+l"(G[2]), "+l"(G[3]), "+l"(Gn[0]), "+l"(Gn[1]), "+l"(Gn[2]), "+l"(Gn[3]), "+r"(pnn), "+r"(sp)
        : "l"(gbev), "l"(streams), "r"(pred)
        : "memory");
}

// MAXR: rows per thread the row loop is unrolled for (ceil(h / 4) <= MAXR); the g_ctx accumulators take 8 registers per row
template <int MAXR>
__global__ void __launch_bounds__(BW_NT, 3)
lift_backward_kernel(const __grid_constant__ HeadMapsCols head_maps, const __grid_constant__ HeadMapsCols grad_maps, const LiftParams P) {
    extern __shared__ __align__(128) unsigned char smem[];
    const BwdLayout L(P.hh);
    const int wtile = blockIdx.x % P.n_wtiles;
    const int img = blockIdx.x / P.n_wtiles;           // (frame, camera): the backward takes the whole batch in one launch
    const int frame = img / P.n_cameras;
    const int w0 = wtile * WT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int hh = L.hh;
    const unsigned char* rec = P.plan_tiles + static_cast<size_t>(blockIdx.x) * PLAN_TILE_BYTES;

    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L.off_bar);
    float* s_prob = reinterpret_cast<float*>(smem + L.off_prob);
    float* s_gprob = reinterpret_cast<float*>(smem + L.off_gprob);
    float* s_ctx = reinterpret_cast<float*>(smem + L.off_ctx);
    unsigned* s_mask = reinterpret_cast<unsigned*>(smem + L.off_mask);
    unsigned short* s_soff = reinterpret_cast<unsigned short*>(smem + L.off_soff);
    if (tid == 0) {
        tma_prefetch_desc(&head_maps.depth);
        tma_prefetch_desc(&head_maps.ctx);
        mbar_init(bar, 1);
        fence_mbar_init();
        const uint32_t prob_bytes = P.use_depth ? static_cast<uint32_t>(hh * DPAD * WT * 4) : 0u;
        mbar_arrive_expect_tx(bar, prob_bytes + static_cast<uint32_t>(hh * 64 * WT * 4));
        if (P.use_depth) tma_load_4d(s_prob, &head_maps.depth, bar, w0, 0, 0, img);
        tma_load_5d(s_ctx, &head_maps.ctx, bar, w0, 0, 0, 0, img);
    }
    for (int i = tid; i < PLAN_PAIRS; i += BW_NT) s_mask[i] = __ldg(reinterpret_cast<const unsigned*>(rec + PLAN_OFF_MASK) + i);
    if (tid < PLAN_STREAMS) s_soff[tid] = __ldg(reinterpret_cast<const unsigned short*>(rec + PLAN_OFF_SOFF) + tid);
    __syncthreads();                                   // plan header staged, the mbarrier is set up
    mbar_wait(bar, 0);                                 // head tile has landed
    softmax_depth<BW_NT>(P, s_prob, hh);
    __syncthreads();

    // ---- main loop: warp = row group, lane = (column, 8-channel lane) ------------------------------------------------------------
    const int col = lane >> 3, cl = lane & 7;
    const int r_lo = plan_group_row(hh, warp);
    const int R = plan_group_row(hh, warp + 1) - r_lo;
    const unsigned upto_lo = (2u << r_lo) - 1u;
    const unsigned upto_hi = (r_lo + R) >= 32 ? 0xffffffffu : ((1u << (r_lo + R)) - 1u);
    const unsigned in_group = upto_hi & ~upto_lo;      // rows r_lo+1 .. r_lo+R-1: where a run may start inside my rows
    const float* gbev = P.grad_bev + static_cast<size_t>(frame) * P.pillars * P.C + cl * BW_CH;   // channel-last
    const int* streams = reinterpret_cast<const int*>(rec + PLAN_OFF_STREAMS);
    const bool b2 = cl & 4, b1 = cl & 2;
    const int jsel = (b2 ? 2 : 0) + (b1 ? 1 : 0);      // the depth (within the group) whose g_prob this lane ends up holding

    unsigned long long gc[MAXR][4];                 // g_ctx of my rows x channel pairs (8cl + 2m, 8cl + 2m + 1)
#pragma unroll
    for (int i = 0; i < MAXR; ++i)
#pragma unroll
        for (int m = 0; m < 4; ++m) gc[i][m] = 0ull;

    // gather pipeline of my four slots: G = current run, Gn = next run (in flight), pnn = pillar of the run after that
    unsigned long long G[BW_ND][4], Gn[BW_ND][4];
    int pnn[BW_ND], sp[BW_ND];
#pragma unroll
    for (int j = 0; j < BW_ND; ++j) {
        sp[j] = s_soff[(warp * WT + col) * BW_ND + j];
#pragma unroll
        for (int m = 0; m < 4; ++m) G[j][m] = Gn[j][m] = 0ull;
    }
    if (R > 0) {
#pragma unroll
        for (int j = 0; j < BW_ND; ++j) {                           // prime: Gn <- run 0, pnn <- pillar of run 1
            pnn[j] = __ldg(streams + sp[j]);
            ++sp[j];
            advance_slot(G[j], Gn[j], pnn[j], sp[j], gbev, streams, 1u);
        }
        float ps[BW_ND] = {0.f, 0.f, 0.f, 0.f};                    // g_prob partial sums of the previous row (reduced one row late)
        // transposing butterfly over the 8 channel lanes: 4 values -> 1 per lane, summed over all 8 lanes.  It runs one row
        // behind the FMAs (its three dependent shuffles hide under the next row's arithmetic).
        auto reduce_and_store = [&](const float (&v4)[BW_ND], int off) {
            const float send0 = b2 ? v4[0] : v4[2], keep0 = b2 ? v4[2] : v4[0];
            const float send1 = b2 ? v4[1] : v4[3], keep1 = b2 ? v4[3] : v4[1];
            const float a0 = keep0 + __shfl_xor_sync(0xffffffffu, send0, 4);
            const float a1 = keep1 + __shfl_xor_sync(0xffffffffu, send1, 4);
            const float send = b1 ? a0 : a1, keep = b1 ? a1 : a0;
            float v = keep + __shfl_xor_sync(0xffffffffu, send, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            if (!(cl & 1)) s_gprob[off + jsel * WT] = v;
        };
        for (int g = 0; g < BW_NG; ++g) {
            unsigned cm[BW_ND], anyj[BW_ND];
            unsigned anyrow = 0;
#pragma unroll
            for (int j = 0; j < BW_ND; ++j) {
                cm[j] = s_mask[((g * BW_ND + j) << 2) + col] & in_group;      // rows where my column's slot j enters another pillar
                anyj[j] = __reduce_or_sync(0xffffffffu, cm[j]);                // ... where any column of the warp does
                anyrow |= anyj[j];
            }
            // the first run of the depth group (g = 0 takes the same path: the primed rows move from Gn to G here)
#pragma unroll
            for (int j = 0; j < BW_ND; ++j) advance_slot(G[j], Gn[j], pnn[j], sp[j], gbev, streams, 1u);
#pragma unroll
            for (int i = 0; i < MAXR; ++i) {
                if (i < R) {
                    const int h = r_lo + i;
                    const float* pr = s_prob + (h * DPAD + g * BW_ND) * WT + col;
                    const float* cx = s_ctx + h * 64 * WT + cl * WT + col;
                    if (i > 0 && ((anyrow >> h) & 1u)) {            // warp-uniform: some slot of some column changes pillar here
#pragma unroll
                        for (int j = 0; j < BW_ND; ++j)
                            if ((anyj[j] >> h) & 1u) advance_slot(G[j], Gn[j], pnn[j], sp[j], gbev, streams, (cm[j] >> h) & 1u);
                    }
                    // the operands of the row after the run changes (loading them before keeps more registers live)
                    float pv[BW_ND];
                    unsigned long long cp[4];
#pragma unroll
                    for (int j = 0; j < BW_ND; ++j) pv[j] = pr[j * WT];
#pragma unroll
                    for (int m = 0; m < 4; ++m) cp[m] = pack2(cx[(2 * m) * 8 * WT], cx[(2 * m + 1) * 8 * WT]);
                    float sj[BW_ND];
#pragma unroll
                    for (int j = 0; j < BW_ND; ++j) {
                        const unsigned long long pp = pack2(pv[j], pv[j]);
#pragma unroll
                        for (int m = 0; m < 4; ++m) ffma2(gc[i][m], pp, G[j][m]);          // g_ctx += prob * G
                        unsigned long long t = mul2(cp[0], G[j][0]);                          // ctx . G over my 8 channels
                        ffma2(t, cp[1], G[j][1]);
                        ffma2(t, cp[2], G[j][2]);
                        ffma2(t, cp[3], G[j][3]);
                        float lo, hi;
                        unpack2(t, lo, hi);
                        sj[j] = lo + hi;
                    }
                    if (P.use_depth) {
                        if (i > 0) reduce_and_store(ps, ((h - 1) * DPAD + g * BW_ND) * WT + col);   // the previous row's g_prob
#pragma unroll
                        for (int j = 0; j < BW_ND; ++j) ps[j] = sj[j];
                    }
                }
            }
            // the last row of the group: its shuffles overlap with the set-up of the next depth group
            if (P.use_depth) reduce_and_store(ps, ((r_lo + R - 1) * DPAD + g * BW_ND) * WT + col);
        }
    }
    // ---- g_ctx registers -> the ctx region, same layout (every thread overwrites exactly the entries only it read) -------------------
#pragma unroll
    for (int i = 0; i < MAXR; ++i) {
        if (i < R) {
            float* cx = s_ctx + (r_lo + i) * 64 * WT + cl * WT + col;
#pragma unroll
            for (int m = 0; m < 4; ++m) {
                float lo, hi;
                unpack2(gc[i][m], lo, hi);
                cx[(2 * m) * 8 * WT] = lo;
                cx[(2 * m + 1) * 8 * WT] = hi;
            }
        }
    }
    __syncthreads();                                   // g_prob of all rows complete

    // ---- softmax backward in place on g_prob: lane = (d mod 8, column) as in the forward softmax ------------------------------------
    if (P.use_depth) {
        const int c8 = lane >> 2, scol = lane & 3;
        for (int row = warp; row < hh; row += BW_NT / 32) {
            const int o = (row * DPAD + c8) * WT + scol;
            float pv[DPAD / 8], gv[DPAD / 8];
            float dot = 0.f;
#pragma unroll
            for (int k = 0; k < DPAD / 8; ++k) {
                pv[k] = s_prob[o + k * 8 * WT];
                gv[k] = s_gprob[o + k * 8 * WT];
                dot = fmaf(pv[k], gv[k], dot);
            }
            dot += __shfl_xor_sync(0xffffffffu, dot, 4);
            dot += __shfl_xor_sync(0xffffffffu, dot, 8);
            dot += __shfl_xor_sync(0xffffffffu, dot, 16);
#pragma unroll
            for (int k = 0; k < DPAD / 8; ++k) s_gprob[o + k * 8 * WT] = pv[k] * (gv[k] - dot);
        }
    }
    fence_proxy_async();       // generic-proxy writes -> visible to the TMA (async proxy)
    __syncthreads();
    if (tid == 0) {
        if (P.use_depth) tma_store_4d(&grad_maps.depth, s_gprob, w0, 0, 0, img);
        tma_store_5d(&grad_maps.ctx, s_ctx, w0, 0, 0, 0, img);
        tma_store_commit_and_wait();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// grad_bev (B', C, X*Y) -> channel-last workspace (B', X*Y, C).  The backward only gathers the rows of pillars that receive a
// point (~1/3 of the grid, clustered around the rig): with the plan's touched map a block of 64 pillars that has none is skipped
// entirely -- neither read nor written.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int TR_PILLARS = 64;
__global__ void __launch_bounds__(256)
nchw_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, const unsigned char* __restrict__ touched, int C,
                    long long pillars, int blocks_per_frame) {
    __shared__ float tile[TR_PILLARS][65];
    const int frame = blockIdx.x / blocks_per_frame;
    const long long p0 = static_cast<long long>(blockIdx.x % blocks_per_frame) * TR_PILLARS;
    const int n_here = static_cast<int>(min(static_cast<long long>(TR_PILLARS), pillars - p0));
    if (touched) {
        const int mine = (threadIdx.x < n_here) ? touched[static_cast<size_t>(frame) * pillars + p0 + threadIdx.x] : 0;
        if (!__syncthreads_or(mine)) return;
    }
    const float* s = src + static_cast<size_t>(frame) * C * pillars + p0;
    for (int i = threadIdx.x; i < C * TR_PILLARS; i += 256) {
        const int c = i / TR_PILLARS, pl = i % TR_PILLARS;
        tile[pl][c] = (pl < n_here) ? s[static_cast<size_t>(c) * pillars + pl] : 0.f;
    }
    __syncthreads();
    float* d = dst + (static_cast<size_t>(frame) * pillars + p0) * C;
    for (int i = threadIdx.x; i < TR_PILLARS * 16; i += 256) {
        const int pl = i >> 4, q = i & 15;
        if (pl < n_here)
            reinterpret_cast<float4*>(d + static_cast<size_t>(pl) * C)[q] =
                make_float4(tile[pl][q * 4 + 0], tile[pl][q * 4 + 1], tile[pl][q * 4 + 2], tile[pl][q * 4 + 3]);
    }
}

size_t lift_backward_relayout_bytes(const LiftParams& P) {
    return P.bev_layout == FIERY_BEV_NCHW ? static_cast<size_t>(P.n_frames) * P.pillars * P.C * sizeof(float) : 0;
}

int launch_lift_backward(const LiftParams& P, const void* head, float* workspace, const void* plan, cudaStream_t stream) {
    HeadMapsCols hm, gm;
    int rc = encode_head_maps_cols(&hm, head, P, BW_CH);
    if (rc != FIERY_OK) return rc;
    rc = encode_head_maps_cols(&gm, P.grad_head, P, BW_CH);
    if (rc != FIERY_OK) return rc;
    LiftParams Q = P;
    unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
    if (P.bev_layout == FIERY_BEV_NCHW) {
        const int bpf = static_cast<int>((P.pillars + TR_PILLARS - 1) / TR_PILLARS);
        const unsigned char* marks = plan ? plan_view(plan, P.n_frames, P.n_cameras, P.n_wtiles, P.pillars, 0).touched : nullptr;
        nchw_to_nhwc_kernel<<<static_cast<unsigned>(bpf) * P.n_frames, 256, 0, stream>>>(P.grad_bev, workspace, marks, P.C, P.pillars, bpf);
        FIERY_CUDA_CHECK(cudaGetLastError());
        Q.grad_bev = workspace;
        ws += (lift_backward_relayout_bytes(P) + 127) & ~static_cast<size_t>(127);
    }
    if (plan) {
        Q.plan_tiles = plan_view(plan, P.n_frames, P.n_cameras, P.n_wtiles, P.pillars, 0).tiles;
    } else {                                          // no plan from the forward: compute the geometry here
        FIERY_REQUIRE(workspace != nullptr, "backward without a plan needs the workspace of fiery_lift_workspace_bytes()");
        rc = launch_lift_plan(Q, ws, nullptr, 1, stream);
        if (rc != FIERY_OK) return rc;
        Q.plan_tiles = ws;
    }
    const BwdLayout L(P.hh);
    FIERY_REQUIRE(L.total <= 227 * 1024, "tile needs %d bytes of shared memory", L.total);
    typedef void (*kernel_t)(const HeadMapsCols, const HeadMapsCols, const LiftParams);
    static const kernel_t kernels[2] = {lift_backward_kernel<7>, lift_backward_kernel<BW_MAXR>};
    static OncePerDevice once;
    rc = once.run([]() -> int {
        for (kernel_t k : kernels) {
            FIERY_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            FIERY_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        }
        return FIERY_OK;
    });
    if (rc != FIERY_OK) return rc;
    const bool small = (P.hh + PLAN_RG - 1) / PLAN_RG <= 7;     // the reference's h = 28: 7 rows per thread
    const long long n_tiles = static_cast<long long>(P.n_frames) * P.n_cameras * P.n_wtiles;
    kernels[small ? 0 : 1]<<<static_cast<unsigned>(n_tiles), BW_NT, L.total, stream>>>(hm, gm, Q);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
