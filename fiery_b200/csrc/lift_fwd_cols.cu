// Forward lift, the tile kernel: depth softmax + depth x context outer product + pillar pooling in one kernel; the frustum volume
// (124 MB/frame in the reference, fiery/models/encoder.py:100) never leaves the SM.
//
// Depth softmax x context outer product (encoder.py:98-100) and the voxel pooling of projection_to_birds_eye_view
// (fiery.py:221-273) for one tile = one camera image x 4 feature columns x all rows x all depths x all channels.  WHERE every
// point lands (get_geometry fiery.py:193-208, indices / mask / ranks fiery.py:236-256) comes from the geometry plan
// (lift_plan.cu), computed once per batch of calibrations and shared with the backward kernel.
//
// Observation the kernel is built on: at fixed (camera, column, depth) the h image rows of a column fall into one BEV pillar,
// or a handful, because Z is collapsed (Z_BOUND has one cell) and cameras are close to level.  So the reference's global
// argsort + cumsum (fiery.py:257, geometry.py:289) becomes a register-resident *segmented* sum along the image column: a
// thread walks the rows and only when the pillar changes (a precomputed event bit) does it flush its partial sum with one
// vector reduction (red.global.add.v2.f32) into a channel-last BEV accumulator.  The 32 lanes of a warp cover the 64 channels
// of a pillar, so each flush is two full 128-byte lines.  ~17k column segments per frame reach L2 instead of 453k points.
//
// The shared-memory layout is chosen so that NOTHING is transposed:
//
//   * the two TMA loads deliver the tile as  prob[row][depth][col4]  and  ctx[row][k][cl][col4]  (channel CPL*cl + k; the
//     channel split is a 5-D tensor map, so the permutation is done by the copy engine).  One 16-byte shared load is then
//     "4 adjacent columns of one (row, depth)" or "... of one (row, channel)";
//   * a thread owns DD depths x 4 columns x 2 channels, held as packed pairs of ADJACENT COLUMNS, so the outer product is
//     8*DD FFMA per row whose operands are exactly the register pairs the loads return;
//   * the tile's pillar runs are read from the plan and expanded into run-end events while the TMA is in flight;
//   * the softmax runs in place on prob (lane = (depth mod 8, column): conflict free, reductions by shuffle);
//   * run ends are detected warp-uniformly (one 32-bit load per row, fetched a row ahead).
#include <string.h>

#include "lift_plan.cuh"

namespace fiery {

constexpr int COLS_NPAIR = DPAD * WT;         // (depth, column) pairs of a tile: each is one image column of points
constexpr int COLS_EVS = 33;                  // event words per unit: rows 0..31 + one that stays 0
constexpr int COLS_PLAN_STAGE = 4096;         // bytes of the tile's plan record staged in shared memory by one bulk copy ...
constexpr int COLS_RUNS_STAGED = (COLS_PLAN_STAGE - PLAN_OFF_RUNS) / 4;   // ... = header + this many runs; later runs are read from global
// A "unit" is DD adjacent depths x the 4 columns of the tile (4*DD pairs = "slots"); the 32 lanes of a unit, one warp, own
// CPL = 2 channels each.  DD trades shared-memory traffic for registers: per image row a unit reads the whole 1 KB context row of
// the tile, so the tile's context traffic is (48 / DD) KB per row.
constexpr int CPL = 2;                        // channels per lane
constexpr int LPU = 64 / CPL;                 // lanes per unit

struct ColsLayout {
    int hh, C;
    int off_bar, off_plan, off_ev, off_prob, off_ctx, off_pillar, total;
    __host__ __device__ ColsLayout(int hh_, int C_, int n_units) : hh(hh_), C(C_) {
        int o = 0;
        off_bar = o;    o += 16;                        // two mbarriers: head tile, plan record
        off_plan = o;   o += COLS_PLAN_STAGE;           // head of the tile's plan record: masks, offsets, the first runs
        off_ev = o;     o += n_units * COLS_EVS * 4;   // run-end events: [unit][row], see expand_plan
        o = (o + 127) & ~127;
        off_prob = o;   o += hh * DPAD * WT * 4;
        o = (o + 127) & ~127;
        off_ctx = o;    o += hh * C * WT * 4;
        o = (o + 127) & ~127;
        off_pillar = o; o += hh * COLS_NPAIR * 4;      // [row][pair = depth*4 + col]
        total = o;
    }
};

// 8-byte asynchronous copy global -> shared (SASS LDGSTS.64): one (channel, row) piece = 4 half-precision columns
// (no L2 policy here: ptxas 12.9 gives the .L2::cache_hint form of this instruction a descriptor operand it never writes)
__device__ __forceinline__ void cp_async_8(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_addr(dst)), "l"(src) : "memory");
}

template <int HALF>
__device__ __forceinline__ float half_of(unsigned long long v) {
    return __uint_as_float(HALF ? static_cast<unsigned>(v >> 32) : static_cast<unsigned>(v));
}

// zero one half of a packed pair where keep == 0 (keep is 0 or ~0): one logic op on one register of the pair, in place
template <int HALF>
__device__ __forceinline__ void clear_half(unsigned long long& v, unsigned keep) {
    v &= HALF ? ((static_cast<unsigned long long>(keep) << 32) | 0xffffffffull) : (0xffffffff00000000ull | keep);
}

// The geometry of the tile comes from the plan (lift_plan.cu: get_geometry + voxel index / mask / rank of every point,
// fiery.py:193-208,236-256, reduced to pillar runs per (depth, column) pair).  Here the runs of the tile are expanded into what the
// pooling loop consumes:
//   ev[unit][row]      bit j (slot j = dd*4 + col: depth DD*unit + dd, column col) set <=> pair j changes pillar between
//                      row-1 and row; bit 4*DD + j: ... and the run that ends sits on a valid pillar (it must be flushed, the
//                      others are only cleared)
//   pillar[row][pair]  written only where it is read: the last row of every run
// thread = (depth, column) pair; a pair has ~2.8 runs on average, so this is a few dozen instructions per thread (the 37
// instructions per POINT of the reference arithmetic are spent once per batch in the plan kernel, not per tile pass).
// DET (the deterministic forward): pillar[row][pair] holds the run's index k in the record's runs[] instead of its pillar -- the row
// of the tile's partial sums the run is stored to -- and -1 for a masked run that reaches the last row.
template <int NT, int DD, bool DET = false>
__device__ __forceinline__ void expand_plan(const ColsLayout& L, unsigned char* smem, const unsigned char* __restrict__ rec) {
    static_assert(NT >= COLS_NPAIR, "one thread per (depth, column) pair at least");
    const int pair = threadIdx.x;
    if (pair >= COLS_NPAIR) return;
    const unsigned char* staged = smem + L.off_plan;
    int* tab = reinterpret_cast<int*>(smem + L.off_pillar) + pair;
    unsigned m = reinterpret_cast<const unsigned*>(staged + PLAN_OFF_MASK)[pair];
    int k = reinterpret_cast<const unsigned short*>(staged + PLAN_OFF_OFF)[pair];
    const int* s_runs = reinterpret_cast<const int*>(staged + PLAN_OFF_RUNS);
    const int* g_runs = reinterpret_cast<const int*>(rec + PLAN_OFF_RUNS);
    auto run = [&](int idx) { return idx < COLS_RUNS_STAGED ? s_runs[idx] : __ldg(g_runs + idx); };
    const int d = pair >> 2, col = pair & 3;
    const int j = (d % DD) * 4 + col;
    unsigned* ev = reinterpret_cast<unsigned*>(smem + L.off_ev) + (d / DD) * COLS_EVS;
    int cur = run(k);
    while (m) {
        const int h = __ffs(m) - 1;                       // rows h-1 | h lie in different pillars
        m &= m - 1;
        const int nxt = run(++k);
        atomicOr(ev + h, (1u << j) | (cur >= 0 ? (1u << (4 * DD + j)) : 0u));
        if constexpr (DET) {
            if (cur >= 0) tab[(h - 1) * COLS_NPAIR] = k - 1;
        } else {
            if (cur >= 0) tab[(h - 1) * COLS_NPAIR] = cur;
        }
        cur = nxt;
    }
    if constexpr (DET) tab[(L.hh - 1) * COLS_NPAIR] = cur >= 0 ? k : -1;
    else tab[(L.hh - 1) * COLS_NPAIR] = cur;              // the run that reaches the last row
}

// constants of the in-tile geometry live where a planned tile stages its plan record
constexpr int GEO_OFF_CAM = 0, GEO_OFF_U = 48, GEO_OFF_V = 64, GEO_OFF_D = 192;

// Calls WITHOUT a plan (a forward-only call whose calibration is new: nothing to share the geometry with): the geometry of the tile
// is evaluated here, while the head tile is in flight -- the tile kernel waits for the copy engine at that point anyway, so this
// costs little, whereas a separate plan kernel in front of every frame group adds a launch and a dependency to every chain.  Same
// evaluator as the plan kernel (geometry.cuh: PillarMap), same result:
// the pillar (rank, fiery.py:236-256; -1 = masked) of every point, evaluated with the reference arithmetic, reduced on the fly to
// what the pooling loop consumes:
//   ev[unit][row]      bit j (slot j = dd*4 + col: depth DD*unit + dd, column col) set <=> pair j changes pillar between
//                      row-1 and row; bit 4*DD + j: ... and the run that ends sits on a valid pillar (it must be flushed, the
//                      others are only cleared)
//   pillar[row][pair]  written only where it is read: the last row of every run
//   touched[pillar]    the layout pass's map of pillars that receive something, marked at every run start
// thread = (pair, row range); the NRS ranges of a pair sit in adjacent lanes and hand their last pillar to the next range.
template <bool POW2, int NT, int DD>
__device__ __forceinline__ void stage_geometry_cols(const LiftParams& P, const ColsLayout& L, unsigned char* smem, int w0,
                                                    unsigned char* touched) {
    constexpr int NRS = NT / COLS_NPAIR >= 4 ? 4 : (NT / COLS_NPAIR >= 2 ? 2 : 1);
    static_assert(NT >= COLS_NPAIR, "one thread per (depth, column) pair at least");
    const float* s_cam = reinterpret_cast<const float*>(smem + L.off_plan + GEO_OFF_CAM);
    const float* s_u = reinterpret_cast<const float*>(smem + L.off_plan + GEO_OFF_U);
    const float* s_v = reinterpret_cast<const float*>(smem + L.off_plan + GEO_OFF_V);
    const float* s_d = reinterpret_cast<const float*>(smem + L.off_plan + GEO_OFF_D);
    int* s_pillar = reinterpret_cast<int*>(smem + L.off_pillar);
    unsigned* s_ev = reinterpret_cast<unsigned*>(smem + L.off_ev);
    CameraTransform T;
#pragma unroll
    for (int i = 0; i < 9; ++i) T.m[i] = s_cam[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) T.t[i] = s_cam[9 + i];
    const PillarMap<POW2> pillar(P.grid);
    const int hh = L.hh;
    const int pair = threadIdx.x / NRS, rs = threadIdx.x % NRS;
    const bool idle = pair >= COLS_NPAIR;                    // NT is not always a multiple of the pair count
    const int d = idle ? 0 : pair >> 2, col = pair & 3;
    const int unit = d / DD, j = (d % DD) * 4 + col;
    const bool split = hh >= 2 * NRS;                       // short columns: one lane of the pair walks all rows
    const int h_lo = idle ? 0 : (split ? (hh * rs) / NRS : 0);
    const int h_hi = idle ? 0 : (split ? (hh * (rs + 1)) / NRS : (rs == 0 ? hh : 0));
    const bool dead = d >= P.D || w0 + col >= P.ww;

    unsigned* ev = s_ev + unit * COLS_EVS;
    int* tab = s_pillar + (idle ? 0 : pair);
    auto run_ends = [&](int h, int before, int now) {        // rows h-1 | h lie in different pillars
        atomicOr(ev + h, (1u << j) | (before >= 0 ? (1u << (4 * DD + j)) : 0u));
        if (before >= 0) tab[(h - 1) * COLS_NPAIR] = before;
        if (touched && now >= 0) touched[now] = 1;          // the layout pass gathers only marked pillars
    };

    int first = -1, prev = -1;
    if (!dead && h_lo < h_hi) {
        const float depth = s_d[d];
        const ColumnTerms ct = column_terms(T, s_u[col], depth);
        int h = h_lo;
#pragma unroll 2
        for (; h < h_hi; ++h) {
            const int cur = pillar(T, ct, s_v[h], depth);
            if (h == h_lo) first = cur;
            else if (cur != prev) run_ends(h, prev, cur);
            prev = cur;
        }
    }
    const int before = __shfl_up_sync(0xffffffffu, prev, 1);   // last pillar of the previous row range of this pair
    if (h_lo < h_hi) {
        if (rs > 0 && split) {
            if (first != before) run_ends(h_lo, before, first);
        } else if (touched && first >= 0) {
            touched[first] = 1;                                     // row 0 starts a run
        }
        if (h_hi == hh) tab[(hh - 1) * COLS_NPAIR] = prev;          // the run that reaches the last row
    }
}


// ---- half-precision head tensors (AMP: Encoder.depth_layer emits fp16, encoder.py:96 under PRECISION 16) ------------------------
// The row pitch of an fp16 plane (w * 2 bytes) is not a multiple of 16 for the reference's w = 60, so the tensor maps cannot
// describe it; a (channel, row) piece of the tile -- 4 columns = 8 bytes, 8-byte aligned because w and the tile edge are
// multiples of 4 -- is fetched with one cp.async into the UPPER HALF of the region the fp32 tile will occupy, in the final
// piece order.  After the geometry phase the pieces are widened in place: every thread reads its pieces, one barrier, every
// thread writes them as fp32 (exact: fp16 -> fp32 conversion, then the same fp32 arithmetic as for an fp32 head, which is what
// autocast does to the reference's softmax and outer product, encoder.py:99-100).
template <int NT>
__device__ __forceinline__ void issue_half_tile(const LiftParams& P, const ColsLayout& L, unsigned char* smem, int img, int w0) {
    const int hh = L.hh;
    const int n_pp = P.use_depth ? hh * DPAD : 0;
    const int n_cp = hh * 64;
    unsigned char* prob_stage = smem + L.off_prob + hh * DPAD * WT * 2;     // upper half of prob[row][depth][col4]
    unsigned char* ctx_stage = smem + L.off_ctx + hh * 64 * WT * 2;              // upper half of ctx[row][k][cl][col4]
    const __half* head = static_cast<const __half*>(P.head_f16);
    const size_t plane = static_cast<size_t>(hh) * P.ww;
    const __half* img_base = head + static_cast<size_t>(img) * P.head_channels * plane + w0;
    const int ctx_ch0 = P.use_depth ? P.D : 0;
    for (int p = threadIdx.x; p < n_pp + n_cp; p += NT) {
        if (p < n_pp) {
            const int row = p / DPAD, d = p - row * DPAD;
            if (d < P.D) cp_async_8(prob_stage + p * 8, img_base + d * plane + static_cast<size_t>(row) * P.ww);
        } else {
            const int q = p - n_pp;
            const int row = q >> 6, r = q & 63;
            const int ch = ctx_ch0 + CPL * (r % LPU) + r / LPU;                     // piece order [k][cl], channel = CPL*cl + k
            cp_async_8(ctx_stage + q * 8, img_base + ch * plane + static_cast<size_t>(row) * P.ww);
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

template <int NT>
__device__ __forceinline__ void widen_half_tile(const LiftParams& P, const ColsLayout& L, unsigned char* smem) {
    constexpr int MAXP = (32 * (DPAD + 64) + NT - 1) / NT;                  // pieces per thread at h = 32
    const int hh = L.hh;
    const int n_pp = P.use_depth ? hh * DPAD : 0;
    const int total = n_pp + hh * 64;
    unsigned char* prob_base = smem + L.off_prob;
    unsigned char* ctx_base = smem + L.off_ctx;
    const int prob_half = hh * DPAD * WT * 2, ctx_half = hh * 64 * WT * 2;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();                                  // every thread's pieces have landed
    uint2 v[MAXP];
#pragma unroll
    for (int i = 0; i < MAXP; ++i) {
        const int p = threadIdx.x + i * NT;
        v[i] = make_uint2(0u, 0u);                     // depth slots >= D stay zero (the tensor maps zero-fill them too)
        if (p < n_pp) {
            if (p % DPAD < P.D) v[i] = *reinterpret_cast<const uint2*>(prob_base + prob_half + p * 8);
        } else if (p < total) {
            v[i] = *reinterpret_cast<const uint2*>(ctx_base + ctx_half + (p - n_pp) * 8);
        }
    }
    __syncthreads();                                  // all pieces are in registers: the fp32 tile may overwrite them
#pragma unroll
    for (int i = 0; i < MAXP; ++i) {
        const int p = threadIdx.x + i * NT;
        if (p < total) {
            const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&v[i].x));
            const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&v[i].y));
            float4* dst = reinterpret_cast<float4*>(p < n_pp ? prob_base + p * 16 : ctx_base + (p - n_pp) * 16);
            *dst = make_float4(lo.x, lo.y, hi.x, hi.y);
        }
    }
    __syncthreads();                                  // the fp32 tile is complete
}

// predicated vector reduction of CPL adjacent channels; HINT: with an L2 `policy` (the scratch accumulator stays in L2 for the layout pass)
template <bool HINT>
__device__ __forceinline__ void red_channels_if(char* dst, const float (&v)[CPL], unsigned bit, uint64_t policy) {
    if (!HINT)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\t@p red.global.add.v2.f32 [%0], {%1, %2};\n\t}"
                     :: "l"(dst), "f"(v[0]), "f"(v[1]), "r"(bit) : "memory");
    else
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\t@p red.global.add.L2::cache_hint.v2.f32 [%0], {%1, %2}, %4;\n\t}"
                     :: "l"(dst), "f"(v[0]), "f"(v[1]), "r"(bit), "l"(policy) : "memory");
}

// the deterministic forward's flush: a predicated plain store of CPL adjacent channels into the run's row of partial sums
__device__ __forceinline__ void st_channels_if(char* dst, const float (&v)[CPL], unsigned bit) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\t@p st.global.v2.f32 [%0], {%1, %2};\n\t}"
                 :: "l"(dst), "f"(v[0]), "f"(v[1]), "r"(bit) : "memory");
}

// One (depth, column) slot of the run-end handling.  `mw` is warp-uniform, so the test is a plain branch; the lanes that own
// the ending run reduce their channels into the accumulator and restart.  The "+ 0.0f" copies are real instructions on
// purpose: they gather the values into the consecutive registers the vector reduction needs HERE, instead of letting the
// register allocator keep the accumulators in that order and un-shuffle them around every FMA pair.
// DET: plp holds run indices and `out` is the tile's rows of partial sums; the run's sum is stored, not reduced.
template <int DD, int SD, int COL, bool HINT, bool DET>
__device__ __forceinline__ void flush_slot(unsigned long long (&acc)[CPL][DD][2], unsigned mw, unsigned own, unsigned flush,
                                           const int* plp, char* out, uint64_t policy) {
    constexpr int j = SD * 4 + COL;
    if (mw & (1u << j)) {
        const unsigned pl = static_cast<unsigned>(plp[j]);
        float v[CPL];
#pragma unroll
        for (int k = 0; k < CPL; ++k) v[k] = __fadd_rn(half_of<COL & 1>(acc[k][SD][COL >> 1]), 0.0f);
        if constexpr (DET) st_channels_if(out + static_cast<size_t>(pl) * (64 * 4), v, flush & (1u << j));
        else red_channels_if<HINT>(out + static_cast<size_t>(pl) * (64 * 4), v, flush & (1u << j), policy);
        const unsigned keep = ((own >> j) & 1u) - 1u;          // 0 where my run ends, ~0 otherwise
#pragma unroll
        for (int k = 0; k < CPL; ++k) clear_half<COL & 1>(acc[k][SD][COL >> 1], keep);
    }
}

template <int DD, int SD, bool HINT, bool DET>
__device__ __forceinline__ void flush_depth(unsigned long long (&acc)[CPL][DD][2], unsigned mw, unsigned own, unsigned flush,
                                            const int* plp, char* out, uint64_t policy) {
    if (mw & (0xfu << (4 * SD))) {
        flush_slot<DD, SD, 0, HINT, DET>(acc, mw, own, flush, plp, out, policy); flush_slot<DD, SD, 1, HINT, DET>(acc, mw, own, flush, plp, out, policy);
        flush_slot<DD, SD, 2, HINT, DET>(acc, mw, own, flush, plp, out, policy); flush_slot<DD, SD, 3, HINT, DET>(acc, mw, own, flush, plp, out, policy);
    }
    if constexpr (SD + 1 < DD) flush_depth<DD, SD + 1, HINT, DET>(acc, mw, own, flush, plp, out, policy);
}

// DD depths per unit, a tile is 48 / DD units of one warp: DD 2 is 768 threads, DD 3 512.  The row loop is unrolled twice for DD 3
// and not at all for DD 2.  Two tiles per SM.
// HINTS: NCHW output, L2 policies on the head loads and the reductions into the scratch (lift_fwd.cu: lanes)
// DET: the deterministic forward (lift_det.cu) -- planned, no hints; every run's sum is stored to row (tile, k) of P.accum, which
// holds det_runs_per_tile(h) rows of 64 channels per tile of the launch.
template <int DD, bool HALF, bool PLANNED, bool HINTS, bool DET>
__global__ void __launch_bounds__((DPAD / DD) * LPU, 2)
lift_forward_cols_kernel(const __grid_constant__ HeadMapsCols head_maps, const LiftParams P) {
    static_assert(!DET || (PLANNED && !HINTS), "the deterministic tile kernel is planned and unhinted");
    constexpr int NU = DPAD / DD;                     // units per tile
    constexpr int NT = NU * LPU;
    constexpr int SLOTS = 4 * DD;
    constexpr int UNR = DD == 3 ? 2 : 1;              // row-loop unroll
    static_assert(DPAD % DD == 0 && SLOTS <= 16, "unsupported unit shape");
    extern __shared__ __align__(128) unsigned char smem[];
    const ColsLayout L(P.hh, P.C, NU);
    const int wtile = blockIdx.x % P.n_wtiles;
    const int img_local = blockIdx.x / P.n_wtiles;    // (frame, camera) within this launch's chunk of frames
    const int img = P.frame0 * P.n_cameras + img_local;
    const int frame = img_local / P.n_cameras;        // chunk-local: indexes the accumulator
    const int w0 = wtile * WT;
    const int tid = threadIdx.x;
    const int hh = L.hh;
    // (img_local indexes the plan's tile records and the accumulator; img the head tensor)

    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L.off_bar);
    const unsigned char* rec = PLANNED ? P.plan_tiles + static_cast<size_t>(blockIdx.x) * PLAN_TILE_BYTES : nullptr;
    if (tid == 0) {
        if (PLANNED) mbar_init(bar + 1, 1);
        if (!HALF) mbar_init(bar, 1);
        fence_mbar_init();
        if (PLANNED) {                                // the tile's geometry: head of its plan record, one bulk copy
            mbar_arrive_expect_tx(bar + 1, COLS_PLAN_STAGE);
            bulk_load_1d(smem + L.off_plan, rec, COLS_PLAN_STAGE, bar + 1);
        }
    }
    if (HALF) {
        issue_half_tile<NT>(P, L, smem, img, w0);
    } else if (tid == 0) {
        tma_prefetch_desc(&head_maps.depth);
        tma_prefetch_desc(&head_maps.ctx);
        const uint32_t prob_bytes = P.use_depth ? static_cast<uint32_t>(hh * DPAD * WT * 4) : 0u;
        mbar_arrive_expect_tx(bar, prob_bytes + static_cast<uint32_t>(hh * L.C * WT * 4));
        if (HINTS) {
            const uint64_t once = l2_evict_first();                                  // the head is read once
            if (P.use_depth) tma_load_4d(smem + L.off_prob, &head_maps.depth, bar, w0, 0, 0, img, once);
            tma_load_5d(smem + L.off_ctx, &head_maps.ctx, bar, w0, 0, 0, 0, img, once);
        } else {
            if (P.use_depth) tma_load_4d(smem + L.off_prob, &head_maps.depth, bar, w0, 0, 0, img);
            tma_load_5d(smem + L.off_ctx, &head_maps.ctx, bar, w0, 0, 0, 0, img);
        }
    }
    {
        unsigned* s_ev = reinterpret_cast<unsigned*>(smem + L.off_ev);
        for (int i = tid; i < NU * COLS_EVS; i += NT) s_ev[i] = 0u;
    }
    if (!PLANNED) {                                   // constants of the in-tile geometry; one lane composes R @ K^-1 (fiery.py:203)
        float* s_u = reinterpret_cast<float*>(smem + L.off_plan + GEO_OFF_U);
        float* s_v = reinterpret_cast<float*>(smem + L.off_plan + GEO_OFF_V);
        float* s_d = reinterpret_cast<float*>(smem + L.off_plan + GEO_OFF_D);
        if (tid < WT) s_u[tid] = (w0 + tid < P.ww) ? P.fu[w0 + tid] : 0.f;
        if (tid >= 32 && tid < 64) s_v[tid - 32] = P.fv[min(tid - 32, hh - 1)];
        if (tid >= 64 && tid < 64 + DPAD) s_d[tid - 64] = (tid - 64 < P.D) ? P.fd[tid - 64] : 0.f;
        if (tid == NT - 1) {
            CameraTransform T;
            load_camera(P.calib_mode, P.calib_a, P.calib_b, img, T);
            float* s_cam = reinterpret_cast<float*>(smem + L.off_plan + GEO_OFF_CAM);
#pragma unroll
            for (int i = 0; i < 9; ++i) s_cam[i] = T.m[i];
#pragma unroll
            for (int i = 0; i < 3; ++i) s_cam[9 + i] = T.t[i];
        }
    }
    __syncthreads();                                  // event words cleared, constants and the mbarriers are set up
    // geometry of the tile (the head tile stays in flight meanwhile): the runs of its plan record, or evaluated here
    if (PLANNED) {
        if (tid < COLS_NPAIR) mbar_wait(bar + 1, 0);
        expand_plan<NT, DD, DET>(L, smem, rec);
    } else {
        unsigned char* touched = P.touched ? P.touched + static_cast<size_t>(frame) * P.pillars : nullptr;
        if (P.grid.pow2[0] && P.grid.pow2[1]) stage_geometry_cols<true, NT, DD>(P, L, smem, w0, touched);
        else stage_geometry_cols<false, NT, DD>(P, L, smem, w0, touched);
    }
    if (HALF) widen_half_tile<NT>(P, L, smem);         // fp16 pieces -> the fp32 tile, in place
    else mbar_wait(bar, 0);                           // head tile has landed
    softmax_depth<NT>(P, reinterpret_cast<float*>(smem + L.off_prob), hh);
    __syncthreads();

    // ---- pooling: thread = (unit of DD depths, 4 columns, channels CPL*cl .. CPL*cl + CPL-1) ---------------------------
    const int unit = tid / LPU;
    const int cl = tid % LPU;
    const float* pp = reinterpret_cast<const float*>(smem + L.off_prob) + unit * DD * WT;
    const float* cp = reinterpret_cast<const float*>(smem + L.off_ctx) + cl * WT;
    const int* plp = reinterpret_cast<const int*>(smem + L.off_pillar) + unit * SLOTS - COLS_NPAIR;          // row h-1
    char* out;
    if constexpr (DET) out = reinterpret_cast<char*>(P.accum + static_cast<size_t>(blockIdx.x) * det_runs_per_tile(hh) * 64 + cl * CPL);
    else out = reinterpret_cast<char*>(P.accum + static_cast<size_t>(frame) * P.pillars * P.C + cl * CPL);
    const unsigned* evp = reinterpret_cast<const unsigned*>(smem + L.off_ev) + unit * COLS_EVS + 1;         // row h+1
    const uint64_t keep = HINTS ? l2_evict_last() : 0;   // the scratch accumulator: the layout pass reads these lines next

    unsigned long long acc[CPL][DD][2];               // [channel k][depth dd][column pair]
#pragma unroll
    for (int k = 0; k < CPL; ++k)
#pragma unroll
        for (int dd = 0; dd < DD; ++dd) acc[k][dd][0] = acc[k][dd][1] = 0ull;

    // own: my slots whose run ends at this row, flush: ... and must be flushed.  mw: slots that end a run anywhere in the
    // warp; a unit is one warp, so that is `own` and every run-end branch is warp-uniform.  Both are fetched one row ahead: the
    // chain load -> branch is long.
    unsigned own = 0, flush = 0, mw = 0;              // row 0 starts every run
#pragma unroll UNR
    for (int h = 0; h < hh; ++h, pp += DPAD * WT, cp += 64 * WT, plp += COLS_NPAIR, ++evp) {
        const unsigned ev_next = *evp;                                // the word after the last row stays 0
        if (mw) flush_depth<DD, 0, HINTS, DET>(acc, mw, own, flush, plp, out, keep);
        ulonglong2 dv[DD];
#pragma unroll
        for (int dd = 0; dd < DD; ++dd) dv[dd] = *reinterpret_cast<const ulonglong2*>(pp + dd * WT);   // columns (0,1) (2,3)
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
            const ulonglong2 c = *reinterpret_cast<const ulonglong2*>(cp + k * LPU * WT);   // channel CPL*cl + k
            // depth x context outer product (encoder.py:100), summed along the column
#pragma unroll
            for (int dd = 0; dd < DD; ++dd) {
                ffma2(acc[k][dd][0], dv[dd].x, c.x);
                ffma2(acc[k][dd][1], dv[dd].y, c.y);
            }
        }
        own = ev_next & ((1u << SLOTS) - 1u);
        flush = ev_next >> SLOTS;
        mw = own;
    }
    // the runs that reach the last row (plp now points at it)
#pragma unroll
    for (int j = 0; j < SLOTS; ++j) {
        const int pl = plp[j];
        float v[CPL];
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
            const unsigned long long a = acc[k][j >> 2][(j & 3) >> 1];
            v[k] = (j & 1) ? half_of<1>(a) : half_of<0>(a);
        }
        if constexpr (DET) st_channels_if(out + static_cast<size_t>(static_cast<unsigned>(pl)) * (64 * 4), v, pl >= 0 ? 1u : 0u);
        else red_channels_if<HINTS>(out + static_cast<size_t>(static_cast<unsigned>(pl)) * (64 * 4), v, pl >= 0 ? 1u : 0u, keep);
    }
}

template <int DD, bool HALF, bool PLANNED, bool HINTS, bool DET>
static int launch_forward_cols_t(const LiftParams& P, const void* head, cudaStream_t stream) {
    constexpr int NU = DPAD / DD, NT = NU * LPU;
    const ColsLayout L(P.hh, P.C, NU);
    auto kernel = lift_forward_cols_kernel<DD, HALF, PLANNED, HINTS, DET>;
    static OncePerDevice once;                        // zero-initialised (static storage)
    int rc = once.run([kernel]() -> int {
        FIERY_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        // ask for the full shared-memory carve-out (two or three tiles of ~75 KB per SM for the reference shape)
        FIERY_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        return FIERY_OK;
    });
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(L.total <= 227 * 1024, "tile needs %d bytes of shared memory", L.total);
    HeadMapsCols maps;
    if (HALF) {
        memset(&maps, 0, sizeof(maps));              // unused: half-precision tiles are fetched with cp.async
        FIERY_REQUIRE(P.head_f16 != nullptr && (reinterpret_cast<uintptr_t>(P.head_f16) & 7) == 0,
                      "half-precision head tensor must be 8-byte aligned");
    } else {
        rc = encode_head_maps_cols(&maps, head, P, CPL);
        if (rc != FIERY_OK) return rc;
    }
    const long long n_tiles = static_cast<long long>(P.n_frames) * P.n_cameras * P.n_wtiles;
    kernel<<<static_cast<unsigned>(n_tiles), NT, L.total, stream>>>(maps, P);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

// L2 hints for NCHW output only: with channel-last output the tile kernel reduces into the caller's output, and hinted there it
// measured slower on an H100 than with the plain instructions
template <int DD, bool HALF, bool PLANNED>
static int launch_layout_t(const LiftParams& P, const void* head, cudaStream_t stream) {
    return P.bev_layout == FIERY_BEV_NCHW ? launch_forward_cols_t<DD, HALF, PLANNED, true, false>(P, head, stream)
                                          : launch_forward_cols_t<DD, HALF, PLANNED, false, false>(P, head, stream);
}

// The deterministic forward's tile kernel (lift_det.cu): P.plan_tiles is required, P.accum receives the runs' partial sums.
int launch_forward_cols_det(const LiftParams& P, const void* head, cudaStream_t stream) {
    FIERY_REQUIRE(P.plan_tiles != nullptr, "the deterministic tile kernel needs a plan");
    return P.head_f16 != nullptr ? launch_forward_cols_t<3, true, true, false, true>(P, head, stream)
                                 : launch_forward_cols_t<3, false, true, false, true>(P, head, stream);
}

// Unit shape (DD depths per unit of one warp, 2 channels per lane).  The pooling loop is bound by shared-memory wavefronts (a
// broadcast LDS.128 costs 2, a 512-byte one 4) and by the run-end control flow, so the shape trades context re-reads (48 / DD per
// row), registers (8 * DD accumulators) and resident warps:
//   * geometry in the tile (no plan): DD = 3 (512 threads) when the grid fills whole waves of 2 tiles per SM; DD = 2 (768 threads, row
//     loop not unrolled) while tiles run alone on an SM, i.e. when the last wave is at most half full;
//   * geometry from a plan: DD = 3 always.
int launch_forward_cols(const LiftParams& P, const void* head, cudaStream_t stream) {
    const bool half = P.head_f16 != nullptr;
    if (P.plan_tiles != nullptr)
        return half ? launch_layout_t<3, true, true>(P, head, stream) : launch_layout_t<3, false, true>(P, head, stream);
    int n_sm = 0, dev = 0;
    FIERY_CUDA_CHECK(cudaGetDevice(&dev));
    FIERY_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    const long long n_tiles = static_cast<long long>(P.n_frames) * P.n_cameras * P.n_wtiles;
    const long long rem = n_tiles % (2ll * n_sm);
    if (!(rem > 0 && rem <= n_sm))
        return half ? launch_layout_t<3, true, false>(P, head, stream) : launch_layout_t<3, false, false>(P, head, stream);
    return half ? launch_layout_t<2, true, false>(P, head, stream) : launch_layout_t<2, false, false>(P, head, stream);
}

}  // namespace fiery
