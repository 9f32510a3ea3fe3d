// Deterministic forward lift: the index over the runs' partial sums and the fixed-order reduction (host side: lift_fwd.cu,
// launch_lift_forward_det).
//
// The default forward flushes every pillar run with a vector reduction into a shared accumulator, so the order in which the runs of
// a pillar are added -- and the last bits of the BEV -- change from call to call.  Here the tile kernel (lift_fwd_cols.cu, DET) stores
// run k of tile t to row t * det_runs_per_tile(h) + k of a partial-sum buffer instead, and the kernels below add the rows of every
// pillar in ascending (tile, k) order:
//   1. det_count_kernel   runs per (frame, pillar), from the plan's runs[] of every tile of the pass
//   2. det_scan_kernel    exclusive scan per frame: where each pillar's list starts; a copy serves as the fill cursor
//   3. det_fill_kernel    the partial-sum row of every valid run into its pillar's list (atomic cursor: any order)
//   4. det_sort_kernel    lists longer than a warp sorted ascending by one CTA (shared memory when the list fits, else in place)
//   5. det_reduce_kernel  one warp per pillar: lists of up to 32 rows are sorted in registers, then the rows are summed in order
// The partial-sum row numbers grow with (tile, k), so the ascending list is the summation order the contract names; it depends on
// the frame's geometry only.
#include "lift_plan.cuh"

namespace fiery {

constexpr int DET_THREADS = 256;
constexpr int SORT_THREADS = 1024;
constexpr int SORT_SMEM = 8192;              // list entries det_sort_kernel sorts in shared memory (longer lists: in place)

// 1. one CTA per tile of the pass
__global__ void __launch_bounds__(DET_THREADS)
det_count_kernel(const unsigned char* __restrict__ tiles, int tiles_per_frame, long long pillars, int* __restrict__ counts) {
    const unsigned char* rec = tiles + static_cast<size_t>(blockIdx.x) * PLAN_TILE_BYTES;
    const int n = static_cast<int>(*reinterpret_cast<const unsigned*>(rec + PLAN_OFF_COUNTS));
    const int* runs = reinterpret_cast<const int*>(rec + PLAN_OFF_RUNS);
    int* c = counts + static_cast<size_t>(blockIdx.x / tiles_per_frame) * pillars;
    for (int k = threadIdx.x; k < n; k += DET_THREADS) {
        const int p = runs[k];
        if (p >= 0) atomicAdd(c + p, 1);
    }
}

// 2. one CTA per frame: counts -> exclusive offsets in place, and the same offsets into cursor
__global__ void __launch_bounds__(1024)
det_scan_kernel(int* __restrict__ start, int* __restrict__ cursor, long long pillars) {
    __shared__ int ws[32];
    __shared__ int carry;
    int* s = start + static_cast<size_t>(blockIdx.x) * pillars;
    int* cur = cursor + static_cast<size_t>(blockIdx.x) * pillars;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long long i0 = 0; i0 < pillars; i0 += 1024) {
        const long long i = i0 + threadIdx.x;
        const int v = i < pillars ? s[i] : 0;
        const int incl = block_inclusive_scan(v, ws);
        const int c = carry;
        if (i < pillars) s[i] = cur[i] = c + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + incl;
        __syncthreads();
    }
}

// 3. one CTA per tile of the pass; a frame's lists live in its own region of list_per_frame entries
__global__ void __launch_bounds__(DET_THREADS)
det_fill_kernel(const unsigned char* __restrict__ tiles, int tiles_per_frame, long long pillars, int runs_per_tile,
                int* __restrict__ cursor, int* __restrict__ lists, long long list_per_frame) {
    const unsigned char* rec = tiles + static_cast<size_t>(blockIdx.x) * PLAN_TILE_BYTES;
    const int n = static_cast<int>(*reinterpret_cast<const unsigned*>(rec + PLAN_OFF_COUNTS));
    const int* runs = reinterpret_cast<const int*>(rec + PLAN_OFF_RUNS);
    const int frame = blockIdx.x / tiles_per_frame;
    int* cur = cursor + static_cast<size_t>(frame) * pillars;
    int* lst = lists + static_cast<size_t>(frame) * list_per_frame;
    const int row0 = blockIdx.x * runs_per_tile;
    for (int k = threadIdx.x; k < n; k += DET_THREADS) {
        const int p = runs[k];
        if (p >= 0) lst[atomicAdd(cur + p, 1)] = row0 + k;
    }
}

// Ascending sort of a[0, n) by the CTA: a bitonic network over the next power of two, every comparator putting the smaller value
// at the lower index, the missing entries [n, pow2) standing for +inf (a comparator that reaches one is a no-op).
__device__ void block_sort_ascending(int* a, int n) {
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k; j >= 2; j >>= 1) {
            const int h = j >> 1;
            for (int c = threadIdx.x; c < (n2 >> 1); c += blockDim.x) {
                const int blk = c / h, off = c - blk * h;
                const int lo = blk * j + off;
                const int hi = j == k ? blk * j + j - 1 - off : lo + h;      // the first step of a stage compares mirrored pairs
                if (hi < n) {
                    const int x = a[lo], y = a[hi];
                    if (y < x) { a[lo] = y; a[hi] = x; }
                }
            }
            __syncthreads();
        }
    }
}

// 4. one CTA per 1024 lists: the lists longer than a warp are queued, then sorted one after the other
__global__ void __launch_bounds__(SORT_THREADS)
det_sort_kernel(const int* __restrict__ start, const int* __restrict__ cursor, int* __restrict__ lists, long long pillars,
                long long n_lists, long long list_per_frame) {
    __shared__ int s_buf[SORT_SMEM];
    __shared__ int s_queue[SORT_THREADS];
    __shared__ int s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const long long i = static_cast<long long>(blockIdx.x) * SORT_THREADS + threadIdx.x;
    if (i < n_lists && cursor[i] - start[i] > 32) s_queue[atomicAdd(&s_n, 1)] = threadIdx.x;
    __syncthreads();
    const int queued = s_n;
    for (int q = 0; q < queued; ++q) {
        const long long li = static_cast<long long>(blockIdx.x) * SORT_THREADS + s_queue[q];
        const int n = cursor[li] - start[li];
        int* a = lists + static_cast<size_t>(li / pillars) * list_per_frame + start[li];
        if (n <= SORT_SMEM) {
            for (int t = threadIdx.x; t < n; t += SORT_THREADS) s_buf[t] = a[t];
            __syncthreads();
            block_sort_ascending(s_buf, n);
            for (int t = threadIdx.x; t < n; t += SORT_THREADS) a[t] = s_buf[t];
        } else {
            block_sort_ascending(a, n);                  // global memory: __syncthreads orders the CTA's own accesses
        }
        __syncthreads();
    }
}

// 5. one warp per (frame, pillar); lane l owns channels 2l, 2l + 1.  Out: the pillar's 64-channel row of `out` (frame-major rows of
// `pillars` pillars), written for every pillar when zero_empty (channel-last output), else only for pillars that receive a run (the
// accumulator in front of the layout pass, which reads only marked rows).
__global__ void __launch_bounds__(DET_THREADS)
det_reduce_kernel(const float* __restrict__ partials, const int* __restrict__ start, const int* __restrict__ cursor,
                  const int* __restrict__ lists, long long pillars, long long n_lists, long long list_per_frame,
                  float* __restrict__ out, int zero_empty) {
    const long long i = static_cast<long long>(blockIdx.x) * (DET_THREADS / 32) + (threadIdx.x >> 5);
    if (i >= n_lists) return;
    const int lane = threadIdx.x & 31;
    const int s0 = start[i];
    const int n = cursor[i] - s0;
    if (n == 0 && !zero_empty) return;
    const int* lst = lists + static_cast<size_t>(i / pillars) * list_per_frame + s0;
    const float2* rows = reinterpret_cast<const float2*>(partials) + lane;
    float2 acc = make_float2(0.f, 0.f);
    for (int t0 = 0; t0 < n; t0 += 32) {
        int v = t0 + lane < n ? __ldg(lst + t0 + lane) : 0x7fffffff;
        if (n <= 32) {                                   // short list: bitonic sort across the warp (longer ones: det_sort_kernel)
#pragma unroll
            for (int k = 2; k <= 32; k <<= 1)
#pragma unroll
                for (int j = k >> 1; j > 0; j >>= 1) {
                    const int o = __shfl_xor_sync(0xffffffffu, v, j);
                    v = (((lane & j) == 0) == ((lane & k) == 0)) ? min(v, o) : max(v, o);
                }
        }
        const int m = min(32, n - t0);
        int u = 0;
        for (; u + 4 <= m; u += 4) {                     // four rows in flight, added in list order
            float2 x[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) x[q] = __ldg(rows + static_cast<size_t>(__shfl_sync(0xffffffffu, v, u + q)) * 32);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                acc.x = __fadd_rn(acc.x, x[q].x);
                acc.y = __fadd_rn(acc.y, x[q].y);
            }
        }
        for (; u < m; ++u) {
            const float2 x = __ldg(rows + static_cast<size_t>(__shfl_sync(0xffffffffu, v, u)) * 32);
            acc.x = __fadd_rn(acc.x, x.x);
            acc.y = __fadd_rn(acc.y, x.y);
        }
    }
    reinterpret_cast<float2*>(out + static_cast<size_t>(i) * 64)[lane] = acc;
}

// Index + reduction of one pass of nf frames whose tiles' partial sums are in `partials`.  start / cursor: nf * pillars ints each;
// lists: nf * list_per_frame ints.  out: see det_reduce_kernel.
int launch_det_reduce(const LiftParams& P, int nf, const unsigned char* tiles, const float* partials, int* start, int* cursor,
                      int* lists, float* out, int zero_empty, cudaStream_t stream) {
    const int tiles_per_frame = P.n_cameras * P.n_wtiles;
    const int runs_per_tile = det_runs_per_tile(P.hh);
    const long long list_per_frame = static_cast<long long>(tiles_per_frame) * runs_per_tile;
    const long long n_lists = static_cast<long long>(nf) * P.pillars;
    const unsigned n_tiles = static_cast<unsigned>(nf) * tiles_per_frame;
    FIERY_CUDA_CHECK(cudaMemsetAsync(start, 0, sizeof(int) * n_lists, stream));
    det_count_kernel<<<n_tiles, DET_THREADS, 0, stream>>>(tiles, tiles_per_frame, P.pillars, start);
    det_scan_kernel<<<nf, 1024, 0, stream>>>(start, cursor, P.pillars);
    det_fill_kernel<<<n_tiles, DET_THREADS, 0, stream>>>(tiles, tiles_per_frame, P.pillars, runs_per_tile, cursor, lists, list_per_frame);
    det_sort_kernel<<<static_cast<unsigned>((n_lists + SORT_THREADS - 1) / SORT_THREADS), SORT_THREADS, 0, stream>>>(
        start, cursor, lists, P.pillars, n_lists, list_per_frame);
    constexpr int WARPS = DET_THREADS / 32;
    det_reduce_kernel<<<static_cast<unsigned>((n_lists + WARPS - 1) / WARPS), DET_THREADS, 0, stream>>>(
        partials, start, cursor, lists, P.pillars, n_lists, list_per_frame, out, zero_empty);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
