// Drop-in kernels for VoxelsSumming (fiery/utils/geometry.py:283-314), the call site at fiery/models/fiery.py:261.
//
// The reference computes a global prefix sum over the rank-sorted (Nm, C) feature rows and differences it at run
// boundaries (geometry.py:289-297).  Here each run is summed directly: a block walks a chunk of consecutive rows with one
// thread per channel, keeps the running sum in a register and emits it when the segment id changes.  Runs that straddle a
// chunk boundary are combined with atomicAdd into the zero-initialised output; interior runs are plain stores.  HBM
// traffic is the algorithmic minimum: read feats once, read ranks once, write (U, C).  The direct sum is also ~100x
// more accurate than cumsum-and-subtract (SURVEY.md section 7, hard part 1).
#include "common.cuh"

namespace fiery {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;                       // rows per thread
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// boundary flag of row i: 1 if it starts a new run (geometry.py:292-293 looks at the same pairs from the other side)
__device__ __forceinline__ int run_start(const int64_t* __restrict__ ranks, int64_t i) {
    return (i > 0 && ranks[i] != ranks[i - 1]) ? 1 : 0;
}

__global__ void __launch_bounds__(SCAN_THREADS)
vs_count_kernel(int64_t n, const int64_t* __restrict__ ranks, int* __restrict__ tile_counts) {
    __shared__ int ws[32];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * SCAN_TILE + static_cast<int64_t>(threadIdx.x) * SCAN_ITEMS;
    int c = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k)
        if (base + k < n) c += run_start(ranks, base + k);
    const int incl = block_inclusive_scan(c, ws);
    if (threadIdx.x == SCAN_THREADS - 1) tile_counts[blockIdx.x] = incl;
}

// exclusive scan of the per-tile counts by one block; also writes the total number of runs
__global__ void __launch_bounds__(1024)
vs_scan_tiles_kernel(int n_tiles, int* __restrict__ tile_counts, int64_t n_rows, int64_t* __restrict__ n_segments) {
    __shared__ int ws[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int start = 0; start < n_tiles; start += 1024) {
        const int i = start + threadIdx.x;
        const int v = (i < n_tiles) ? tile_counts[i] : 0;
        const int incl = block_inclusive_scan(v, ws);
        const int c = carry;
        if (i < n_tiles) tile_counts[i] = c + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *n_segments = n_rows > 0 ? static_cast<int64_t>(carry) + 1 : 0;
}

__global__ void __launch_bounds__(SCAN_THREADS)
vs_assign_kernel(int64_t n, const int64_t* __restrict__ ranks, const int* __restrict__ tile_offsets,
                 int32_t* __restrict__ seg) {
    __shared__ int ws[32];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * SCAN_TILE + static_cast<int64_t>(threadIdx.x) * SCAN_ITEMS;
    int f[SCAN_ITEMS];
    int c = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        f[k] = (base + k < n) ? run_start(ranks, base + k) : 0;
        c += f[k];
    }
    const int incl = block_inclusive_scan(c, ws);
    int run = tile_offsets[blockIdx.x] + incl - c;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        run += f[k];
        if (base + k < n) seg[base + k] = run;
    }
}

// ---- forward ---------------------------------------------------------------------------------------------------------
constexpr int VS_ROWS = 64;      // rows per chunk

__global__ void vs_forward_kernel(int64_t n_rows, int C, int64_t stride, const float* __restrict__ feats,
                                  const int64_t* __restrict__ coords, const int32_t* __restrict__ seg,
                                  float* __restrict__ sums, int64_t* __restrict__ coords_out) {
    const int c = threadIdx.x;                                             // channel
    const int64_t chunk = static_cast<int64_t>(blockIdx.x) * blockDim.y + threadIdx.y;
    const int64_t r0 = chunk * VS_ROWS;
    if (r0 >= n_rows) return;
    const int64_t r1 = min(n_rows, r0 + VS_ROWS);
    const bool live = c < C;
    const int first_seg = seg[r0];
    int cur = first_seg;
    float acc = 0.f;
#pragma unroll 8
    for (int64_t r = r0; r < r1; ++r) {
        const int s = seg[r];
        const float x = live ? feats[r * stride + c] : 0.f;
        if (s != cur) {
            if (live) {
                if (cur == first_seg) atomicAdd(sums + static_cast<int64_t>(cur) * C + c, acc);   // may continue a run of the previous chunk
                else sums[static_cast<int64_t>(cur) * C + c] = acc;
            }
            if (c < 3) coords_out[static_cast<int64_t>(cur) * 3 + c] = coords[(r - 1) * 3 + c];  // last row of the run, geometry.py:295
            cur = s;
            acc = 0.f;
        }
        acc += x;
    }
    if (live) atomicAdd(sums + static_cast<int64_t>(cur) * C + c, acc);                           // may continue in the next chunk
    const bool run_ends_here = (r1 == n_rows) || (seg[r1] != cur);
    if (run_ends_here && c < 3) coords_out[static_cast<int64_t>(cur) * 3 + c] = coords[(r1 - 1) * 3 + c];
}

// ---- deterministic forward ------------------------------------------------------------------------------------------
// The same walk, but a run that crosses a chunk edge is not combined with atomics: chunk q stores the piece of its first run to
// edge[q][0] when that run continues from chunk q-1, and the piece of its last run to edge[q][1] when that run starts in chunk q and
// continues into chunk q+1.  Runs that start and end inside a chunk keep their plain stores.  vs_join_kernel then adds the pieces of
// every straddling run in chunk order.
__device__ __forceinline__ int64_t vs_chunk_end(int64_t q, int64_t n_rows) { return min(n_rows, (q + 1) * VS_ROWS); }

__global__ void vs_forward_det_kernel(int64_t n_rows, int C, int64_t stride, const float* __restrict__ feats,
                                      const int64_t* __restrict__ coords, const int32_t* __restrict__ seg,
                                      float* __restrict__ sums, int64_t* __restrict__ coords_out, float* __restrict__ edge) {
    const int c = threadIdx.x;                                             // channel
    const int64_t chunk = static_cast<int64_t>(blockIdx.x) * blockDim.y + threadIdx.y;
    const int64_t r0 = chunk * VS_ROWS;
    if (r0 >= n_rows) return;
    const int64_t r1 = vs_chunk_end(chunk, n_rows);
    const bool live = c < C;
    const int first_seg = seg[r0];
    const bool open = r0 > 0 && seg[r0 - 1] == first_seg;                 // the first run continues one of the previous chunk
    float* piece = edge + chunk * 2 * C + c;
    int cur = first_seg;
    float acc = 0.f;
#pragma unroll 8
    for (int64_t r = r0; r < r1; ++r) {
        const int s = seg[r];
        const float x = live ? feats[r * stride + c] : 0.f;
        if (s != cur) {
            if (live) {
                if (cur == first_seg && open) piece[0] = acc;
                else sums[static_cast<int64_t>(cur) * C + c] = acc;
            }
            if (c < 3) coords_out[static_cast<int64_t>(cur) * 3 + c] = coords[(r - 1) * 3 + c];  // last row of the run, geometry.py:295
            cur = s;
            acc = 0.f;
        }
        acc += x;
    }
    const bool run_ends_here = (r1 == n_rows) || (seg[r1] != cur);
    if (live) {
        if (cur == first_seg && open) piece[0] = acc;
        else if (run_ends_here) sums[static_cast<int64_t>(cur) * C + c] = acc;
        else piece[C] = acc;
    }
    if (run_ends_here && c < 3) coords_out[static_cast<int64_t>(cur) * 3 + c] = coords[(r1 - 1) * 3 + c];
}

// One thread per (chunk, channel): a chunk whose last run starts in it and continues sums that run's pieces -- its own edge[q][1], then
// edge[j][0] of the chunks j = q+1 .. the chunk where the run ends, in that order.  The end row is found by bisection (seg ascends).
__global__ void vs_join_kernel(int64_t n_rows, int C, const int32_t* __restrict__ seg, const float* __restrict__ edge,
                               float* __restrict__ sums) {
    const int c = threadIdx.x;
    const int64_t q = static_cast<int64_t>(blockIdx.x) * blockDim.y + threadIdx.y;
    const int64_t r0 = q * VS_ROWS;
    if (r0 >= n_rows || c >= C) return;
    const int64_t r1 = vs_chunk_end(q, n_rows);
    if (r1 == n_rows) return;
    const int s = seg[r1 - 1];
    if (seg[r1] != s) return;                                              // the last run ends in this chunk
    if (seg[r0] == s && r0 > 0 && seg[r0 - 1] == s) return;                // ... or started before it: a middle piece
    int64_t lo = r1, hi = n_rows;                                          // first row past the run
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (seg[mid] == s) lo = mid + 1;
        else hi = mid;
    }
    const int64_t last = (lo - 1) / VS_ROWS;
    float acc = edge[q * 2 * C + C + c];
    int64_t j = q + 1;
    for (; j + 4 <= last + 1; j += 4) {                                    // four pieces in flight, added in chunk order
        float x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) x[u] = edge[(j + u) * 2 * C + c];
#pragma unroll
        for (int u = 0; u < 4; ++u) acc += x[u];
    }
    for (; j <= last; ++j) acc += edge[j * 2 * C + c];
    sums[static_cast<int64_t>(s) * C + c] = acc;
}

// ---- backward: grad_feats[i] = grad_sums[seg[i]] (geometry.py:305-314) ----------------------------------------------
__global__ void vs_backward_kernel(int64_t n_rows, int C, const float* __restrict__ grad_sums,
                                   const int32_t* __restrict__ seg, float* __restrict__ grad_feats) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = n_rows * C;
    if (i >= total) return;
    const int64_t r = i / C;
    const int c = static_cast<int>(i % C);
    grad_feats[i] = grad_sums[static_cast<int64_t>(seg[r]) * C + c];
}

// ---- host ---------------------------------------------------------------------------------------------------------
// Scratch of the plan (per-tile run counts + the total), cached per host thread and device and grown on demand: the plan
// synchronises its stream before it returns, so the buffer is idle between calls.  (A cudaMallocAsync/cudaFreeAsync pair per
// call costs from 0.3 ms to over 100 ms when the default pool hands its memory back at every synchronise.)
struct PlanScratch {
    int* counts = nullptr;
    size_t bytes = 0;
    int64_t* pinned_total = nullptr;
};

int vs_plan(int64_t n_rows, const int64_t* ranks, int32_t* seg, int64_t* host_n, cudaStream_t stream) {
    static thread_local PlanScratch scratch[16];
    int dev = 0;
    FIERY_CUDA_CHECK(cudaGetDevice(&dev));
    FIERY_REQUIRE(dev >= 0 && dev < 16, "device %d out of range", dev);
    PlanScratch& S = scratch[dev];
    const int n_tiles = static_cast<int>((n_rows + SCAN_TILE - 1) / SCAN_TILE);
    const int padded = (n_tiles + 3) & ~3;                       // keeps the trailing int64 16-byte aligned
    const size_t need = sizeof(int) * padded + sizeof(int64_t) * 2;
    if (S.bytes < need) {
        if (S.counts) FIERY_CUDA_CHECK(cudaFree(S.counts));
        S.counts = nullptr;
        S.bytes = 0;
        const size_t grow = need * 2 > (1u << 16) ? need * 2 : (1u << 16);
        FIERY_CUDA_CHECK(cudaMalloc(&S.counts, grow));
        S.bytes = grow;
    }
    if (!S.pinned_total) FIERY_CUDA_CHECK(cudaHostAlloc(&S.pinned_total, sizeof(int64_t), cudaHostAllocDefault));
    int* tile_counts = S.counts;
    int64_t* d_n = reinterpret_cast<int64_t*>(tile_counts + padded);
    vs_count_kernel<<<n_tiles, SCAN_THREADS, 0, stream>>>(n_rows, ranks, tile_counts);
    vs_scan_tiles_kernel<<<1, 1024, 0, stream>>>(n_tiles, tile_counts, n_rows, d_n);
    vs_assign_kernel<<<n_tiles, SCAN_THREADS, 0, stream>>>(n_rows, ranks, tile_counts, seg);
    FIERY_CUDA_CHECK(cudaGetLastError());
    FIERY_CUDA_CHECK(cudaMemcpyAsync(S.pinned_total, d_n, sizeof(int64_t), cudaMemcpyDeviceToHost, stream));
    FIERY_CUDA_CHECK(cudaStreamSynchronize(stream));   // U sizes the outputs (the reference syncs here too, geometry.py:295)
    *host_n = *S.pinned_total;
    return FIERY_OK;
}

int vs_forward(int64_t n_rows, int C, int64_t stride, const float* feats, const int64_t* coords, const int32_t* seg,
               int64_t n_seg, float* sums, int64_t* coords_out, cudaStream_t stream) {
    FIERY_REQUIRE(C <= 1024, "channels=%d exceeds 1024", C);
    FIERY_CUDA_CHECK(cudaMemsetAsync(sums, 0, sizeof(float) * n_seg * C, stream));
    const int tx = ((C < 3 ? 3 : C) + 31) & ~31;
    const int ty = tx >= 256 ? 1 : 256 / tx;
    const int64_t chunks = (n_rows + VS_ROWS - 1) / VS_ROWS;
    const dim3 block(tx, ty);
    vs_forward_kernel<<<static_cast<unsigned>((chunks + ty - 1) / ty), block, 0, stream>>>(n_rows, C, stride, feats, coords,
                                                                                        seg, sums, coords_out);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

size_t vs_det_workspace_bytes(int64_t n_rows, int C) {
    return static_cast<size_t>((n_rows + VS_ROWS - 1) / VS_ROWS) * 2 * C * sizeof(float);
}

// Every run is written exactly once (a plain store in its chunk, or by vs_join_kernel), so `sums` needs no zero-fill.
int vs_forward_det(int64_t n_rows, int C, int64_t stride, const float* feats, const int64_t* coords, const int32_t* seg,
                   float* sums, int64_t* coords_out, float* edge, cudaStream_t stream) {
    FIERY_REQUIRE(C <= 1024, "channels=%d exceeds 1024", C);
    const int tx = ((C < 3 ? 3 : C) + 31) & ~31;
    const int ty = tx >= 256 ? 1 : 256 / tx;
    const int64_t chunks = (n_rows + VS_ROWS - 1) / VS_ROWS;
    const dim3 block(tx, ty);
    const unsigned grid = static_cast<unsigned>((chunks + ty - 1) / ty);
    vs_forward_det_kernel<<<grid, block, 0, stream>>>(n_rows, C, stride, feats, coords, seg, sums, coords_out, edge);
    vs_join_kernel<<<grid, block, 0, stream>>>(n_rows, C, seg, edge, sums);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

int vs_backward(int64_t n_rows, int C, const float* grad_sums, const int32_t* seg, float* grad_feats, cudaStream_t stream) {
    const int64_t total = n_rows * C;
    vs_backward_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(n_rows, C, grad_sums, seg, grad_feats);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
