// Microbenchmark: why is the accumulator -> NCHW finalize pass slow?  Variants isolate reads / zero-writes / store shape.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o finalize_variants finalize_variants.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} }while(0)

constexpr int C = 64, P = 128, STRIDE = 68;

template <bool READ, bool ZERO, int STORE>   // STORE: 0 = 16B per lane over channels (current), 1 = scalar coalesced rows, 2 = float4 coalesced rows, 3 = none
__global__ void __launch_bounds__(256) fin(float* __restrict__ accum, unsigned char* __restrict__ flags, float* __restrict__ bev,
                                           long long pillars, int bpf) {
    __shared__ __align__(16) float tile[P * STRIDE];
    __shared__ unsigned char sflag[P];
    const int frame = blockIdx.x / bpf;
    const long long p0 = (long long)(blockIdx.x % bpf) * P;
    const int n_here = (int)min((long long)P, pillars - p0);
    const int tid = threadIdx.x;
    unsigned char* f = flags + (size_t)frame * pillars + p0;
    if (tid < P) { unsigned char v = 0; if (tid < n_here) { v = f[tid]; } sflag[tid] = v; }
    __syncthreads();
    float* src = accum + ((size_t)frame * pillars + p0) * C;
    float4 v[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int i = it * 256 + tid; const int pl = i >> 4, q = i & 15;
        v[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (READ && sflag[pl]) v[it] = *(reinterpret_cast<float4*>(src + (size_t)pl * C) + q);
    }
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int i = it * 256 + tid; const int pl = i >> 4, q = i & 15;
        if (ZERO && sflag[pl]) *(reinterpret_cast<float4*>(src + (size_t)pl * C) + q) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(tile + pl * STRIDE + q * 4) = v[it];
    }
    __syncthreads();
    if (STORE == 0) {
        const int c = tid & 63, grp = tid >> 6;
        float* dst = bev + ((size_t)frame * C + c) * pillars + p0;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int pl0 = (it * 4 + grp) * 8;
            float w[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) w[k] = tile[(pl0 + k) * STRIDE + c];
            if (pl0 + 8 <= n_here) {
                reinterpret_cast<float4*>(dst + pl0)[0] = make_float4(w[0], w[1], w[2], w[3]);
                reinterpret_cast<float4*>(dst + pl0)[1] = make_float4(w[4], w[5], w[6], w[7]);
            }
        }
    } else if (STORE == 1) {
        float* dst = bev + (size_t)frame * C * pillars + p0;
        for (int i = tid; i < C * P; i += 256) {
            const int c = i / P, pl = i % P;
            if (pl < n_here) dst[(size_t)c * pillars + pl] = tile[pl * STRIDE + c];
        }
    } else if (STORE == 2) {
        float* dst = bev + (size_t)frame * C * pillars + p0;
        for (int i = tid; i < C * P / 4; i += 256) {
            const int c = i / (P / 4), pq = i % (P / 4);
            if (pq * 4 + 4 <= n_here)
                reinterpret_cast<float4*>(dst + (size_t)c * pillars)[pq] =
                    make_float4(tile[(pq * 4 + 0) * STRIDE + c], tile[(pq * 4 + 1) * STRIDE + c], tile[(pq * 4 + 2) * STRIDE + c], tile[(pq * 4 + 3) * STRIDE + c]);
        }
    }
}

// S3: one thread per pillar, strided 16-byte loads through L1, coalesced scalar stores, no shared memory
template <bool ZERO>
__global__ void __launch_bounds__(256) fin_s3(float* __restrict__ accum, unsigned char* __restrict__ flags, float* __restrict__ bev,
                                             long long pillars, int bpf) {
    const int frame = blockIdx.x / bpf;
    const long long pl = (long long)(blockIdx.x % bpf) * 256 + threadIdx.x;
    if (pl >= pillars) return;
    unsigned char* f = flags + (size_t)frame * pillars + pl;
    float4 v[16];
    if (*f) {
        float4* row = reinterpret_cast<float4*>(accum + ((size_t)frame * pillars + pl) * C);
#pragma unroll
        for (int q = 0; q < 16; ++q) v[q] = row[q];
        if (ZERO) {
#pragma unroll
            for (int q = 0; q < 16; ++q) row[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    } else {
#pragma unroll
        for (int q = 0; q < 16; ++q) v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float* dst = bev + (size_t)frame * C * pillars + pl;
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        dst[(size_t)(4 * q + 0) * pillars] = v[q].x; dst[(size_t)(4 * q + 1) * pillars] = v[q].y;
        dst[(size_t)(4 * q + 2) * pillars] = v[q].z; dst[(size_t)(4 * q + 3) * pillars] = v[q].w;
    }
}

// scatter-accumulate into flagged pillars like the lift kernel does: one 16-byte vector reduction per (pillar, 4 channels)
template <int MODE>   // 0: red.global.add.v4.f32, 1: 4 x scalar atomicAdd, 2: plain load+store (no atomic; single contribution)
__global__ void red_k(float* __restrict__ accum, const unsigned char* __restrict__ flags, long long total_pillars, int reps) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long pl = i >> 4; const int q = i & 15;
    if (pl >= total_pillars || !flags[pl]) return;
    float* dst = accum + pl * C + q * 4;
    for (int r = 0; r < reps; ++r) {
        if (MODE == 0) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(1.f), "f"(2.f), "f"(3.f), "f"(4.f) : "memory");
        else if (MODE == 1) { atomicAdd(dst, 1.f); atomicAdd(dst + 1, 2.f); atomicAdd(dst + 2, 3.f); atomicAdd(dst + 3, 4.f); }
        else { float4 v = *reinterpret_cast<float4*>(dst); v.x += 1.f; v.y += 2.f; v.z += 3.f; v.w += 4.f; *reinterpret_cast<float4*>(dst) = v; }
    }
}

__global__ void copy_k(const float4* a, float4* b, size_t n) { size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; if (i < n) b[i] = a[i]; }
__global__ void fill_k(float4* b, size_t n, float v) { size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; if (i < n) b[i] = make_float4(v, v, v, v); }

int main() {
    const int frames = 9; const long long pillars = 40000; const int bpf = (int)((pillars + P - 1) / P);
    size_t nacc = (size_t)frames * pillars * C;
    float *acc, *bev, *flush; unsigned char* flags;
    CK(cudaMalloc(&acc, nacc * 4)); CK(cudaMalloc(&bev, nacc * 4)); CK(cudaMalloc(&flags, frames * pillars)); CK(cudaMalloc(&flush, 256 << 20));
    std::vector<unsigned char> hf(frames * pillars);
    srand(1); for (auto& x : hf) x = (rand() % 100) < 55;
    CK(cudaMemcpy(flags, hf.data(), hf.size(), cudaMemcpyHostToDevice));
    CK(cudaMemset(acc, 0, nacc * 4));
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    auto timeit = [&](const char* name, auto launch) {
        float best = 1e9, sum = 0; const int reps = 6;
        for (int r = 0; r < reps; ++r) {
            fill_k<<<(unsigned)(((256u << 20) / 16 + 255) / 256), 256>>>((float4*)flush, (256u << 20) / 16, 1.f);
            cudaEventRecord(a); launch(); cudaEventRecord(b); CK(cudaEventSynchronize(b));
            float ms; cudaEventElapsedTime(&ms, a, b); if (r) { sum += ms; best = ms < best ? ms : best; }
        }
        printf("%-48s mean %8.2f us  best %8.2f us\n", name, sum / (reps - 1) * 1e3, best * 1e3);
    };
    const unsigned grid = bpf * frames;
    timeit("copy 92MB->92MB (float4)", [&] { copy_k<<<(unsigned)((nacc / 4 + 255) / 256), 256>>>((float4*)acc, (float4*)bev, nacc / 4); });
    timeit("fill 92MB", [&] { fill_k<<<(unsigned)((nacc / 4 + 255) / 256), 256>>>((float4*)bev, nacc / 4, 0.f); });
    timeit("A read+zero, store16B-per-lane (current)", [&] { fin<true, true, 0><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    timeit("B read, no zero, store16B-per-lane", [&] { fin<true, false, 0><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    timeit("C no read, no zero, store16B-per-lane", [&] { fin<false, false, 0><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    timeit("D read+zero, scalar coalesced rows", [&] { fin<true, true, 1><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    timeit("E read+zero, float4 coalesced rows", [&] { fin<true, true, 2><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    timeit("F no read, float4 coalesced rows", [&] { fin<false, false, 2><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    const int bpf3 = (int)((pillars + 255) / 256);
    timeit("S3 thread-per-pillar read+zero", [&] { fin_s3<true><<<bpf3 * frames, 256>>>(acc, flags, bev, pillars, bpf3); });
    timeit("S3 thread-per-pillar read, no zero", [&] { fin_s3<false><<<bpf3 * frames, 256>>>(acc, flags, bev, pillars, bpf3); });
    timeit("G read+zero, no store", [&] { fin<true, true, 3><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    timeit("H read only, no store", [&] { fin<true, false, 3><<<grid, 256>>>(acc, flags, bev, pillars, bpf); });
    // ---- does a preceding scatter of vector reductions slow the finalize down? ----
    const long long tp = (long long)frames * pillars;
    const unsigned rgrid = (unsigned)((tp * 16 + 255) / 256);
    auto timeit2 = [&](const char* name, auto pre, auto launch, bool flush_between) {
        float sum = 0, best = 1e9; const int reps = 5;
        for (int r = 0; r < reps; ++r) {
            fill_k<<<(unsigned)(((256u << 20) / 16 + 255) / 256), 256>>>((float4*)flush, (256u << 20) / 16, 1.f);
            pre();
            if (flush_between) fill_k<<<(unsigned)(((256u << 20) / 16 + 255) / 256), 256>>>((float4*)flush, (256u << 20) / 16, 1.f);
            cudaEventRecord(a); launch(); cudaEventRecord(b); CK(cudaEventSynchronize(b));
            float ms; cudaEventElapsedTime(&ms, a, b); if (r) { sum += ms; best = ms < best ? ms : best; }
        }
        printf("%-60s mean %8.2f us  best %8.2f us\n", name, sum / (reps - 1) * 1e3, best * 1e3);
    };
    auto finA = [&] { fin<true, true, 0><<<grid, 256>>>(acc, flags, bev, pillars, bpf); };
    timeit2("red.v4 x3 kernel itself", [&] {}, [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, false);
    timeit2("atomicAdd x3 kernel itself", [&] {}, [&] { red_k<1><<<rgrid, 256>>>(acc, flags, tp, 3); }, false);
    timeit2("ld+st kernel itself", [&] {}, [&] { red_k<2><<<rgrid, 256>>>(acc, flags, tp, 1); }, false);
    timeit2("A after red.v4 x3 (no flush between)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, finA, false);
    timeit2("A after red.v4 x3 (L2 flushed between)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, finA, true);
    timeit2("A after scalar atomicAdd x3 (no flush)", [&] { red_k<1><<<rgrid, 256>>>(acc, flags, tp, 3); }, finA, false);
    timeit2("A after plain ld+st (no flush)", [&] { red_k<2><<<rgrid, 256>>>(acc, flags, tp, 1); }, finA, false);
    timeit2("S3 after red.v4 x3 (no flush)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, [&] { fin_s3<true><<<bpf3 * frames, 256>>>(acc, flags, bev, pillars, bpf3); }, false);
    timeit2("S3 after red.v4 x3 (L2 flushed)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, [&] { fin_s3<true><<<bpf3 * frames, 256>>>(acc, flags, bev, pillars, bpf3); }, true);
    timeit2("H (read only) after red.v4 x3 (no flush)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, [&] { fin<true, false, 3><<<grid, 256>>>(acc, flags, bev, pillars, bpf); }, false);
    timeit2("G (read+zero) after red.v4 x3 (no flush)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, [&] { fin<true, true, 3><<<grid, 256>>>(acc, flags, bev, pillars, bpf); }, false);
    timeit2("C (stores only) after red.v4 x3 (no flush)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, [&] { fin<false, false, 0><<<grid, 256>>>(acc, flags, bev, pillars, bpf); }, false);
    timeit2("fill 92MB after red.v4 x3 (no flush)", [&] { red_k<0><<<rgrid, 256>>>(acc, flags, tp, 3); }, [&] { fill_k<<<(unsigned)((nacc / 4 + 255) / 256), 256>>>((float4*)bev, nacc / 4, 0.f); }, false);
    return 0;
}
