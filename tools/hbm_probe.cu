// hbm_probe.cu -- what does ONE H100's HBM deliver for write-heavy SM traffic, by access pattern?
//
// The Crossword distribute kernel (cfg 4) writes 5 bytes for every byte it reads and stays below the measured copy
// bandwidth; making it more parallel made it slower (tools/distribute_ab.py compares the variants).  This probe separates
// the memory system's ceiling from the kernel's own structure:
//   fill        write-only, grid-stride 128-bit stores (st.global / .cs / .wt)
//   fan K       every thread loads one 16-byte vector and stores it to K destination streams that are `gap` bytes apart
//               (K = 1: copy; K = 5: the distribute ratio) -- flat grid-stride, i.e. the friendliest possible layout
//   rows K      the distribute layout: a warp owns a "codeword" of `cols` columns, walks it 32 (or 64) columns per pass and
//               writes each column to K destination slots in K far-apart logs (+ row pitch), codewords of a CTA far apart
// Reported: total DRAM bytes moved (reads + writes) / time, best of 5.
//
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/hbm_probe tools/hbm_probe.cu
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>

#define CK(x)                                                                                                   \
    do {                                                                                                        \
        cudaError_t e_ = (x);                                                                                   \
        if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } \
    } while (0)

__device__ __forceinline__ uint4 ldg128(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
template <int MODE>
__device__ __forceinline__ void stg128(void *p, const uint4 &v) {
    if (MODE == 0) asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    else if (MODE == 1) asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    else asm volatile("st.global.wt.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(256) fill_kernel(uint4 *dst, size_t nvec) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    const uint4 v = make_uint4(threadIdx.x, blockIdx.x, 3u, 4u);
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) stg128<MODE>(dst + i, v);
}

template <int MODE, int K>
__global__ void __launch_bounds__(256) fan_kernel(const uint4 *__restrict__ src, uint4 *dst, size_t nvec, size_t gap_vec) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
        const uint4 v = ldg128(src + i);
#pragma unroll
        for (int k = 0; k < K; ++k) stg128<MODE>(dst + k * gap_vec + i, v);
    }
}

// warp per codeword of `cols` columns; K destination logs `gap` apart; codeword g's slot at g*cols within each log
template <int MODE, int K, int U>
__global__ void __launch_bounds__(256) rows_kernel(const uint4 *__restrict__ src, uint4 *dst, size_t ncw, uint32_t cols, size_t gap_vec) {
    const uint32_t lane = threadIdx.x & 31u;
    const size_t warp = (size_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5, nwarps = (size_t(gridDim.x) * blockDim.x) >> 5;
    for (size_t g = warp; g < ncw; g += nwarps) {
        const uint4 *s = src + g * cols;
        uint4 *d = dst + g * cols;
        for (uint32_t v0 = 0; v0 < cols; v0 += 32u * U) {
            uint4 x[U];
#pragma unroll
            for (int u = 0; u < U; ++u) x[u] = (v0 + u * 32u + lane < cols) ? ldg128(s + v0 + u * 32u + lane) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (v0 + u * 32u + lane < cols) {
#pragma unroll
                    for (int k = 0; k < K; ++k) stg128<MODE>(d + k * gap_vec + v0 + u * 32u + lane, x[u]);
                }
        }
    }
}

template <typename F>
static double best_of(F &&launch, double bytes) {
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    double best = 0;
    for (int rep = 0; rep < 6; ++rep) {
        CK(cudaEventRecord(a)); launch(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
        float ms; CK(cudaEventElapsedTime(&ms, a, b));
        const double gbs = bytes / (ms * 1e-3) / 1e9;
        if (rep > 0 && gbs > best) best = gbs;
    }
    return best;
}

int main() {
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    const size_t SRC = size_t(8) << 30, K = 5, GAP = size_t(9) << 30;         // 8 GiB source, five 9-GiB-apart destination logs
    uint8_t *src, *dst;
    CK(cudaMalloc(&src, SRC)); CK(cudaMalloc(&dst, K * GAP));
    CK(cudaMemset(src, 0x3c, SRC));
    const size_t nvec = SRC / 16, gap_vec = GAP / 16;
    printf("# %s, %d SMs; source 8 GiB, destinations 9 GiB apart; GB/s of DRAM traffic (reads + writes), best of 5\n", prop.name, sms);
    printf("memset (cudaMemsetAsync)                                  %8.0f\n", best_of([&] { CK(cudaMemsetAsync(dst, 1, SRC)); }, double(SRC)));
    for (int ctas : {4, 8, 16}) {
        printf("fill  st.global     %2d CTAs/SM                             %8.0f\n", ctas, best_of([&] { fill_kernel<0><<<sms * ctas, 256>>>((uint4 *)dst, nvec); }, double(SRC)));
        printf("fill  st.global.cs  %2d CTAs/SM                             %8.0f\n", ctas, best_of([&] { fill_kernel<1><<<sms * ctas, 256>>>((uint4 *)dst, nvec); }, double(SRC)));
    }
    printf("fill  st.global.wt   8 CTAs/SM                             %8.0f\n", best_of([&] { fill_kernel<2><<<sms * 8, 256>>>((uint4 *)dst, nvec); }, double(SRC)));
    for (int ctas : {8, 32}) {
        printf("fan 1 (copy)   st.cs %2d CTAs/SM                            %8.0f\n", ctas, best_of([&] { fan_kernel<1, 1><<<sms * ctas, 256>>>((const uint4 *)src, (uint4 *)dst, nvec, gap_vec); }, 2.0 * SRC));
        printf("fan 2          st.cs %2d CTAs/SM                            %8.0f\n", ctas, best_of([&] { fan_kernel<1, 2><<<sms * ctas, 256>>>((const uint4 *)src, (uint4 *)dst, nvec, gap_vec); }, 3.0 * SRC));
        printf("fan 5          st.cs %2d CTAs/SM                            %8.0f\n", ctas, best_of([&] { fan_kernel<1, 5><<<sms * ctas, 256>>>((const uint4 *)src, (uint4 *)dst, nvec, gap_vec); }, 6.0 * SRC));
        printf("fan 5          st    %2d CTAs/SM                            %8.0f\n", ctas, best_of([&] { fan_kernel<0, 5><<<sms * ctas, 256>>>((const uint4 *)src, (uint4 *)dst, nvec, gap_vec); }, 6.0 * SRC));
    }
    for (uint32_t cols : {86u, 342u, 1366u}) {        // 4 KB / 16 KB / 64 KB payloads at RS(3,2)
        const size_t ncw = nvec / cols;
        const double bytes = 6.0 * double(ncw) * cols * 16;
        for (int ctas : {3, 6}) {
            printf("rows 5 x %4u cols, st.cs, 1 col/pass, %d CTAs/SM            %8.0f\n", cols, ctas, best_of([&] { rows_kernel<1, 5, 1><<<sms * ctas * 4, 256>>>((const uint4 *)src, (uint4 *)dst, ncw, cols, gap_vec); }, bytes));
            printf("rows 5 x %4u cols, st.cs, 2 col/pass, %d CTAs/SM            %8.0f\n", cols, ctas, best_of([&] { rows_kernel<1, 5, 2><<<sms * ctas * 4, 256>>>((const uint4 *)src, (uint4 *)dst, ncw, cols, gap_vec); }, bytes));
            printf("rows 5 x %4u cols, st,    2 col/pass, %d CTAs/SM            %8.0f\n", cols, ctas, best_of([&] { rows_kernel<0, 5, 2><<<sms * ctas * 4, 256>>>((const uint4 *)src, (uint4 *)dst, ncw, cols, gap_vec); }, bytes));
        }
    }
    return 0;
}
