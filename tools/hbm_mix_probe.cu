// hbm_mix_probe.cu -- what does ONE H100's HBM deliver for the traffic mix of the RS(3,2) accept step?
//
// The fused accept step (bench.py cfg3) reads a 4096 B payload and writes two 1376 B padded parity rows per group,
// 2^20 groups: 59 % reads, 41 % writes.  The copy bandwidth (1:1) is not its ceiling.  This probe times flat
// streaming kernels at exactly that shape, with no arithmetic beyond the XORs that keep the loads live:
//   mix 3:2   item i reads row i (256 x 16 B) and writes 86 x 16 B to each of two planes (thread per output column)
//   read      the 4 GiB of payload rows, XOR-reduced per thread
//   write     the two parity planes (2 x 2^20 x 1376 B)
//   copy 1:1  the 4 GiB of payload rows to a second buffer
// Each at a few CTAs-per-SM settings; every (kernel, setting) is timed with CUDA events over 12 launches, the first
// dropped.  Reported: DRAM bytes moved (reads + writes) / time, best and median, and the time of the best launch.
// The last line is JSON with the best of each kind.
//
// Build + run: python tools/hbm_mix_probe.py   (nvcc -O3 -gencode arch=compute_90a,code=sm_90a, into a temp dir)
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                                                   \
    do {                                                                                                        \
        cudaError_t e_ = (x);                                                                                   \
        if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } \
    } while (0)

constexpr uint32_t kRowVec = 256;    // 4096 B payload row
constexpr uint32_t kOutVec = 86;     // 1376 B padded parity row (RS(3,2): L = 1366)

__device__ __forceinline__ uint4 ldg128(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg128_cs(void *p, const uint4 &v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 x4(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }

// thread <-> (item, output column) flat grid-stride; column c reads vectors c, c + 86, c + 172 of the row
__global__ void __launch_bounds__(256) mix_kernel(const uint4 *__restrict__ src, uint4 *out0, uint4 *out1, uint64_t n) {
    const uint64_t total = n * kOutVec, stride = uint64_t(gridDim.x) * blockDim.x;
    for (uint64_t t = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += stride) {
        const uint64_t i = t / kOutVec;
        const uint32_t c = uint32_t(t - i * kOutVec);
        const uint4 *row = src + i * kRowVec;
        const uint4 a = ldg128(row + c), b = ldg128(row + c + kOutVec);
        uint4 v = x4(a, b);
        if (c + 2 * kOutVec < kRowVec) v = x4(v, ldg128(row + c + 2 * kOutVec));
        stg128_cs(out0 + t, v);
        stg128_cs(out1 + t, x4(a, v));
    }
}

// the accept kernels' layout: a CTA of 96 threads per item, items strided over the grid
__global__ void __launch_bounds__(96) mix_row_kernel(const uint4 *__restrict__ src, uint4 *out0, uint4 *out1, uint64_t n) {
    const uint32_t c = threadIdx.x;
    if (c >= kOutVec) return;
    for (uint64_t i = blockIdx.x; i < n; i += gridDim.x) {
        const uint4 *row = src + i * kRowVec;
        const uint4 a = ldg128(row + c), b = ldg128(row + c + kOutVec);
        uint4 v = x4(a, b);
        if (c + 2 * kOutVec < kRowVec) v = x4(v, ldg128(row + c + 2 * kOutVec));
        stg128_cs(out0 + i * kOutVec + c, v);
        stg128_cs(out1 + i * kOutVec + c, x4(a, v));
    }
}

__global__ void __launch_bounds__(256) read_kernel(const uint4 *__restrict__ src, uint4 *sink, uint64_t nvec) {
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    uint4 acc = make_uint4(0, 0, 0, 0);
    for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) acc = x4(acc, ldg128(src + i));
    if ((acc.x ^ acc.y ^ acc.z ^ acc.w) == 0x9e3779b9u) sink[threadIdx.x] = acc;     // keeps the loads live
}

__global__ void __launch_bounds__(256) write_kernel(uint4 *dst, uint64_t nvec) {
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    const uint4 v = make_uint4(threadIdx.x, blockIdx.x, 3u, 4u);
    for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) stg128_cs(dst + i, v);
}

__global__ void __launch_bounds__(256) copy_kernel(const uint4 *__restrict__ src, uint4 *dst, uint64_t nvec) {
    const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
    for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) stg128_cs(dst + i, ldg128(src + i));
}

struct Result { double best_gbs, med_gbs, best_ms; };

template <typename F>
static Result timed(F &&launch, double bytes) {
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    std::vector<double> ms;
    for (int rep = 0; rep < 12; ++rep) {
        CK(cudaEventRecord(a)); launch(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
        CK(cudaGetLastError());
        float t; CK(cudaEventElapsedTime(&t, a, b));
        if (rep > 0) ms.push_back(t);
    }
    CK(cudaEventDestroy(a)); CK(cudaEventDestroy(b));
    std::sort(ms.begin(), ms.end());
    const double med = ms[ms.size() / 2];
    return {bytes / (ms[0] * 1e-3) / 1e9, bytes / (med * 1e-3) / 1e9, ms[0]};
}

int main() {
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    const uint64_t n = 1ull << 20;
    const uint64_t in_bytes = n * kRowVec * 16, plane_bytes = n * kOutVec * 16;
    uint8_t *src, *dst, *par;
    CK(cudaMalloc(&src, in_bytes)); CK(cudaMalloc(&dst, in_bytes)); CK(cudaMalloc(&par, 2 * plane_bytes));
    CK(cudaMemset(src, 0x3c, in_bytes)); CK(cudaMemset(par, 0, 2 * plane_bytes));
    uint4 *p0 = reinterpret_cast<uint4 *>(par), *p1 = reinterpret_cast<uint4 *>(par + plane_bytes);
    const double mix_bytes = double(in_bytes + 2 * plane_bytes);
    printf("# %s, %d SMs; 2^20 items: read 4096 B + write 2 x 1376 B each; GB/s of DRAM traffic (reads + writes), "
           "11 timed launches\n", prop.name, sms);
    printf("%-44s %9s %9s %9s\n", "kernel", "best", "median", "best ms");
    Result best_mix{0, 0, 0}, best_read{0, 0, 0}, best_write{0, 0, 0}, best_copy{0, 0, 0};
    auto row = [](const char *name, int cps, const Result &r, Result &keep) {
        printf("%-32s %2d CTAs/SM %9.0f %9.0f %9.3f\n", name, cps, r.best_gbs, r.med_gbs, r.best_ms);
        if (r.best_gbs > keep.best_gbs) keep = r;
    };
    for (int cps : {4, 8, 16})
        row("mix 3:2  flat, 256 thr", cps, timed([&] { mix_kernel<<<sms * cps, 256>>>((const uint4 *)src, p0, p1, n); }, mix_bytes), best_mix);
    for (int cps : {8, 16, 20})
        row("mix 3:2  row, 96 thr/item", cps, timed([&] { mix_row_kernel<<<sms * cps, 96>>>((const uint4 *)src, p0, p1, n); }, mix_bytes), best_mix);
    for (int cps : {4, 8, 16})
        row("read     flat, 256 thr", cps, timed([&] { read_kernel<<<sms * cps, 256>>>((const uint4 *)src, (uint4 *)dst, in_bytes / 16); }, double(in_bytes)), best_read);
    for (int cps : {4, 8, 16})
        row("write    flat, 256 thr", cps, timed([&] { write_kernel<<<sms * cps, 256>>>(p0, 2 * plane_bytes / 16); }, double(2 * plane_bytes)), best_write);
    for (int cps : {4, 8, 16})
        row("copy 1:1 flat, 256 thr", cps, timed([&] { copy_kernel<<<sms * cps, 256>>>((const uint4 *)src, (uint4 *)dst, in_bytes / 16); }, 2.0 * in_bytes), best_copy);
    printf("{\"card\": \"%s\", \"items\": %llu, \"mix32_gbs\": %.1f, \"mix32_ms\": %.4f, \"mix32_median_gbs\": %.1f, "
           "\"read_gbs\": %.1f, \"write_gbs\": %.1f, \"copy_gbs\": %.1f}\n",
           prop.name, (unsigned long long)n, best_mix.best_gbs, best_mix.best_ms, best_mix.med_gbs, best_read.best_gbs,
           best_write.best_gbs, best_copy.best_gbs);
    CK(cudaFree(src)); CK(cudaFree(dst)); CK(cudaFree(par));
    return 0;
}
