// nvlink_probe.cu -- how fast can ONE H100 move bytes into / out of a peer's HBM over NVLink, by mechanism?
//
// Decides how the multi-GPU accept step should deliver shard planes to the simulated follower replicas
// (DESIGN.md section 6).  Single process, two GPUs (0 and 1) with peer access; every test moves BYTES per
// direction, best of REPS, unidirectional (0 -> 1) and bidirectional (0 -> 1 and 1 -> 0 at the same time):
//   ce        cudaMemcpyPeerAsync (copy engine)
//   st        SM push: ld.global.nc local, st.global{,.cs,.wt} v4 to the peer, `unroll` vectors in flight per thread
//   ld        SM pull: ld.global.nc v4 from the peer, st.global.cs local
//   bulk      SM push through shared memory: cp.async.bulk global->shared (local), cp.async.bulk shared->global (peer),
//             a ring of `stages` tiles of `tile` bytes per CTA (TMA 1-D bulk copies, one elected thread issues)
//   rows      the encode kernel's pattern: a CTA walks "codewords", each thread stores one 16-byte column into each
//             of 4 peer planes (row pitch 1376 B) -- with and without the final per-CTA system fence
//
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/nvlink_probe tools/nvlink_probe.cu
// Run:   ./tools/nvlink_probe   (on a box with two peer-capable GPUs)
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                                  \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) {                                                               \
            fprintf(stderr, "CUDA error %s at %s:%d: %s\n", #x, __FILE__, __LINE__, cudaGetErrorString(e_)); \
            exit(1);                                                                           \
        }                                                                                      \
    } while (0)

static constexpr size_t BYTES = size_t(2) << 30;   // per direction
static constexpr int REPS = 5;

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

// flat copy: grid-stride over 16-byte vectors, U vectors in flight per thread
template <int MODE, int U>
__global__ void __launch_bounds__(256) copy_kernel(const uint4 *__restrict__ src, uint4 *__restrict__ dst, size_t nvec) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    for (; i + (U - 1) * stride < nvec; i += U * stride) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) v[u] = ldg128(src + i + u * stride);
#pragma unroll
        for (int u = 0; u < U; ++u) stg128<MODE>(dst + i + u * stride, v[u]);
    }
    for (; i < nvec; i += stride) stg128<MODE>(dst + i, ldg128(src + i));
}

// ---- bulk (TMA 1-D) ring: global(local) -> shared -> global(peer) ---------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nWAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *gdst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// one warp per CTA drives the ring (TMA needs no other threads); STAGES tiles of `tile` bytes
template <int STAGES>
__global__ void __launch_bounds__(32) bulk_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, size_t bytes, uint32_t tile) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t full[STAGES];
    const size_t ntiles = bytes / tile;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    if (threadIdx.x != 0) return;
    // tiles t = blockIdx.x, + gridDim.x, ...; stage s = it % STAGES
    size_t t = blockIdx.x;
    uint32_t it = 0;
    // prologue: fill the ring
    size_t tf = t;
    for (int s = 0; s < STAGES && tf < ntiles; ++s, tf += gridDim.x) {
        mbar_expect_tx(&full[s], tile);
        bulk_g2s(smem + size_t(s) * tile, src + tf * tile, tile, &full[s]);
    }
    for (; t < ntiles; t += gridDim.x, ++it) {
        const int s = it % STAGES;
        mbar_wait(&full[s], (it / STAGES) & 1u);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        bulk_s2g(dst + t * tile, smem + size_t(s) * tile, tile);
        bulk_commit();
        // refill this stage once its store has finished READING shared memory
        if (tf < ntiles) {
            bulk_wait_read<0>();
            mbar_expect_tx(&full[s], tile);
            bulk_g2s(smem + size_t(s) * tile, src + tf * tile, tile, &full[s]);
            tf += gridDim.x;
        }
    }
    bulk_wait_all();
}

// ---- the row kernel's store pattern: 4 peer planes, 86 columns of 16 B per codeword --------------------------
template <int MODE, bool FENCE>
__global__ void __launch_bounds__(128, 8) rows_kernel(const uint8_t *__restrict__ src, uint8_t *p0, uint8_t *p1, uint8_t *p2, uint8_t *p3,
                                                      uint32_t n, uint32_t vpc, uint32_t pitch) {
    const uint32_t v = threadIdx.x;
    for (uint32_t g = blockIdx.x; g < n; g += gridDim.x) {
        if (v >= vpc) continue;
        const uint8_t *s = src + size_t(g) * 4u * pitch + v * 16u;
        const uint4 a = ldg128(s), b = ldg128(s + pitch), c = ldg128(s + 2 * pitch), d = ldg128(s + 3 * pitch);
        const size_t o = size_t(g) * pitch + v * 16u;
        stg128<MODE>(p0 + o, a);
        stg128<MODE>(p1 + o, b);
        stg128<MODE>(p2 + o, c);
        stg128<MODE>(p3 + o, d);
    }
    if (FENCE) __threadfence_system();
}

struct Side {
    int dev, peer;
    uint8_t *local, *remote;   // local source buffer; destination buffer in the PEER's memory
    uint8_t *local_dst;        // destination buffer in local memory (for pulls), source = peer's `local`
    uint8_t *peer_src;
    cudaStream_t st;
    cudaEvent_t a, b;
};

template <typename F>
static void run(const char *name, Side *sides, int nsides, size_t bytes, F &&launch) {
    double best = 0;
    for (int rep = 0; rep < REPS + 1; ++rep) {
        for (int s = 0; s < nsides; ++s) { CK(cudaSetDevice(sides[s].dev)); CK(cudaDeviceSynchronize()); }
        for (int s = 0; s < nsides; ++s) { CK(cudaSetDevice(sides[s].dev)); CK(cudaEventRecord(sides[s].a, sides[s].st)); launch(sides[s]); CK(cudaEventRecord(sides[s].b, sides[s].st)); }
        float worst = 0;
        for (int s = 0; s < nsides; ++s) {
            CK(cudaSetDevice(sides[s].dev));
            CK(cudaEventSynchronize(sides[s].b));
            float ms; CK(cudaEventElapsedTime(&ms, sides[s].a, sides[s].b));
            if (ms > worst) worst = ms;
        }
        const double gbs = double(bytes) / (worst * 1e-3) / 1e9;
        if (rep > 0 && gbs > best) best = gbs;
    }
    printf("%-58s %s  %8.1f GB/s per direction\n", name, nsides == 2 ? "bidir" : "unidir", best);
    fflush(stdout);
}

int main() {
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (ndev < 2) { printf("need 2 GPUs, have %d\n", ndev); return 0; }
    Side sd[2];
    for (int i = 0; i < 2; ++i) {
        CK(cudaSetDevice(i));
        int can = 0; CK(cudaDeviceCanAccessPeer(&can, i, 1 - i));
        if (!can) { printf("no peer access %d -> %d\n", i, 1 - i); return 0; }
        CK(cudaDeviceEnablePeerAccess(1 - i, 0));
    }
    uint8_t *src[2], *dst[2];
    for (int i = 0; i < 2; ++i) {
        CK(cudaSetDevice(i));
        CK(cudaMalloc(&src[i], BYTES)); CK(cudaMalloc(&dst[i], BYTES));
        CK(cudaMemset(src[i], 0x5a + i, BYTES)); CK(cudaMemset(dst[i], 0, BYTES));
        CK(cudaStreamCreateWithFlags(&sd[i].st, cudaStreamNonBlocking));
        CK(cudaEventCreate(&sd[i].a)); CK(cudaEventCreate(&sd[i].b));
    }
    for (int i = 0; i < 2; ++i) {
        sd[i].dev = i; sd[i].peer = 1 - i; sd[i].local = src[i]; sd[i].remote = dst[1 - i];
        sd[i].local_dst = dst[i]; sd[i].peer_src = src[1 - i];
    }
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    printf("# %s, %d SMs, %zu MiB per direction, best of %d\n", prop.name, sms, BYTES >> 20, REPS);
    const size_t nvec = BYTES / 16;
    char name[160];
    for (int nsides = 1; nsides <= 2; ++nsides) {
        // local copy (HBM reference)
        run("local copy kernel (st.cs, unroll 4, SMs x 16 CTAs)", sd, nsides, BYTES,
            [&](Side &s) { copy_kernel<1, 4><<<sms * 16, 256, 0, s.st>>>((const uint4 *)s.local, (uint4 *)s.local_dst, nvec); });
        run("ce   cudaMemcpyPeerAsync", sd, nsides, BYTES,
            [&](Side &s) { CK(cudaMemcpyPeerAsync(s.remote, s.peer, s.local, s.dev, BYTES, s.st)); });
        for (int ctas : {1, 2, 4, 8, 16}) {
            snprintf(name, sizeof name, "st   push st.global        unroll 4, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<0, 4><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.local, (uint4 *)s.remote, nvec); });
        }
        for (int ctas : {2, 8}) {
            snprintf(name, sizeof name, "st   push st.global.cs     unroll 4, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<1, 4><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.local, (uint4 *)s.remote, nvec); });
            snprintf(name, sizeof name, "st   push st.global.wt     unroll 4, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<2, 4><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.local, (uint4 *)s.remote, nvec); });
            snprintf(name, sizeof name, "st   push st.global        unroll 1, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<0, 1><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.local, (uint4 *)s.remote, nvec); });
            snprintf(name, sizeof name, "st   push st.global        unroll 8, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<0, 8><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.local, (uint4 *)s.remote, nvec); });
        }
        for (int ctas : {1, 2, 4, 8, 16}) {
            snprintf(name, sizeof name, "ld   pull ld.global.nc     unroll 4, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<1, 4><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.peer_src, (uint4 *)s.local_dst, nvec); });
        }
        for (int ctas : {8}) {
            snprintf(name, sizeof name, "ld   pull ld.global.nc     unroll 8, %d CTAs/SM", ctas);
            run(name, sd, nsides, BYTES, [&](Side &s) { copy_kernel<1, 8><<<sms * ctas, 256, 0, s.st>>>((const uint4 *)s.peer_src, (uint4 *)s.local_dst, nvec); });
        }
        for (uint32_t tile : {1376u, 4096u, 16384u, 32768u}) {
            for (int ctas : {1, 2, 4}) {
                const size_t moved = (BYTES / tile) * tile;
                snprintf(name, sizeof name, "bulk push cp.async.bulk    tile %5u B x 4 stages, %d CTAs/SM", tile, ctas);
                run(name, sd, nsides, moved, [&](Side &s) {
                    CK(cudaFuncSetAttribute(bulk_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 32768));
                    bulk_kernel<4><<<sms * ctas, 32, 4 * tile, s.st>>>(s.local, s.remote, BYTES, tile);
                });
            }
        }
        {
            const uint32_t pitch = 1376, vpc = 86;
            const uint32_t n = uint32_t(BYTES / (4 * pitch));
            const size_t moved = size_t(n) * 4 * pitch;
            const size_t plane = size_t(n) * pitch;
            for (int waves : {1, 8, 64}) {
                const uint32_t grid = sms * 8 * waves;
                snprintf(name, sizeof name, "rows 4 planes x 86 cols, st.global.cs, no fence, %d waves", waves);
                run(name, sd, nsides, moved, [&](Side &s) { rows_kernel<1, false><<<grid, 96, 0, s.st>>>(s.local, s.remote, s.remote + plane, s.remote + 2 * plane, s.remote + 3 * plane, n, vpc, pitch); });
                snprintf(name, sizeof name, "rows 4 planes x 86 cols, st.global,    no fence, %d waves", waves);
                run(name, sd, nsides, moved, [&](Side &s) { rows_kernel<0, false><<<grid, 96, 0, s.st>>>(s.local, s.remote, s.remote + plane, s.remote + 2 * plane, s.remote + 3 * plane, n, vpc, pitch); });
                snprintf(name, sizeof name, "rows 4 planes x 86 cols, st.global.cs, sys fence, %d waves", waves);
                run(name, sd, nsides, moved, [&](Side &s) { rows_kernel<1, true><<<grid, 96, 0, s.st>>>(s.local, s.remote, s.remote + plane, s.remote + 2 * plane, s.remote + 3 * plane, n, vpc, pitch); });
            }
        }
    }
    // sanity: the last bulk / rows runs really delivered the bytes
    CK(cudaSetDevice(1));
    std::vector<uint8_t> h(4096);
    CK(cudaMemcpy(h.data(), dst[1], h.size(), cudaMemcpyDeviceToHost));
    printf("# dst[1][0..3] = %02x %02x %02x %02x (expect 5a)\n", h[0], h[1], h[2], h[3]);
    return 0;
}
