// capi.cu -- the extern "C" boundary declared in include/summerset_b200.h.
//
// Host-side logic only: handle management, argument checks that mirror the crate's error
// behaviour, coefficient-program construction, H2D/D2H plumbing for the host-buffer entry points.
// All arithmetic on shard bytes and vote masks happens in the kernels (rs_kernels.cu,
// tally_kernels.cu).  There is no CPU fallback anywhere in this file.
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <mutex>
#include <new>

#include "gf256.hpp"
#include "ss_internal.hpp"

namespace ssb {

// ---- errors -----------------------------------------------------------------------------------
// One buffer per calling thread: two coders driven from two tokio worker threads never see each other's text, and the
// pointer ss_last_error() returns stays valid until the next failing call on the same thread.
static thread_local char g_err[512] = "";

int set_error(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int cuda_error(cudaError_t e, const char *what, const char *file, int line) {
    // A failed runtime call also leaves its error as the thread's last error.  Clear it: otherwise the next successful
    // call reports it again from the cudaGetLastError() after its first kernel launch.
    cudaGetLastError();
    const char *base = strrchr(file, '/');
    const int code = (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorNoKernelImageForDevice)
                         ? SS_ERR_NO_DEVICE
                         : (e == cudaErrorMemoryAllocation ? SS_ERR_OUT_OF_MEMORY : SS_ERR_CUDA);
    return set_error(code, "CUDA error %d (%s) in %s at %s:%d", static_cast<int>(e), cudaGetErrorString(e), what,
                     base ? base + 1 : file, line);
}

int ctx_bind(ss_ctx *ctx) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (ctx->closing.load()) return set_error(SS_ERR_INVALID_ARG, "context was destroyed (a handle outlived it)");
    SS_CUDA(cudaSetDevice(ctx->device));
    return SS_OK;
}

int ctx_scratch(ss_ctx *ctx, size_t bytes, void **out) {
    if (bytes > ctx->scratch_bytes) {
        // the old block may still be in use by queued kernels: drain before freeing
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        if (ctx->scratch) SS_CUDA(cudaFree(ctx->scratch));
        ctx->scratch = nullptr;
        ctx->scratch_bytes = 0;
        size_t want = bytes < (1u << 20) ? (1u << 20) : bytes;
        SS_CUDA(cudaMalloc(&ctx->scratch, want));
        ctx->scratch_bytes = want;
    }
    *out = ctx->scratch;
    return SS_OK;
}

// grow-only pinned host staging for the single-codeword calls: the caller's shard slices are pageable memory, and one
// pinned H2D + one pinned D2H cost far less than d + p pageable copies (each of which the driver stages anyway)
static int ctx_pinned(ss_ctx *ctx, size_t bytes, uint8_t **out) {
    if (bytes > ctx->pinned_bytes) {
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        if (ctx->pinned) SS_CUDA(cudaFreeHost(ctx->pinned));
        ctx->pinned = nullptr;
        ctx->pinned_bytes = 0;
        size_t want = bytes < (1u << 20) ? (1u << 20) : bytes;
        SS_CUDA(cudaHostAlloc(&ctx->pinned, want, cudaHostAllocDefault));
        ctx->pinned_bytes = want;
    }
    *out = static_cast<uint8_t *>(ctx->pinned);
    return SS_OK;
}
constexpr size_t kStagedCallLimit = size_t(8) << 20;    // larger codewords copy straight from the caller's slices

static int pipeline_init(ss_ctx *ctx) {
    if (ctx->pipeline_ready) return SS_OK;
    SS_CUDA(cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking));
    SS_CUDA(cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
    for (int i = 0; i < ss_ctx::kStages; ++i) {
        SS_CUDA(cudaEventCreateWithFlags(&ctx->ev_h2d[i], cudaEventDisableTiming));
        SS_CUDA(cudaEventCreateWithFlags(&ctx->ev_kernel[i], cudaEventDisableTiming));
        SS_CUDA(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming));
    }
    ctx->pipeline_ready = true;
    return SS_OK;
}

static int pipeline_staging(ss_ctx *ctx, size_t in_bytes, size_t out_bytes) {
    SS_TRY(pipeline_init(ctx));
    if (in_bytes > ctx->stage_in_bytes) {
        for (int i = 0; i < ss_ctx::kStages; ++i) {
            if (ctx->stage_in[i]) SS_CUDA(cudaFree(ctx->stage_in[i]));
            ctx->stage_in[i] = nullptr;
            SS_CUDA(cudaMalloc(&ctx->stage_in[i], in_bytes));
        }
        ctx->stage_in_bytes = in_bytes;
    }
    if (out_bytes > ctx->stage_out_bytes) {
        for (int i = 0; i < ss_ctx::kStages; ++i) {
            if (ctx->stage_out[i]) SS_CUDA(cudaFree(ctx->stage_out[i]));
            ctx->stage_out[i] = nullptr;
            SS_CUDA(cudaMalloc(&ctx->stage_out[i], out_bytes));
        }
        ctx->stage_out_bytes = out_bytes;
    }
    return SS_OK;
}

// ---- coefficient programs -----------------------------------------------------------------------
// header + splats[p*d*8] + hmask[p*d*8] + (d <= 4) transposed masks hmT[p*8*4] (one uint4 = the masks of all
// inputs for one (output, bit) pair)
static size_t prog_bytes(int d, int p) {
    return sizeof(ProgHeader) + 2 * size_t(p) * size_t(d) * 8 * 4 + (d <= 4 ? size_t(p) * 8 * 4 * 4 : 0);
}

// fills, for coefficient c = c[j][i] of a (p x d) program: the bit-plane splats, the Horner bit masks
// (stored p*d*8 words after the splats) and the running top bit of row j
static void fill_coef(uint8_t *prog, int d, int p, int j, int i, uint8_t c) {
    ProgHeader *h = reinterpret_cast<ProgHeader *>(prog);
    uint32_t *splat = reinterpret_cast<uint32_t *>(prog + sizeof(ProgHeader));
    uint32_t *hmask = splat + size_t(p) * d * 8;
    for (int k = 0; k < 8; ++k) {
        const uint32_t b = gf::mul(c, static_cast<uint8_t>(1u << k));
        splat[(size_t(j) * d + i) * 8 + k] = b * 0x01010101u;
        hmask[(size_t(j) * d + i) * 8 + k] = ((c >> k) & 1u) ? 0xffffffffu : 0u;
        if (d <= 4) (hmask + size_t(p) * d * 8)[(size_t(j) * 8 + k) * 4 + i] = ((c >> k) & 1u) ? 0xffffffffu : 0u;
        if (((c >> k) & 1u) && k > h->top[j]) h->top[j] = static_cast<uint8_t>(k);
        if (j < 2 && h->top[j] > h->topT[j]) h->topT[j] = h->top[j];
    }
}

// program for `present` pattern: outputs = missing data shards (then missing parity unless data_only)
static void build_decode_program(const gf::Matrix &M, int d, int p, uint32_t present, bool data_only,
                                 uint8_t *out) {
    const int t = d + p;
    memset(out, 0, prog_bytes(d, p));
    ProgHeader *h = reinterpret_cast<ProgHeader *>(out);
    int src[kMaxD], ns = 0;
    for (int i = 0; i < t && ns < d; ++i)
        if ((present >> i) & 1u) src[ns++] = i;
    if (ns < d) { h->valid = 0; return; }        // crate: Error::TooFewShardsPresent
    h->valid = 1;
    for (int i = 0; i < d; ++i) h->src[i] = static_cast<uint8_t>(src[i]);
    gf::Matrix sub(d, d), dec;
    for (int r = 0; r < d; ++r)
        for (int c = 0; c < d; ++c) sub.at(r, c) = M.at(src[r], c);
    if (!sub.inverse(dec)) { h->valid = 0; return; }   // cannot happen for an MDS matrix
    int n_out = 0;
    for (int r = 0; r < d; ++r) {
        if ((present >> r) & 1u) continue;
        h->dst[n_out] = static_cast<uint8_t>(r);
        for (int i = 0; i < d; ++i) fill_coef(out, d, p, n_out, i, dec.at(r, i));
        ++n_out;
    }
    h->n_missing_data = static_cast<uint8_t>(n_out);
    // XOR chain (d <= 4 fast path only): when exactly two data shards r0 < r1 are missing and the all-ones parity
    // row (index d) is among the sources, d_r1 = p_0 ^ d_r0 ^ (the available data shards): the second output
    // needs no dense row, only XORs of sources plus the first output.
    if (d <= 4 && n_out == 2) {
        bool ones = true;
        for (int c = 0; c < d; ++c) ones = ones && M.at(d, c) == 1;
        bool has_p0 = false;
        for (int i = 0; i < d; ++i) has_p0 = has_p0 || src[i] == d;
        if (ones && has_p0) {
            uint32_t *hmT = reinterpret_cast<uint32_t *>(out + sizeof(ProgHeader)) + 2 * size_t(p) * d * 8;
            for (int k = 0; k < 8; ++k)
                for (int i = 0; i < 4; ++i) hmT[(size_t(1) * 8 + k) * 4 + i] = 0u;
            for (int i = 0; i < d; ++i)                                   // p_0 and the available data shards only
                if (src[i] <= d) hmT[(size_t(1) * 8 + 0) * 4 + i] = 0xffffffffu;
            h->topT[1] = 0;
            h->chain1 = 1;
        }
    }
    if (!data_only) {
        for (int q = d; q < t; ++q) {
            if ((present >> q) & 1u) continue;
            h->dst[n_out] = static_cast<uint8_t>(q);
            // parity row q over the d sources = M[q] * dec
            for (int i = 0; i < d; ++i) {
                uint8_t c = 0;
                for (int k = 0; k < d; ++k) c ^= gf::mul(M.at(q, k), dec.at(k, i));
                fill_coef(out, d, p, n_out, i, c);
            }
            ++n_out;
        }
    }
    h->n_out = static_cast<uint8_t>(n_out);
}

static void build_encode_program(const gf::Matrix &M, int d, int p, uint8_t *out) {
    memset(out, 0, prog_bytes(d, p));
    ProgHeader *h = reinterpret_cast<ProgHeader *>(out);
    h->valid = 1;
    h->n_out = static_cast<uint8_t>(p);
    for (int i = 0; i < d; ++i) h->src[i] = static_cast<uint8_t>(i);
    for (int j = 0; j < p; ++j) {
        h->dst[j] = static_cast<uint8_t>(j);      // relative to the parity base
        for (int i = 0; i < d; ++i) fill_coef(out, d, p, j, i, M.at(d + j, i));
    }
}

static int check_shard_args(const ss_rs_coder *c, const void *shards, size_t n_shards, size_t shard_len) {
    if (c == nullptr || shards == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder or shard array");
    const size_t t = size_t(c->d + c->p);
    if (n_shards < t) return set_error(SS_ERR_TOO_FEW_SHARDS, "too few shards: %zu < %zu", n_shards, t);
    if (n_shards > t) return set_error(SS_ERR_TOO_MANY_SHARDS, "too many shards: %zu > %zu", n_shards, t);
    if (shard_len == 0) return set_error(SS_ERR_EMPTY_SHARD, "empty shard");
    if (shard_len >= 0x7fffffffull / size_t(c->d))
        return set_error(SS_ERR_INVALID_ARG, "shard too large for one call: %zu bytes", shard_len);
    return SS_OK;
}

// validates the wait half of an ss_step_sync and turns it into the kernels' argument
int make_flag_wait(ss_ctx *ctx, const ss_step_sync *sync, dev::FlagWait *out) {
    *out = dev::FlagWait{nullptr, 0, 0, 0, nullptr};
    if (sync == nullptr) return SS_OK;
    if (sync->n_wait > 32 || sync->n_signal > 32) return set_error(SS_ERR_INVALID_ARG, "at most 32 wait / signal flags");
    if (sync->n_wait != 0 && sync->wait_flags == nullptr) return set_error(SS_ERR_INVALID_ARG, "null wait_flags");
    if (sync->n_signal != 0 && sync->signal_flags == nullptr) return set_error(SS_ERR_INVALID_ARG, "null signal_flags");
    if (sync->n_wait == 0 || sync->wait_value == 0) return SS_OK;        // counters start at 0: nothing to wait for
    out->flags = sync->wait_flags; out->n = sync->n_wait; out->value = sync->wait_value;
    out->timeout_ns = 2000000000ull;
    out->status = ctx->dev_status;
    return SS_OK;
}

// frees everything the context owns; only called once no coder / engine handle refers to it any more
static void ctx_teardown(ss_ctx *ctx) {
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->pipeline_ready) {
        cudaStreamSynchronize(ctx->h2d_stream);
        cudaStreamSynchronize(ctx->d2h_stream);
        for (int i = 0; i < ss_ctx::kStages; ++i) {
            cudaEventDestroy(ctx->ev_h2d[i]);
            cudaEventDestroy(ctx->ev_kernel[i]);
            cudaEventDestroy(ctx->ev_done[i]);
        }
        cudaStreamDestroy(ctx->h2d_stream);
        cudaStreamDestroy(ctx->d2h_stream);
    }
    for (int i = 0; i < ss_ctx::kStages; ++i) {
        if (ctx->stage_in[i]) cudaFree(ctx->stage_in[i]);
        if (ctx->stage_out[i]) cudaFree(ctx->stage_out[i]);
    }
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    if (ctx->dev_status) cudaFree(ctx->dev_status);
    if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

// The context holds one reference to itself (dropped by ss_ctx_destroy) and every coder / engine one more: whoever drops
// the last one tears it down, so destroy and the handles' destroy calls may come in any order and from any threads.
void ctx_retain(ss_ctx *ctx) { ctx->live_handles.fetch_add(1); }
void ctx_release(ss_ctx *ctx) {
    if (ctx->live_handles.fetch_sub(1) == 1) ctx_teardown(ctx);
}


}  // namespace ssb

using namespace ssb;

// =================================================================================================
extern "C" {

int ss_version(void) { return SS_VERSION; }

const char *ss_last_error(void) { return g_err; }

const char *ss_strerror(int code) {
    switch (code) {
        case SS_OK: return "ok";
        case SS_ERR_TOO_FEW_SHARDS: return "too few shards";
        case SS_ERR_TOO_MANY_SHARDS: return "too many shards";
        case SS_ERR_TOO_FEW_DATA_SHARDS: return "too few data shards";
        case SS_ERR_TOO_MANY_DATA_SHARDS: return "too many data shards";
        case SS_ERR_TOO_FEW_PARITY_SHARDS: return "too few parity shards";
        case SS_ERR_TOO_MANY_PARITY_SHARDS: return "too many parity shards";
        case SS_ERR_TOO_FEW_BUFFER_SHARDS: return "too few buffer shards";
        case SS_ERR_TOO_MANY_BUFFER_SHARDS: return "too many buffer shards";
        case SS_ERR_INCORRECT_SHARD_SIZE: return "incorrect shard size";
        case SS_ERR_TOO_FEW_SHARDS_PRESENT: return "too few shards present";
        case SS_ERR_EMPTY_SHARD: return "empty shard";
        case SS_ERR_INVALID_SHARD_FLAGS: return "invalid shard flags";
        case SS_ERR_INVALID_INDEX: return "invalid index";
        case SS_ERR_INVALID_ARG: return "invalid argument";
        case SS_ERR_UNSUPPORTED: return "unsupported configuration";
        case SS_ERR_OUT_OF_MEMORY: return "out of device memory";
        case SS_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (no CPU fallback)";
        case SS_ERR_CUDA: return "CUDA error";
        default: return "unknown error";
    }
}

// ---- context ------------------------------------------------------------------------------------
static int ctx_create_common(int device, void *stream, bool borrow, ss_ctx **out) {
    if (out == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        return set_error(SS_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback",
                         e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    }
    if (device < 0 || device >= count) return set_error(SS_ERR_INVALID_ARG, "device %d out of range [0,%d)", device, count);
    cudaDeviceProp prop;
    SS_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return set_error(SS_ERR_NO_DEVICE, "device %d is sm_%d%d; kernels are built for sm_90a only", device, prop.major,
                         prop.minor);
    SS_CUDA(cudaSetDevice(device));
    ss_ctx *ctx = new (std::nothrow) ss_ctx();
    if (!ctx) return set_error(SS_ERR_OUT_OF_MEMORY, "host allocation failed");
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if (borrow) {
        ctx->stream = static_cast<cudaStream_t>(stream);
        ctx->owns_stream = false;
    } else {
        e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) { delete ctx; return cuda_error(e, "cudaStreamCreateWithFlags", __FILE__, __LINE__); }
        ctx->owns_stream = true;
    }
    e = cudaMalloc(reinterpret_cast<void **>(&ctx->dev_status), 256);
    // on the context's stream, which a non-blocking stream needs: the legacy default stream is not ordered before it
    if (e == cudaSuccess) e = cudaMemsetAsync(ctx->dev_status, 0, 256, ctx->stream);
    if (e != cudaSuccess) {
        if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
        delete ctx;
        return cuda_error(e, "allocate device status word", __FILE__, __LINE__);
    }
    *out = ctx;
    return SS_OK;
}

int ss_ctx_create(int device, ss_ctx **out) { return ctx_create_common(device, nullptr, false, out); }
int ss_ctx_create_on_stream(int device, void *cuda_stream, ss_ctx **out) {
    return ctx_create_common(device, cuda_stream, true, out);
}

// Handles created on a context (coders, engines) keep it alive: destroying the context first only marks it closed,
// and the last handle's destroy call tears it down (either order is safe, e.g. Python garbage collection).
int ss_ctx_destroy(ss_ctx *ctx) {
    if (ctx == nullptr) return SS_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->closing.exchange(true)) return SS_OK;     // a second destroy while handles keep the context alive
    ctx_release(ctx);                                  // the context's own reference
    return SS_OK;
}

int ss_ctx_sync(ss_ctx *ctx) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    return SS_OK;
}

void *ss_ctx_stream(ss_ctx *ctx) { return ctx ? static_cast<void *>(ctx->stream) : nullptr; }
int ss_ctx_sm_count(ss_ctx *ctx) { return ctx ? ctx->sm_count : 0; }
uint64_t ss_ctx_launch_count(ss_ctx *ctx) { return ctx ? ctx->launches : 0; }

int ss_dev_alloc(ss_ctx *ctx, size_t bytes, void **dptr) {
    SS_TRY(ctx_bind(ctx));
    if (dptr == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    SS_CUDA(cudaMalloc(dptr, bytes ? bytes : 1));
    return SS_OK;
}
int ss_dev_free(ss_ctx *ctx, void *dptr) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaFree(dptr));
    return SS_OK;
}
int ss_dev_memset(ss_ctx *ctx, void *dptr, int value, size_t bytes) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaMemsetAsync(dptr, value, bytes, ctx->stream));
    return SS_OK;
}
int ss_host_alloc(ss_ctx *ctx, size_t bytes, void **hptr) {
    SS_TRY(ctx_bind(ctx));
    if (hptr == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    SS_CUDA(cudaHostAlloc(hptr, bytes ? bytes : 1, cudaHostAllocDefault));
    return SS_OK;
}
int ss_host_alloc_wc(ss_ctx *ctx, size_t bytes, void **hptr) {
    SS_TRY(ctx_bind(ctx));
    if (hptr == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    SS_CUDA(cudaHostAlloc(hptr, bytes ? bytes : 1, cudaHostAllocWriteCombined));
    return SS_OK;
}
int ss_host_free(ss_ctx *ctx, void *hptr) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaFreeHost(hptr));
    return SS_OK;
}
int ss_copy_h2d(ss_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return SS_OK;
}
int ss_copy_d2h(ss_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    return SS_OK;
}

int ss_copy_d2d(ss_ctx *ctx, void *dst_dev, const void *src_dev, size_t bytes) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaMemcpyAsync(dst_dev, src_dev, bytes, cudaMemcpyDefault, ctx->stream));
    return SS_OK;
}

int ss_ipc_export(ss_ctx *ctx, void *dptr, uint8_t handle[SS_IPC_HANDLE_BYTES]) {
    SS_TRY(ctx_bind(ctx));
    if (dptr == nullptr || handle == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == SS_IPC_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    SS_CUDA(cudaIpcGetMemHandle(&h, dptr));
    memcpy(handle, &h, sizeof(h));
    return SS_OK;
}

int ss_ipc_open(ss_ctx *ctx, const uint8_t handle[SS_IPC_HANDLE_BYTES], void **dptr) {
    SS_TRY(ctx_bind(ctx));
    if (dptr == nullptr || handle == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    SS_CUDA(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
    return SS_OK;
}

int ss_ipc_close(ss_ctx *ctx, void *dptr) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaIpcCloseMemHandle(dptr));
    return SS_OK;
}

// ---- coder --------------------------------------------------------------------------------------
int ss_rs_coder_create(ss_ctx *ctx, int d, int p, ss_rs_coder **out) {
    if (out == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    *out = nullptr;
    SS_TRY(ctx_bind(ctx));
    // crate ReedSolomon::new error order
    if (d <= 0) return set_error(SS_ERR_TOO_FEW_DATA_SHARDS, "too few data shards: %d", d);
    if (p <= 0) return set_error(SS_ERR_TOO_FEW_PARITY_SHARDS, "too few parity shards: %d", p);
    if (d + p > 256) return set_error(SS_ERR_TOO_MANY_SHARDS, "too many shards: %d + %d > 256", d, p);
    ss_rs_coder *c = new (std::nothrow) ss_rs_coder();
    if (!c) return set_error(SS_ERR_OUT_OF_MEMORY, "host allocation failed");
    c->ctx = ctx; c->d = d; c->p = p;
    ctx_retain(ctx);
    gf::Matrix M;

    try {
        M = gf::coding_matrix(d, p);
    } catch (const std::exception &ex) {
        ctx_release(ctx);
        delete c;
        return set_error(SS_ERR_INVALID_ARG, "matrix construction failed: %s", ex.what());
    }
    c->matrix = M.v;
    c->is_rs32 = (d == 3 && p == 2 && M.at(3, 0) == 1 && M.at(3, 1) == 1 && M.at(3, 2) == 1 && M.at(4, 0) == 0x0f &&
                  M.at(4, 1) == 0x08 && M.at(4, 2) == 0x06);
    c->batch_ok = (d <= kMaxD && p <= kMaxP);
    c->dec_ok = c->batch_ok && (d + p <= 12);
    c->prog_stride = prog_bytes(d, p);
    if (c->batch_ok) {
        std::vector<uint8_t> buf(c->prog_stride);
        build_encode_program(M, d, p, buf.data());
        cudaError_t e = cudaMalloc(&c->enc_prog, buf.size());
        if (e == cudaSuccess) e = cudaMemcpy(c->enc_prog, buf.data(), buf.size(), cudaMemcpyHostToDevice);
        c->static_code = ssb::match_static_code(d, p, c->matrix.data());
        if (e == cudaSuccess && d <= 8) {
            std::vector<uint32_t> t8(size_t(p) * 8 * 8, 0u);
            for (int j = 0; j < p; ++j) {
                int top = 0;
                for (int i = 0; i < d; ++i)
                    for (int k = 0; k < 8; ++k)
                        if ((M.at(d + j, i) >> k) & 1) { t8[(size_t(j) * 8 + k) * 8 + i] = 0xffffffffu; if (k > top) top = k; }
                c->enc_top[j] = static_cast<uint8_t>(top);
            }
            e = cudaMalloc(&c->enc_hmT8, t8.size() * 4);
            if (e == cudaSuccess) e = cudaMemcpy(c->enc_hmT8, t8.data(), t8.size() * 4, cudaMemcpyHostToDevice);
        }
        if (e != cudaSuccess) { ss_rs_coder_destroy(c); return cuda_error(e, "upload encode program", __FILE__, __LINE__); }
    }
    if (c->dec_ok) {
        const size_t npat = size_t(1) << (d + p);
        std::vector<uint8_t> all(npat * c->prog_stride), dat(npat * c->prog_stride);
        for (size_t pat = 0; pat < npat; ++pat) {
            build_decode_program(M, d, p, static_cast<uint32_t>(pat), false, all.data() + pat * c->prog_stride);
            build_decode_program(M, d, p, static_cast<uint32_t>(pat), true, dat.data() + pat * c->prog_stride);
        }
        if (d <= 4) {
            // compact copies for the small-code kernel: header fields + the transposed mask rows only
            c->fast_stride = sizeof(FastProgHeader) + size_t(p) * 8 * 16;
            std::vector<uint8_t> fa(npat * c->fast_stride, 0), fd(npat * c->fast_stride, 0);
            auto compact = [&](const std::vector<uint8_t> &full, std::vector<uint8_t> &fast) {
                for (size_t pat = 0; pat < npat; ++pat) {
                    const uint8_t *src = full.data() + pat * c->prog_stride;
                    const ProgHeader *h = reinterpret_cast<const ProgHeader *>(src);
                    uint8_t *dst = fast.data() + pat * c->fast_stride;
                    FastProgHeader *f = reinterpret_cast<FastProgHeader *>(dst);
                    f->valid = h->valid; f->n_out = h->n_out; f->chain1 = h->chain1;
                    for (int i = 0; i < 4; ++i) f->src[i] = h->src[i];
                    for (int j = 0; j < kMaxP; ++j) { f->dst[j] = h->dst[j]; f->top[j] = j < 2 ? h->topT[j] : h->top[j]; }
                    memcpy(dst + sizeof(FastProgHeader), src + sizeof(ProgHeader) + 2 * size_t(p) * d * 8 * 4, size_t(p) * 8 * 16);
                }
            };
            compact(all, fa);
            compact(dat, fd);
            cudaError_t e2 = cudaMalloc(&c->fast_progs, fa.size());
            if (e2 == cudaSuccess) e2 = cudaMalloc(&c->fast_progs_data, fd.size());
            if (e2 == cudaSuccess) e2 = cudaMemcpy(c->fast_progs, fa.data(), fa.size(), cudaMemcpyHostToDevice);
            if (e2 == cudaSuccess) e2 = cudaMemcpy(c->fast_progs_data, fd.data(), fd.size(), cudaMemcpyHostToDevice);
            if (e2 != cudaSuccess) { ss_rs_coder_destroy(c); return cuda_error(e2, "upload compact decode programs", __FILE__, __LINE__); }
        }
        cudaError_t e = cudaMalloc(&c->dec_progs, all.size());
        if (e == cudaSuccess) e = cudaMalloc(&c->dec_progs_data, dat.size());
        if (e == cudaSuccess) e = cudaMemcpy(c->dec_progs, all.data(), all.size(), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(c->dec_progs_data, dat.data(), dat.size(), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { ss_rs_coder_destroy(c); return cuda_error(e, "upload decode programs", __FILE__, __LINE__); }
    }
    *out = c;
    return SS_OK;
}

int ss_rs_coder_destroy(ss_rs_coder *c) {
    if (c == nullptr) return SS_OK;
    if (c->ctx) {
        cudaSetDevice(c->ctx->device);
        cudaStreamSynchronize(c->ctx->stream);
    }
    if (c->enc_prog) cudaFree(c->enc_prog);
    if (c->enc_hmT8) cudaFree(c->enc_hmT8);
    if (c->dec_progs) cudaFree(c->dec_progs);
    if (c->dec_progs_data) cudaFree(c->dec_progs_data);
    if (c->fast_progs) cudaFree(c->fast_progs);
    if (c->fast_progs_data) cudaFree(c->fast_progs_data);
    jit_release(c);
    if (c->ctx) ctx_release(c->ctx);
    delete c;
    return SS_OK;
}

int ss_rs_data_shard_count(const ss_rs_coder *c) { return c ? c->d : 0; }
int ss_rs_parity_shard_count(const ss_rs_coder *c) { return c ? c->p : 0; }
int ss_rs_total_shard_count(const ss_rs_coder *c) { return c ? c->d + c->p : 0; }
int ss_rs_coder_matrix(const ss_rs_coder *c, uint8_t *out) {
    if (c == nullptr || out == nullptr) return set_error(SS_ERR_INVALID_ARG, "null argument");
    memcpy(out, c->matrix.data(), c->matrix.size());
    return SS_OK;
}
int ss_rs_set_variant(ss_rs_coder *c, int variant) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    c->variant = variant;
    return SS_OK;
}
const char *ss_rs_last_kernel(const ss_rs_coder *c) { return c ? c->last_kernel : "none"; }

// ---- one codeword, host slices --------------------------------------------------------------------
// Device layout used for single-codeword calls: shard j at scratch + j*ds, ds = round_up(L,16).
int ss_rs_encode(ss_rs_coder *c, uint8_t *const *shards, size_t n_shards, size_t shard_len) {
    SS_TRY(check_shard_args(c, shards, n_shards, shard_len));
    ss_ctx *ctx = c->ctx;
    SS_TRY(ctx_bind(ctx));
    const int d = c->d, p = c->p;
    const size_t L = shard_len, ds = (L + 15) & ~size_t(15);
    const size_t par_at = (size_t(d) * L + 255) & ~size_t(255);
    void *scr = nullptr;
    SS_TRY(ctx_scratch(ctx, par_at + size_t(p) * ds, &scr));
    uint8_t *d_data = static_cast<uint8_t *>(scr);
    uint8_t *d_par = d_data + par_at;
    const bool staged = size_t(d) * L + size_t(p) * ds <= kStagedCallLimit;
    uint8_t *pin = nullptr;
    if (staged) {
        SS_TRY(ctx_pinned(ctx, size_t(d) * L + size_t(p) * ds, &pin));
        for (int i = 0; i < d; ++i) memcpy(pin + size_t(i) * L, shards[i], L);
        SS_CUDA(cudaMemcpyAsync(d_data, pin, size_t(d) * L, cudaMemcpyHostToDevice, ctx->stream));
    } else {
        for (int i = 0; i < d; ++i)
            SS_CUDA(cudaMemcpyAsync(d_data + size_t(i) * L, shards[i], L, cudaMemcpyHostToDevice, ctx->stream));
    }
    EncGeom g{};
    g.data = d_data; g.data_off = nullptr; g.data_len = nullptr; g.data_stride = size_t(d) * L;
    g.uni_len = static_cast<uint32_t>(size_t(d) * L);
    g.parity = d_par; g.plane_stride = ds; g.par_off = nullptr; g.shard_stride = ds; g.n = 1;
    g.flags = SS_RS_OUT_PADDED16;
    SS_TRY(launch_rs_encode(c, g, nullptr));
    if (staged) {
        uint8_t *pout = pin + size_t(d) * L;
        SS_CUDA(cudaMemcpyAsync(pout, d_par, size_t(p) * ds, cudaMemcpyDeviceToHost, ctx->stream));
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        for (int j = 0; j < p; ++j) memcpy(shards[d + j], pout + size_t(j) * ds, L);
        return SS_OK;
    }
    for (int j = 0; j < p; ++j)
        SS_CUDA(cudaMemcpyAsync(shards[d + j], d_par + size_t(j) * ds, L, cudaMemcpyDeviceToHost, ctx->stream));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    return SS_OK;
}

static int reconstruct_one(ss_rs_coder *c, uint8_t *const *shards, uint8_t *present, size_t n_shards,
                           size_t shard_len, int data_only) {
    SS_TRY(check_shard_args(c, shards, n_shards, shard_len));
    if (present == nullptr) return set_error(SS_ERR_INVALID_ARG, "null present array");
    ss_ctx *ctx = c->ctx;
    SS_TRY(ctx_bind(ctx));
    const int d = c->d, p = c->p, t = d + p;
    int np = 0;
    for (int i = 0; i < t; ++i) np += present[i] ? 1 : 0;
    if (np == t) return SS_OK;                       // crate: nothing to do
    if (np < d) return set_error(SS_ERR_TOO_FEW_SHARDS_PRESENT, "too few shards present: %d < %d", np, d);
    const int upto = data_only ? d : t;
    int nmiss = 0;
    for (int i = 0; i < upto; ++i) nmiss += present[i] ? 0 : 1;
    if (nmiss == 0) return SS_OK;                    // reconstruct_data with every data shard present: nothing to regenerate
    if (!c->dec_ok)
        return set_error(SS_ERR_UNSUPPORTED, "reconstruct needs d+p <= 12 on this build (coder is %d,%d)", d, p);
    const size_t L = shard_len, ds = (L + 15) & ~size_t(15);
    const size_t meta = 256;
    void *scr = nullptr;
    SS_TRY(ctx_scratch(ctx, meta + size_t(t) * ds, &scr));
    uint8_t *d_meta = static_cast<uint8_t *>(scr);
    uint8_t *d_sh = d_meta + meta;
    uint32_t pat = 0;
    for (int i = 0; i < t; ++i)
        if (present[i]) pat |= 1u << i;
    struct Meta { uint64_t off; uint32_t len; uint32_t pat; int32_t status; } h = {0, static_cast<uint32_t>(size_t(d) * L), pat, 0};
    const bool staged = meta + size_t(t) * ds <= kStagedCallLimit;
    uint8_t *pin = nullptr;
    if (staged) {
        // one pinned image of the metadata block + all shard slots up, one image down
        SS_TRY(ctx_pinned(ctx, meta + size_t(t) * ds, &pin));
        memset(pin, 0, meta);
        memcpy(pin, &h, sizeof(h));
        for (int i = 0; i < t; ++i)
            if (present[i]) memcpy(pin + meta + size_t(i) * ds, shards[i], L);
        SS_CUDA(cudaMemcpyAsync(d_meta, pin, meta + size_t(t) * ds, cudaMemcpyHostToDevice, ctx->stream));
    } else {
        SS_CUDA(cudaMemcpyAsync(d_meta, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
        for (int i = 0; i < t; ++i)
            if (present[i])
                SS_CUDA(cudaMemcpyAsync(d_sh + size_t(i) * ds, shards[i], L, cudaMemcpyHostToDevice, ctx->stream));
    }
    SS_TRY(launch_rs_reconstruct(c, d_sh, ds, reinterpret_cast<const uint64_t *>(d_meta),
                                 reinterpret_cast<const uint32_t *>(d_meta + 8),
                                 reinterpret_cast<const uint32_t *>(d_meta + 12), 1, data_only,
                                 reinterpret_cast<int32_t *>(d_meta + 16), SS_RS_OUT_PADDED16));
    if (staged) {
        SS_CUDA(cudaMemcpyAsync(pin + meta, d_sh, size_t(t) * ds, cudaMemcpyDeviceToHost, ctx->stream));
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
        for (int i = 0; i < upto; ++i)
            if (!present[i]) memcpy(shards[i], pin + meta + size_t(i) * ds, L);
    } else {
        for (int i = 0; i < upto; ++i)
            if (!present[i])
                SS_CUDA(cudaMemcpyAsync(shards[i], d_sh + size_t(i) * ds, L, cudaMemcpyDeviceToHost, ctx->stream));
        SS_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    for (int i = 0; i < upto; ++i) present[i] = 1;
    return SS_OK;
}

int ss_rs_reconstruct(ss_rs_coder *c, uint8_t *const *shards, uint8_t *present, size_t n_shards, size_t shard_len) {
    return reconstruct_one(c, shards, present, n_shards, shard_len, 0);
}
int ss_rs_reconstruct_data(ss_rs_coder *c, uint8_t *const *shards, uint8_t *present, size_t n_shards,
                           size_t shard_len) {
    return reconstruct_one(c, shards, present, n_shards, shard_len, 1);
}

int ss_rs_verify(ss_rs_coder *c, const uint8_t *const *shards, size_t n_shards, size_t shard_len, int *ok) {
    SS_TRY(check_shard_args(c, shards, n_shards, shard_len));
    if (ok == nullptr) return set_error(SS_ERR_INVALID_ARG, "null ok pointer");
    const int d = c->d, p = c->p;
    // recomputed-parity staging lives in the coder (grow-only): no allocation per call
    if (c->verify_buf.size() < size_t(p) * shard_len) c->verify_buf.resize(size_t(p) * shard_len);
    c->verify_ptrs.resize(size_t(d + p));
    for (int i = 0; i < d; ++i) c->verify_ptrs[i] = const_cast<uint8_t *>(shards[i]);
    for (int j = 0; j < p; ++j) c->verify_ptrs[d + j] = c->verify_buf.data() + size_t(j) * shard_len;
    SS_TRY(ss_rs_encode(c, c->verify_ptrs.data(), n_shards, shard_len));    // parity recomputed on the GPU
    *ok = 1;
    for (int j = 0; j < p; ++j)
        if (memcmp(c->verify_ptrs[d + j], shards[d + j], shard_len) != 0) { *ok = 0; break; }
    return SS_OK;
}

// ---- batched, device-resident ---------------------------------------------------------------------
int ss_rs_encode_batch_dev(ss_rs_coder *c, const uint8_t *data, const uint64_t *data_off, const uint32_t *data_len,
                           uint64_t n, uint8_t *parity, uint64_t plane_stride, const uint64_t *par_off, uint32_t flags) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n == 0) return SS_OK;
    if (!data || !data_off || !data_len || !parity || !par_off) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    EncGeom g{};
    g.data = data; g.data_off = data_off; g.data_len = data_len; g.parity = parity; g.plane_stride = plane_stride;
    g.par_off = par_off; g.n = n; g.flags = flags;
    return launch_rs_encode(c, g, nullptr);
}

int ss_rs_encode_uniform_dev(ss_rs_coder *c, const uint8_t *data, uint64_t data_stride, uint32_t data_len, uint64_t n,
                             uint8_t *parity, uint64_t plane_stride, uint64_t shard_stride, uint32_t flags) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n == 0 || data_len == 0) return SS_OK;
    if (!data || !parity) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    EncGeom g{};
    g.data = data; g.data_off = nullptr; g.data_stride = data_stride; g.uni_len = data_len; g.parity = parity;
    g.plane_stride = plane_stride; g.shard_stride = shard_stride; g.n = n; g.flags = flags;
    return launch_rs_encode(c, g, nullptr);
}

int ss_rs_reconstruct_batch_dev(ss_rs_coder *c, uint8_t *shards, uint64_t plane_stride, const uint64_t *off,
                                const uint32_t *data_len, const uint32_t *present, uint64_t n, int data_only,
                                int32_t *status, uint32_t flags) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n == 0) return SS_OK;
    if (!shards || !off || !data_len || !present || !status) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_rs_reconstruct(c, shards, plane_stride, off, data_len, present, n, data_only, status, flags);
}

int ss_rs_reconstruct_uniform_dev(ss_rs_coder *c, uint8_t *shards, uint64_t plane_stride, uint64_t shard_stride,
                                  uint32_t data_len, const uint32_t *present, uint64_t n, int data_only, int32_t *status) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n == 0) return SS_OK;
    if (!shards || !present || !status) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (!c->batch_ok || !c->dec_ok)
        return set_error(SS_ERR_UNSUPPORTED, "batched reconstruct needs d+p <= 12 (coder is %d,%d)", c->d, c->p);
    return launch_rs_reconstruct_uniform(c, shards, plane_stride, shard_stride, data_len, present, n, data_only, status);
}

int ss_accept_step_fused_dev(ss_rs_coder *c, const uint8_t *data, uint64_t data_stride, uint32_t data_len,
                             uint64_t n_groups, uint8_t *parity, uint64_t plane_stride, uint64_t shard_stride,
                             uint32_t flags, const uint64_t *planes, uint32_t n_replicas, uint32_t threshold,
                             uint64_t *committed, uint32_t *commit_bar) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n_groups == 0) return SS_OK;
    if (!data || !parity || !planes || !committed) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (n_replicas == 0 || n_replicas > 16) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..16");
    EncGeom g{};
    g.data = data; g.data_off = nullptr; g.data_stride = data_stride; g.uni_len = data_len; g.parity = parity;
    g.plane_stride = plane_stride; g.shard_stride = shard_stride; g.n = n_groups; g.flags = flags;
    TallyArgs t;
    t.planes = planes; t.R = n_replicas; t.threshold = threshold; t.G = n_groups; t.committed = committed;
    t.commit_bar = commit_bar;
    return launch_rs_encode(c, g, &t);
}

int ss_accept_step_replicate_dev(ss_rs_coder *c, const uint8_t *data, uint64_t data_stride, uint32_t data_len,
                                 uint64_t n_groups, uint8_t *const *shard_planes, uint64_t shard_stride,
                                 const uint64_t *planes, uint32_t n_replicas, uint32_t threshold,
                                 uint64_t *committed, uint32_t *commit_bar, const ss_step_sync *sync) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n_groups == 0) return SS_OK;
    if (!data || !shard_planes) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    const int d = c->d, nsh = c->d + c->p;
    if (d > 8 || nsh > 16) return set_error(SS_ERR_UNSUPPORTED, "replicate step needs d <= 8 data shards (coder is %d,%d)", c->d, c->p);
    const uint64_t L = (uint64_t(data_len) + d - 1) / d, vpc = (L + 15) / 16;
    if (data_len == 0 || ((reinterpret_cast<uintptr_t>(data) | data_stride | shard_stride) & 15u) || shard_stride < vpc * 16)
        return set_error(SS_ERR_UNSUPPORTED, "replicate step needs 16-byte aligned uniform payloads and padded shard slots");
    for (int j = 0; j < nsh; ++j)
        if (shard_planes[j] == nullptr || (reinterpret_cast<uintptr_t>(shard_planes[j]) & 15u))
            return set_error(SS_ERR_INVALID_ARG, "shard plane %d is null or not 16-byte aligned", j);
    EncGeom g{};
    g.data = data; g.data_off = nullptr; g.data_stride = data_stride; g.uni_len = data_len;
    g.parity = shard_planes[d]; g.plane_stride = 16; g.shard_stride = shard_stride; g.n = n_groups;
    g.flags = SS_RS_OUT_PADDED16 | SS_RS_EMIT_DATA;
    g.plane_ptrs = shard_planes;
    SS_TRY(make_flag_wait(c->ctx, sync, &g.wait));
    TallyArgs t;
    const bool with_tally = planes != nullptr;
    if (with_tally) {
        if (!committed) return set_error(SS_ERR_INVALID_ARG, "null committed buffer");
        if (n_replicas == 0 || n_replicas > 16) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..16");
        t.planes = planes; t.R = n_replicas; t.threshold = threshold; t.G = n_groups; t.committed = committed;
        t.commit_bar = commit_bar;
    }
    const int saved = c->variant;
    if ((c->variant & 15) == 1 || (c->variant & 15) == 5) c->variant &= ~15;     // the flat / bit-plane kernels have no peer-plane mode
    const int rc = launch_rs_encode(c, g, with_tally ? &t : nullptr);
    c->variant = saved;
    if (rc != SS_OK) return rc;
    return launch_flag_signal(c->ctx, sync);
}

int ss_follower_ack_dev(ss_ctx *ctx, const uint64_t *ack_src, uint64_t *const *ack_dst, uint32_t R, uint64_t G,
                        const ss_step_sync *sync) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (!ack_src || !ack_dst) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (R == 0 || R > 16) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..16");
    dev::FlagWait w;
    SS_TRY(make_flag_wait(ctx, sync, &w));
    SS_TRY(launch_follower_ack(ctx, ack_src, ack_dst, R, G, w));
    return launch_flag_signal(ctx, sync);
}

int ss_flags_signal_dev(ss_ctx *ctx, const ss_step_sync *sync) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    dev::FlagWait w;
    SS_TRY(make_flag_wait(ctx, sync, &w));        // validates both halves
    return launch_flag_signal(ctx, sync);
}

int ss_flags_wait_dev(ss_ctx *ctx, const ss_step_sync *sync) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    dev::FlagWait w;
    SS_TRY(make_flag_wait(ctx, sync, &w));
    return launch_flag_wait(ctx, w);
}

int ss_event_create(ss_ctx *ctx, void **event) {
    SS_TRY(ctx_bind(ctx));
    if (event == nullptr) return set_error(SS_ERR_INVALID_ARG, "null out pointer");
    cudaEvent_t ev;
    SS_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    *event = ev;
    return SS_OK;
}
int ss_event_destroy(ss_ctx *ctx, void *event) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaEventDestroy(static_cast<cudaEvent_t>(event)));
    return SS_OK;
}
int ss_event_record(ss_ctx *ctx, void *event) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(event), ctx->stream));
    return SS_OK;
}
int ss_event_wait(ss_ctx *ctx, void *event) {
    SS_TRY(ctx_bind(ctx));
    SS_CUDA(cudaStreamWaitEvent(ctx->stream, static_cast<cudaEvent_t>(event), 0));
    return SS_OK;
}

int ss_ctx_device_status(ss_ctx *ctx, uint32_t *status) {
    SS_TRY(ctx_bind(ctx));
    if (status == nullptr) return set_error(SS_ERR_INVALID_ARG, "null status pointer");
    SS_CUDA(cudaMemcpyAsync(status, ctx->dev_status, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    SS_CUDA(cudaMemsetAsync(ctx->dev_status, 0, sizeof(uint32_t), ctx->stream));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    return SS_OK;
}

// ---- host-buffer batch encode (+ optional fused tally): chunked, copy/compute overlapped -----------------
// Per chunk of C codewords: H2D of the payloads (and of the chunk's R ack-plane slices) on the copy-in stream, ONE
// fused kernel on the context's stream, D2H of the parity slices (and commit words / commit_bar) on the copy-out
// stream; three staging buffers deep, so chunk k+1 uploads and chunk k-1 downloads while chunk k computes.
static int encode_uniform_host(ss_rs_coder *c, const uint8_t *data, uint64_t data_stride, uint32_t data_len, uint64_t n,
                               uint8_t *parity, uint64_t plane_stride, uint64_t shard_stride, const uint64_t *planes,
                               uint32_t R, uint32_t threshold, uint64_t *committed, uint32_t *commit_bar) {
    ss_ctx *ctx = c->ctx;
    SS_TRY(ctx_bind(ctx));
    const int d = c->d, p = c->p;
    const bool tally = planes != nullptr;
    const uint64_t L = (uint64_t(data_len) + d - 1) / d, ds = (L + 15) & ~uint64_t(15);
    if (data_stride < data_len || shard_stride < L) return set_error(SS_ERR_INVALID_ARG, "stride shorter than element");
    // chunk: 16 MiB of payload by default; SS_E2E_CHUNK_MB overrides, for tuning
    uint64_t chunk_mb = 16;
    if (const char *e = getenv("SS_E2E_CHUNK_MB")) { const long v = atol(e); if (v >= 1 && v <= 4096) chunk_mb = static_cast<uint64_t>(v); }
    uint64_t C = (chunk_mb << 20) / data_stride;
    if (C < 2) C = 2;
    C &= ~uint64_t(1);                      // even: the chunk's ack-plane slices stay 16-byte aligned
    if (C > n) C = n;
    const uint64_t in_stride_dev = (data_stride + 15) & ~uint64_t(15);
    const bool in_contig = (in_stride_dev == data_stride);
    const uint64_t in_pay = (C * in_stride_dev + 256 + 255) & ~uint64_t(255);
    const uint64_t out_par = (uint64_t(p) * C * ds + 255) & ~uint64_t(255);
    const uint64_t out_cm = (C * 8 + 255) & ~uint64_t(255);
    SS_TRY(pipeline_staging(ctx, in_pay + (tally ? uint64_t(R) * C * 8 : 0), out_par + (tally ? out_cm + C * 4 : 0)));
    const uint64_t nchunks = (n + C - 1) / C;
    for (uint64_t k = 0; k < nchunks; ++k) {
        const int b = static_cast<int>(k % ss_ctx::kStages);
        const uint64_t g0 = k * C, nc = (n - g0) < C ? (n - g0) : C;
        uint8_t *din = static_cast<uint8_t *>(ctx->stage_in[b]);
        uint8_t *dout = static_cast<uint8_t *>(ctx->stage_out[b]);
        uint64_t *dpl = reinterpret_cast<uint64_t *>(din + in_pay);
        uint64_t *dcm = reinterpret_cast<uint64_t *>(dout + out_par);
        uint32_t *dbar = reinterpret_cast<uint32_t *>(dout + out_par + out_cm);
        if (k >= ss_ctx::kStages) SS_CUDA(cudaStreamWaitEvent(ctx->h2d_stream, ctx->ev_done[b], 0));
        if (in_contig)      // up to the last payload's end, not its row's: the caller's buffer may stop there
            SS_CUDA(cudaMemcpyAsync(din, data + g0 * data_stride, (nc - 1) * data_stride + data_len, cudaMemcpyHostToDevice,
                                    ctx->h2d_stream));
        else
            SS_CUDA(cudaMemcpy2DAsync(din, in_stride_dev, data + g0 * data_stride, data_stride, data_len, nc,
                                      cudaMemcpyHostToDevice, ctx->h2d_stream));
        if (tally)      // R slices of nc words, packed as planes[r*nc + g] on the device
            SS_CUDA(cudaMemcpy2DAsync(dpl, nc * 8, planes + g0, n * 8, nc * 8, R, cudaMemcpyHostToDevice, ctx->h2d_stream));
        SS_CUDA(cudaEventRecord(ctx->ev_h2d[b], ctx->h2d_stream));
        SS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[b], 0));
        EncGeom g{};
        g.data = din; g.data_off = nullptr; g.data_stride = in_stride_dev; g.uni_len = data_len; g.parity = dout;
        g.plane_stride = C * ds; g.shard_stride = ds; g.n = nc; g.flags = SS_RS_OUT_PADDED16;
        TallyArgs t;
        if (tally) { t.planes = dpl; t.R = R; t.threshold = threshold; t.G = nc; t.committed = dcm; t.commit_bar = commit_bar ? dbar : nullptr; }
        SS_TRY(launch_rs_encode(c, g, tally ? &t : nullptr));
        SS_CUDA(cudaEventRecord(ctx->ev_kernel[b], ctx->stream));
        SS_CUDA(cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_kernel[b], 0));
        for (int j = 0; j < p; ++j) {
            uint8_t *hdst = parity + uint64_t(j) * plane_stride + g0 * shard_stride;
            const uint8_t *dsrc = dout + uint64_t(j) * C * ds;
            if (shard_stride == ds)
                SS_CUDA(cudaMemcpyAsync(hdst, dsrc, nc * ds, cudaMemcpyDeviceToHost, ctx->d2h_stream));
            else
                SS_CUDA(cudaMemcpy2DAsync(hdst, shard_stride, dsrc, ds, L, nc, cudaMemcpyDeviceToHost, ctx->d2h_stream));
        }
        if (tally) {
            SS_CUDA(cudaMemcpyAsync(committed + g0, dcm, nc * 8, cudaMemcpyDeviceToHost, ctx->d2h_stream));
            if (commit_bar) SS_CUDA(cudaMemcpyAsync(commit_bar + g0, dbar, nc * 4, cudaMemcpyDeviceToHost, ctx->d2h_stream));
        }
        SS_CUDA(cudaEventRecord(ctx->ev_done[b], ctx->d2h_stream));
    }
    SS_CUDA(cudaStreamSynchronize(ctx->d2h_stream));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    return SS_OK;
}

int ss_rs_encode_uniform(ss_rs_coder *c, const uint8_t *data, uint64_t data_stride, uint32_t data_len, uint64_t n,
                         uint8_t *parity, uint64_t plane_stride, uint64_t shard_stride) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n == 0 || data_len == 0) return SS_OK;
    if (!data || !parity) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return encode_uniform_host(c, data, data_stride, data_len, n, parity, plane_stride, shard_stride, nullptr, 0, 0, nullptr,
                               nullptr);
}

int ss_accept_step_fused(ss_rs_coder *c, const uint8_t *data, uint64_t data_stride, uint32_t data_len, uint64_t n_groups,
                         uint8_t *parity, uint64_t plane_stride, uint64_t shard_stride, const uint64_t *planes,
                         uint32_t n_replicas, uint32_t threshold, uint64_t *committed, uint32_t *commit_bar) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n_groups == 0) return SS_OK;
    if (!data || !parity || !planes || !committed) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    if (data_len == 0) return set_error(SS_ERR_INVALID_ARG, "null codewords cannot be encoded");
    if (n_replicas == 0 || n_replicas > 16) return set_error(SS_ERR_INVALID_ARG, "n_replicas must be 1..16");
    return encode_uniform_host(c, data, data_stride, data_len, n_groups, parity, plane_stride, shard_stride, planes, n_replicas,
                               threshold, committed, commit_bar);
}

// ---- tallies ----------------------------------------------------------------------------------------
int ss_tally_planes_dev(ss_ctx *ctx, const uint64_t *planes, uint32_t R, uint64_t G, uint32_t thr, uint64_t *committed,
                        uint32_t *commit_bar) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (G == 0) return SS_OK;
    if (!planes || !committed) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_tally_planes(ctx, planes, R, G, thr, committed, commit_bar);
}

int ss_tally_planes(ss_ctx *ctx, const uint64_t *planes, uint32_t R, uint64_t G, uint32_t thr, uint64_t *committed,
                    uint32_t *commit_bar) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (G == 0) return SS_OK;
    if (!planes || !committed) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    SS_TRY(ctx_bind(ctx));
    const size_t in_b = size_t(R) * G * 8, out_b = G * 8, bar_b = commit_bar ? G * 4 : 0;
    void *scr = nullptr;
    SS_TRY(ctx_scratch(ctx, in_b + out_b + bar_b, &scr));
    uint64_t *d_pl = static_cast<uint64_t *>(scr);
    uint64_t *d_cm = d_pl + size_t(R) * G;
    uint32_t *d_bar = commit_bar ? reinterpret_cast<uint32_t *>(d_cm + G) : nullptr;
    SS_CUDA(cudaMemcpyAsync(d_pl, planes, in_b, cudaMemcpyHostToDevice, ctx->stream));
    SS_TRY(launch_tally_planes(ctx, d_pl, R, G, thr, d_cm, d_bar));
    SS_CUDA(cudaMemcpyAsync(committed, d_cm, out_b, cudaMemcpyDeviceToHost, ctx->stream));
    if (commit_bar) SS_CUDA(cudaMemcpyAsync(commit_bar, d_bar, bar_b, cudaMemcpyDeviceToHost, ctx->stream));
    SS_CUDA(cudaStreamSynchronize(ctx->stream));
    return SS_OK;
}

int ss_tally_masks_dev(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, uint64_t n, uint32_t thr,
                       uint64_t *commit_bits) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (n == 0) return SS_OK;
    if (!masks || !commit_bits) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_tally_masks(ctx, masks, mask_bytes, n, thr, commit_bits);
}

int ss_ack_ingest_dev(ss_ctx *ctx, const uint32_t *rec_group, const uint8_t *rec_slot, const uint8_t *rec_peer,
                      const uint64_t *rec_ballot, uint64_t n_records, const uint64_t *bal_prepared,
                      const uint64_t *inst_bal, const uint64_t *accepting, uint32_t R, uint64_t G, uint64_t *planes) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (n_records == 0) return SS_OK;
    if (!rec_group || !rec_slot || !rec_peer || !rec_ballot || !bal_prepared || !inst_bal || !accepting || !planes)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_ack_ingest(ctx, rec_group, rec_slot, rec_peer, rec_ballot, n_records, bal_prepared, inst_bal,
                             accepting, nullptr, R, G, planes);
}

int ss_tally_crossword_dev(ss_ctx *ctx, const void *masks, uint32_t mask_bytes, const uint8_t *policy_idx, uint64_t n,
                           const uint32_t *policies_host, uint32_t n_policies, uint32_t n_replicas, uint32_t T,
                           uint32_t d, uint32_t majority, uint32_t f, int balanced, uint64_t *commit_bits) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (n == 0) return SS_OK;
    if (!masks || !policy_idx || !policies_host || !commit_bits) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_tally_crossword(ctx, masks, mask_bytes, policy_idx, n, policies_host, n_policies, n_replicas, T, d,
                                  majority, f, balanced, commit_bits);
}

int ss_raft_commit_scan_dev(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G,
                            const uint32_t *last_commit, const uint32_t *log_end, const uint32_t *curr_term,
                            const uint32_t *terms, uint32_t window, uint32_t threshold, uint32_t *new_commit,
                            uint32_t *window_overflow) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (G == 0) return SS_OK;
    if ((!match && n_peers) || !last_commit || !log_end || !curr_term || !terms || !new_commit)
        return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_raft_scan(ctx, match, n_peers, G, last_commit, log_end, curr_term, terms, window, threshold,
                            new_commit, window_overflow);
}

int ss_crossword_distribute_dev(ss_rs_coder *c, const uint8_t *data, const uint64_t *data_off, const uint32_t *data_len,
                                const uint8_t *spr, const uint64_t *rep_off, uint64_t n, uint8_t *const *replica_logs,
                                uint32_t n_replicas) {
    if (c == nullptr) return set_error(SS_ERR_INVALID_ARG, "null coder");
    if (n == 0) return SS_OK;
    if (!data || !data_off || !data_len || !spr || !rep_off || !replica_logs) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_crossword_distribute(c, data, data_off, data_len, spr, rep_off, n, replica_logs, n_replicas);
}

int ss_frame_accept_batch_dev(ss_ctx *ctx, const uint8_t *shard_plane, uint64_t shard_stride, uint32_t shard_idx, uint32_t d,
                              uint32_t p, uint32_t data_len, uint32_t msg_variant, const uint64_t *slot,
                              const uint64_t *ballot, uint64_t n, uint8_t *out, uint64_t frame_stride, uint64_t *frame_off,
                              uint32_t *frame_len) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (n == 0) return SS_OK;
    if (!shard_plane || !slot || !ballot || !out || !frame_off || !frame_len) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_frame_accept(ctx, shard_plane, shard_stride, shard_idx, d, p, data_len, msg_variant, slot, ballot, n, out,
                               frame_stride, frame_off, frame_len);
}

int ss_gossip_plan_dev(ss_ctx *ctx, uint32_t me, uint32_t population, uint32_t d, const uint8_t *src_peer, const uint32_t *avail,
                       const uint8_t *policy_idx, const uint32_t *policies_host, uint32_t n_policies, uint32_t peer_alive,
                       uint64_t N, uint32_t *targets, uint32_t *excl) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (N == 0) return SS_OK;
    if (!src_peer || !avail || !policy_idx || !policies_host || !targets || !excl) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_gossip_plan(ctx, me, population, d, src_peer, avail, policy_idx, policies_host, n_policies, peer_alive, N,
                              targets, excl);
}

int ss_raft_kth_match_dev(ss_ctx *ctx, const uint32_t *match, uint32_t n_peers, uint64_t G, uint32_t k, uint32_t *out) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (G == 0) return SS_OK;
    if (!match || !out) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_kth_match(ctx, match, n_peers, G, k, out);
}

int ss_prepare_merge_dev(ss_ctx *ctx, const uint64_t *vote_bal, const uint32_t *vote_mask, uint32_t R, uint64_t N,
                         const uint8_t *acks_cnt, uint32_t d, uint32_t population, uint32_t f, uint64_t *max_bal,
                         uint32_t *merged, uint8_t *action) {
    if (ctx == nullptr) return set_error(SS_ERR_INVALID_ARG, "null context");
    if (N == 0) return SS_OK;
    if (!vote_bal || !vote_mask || !acks_cnt || !max_bal || !merged || !action) return set_error(SS_ERR_INVALID_ARG, "null buffer");
    return launch_prepare_merge(ctx, vote_bal, vote_mask, R, N, acks_cnt, d, population, f, max_bal, merged, action);
}

}  // extern "C"
