// jit.cu -- run-time specialisation of the row / packed encode kernels for codes that have no compile-time table.
//
// The protocols' own codes (ReedSolomon::new(majority, population - majority), populations 3..9) are compile-time
// tables (static_codes.hpp).  Any other (d <= 8, p <= 8) matrix -- Crossword with rs_total_shards > population,
// crossword/mod.rs:805-830 -- used to run the same kernels with coefficient MASKS fetched per bit level, at about half
// the speed (DESIGN.md section 3).  Here the coder's parity rows are handed to NVRTC as preprocessor constants and
// horner_row_kernels.cuh is compiled for exactly that matrix, once per coder (lazily, ~1 s): every code then runs the
// fully unrolled kernels with its coefficients as immediates.  NVRTC is NVIDIA's run-time CUDA compiler (libnvrtc, part
// of the toolkit): the kernels remain the hand-written ones of this repository; nothing is traced or generated.
//
// libnvrtc is opened with dlopen on first use, so the library has no load-time dependency on it; if it is missing or
// the compilation fails the coder keeps the run-time-mask kernels (still GPU kernels) and says so in
// ss_rs_jit_status().  The CUBIN is loaded and launched through the CUDA runtime's library API
// (cudaLibraryLoadData / cudaLibraryGetKernel / cudaLaunchKernel): no driver-API linkage.
#include <dlfcn.h>
#include <nvrtc.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "gf256.hpp"
#include "ss_internal.hpp"
#include "static_codes.hpp"

namespace ssb {

static const char *kJitSource =
#include "jit_source.inc"
    ;

struct NvrtcApi {
    void *handle = nullptr;
    nvrtcResult (*CreateProgram)(nvrtcProgram *, const char *, const char *, int, const char *const *, const char *const *) = nullptr;
    nvrtcResult (*DestroyProgram)(nvrtcProgram *) = nullptr;
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char *const *) = nullptr;
    nvrtcResult (*AddNameExpression)(nvrtcProgram, const char *) = nullptr;
    nvrtcResult (*GetLoweredName)(nvrtcProgram, const char *, const char **) = nullptr;
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t *) = nullptr;
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char *) = nullptr;
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t *) = nullptr;
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char *) = nullptr;
    const char *(*GetErrorString)(nvrtcResult) = nullptr;
    bool ok = false;
};

static NvrtcApi &nvrtc_api() {
    static NvrtcApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"};
        for (const char *n : names) {
            api.handle = dlopen(n, RTLD_NOW | RTLD_LOCAL);
            if (api.handle) break;
        }
        if (!api.handle) return;
#define SS_NVRTC_SYM(field, sym) *reinterpret_cast<void **>(&api.field) = dlsym(api.handle, sym)
        SS_NVRTC_SYM(CreateProgram, "nvrtcCreateProgram");
        SS_NVRTC_SYM(DestroyProgram, "nvrtcDestroyProgram");
        SS_NVRTC_SYM(CompileProgram, "nvrtcCompileProgram");
        SS_NVRTC_SYM(AddNameExpression, "nvrtcAddNameExpression");
        SS_NVRTC_SYM(GetLoweredName, "nvrtcGetLoweredName");
        SS_NVRTC_SYM(GetCUBINSize, "nvrtcGetCUBINSize");
        SS_NVRTC_SYM(GetCUBIN, "nvrtcGetCUBIN");
        SS_NVRTC_SYM(GetProgramLogSize, "nvrtcGetProgramLogSize");
        SS_NVRTC_SYM(GetProgramLog, "nvrtcGetProgramLog");
        SS_NVRTC_SYM(GetErrorString, "nvrtcGetErrorString");
#undef SS_NVRTC_SYM
        api.ok = api.CreateProgram && api.DestroyProgram && api.CompileProgram && api.AddNameExpression && api.GetLoweredName &&
                 api.GetCUBINSize && api.GetCUBIN && api.GetProgramLogSize && api.GetProgramLog && api.GetErrorString;
    });
    return api;
}

// resident 256-thread CTAs of the row kernel by code width (the launcher's default register budgets)
static int row_min_blocks(int d) { return d <= 4 ? 12 : d == 5 ? 10 : d == 6 ? 8 : 6; }

// Compiles ONE instance of horner_row_kernels.cuh for the given parity rows (p x d, row-major).  No GPU is needed.
// which: 0 row<128 threads>, 1 row<256>, 2 packed<aligned, pipelined>, 3 packed<unaligned, pipelined>, 4 packed<unaligned>.
int jit_compile(int d, int p, const uint8_t *rows, int which, std::vector<char> &cubin, std::string &name, std::string &log) {
    NvrtcApi &rt = nvrtc_api();
    if (!rt.ok) { log = "libnvrtc could not be loaded"; return SS_ERR_UNSUPPORTED; }
    if (d < 1 || d > 8 || p < 1 || p > 8 || which < 0 || which > 4) { log = "run-time specialisation covers d <= 8, p <= 8"; return SS_ERR_UNSUPPORTED; }
    std::string coefs;
    char tmp[16];
    for (int i = 0; i < d * p; ++i) {
        snprintf(tmp, sizeof tmp, "%s0x%02xu", i ? "," : "", rows[i]);
        coefs += tmp;
    }
    const std::string def_d = "-DSS_JIT_D=" + std::to_string(d), def_p = "-DSS_JIT_P=" + std::to_string(p), def_c = "-DSS_JIT_COEFS=" + coefs;
    const char *opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", def_d.c_str(), def_p.c_str(), def_c.c_str()};
    nvrtcProgram prog = nullptr;
    nvrtcResult r = rt.CreateProgram(&prog, kJitSource, "summerset_b200_jit.cu", 0, nullptr, nullptr);
    if (r != NVRTC_SUCCESS) { log = std::string("nvrtcCreateProgram: ") + rt.GetErrorString(r); return SS_ERR_UNSUPPORTED; }
    const std::string D = std::to_string(d);
    const std::string exprs[5] = {
        "&ssb::horner_encode_row_kernel<" + D + ", ssb::kCodeJit, 128, " + std::to_string(row_min_blocks(d)) + ">",
        "&ssb::horner_encode_row_kernel<" + D + ", ssb::kCodeJit, 256, 3>",
        "&ssb::horner_encode_packed_kernel<" + D + ", ssb::kCodeJit, true, true>",
        "&ssb::horner_encode_packed_kernel<" + D + ", ssb::kCodeJit, false, true>",
        "&ssb::horner_encode_packed_kernel<" + D + ", ssb::kCodeJit, false, false>"};
    rt.AddNameExpression(prog, exprs[which].c_str());
    r = rt.CompileProgram(prog, 5, opts);
    size_t ls = 0;
    rt.GetProgramLogSize(prog, &ls);
    if (ls > 1) { log.resize(ls); rt.GetProgramLog(prog, &log[0]); }
    if (r != NVRTC_SUCCESS) {
        log = std::string("nvrtcCompileProgram: ") + rt.GetErrorString(r) + "\n" + log;
        rt.DestroyProgram(&prog);
        return SS_ERR_UNSUPPORTED;
    }
    const char *low = nullptr;
    if (rt.GetLoweredName(prog, exprs[which].c_str(), &low) != NVRTC_SUCCESS || low == nullptr) {
        log = "nvrtcGetLoweredName failed for " + exprs[which];
        rt.DestroyProgram(&prog);
        return SS_ERR_UNSUPPORTED;
    }
    name = low;
    size_t cs = 0;
    rt.GetCUBINSize(prog, &cs);
    cubin.resize(cs);
    r = rt.GetCUBIN(prog, cubin.data());
    rt.DestroyProgram(&prog);
    if (r != NVRTC_SUCCESS || cs == 0) { log = "nvrtcGetCUBIN failed"; return SS_ERR_UNSUPPORTED; }
    return SS_OK;
}

// lazily compiles + loads ONE specialised kernel of the coder (the geometry in use decides which); SS_OK when ready
int jit_ensure(ss_rs_coder *c, int which) {
    if (c->jit_state[which] > 0) return SS_OK;
    if (c->jit_state[which] < 0) return SS_ERR_UNSUPPORTED;
    c->jit_state[which] = -1;
    std::vector<char> cubin;
    std::string name, log;
    const uint8_t *rows = c->matrix.data() + size_t(c->d) * c->d;
    if (jit_compile(c->d, c->p, rows, which, cubin, name, log) != SS_OK) { c->jit_message = log; return SS_ERR_UNSUPPORTED; }
    cudaLibrary_t lib = nullptr;
    cudaError_t e = cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
    if (e != cudaSuccess) {
        cudaGetLastError();
        c->jit_message = std::string("cudaLibraryLoadData: ") + cudaGetErrorString(e);
        return SS_ERR_UNSUPPORTED;
    }
    cudaKernel_t k = nullptr;
    e = cudaLibraryGetKernel(&k, lib, name.c_str());
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaLibraryUnload(lib);
        c->jit_message = std::string("cudaLibraryGetKernel(") + name + "): " + cudaGetErrorString(e);
        return SS_ERR_UNSUPPORTED;
    }
    c->jit_kernel[which] = k;
    c->jit_library[which] = lib;
    c->jit_state[which] = 1;
    c->jit_message = "specialised by NVRTC (" + name + ", " + std::to_string(cubin.size()) + " bytes of sm_90a code)";
    return SS_OK;
}

void jit_release(ss_rs_coder *c) {
    for (int i = 0; i < 5; ++i) {
        if (c->jit_library[i]) cudaLibraryUnload(static_cast<cudaLibrary_t>(c->jit_library[i]));
        c->jit_library[i] = nullptr;
        c->jit_state[i] = 0;
    }
}

}  // namespace ssb

extern "C" {

// Compiles the specialised kernels for RS(d, p) exactly as a coder would, without touching a GPU: returns the CUBIN size
// (> 0) or a negative error code with the compiler log in `log`.  Used by the CPU test-suite and by INTEGRATION checks.
long ss_jit_selftest(int d, int p, char *log, size_t log_cap) {
    if (log && log_cap) log[0] = 0;
    ssb::gf::Matrix M;
    try {
        M = ssb::gf::coding_matrix(d, p);
    } catch (const std::exception &ex) {
        if (log && log_cap) snprintf(log, log_cap, "%s", ex.what());
        return SS_ERR_INVALID_ARG;
    }
    long total = 0;
    for (int which = 0; which < 5; ++which) {          // every instance a coder may ask for
        std::vector<char> cubin;
        std::string name, msg;
        const int rc = ssb::jit_compile(d, p, M.v.data() + size_t(d) * d, which, cubin, name, msg);
        if (rc != SS_OK) {
            if (log && log_cap) snprintf(log, log_cap, "%s", msg.c_str());
            return rc;
        }
        total += static_cast<long>(cubin.size());
    }
    return total;
}

const char *ss_rs_jit_status(const ss_rs_coder *c) {
    if (c == nullptr) return "null coder";
    if (c->static_code >= 0 || c->is_rs32) return "compile-time code table (no run-time specialisation needed)";
    if (c->jit_message.empty()) return "not specialised yet (happens on the first batched encode)";
    return c->jit_message.c_str();
}

}  // extern "C"
