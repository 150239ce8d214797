// jit.cu — run-time specialisation of kernels with NVRTC for sm_90a.
//
// Trino compiles every filter/projection/accumulator into JVM bytecode at plan time
// (M/sql/gen/ExpressionCompiler.java:50-85, M/operator/aggregation/AccumulatorCompiler.java).  The GPU analogue is
// to specialise the hand-written kernel bodies of device_lib.cuh for the concrete row program: the generated
// translation unit is device_lib.cuh (embedded verbatim) + a small struct of straight-line typed code, compiled
// once per distinct program (cached) to a cubin and launched through the driver API on the ctx stream.
// libnvrtc / libcuda are resolved with dlopen so libtrino_gpu.so carries no link-time dependency on them; when
// NVRTC is not present the callers keep using the ahead-of-time interpreter kernels.
#include <dlfcn.h>

#include <mutex>
#include <unordered_map>

#include "jit.cuh"

namespace {

const char* kPrelude =
#include "device_lib_str.inc"
    ;

typedef struct _nvrtcProgram* nvrtcProgram;
typedef struct CUmod_st* CUmodule;
typedef struct CUfunc_st* CUfunction;

struct Api {
    bool tried = false, ok = false, rtc_ok = false;
    std::string why;
    int (*nvrtcCreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    int (*nvrtcCompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
    int (*nvrtcGetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
    int (*nvrtcGetProgramLog)(nvrtcProgram, char*) = nullptr;
    int (*nvrtcGetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
    int (*nvrtcGetCUBIN)(nvrtcProgram, char*) = nullptr;
    int (*nvrtcDestroyProgram)(nvrtcProgram*) = nullptr;
    int (*cuModuleLoadData)(CUmodule*, const void*) = nullptr;
    int (*cuModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
    int (*cuLaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, cudaStream_t, void**, void**) = nullptr;
    int (*cuOccupancyMaxActiveBlocksPerMultiprocessor)(int*, CUfunction, int, size_t) = nullptr;
    int (*cuFuncSetAttribute)(CUfunction, int, int) = nullptr;
    int (*cuGetErrorString)(int, const char**) = nullptr;
};

Api g_api;
std::mutex g_mu;
std::unordered_map<std::string, CUfunction> g_cache;   // key: device + kernel name + source

void* open_first(const char* const* names)
{
    for (int i = 0; names[i]; i++) {
        void* h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
        if (h) return h;
    }
    return nullptr;
}

void load_api()
{
    if (g_api.tried) return;
    g_api.tried = true;
    if (getenv("TGPU_DISABLE_JIT")) { g_api.why = "disabled by TGPU_DISABLE_JIT"; return; }
    const char* rtc_names[] = {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so", nullptr};
    const char* cu_names[] = {"libcuda.so.1", "libcuda.so", nullptr};
    void* rtc = open_first(rtc_names);
    void* cu = open_first(cu_names);
    if (!rtc) { g_api.why = "libnvrtc.so.12 not found"; return; }
#define LOAD(h, name)                                                     \
    *(void**)(&g_api.name) = dlsym(h, #name);                              \
    if (!g_api.name) { g_api.why = std::string("missing symbol ") + #name; return; }
    LOAD(rtc, nvrtcCreateProgram) LOAD(rtc, nvrtcCompileProgram) LOAD(rtc, nvrtcGetProgramLogSize) LOAD(rtc, nvrtcGetProgramLog)
    LOAD(rtc, nvrtcGetCUBINSize) LOAD(rtc, nvrtcGetCUBIN) LOAD(rtc, nvrtcDestroyProgram)
    g_api.rtc_ok = true;
    if (!cu) { g_api.why = "libcuda.so.1 not found"; return; }
    LOAD(cu, cuModuleLoadData) LOAD(cu, cuModuleGetFunction) LOAD(cu, cuLaunchKernel) LOAD(cu, cuFuncSetAttribute) LOAD(cu, cuGetErrorString) LOAD(cu, cuOccupancyMaxActiveBlocksPerMultiprocessor)
#undef LOAD
    g_api.ok = true;
}

}  // namespace

namespace tg {

bool jit_available()
{
    std::lock_guard<std::mutex> lock(g_mu);
    load_api();
    return g_api.ok;
}

const char* jit_unavailable_reason()
{
    return g_api.why.c_str();
}

// compile (prelude + body) for sm_90a; returns the cubin.  Needs no GPU: used by the CPU tests as well.
int jit_compile_cubin(tgpu_ctx* ctx, const std::string& body, std::string* cubin)
{
    {
        std::lock_guard<std::mutex> lock(g_mu);
        load_api();
    }
    if (!g_api.rtc_ok) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "NVRTC unavailable: %s", g_api.why.c_str());
    std::string src = std::string(kPrelude) + "\n" + body;
    nvrtcProgram prog = nullptr;
    int r = g_api.nvrtcCreateProgram(&prog, src.c_str(), "tgpu_jit.cu", 0, nullptr, nullptr);
    if (r != 0) return tg_fail(ctx, TGPU_ERR_CUDA, "nvrtcCreateProgram failed (%d)", r);
    const char* opts[] = {"--gpu-architecture=sm_90a", "--std=c++17", "--fmad=false", "-lineinfo", "-default-device"};
    r = g_api.nvrtcCompileProgram(prog, 5, opts);
    if (r != 0) {
        size_t n = 0;
        g_api.nvrtcGetProgramLogSize(prog, &n);
        std::string log(n + 1, '\0');
        if (n) g_api.nvrtcGetProgramLog(prog, &log[0]);
        g_api.nvrtcDestroyProgram(&prog);
        return tg_fail(ctx, TGPU_ERR_CUDA, "NVRTC compilation failed (%d): %.900s", r, log.c_str());
    }
    size_t n = 0;
    g_api.nvrtcGetCUBINSize(prog, &n);
    cubin->assign(n, '\0');
    g_api.nvrtcGetCUBIN(prog, &(*cubin)[0]);
    g_api.nvrtcDestroyProgram(&prog);
    return TGPU_OK;
}

int jit_selftest(const int32_t* channel_types, int32_t num_channels, const std::function<std::string(const int* elems)>& gen, int64_t* cubin_bytes,
                 char* source_out, int64_t source_cap)
{
    int elems[TGPU_MAX_CHANNELS] = {0};
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        DevColumn col;
        col.type = channel_types[c];
        elems[c] = col.elem_size();
    }
    auto copy_out = [&](const std::string& text) {
        if (source_out && source_cap > 0) { strncpy(source_out, text.c_str(), (size_t)source_cap - 1); source_out[source_cap - 1] = 0; }
    };
    const std::string src = gen(elems);
    copy_out(src);
    tgpu_ctx host;
    std::string cubin;
    const int st = jit_compile_cubin(&host, src, &cubin);
    if (st != TGPU_OK) { copy_out(host.err); return st; }
    *cubin_bytes = (int64_t)cubin.size();
    return TGPU_OK;
}

int jit_get_function(tgpu_ctx* ctx, const std::string& body, const char* kernel_name, void** fn_out)
{
    std::string key = std::to_string(ctx->device) + "|" + kernel_name + "|" + body;
    {
        std::lock_guard<std::mutex> lock(g_mu);
        auto it = g_cache.find(key);
        if (it != g_cache.end()) { *fn_out = (void*)it->second; return TGPU_OK; }
    }
    std::string cubin;
    TG_TRY(jit_compile_cubin(ctx, body, &cubin));
    CUmodule mod = nullptr;
    int r = g_api.cuModuleLoadData(&mod, cubin.data());
    if (r != 0) {
        const char* msg = nullptr;
        g_api.cuGetErrorString(r, &msg);
        return tg_fail(ctx, TGPU_ERR_CUDA, "cuModuleLoadData failed: %s", msg ? msg : "?");
    }
    CUfunction fn = nullptr;
    r = g_api.cuModuleGetFunction(&fn, mod, kernel_name);
    if (r != 0) return tg_fail(ctx, TGPU_ERR_CUDA, "cuModuleGetFunction(%s) failed (%d)", kernel_name, r);
    {
        std::lock_guard<std::mutex> lock(g_mu);
        g_cache[key] = fn;
    }
    *fn_out = (void*)fn;
    return TGPU_OK;
}

int jit_blocks_per_sm(void* fn, int block, size_t smem)
{
    int n = 0;
    if (!g_api.cuOccupancyMaxActiveBlocksPerMultiprocessor || g_api.cuOccupancyMaxActiveBlocksPerMultiprocessor(&n, (CUfunction)fn, block, smem) != 0 || n < 1) return 4;
    return n;
}

int jit_launch(tgpu_ctx* ctx, void* fn, int grid, int block, size_t smem, void** params)
{
    if (smem > 48 * 1024) {
        int r = g_api.cuFuncSetAttribute((CUfunction)fn, 8 /* CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES */, (int)smem);
        if (r != 0) return tg_fail(ctx, TGPU_ERR_CUDA, "cuFuncSetAttribute(max dynamic smem %zu) failed (%d)", smem, r);
    }
    int r = g_api.cuLaunchKernel((CUfunction)fn, (unsigned)grid, 1, 1, (unsigned)block, 1, 1, (unsigned)smem, ctx->stream, params, nullptr);
    ctx->launches++;
    if (r != 0) {
        const char* msg = nullptr;
        g_api.cuGetErrorString(r, &msg);
        return tg_fail(ctx, TGPU_ERR_CUDA, "cuLaunchKernel failed: %s", msg ? msg : "?");
    }
    return TGPU_OK;
}

}  // namespace tg
