// Error plumbing, the kernel launch helper with its per-device state, and small utility kernels shared by the C ABI.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace stb {
unsigned long long launches();

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }

static unsigned long long g_launches = 0;
unsigned long long launches() { return g_launches; }

// ---- event profiler ----
struct ProfRec { const char* name; cudaEvent_t e0, e1; double bytes, flops; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
static std::vector<cudaEvent_t> g_events;
static cudaEvent_t take_event() {
    if (!g_events.empty()) { cudaEvent_t e = g_events.back(); g_events.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
}
ProfScope::ProfScope(const char* name, cudaStream_t s, double bytes, double flops) : slot(-1), st(s) {
    if (!g_prof_on) return;
    ProfRec r{name, take_event(), take_event(), bytes, flops};
    cudaEventRecord(r.e0, st);
    slot = (int)g_prof.size();
    g_prof.push_back(r);
}
ProfScope::~ProfScope() {
    if (slot >= 0) cudaEventRecord(g_prof[slot].e1, st);
}

// ---- launch policy (common.cuh: LaunchSpec) ----

// STB_PDL=0 turns programmatic dependent launch off for every kernel (the in-kernel griddepcontrol instructions are then
// no-ops); unset or any other value leaves it on.
static bool pdl_enabled() {
    static const bool on = [] {
        const char* e = getenv("STB_PDL");
        return !(e && strcmp(e, "0") == 0);
    }();
    return on;
}

int& launch_priority() {
    static thread_local int p = 0;
    return p;
}

// Per-device state.  Function attributes and SM counts belong to a device, and a process may drive models on several.
struct FuncSmem {
    size_t opted;      // dynamic shared memory the kernel may currently be launched with
    size_t limit;      // the device's opt-in limit minus the kernel's static shared memory
    bool carveout;     // the largest carveout is set
};
static std::mutex g_dev_mu;
static std::map<int, int> g_sms;                                     // device ordinal -> multiprocessor count
static std::map<std::pair<const void*, int>, FuncSmem> g_smem;       // (kernel, device ordinal) -> shared memory

int sm_count() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    std::lock_guard<std::mutex> lk(g_dev_mu);
    int& n = g_sms[dev];
    if (n == 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
    return n;
}

// the entry of `kernel` on the current device; the caller holds g_dev_mu
static int func_smem(const void* kernel, FuncSmem** out) {
    int dev = 0;
    STB_CUDA_OK(cudaGetDevice(&dev));
    auto it = g_smem.find({kernel, dev});
    if (it == g_smem.end()) {
        cudaFuncAttributes fa;
        int optin = 0;
        STB_CUDA_OK(cudaFuncGetAttributes(&fa, kernel));
        STB_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        const FuncSmem f = {(size_t)fa.maxDynamicSharedSizeBytes, (size_t)optin - fa.sharedSizeBytes, false};
        it = g_smem.emplace(std::make_pair(kernel, dev), f).first;
    }
    *out = &it->second;
    return STB_OK;
}

int max_dynamic_smem(const void* kernel, size_t* limit) {
    std::lock_guard<std::mutex> lk(g_dev_mu);
    FuncSmem* f = nullptr;
    STB_TRY(func_smem(kernel, &f));
    *limit = f->limit;
    return STB_OK;
}

static int opt_in_smem(const void* kernel, size_t smem, bool max_carveout) {
    std::lock_guard<std::mutex> lk(g_dev_mu);
    FuncSmem* f = nullptr;
    STB_TRY(func_smem(kernel, &f));
    if (smem > f->opted) {
        STB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        f->opted = smem;
    }
    if (max_carveout && !f->carveout) {
        STB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        f->carveout = true;
    }
    return STB_OK;
}

int launch_kernel(const void* kernel, const LaunchSpec& s, void** args) {
    if (s.smem > 0 || s.max_carveout) STB_TRY(opt_in_smem(kernel, s.smem, s.max_carveout));
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = s.grid;
    cfg.blockDim = s.block;
    cfg.dynamicSmemBytes = s.smem;
    cfg.stream = s.stream;
    cudaLaunchAttribute attr[3];
    unsigned n = 0;
    if (s.cluster > 0) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = s.cluster;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    if (s.pdl && pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    const int priority = launch_priority();
    if (priority != 0) {
        attr[n].id = cudaLaunchAttributePriority;
        attr[n].val.priority = priority;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    cudaError_t e = cudaLaunchKernelExC(&cfg, kernel, args);
    ++g_launches;
    const cudaError_t latched = cudaGetLastError();      // also clears the launch's own error
    if (e == cudaSuccess) e = latched;
    if (e != cudaSuccess) {
        set_error("%s:%d: kernel launch -> %s", s.file, s.line, cudaGetErrorString(e));
        return STB_ERR_CUDA;
    }
    return STB_OK;
}

// fp32 [rows][cols] -> fp16 hi (+ lo) planes.  8 elements per thread, 128-bit loads/stores where aligned.
__global__ void split_f16_kernel(const float* __restrict__ src, long long rows, int cols, long long src_ld,
                                 __half* __restrict__ hi, __half* __restrict__ lo, long long dst_ld) {
    const long long total = rows * (long long)cols;
    for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x); i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cols;
        const int c = (int)(i - r * cols);
        __half h, l;
        split_f16(src[r * src_ld + c], h, l);
        hi[r * dst_ld + c] = h;
        if (lo != nullptr) lo[r * dst_ld + c] = l;
    }
}

// y = a * x + b * y
__global__ void axpby_kernel(float* __restrict__ y, const float* __restrict__ x, float a, float b, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        y[i] = a * x[i] + b * y[i];
}

}  // namespace stb

extern "C" int stb_axpby(float* y, const float* x, float a, float b, long long n, void* stream) {
    STB_REQUIRE(y && x && n >= 0, "stb_axpby: bad arguments");
    if (n == 0) return STB_OK;
    const int cap = stb::sm_count() * 8;
    const int grid = (int)((n + 255) / 256 < cap ? (n + 255) / 256 : cap);
    return stb::launch(stb::axpby_kernel, {grid, 256, 0, (cudaStream_t)stream}, y, x, a, b, n);
}

extern "C" const char* stb_last_error(void) { return stb::get_error(); }
extern "C" int stb_abi_version(void) { return 7; }
extern "C" unsigned long long stb_launch_count(void) { return stb::launches(); }

extern "C" int stb_split_f16(const float* src, long long rows, int cols, long long src_ld, void* hi, void* lo,
                             long long dst_ld, void* stream) {
    STB_REQUIRE(src && hi && rows >= 0 && cols > 0, "stb_split_f16: bad arguments");
    if (rows == 0) return STB_OK;
    const long long total = rows * (long long)cols;
    int blocks = (int)((total + 255) / 256);
    const int cap = stb::sm_count() * 16;
    if (blocks > cap) blocks = cap;
    return stb::launch(stb::split_f16_kernel, {blocks, 256, 0, (cudaStream_t)stream}, src, rows, cols, src_ld, (__half*)hi,
                       (__half*)lo, dst_ld);
}

extern "C" void stb_prof_enable(int on) { stb::g_prof_on = on != 0; }

// Synchronises, aggregates the records since the last call per kernel name into `buf` as JSON
// {"name": {"n": launches, "ms": total, "bytes": algorithmic, "flops": algorithmic}, ...}, then clears them.
extern "C" int stb_prof_report(char* buf, size_t buf_bytes) {
    STB_CUDA_OK(cudaDeviceSynchronize());
    struct Agg { long long n = 0; double ms = 0, bytes = 0, flops = 0; };
    std::map<std::string, Agg> agg;
    for (auto& r : stb::g_prof) {
        float t = 0;
        cudaEventElapsedTime(&t, r.e0, r.e1);
        Agg& a = agg[r.name];
        a.n += 1; a.ms += t; a.bytes += r.bytes; a.flops += r.flops;
        stb::g_events.push_back(r.e0);
        stb::g_events.push_back(r.e1);
    }
    stb::g_prof.clear();
    std::string out = "{";
    bool first = true;
    for (auto& kv : agg) {
        char tmp[256];
        snprintf(tmp, sizeof(tmp), "%s\"%s\": {\"n\": %lld, \"ms\": %.6f, \"bytes\": %.0f, \"flops\": %.0f}", first ? "" : ", ",
                 kv.first.c_str(), kv.second.n, kv.second.ms, kv.second.bytes, kv.second.flops);
        out += tmp;
        first = false;
    }
    out += "}";
    STB_REQUIRE(buf && out.size() + 1 <= buf_bytes, "stb_prof_report: buffer too small (%zu needed)", out.size() + 1);
    memcpy(buf, out.c_str(), out.size() + 1);
    return STB_OK;
}
