// Error plumbing, device attributes and small utility kernels shared by the C ABI.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
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
void count_launch() { ++g_launches; }
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

// STB_PDL: bit 0 = programmatic dependent launch for the ordinary kernels (launch_pdl), bit 1 = for the cluster kernel of
// the decode-step linears.  Default 3 (both); 0 disables it everywhere (the in-kernel griddepcontrol instructions are then no-ops).
bool pdl_enabled(int kind) {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("STB_PDL");
        v = (e && e[0]) ? atoi(e) : 3;
    }
    return (v >> kind) & 1;
}

int& launch_priority() {
    static thread_local int p = 0;
    return p;
}

int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
            n = 132;
    }
    return n;
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
    stb::axpby_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(y, x, a, b, n);
    STB_LAUNCH_OK();
    return STB_OK;
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
    stb::split_f16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, rows, cols, src_ld, (__half*)hi, (__half*)lo, dst_ld);
    STB_LAUNCH_OK();
    return STB_OK;
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
