// Shared device/host helpers for the H100 (sm_90a) kernels of the stable-ts word-timestamp hot path.
// Everything here is hand-written for sm_90a: mbarrier / TMA / wgmma inline PTX, warp-shuffle reductions,
// split-fp16 ("hi + lo") helpers used to run fp32-accurate GEMMs on the fp16 tensor pipe.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/stablets_b200.h"

// NO kernel parameter of this library is restrict-qualified.  Under programmatic dependent launch a kernel reads its
// predecessor's output after griddepcontrol.wait; with `const T* __restrict__` parameters nvcc turns such reads into
// ld.global.nc, and -- invariant loads carry no memory dependence -- schedules them ABOVE the wait (round 2, seen in SASS:
// LDG.E.CONSTANT of the token id and of the position counter before ACQBULK in embed_step_kernel; under CUDA-graph replay
// the step then embedded the PREVIOUS token).  The qualifier stays in the sources as documentation of intent and is erased
// here; data that really is constant for a kernel's lifetime (weights, biases, tables) is read with explicit __ldg().
// tools/check_pdl_sass.py lists every non-coherent load that precedes a kernel's wait.
#define __restrict__

namespace stb {

// ---- host-side error plumbing (thread-local message returned by stb_last_error) ----
void set_error(const char* fmt, ...);
const char* get_error();

#define STB_CUDA_OK(expr)                                                                              \
    do {                                                                                               \
        cudaError_t e__ = (expr);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            stb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__));      \
            (void)cudaGetLastError(); /* do not leave the error latched for an unrelated later launch check */ \
            return STB_ERR_CUDA;                                                                       \
        }                                                                                              \
    } while (0)

#define STB_REQUIRE(cond, ...)                                                                         \
    do {                                                                                               \
        if (!(cond)) {                                                                                 \
            stb::set_error(__VA_ARGS__);                                                               \
            return STB_ERR_ARG;                                                                        \
        }                                                                                              \
    } while (0)

#define STB_TRY(expr)                                                                                  \
    do {                                                                                               \
        int r__ = (expr);                                                                              \
        if (r__ != STB_OK) return r__;                                                                 \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Optional per-launch CUDA-event profiling (stb_prof_enable): events are recorded on the launching stream around one
// kernel; stb_prof_report() aggregates time / algorithmic bytes / algorithmic FLOPs per kernel name.
struct ProfScope {
    ProfScope(const char* name, cudaStream_t st, double bytes = 0.0, double flops = 0.0);
    ~ProfScope();
    int slot;
    cudaStream_t st;
};
int sm_count();   // cudaDevAttrMultiProcessorCount of the current device, cached per device ordinal

// launch priority of the kernels launched next by this host thread (cudaLaunchAttributePriority; 0 = the stream's own).
// The decode step raises it for its latency-bound linear layers: under programmatic dependent launch the next kernel's CTAs
// can become resident while the previous kernel's tail still runs, and the block scheduler then serves the higher-priority
// CTAs first.  Not measured against priority 0.
int& launch_priority();

// ---------------------------------------------------------------------------------------------------------
// Kernel launches.  Every kernel of this library is launched with stb::launch, which owns the launch policy (misc.cu):
//  - programmatic dependent launch (PDL, `pdl`): the kernel may start while its predecessor in the stream is still
//    running, so it must execute pdl_wait() before touching anything the predecessor writes; a kernel without that wait
//    must not set `pdl`.  pdl_trigger() lets the NEXT kernel start early.  Both are no-ops for ordinary launches, and
//    STB_PDL=0 turns PDL off for every launch.
//  - the thread-block cluster (`cluster` = x-size; 0 = an ordinary launch, 1 = a cluster of one CTA);
//  - launch_priority(), when it is not 0;
//  - the opt-in to more dynamic shared memory than a kernel is allowed by default, per (kernel, device), and the
//    largest shared-memory carveout when `max_carveout` is set;
//  - one count per launch for stb_launch_count(), and the launch error check (the latched error is cleared).
// ---------------------------------------------------------------------------------------------------------
struct LaunchSpec {
    dim3 grid, block;
    size_t smem = 0;                            // dynamic shared memory, bytes
    cudaStream_t stream = nullptr;
    bool pdl = false;
    unsigned cluster = 0;
    bool max_carveout = false;
    const char* file = __builtin_FILE();        // the call site, named by the launch error
    int line = __builtin_LINE();
};

int launch_kernel(const void* kernel, const LaunchSpec& spec, void** args);
// largest dynamic shared memory `kernel` can be launched with on the current device (the device's opt-in limit minus
// the kernel's static shared memory)
int max_dynamic_smem(const void* kernel, size_t* limit);

// Returns STB_OK or STB_ERR_CUDA (message in stb_last_error).
template <typename... KArgs, typename... Args>
static inline int launch(void (*kernel)(KArgs...), const LaunchSpec& spec, Args... args) {
    return [&](KArgs... a) {
        void* p[] = {(void*)&a...};
        return launch_kernel((const void*)kernel, spec, p);
    }(static_cast<KArgs>(args)...);
}

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------
// warp helpers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// fp32 -> (hi, lo) fp16 pair with hi + lo == x to ~2^-22 relative.
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// ---------------------------------------------------------------------------------------------------------
// mbarrier / TMA / wgmma PTX (sm_90a)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait (~2 s of SM clock): a protocol bug must trap (launch error) rather than hang the GPU machine.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {
            printf("stb: mbarrier timeout tag=%d block=(%d,%d,%d) thread=%d parity=%u\n", tag, blockIdx.x, blockIdx.y,
                   blockIdx.z, threadIdx.x, parity);
            __trap();
        }
    }
}

// The same bounded wait for every warp of a kernel that issues wgmma: ptxas serialises the wgmma.mma_async of a kernel that
// contains any function call, and printf is one, so a timeout here traps without a message.
__device__ __forceinline__ void mbar_wait_mma(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---- wgmma (sm_90a): D[registers] (+)= A * B, fp16 inputs, fp32 accumulate, issued by all 128 threads of a warpgroup.
// The accumulator of an m64nN tile is spread over the warpgroup: thread t holds, for every 8-column group j < N / 8,
//   d[4j + 0], d[4j + 1]  at row 16 (t / 32) + (t % 32) / 4,      columns 8j + 2 (t % 4) + {0, 1}
//   d[4j + 2], d[4j + 3]  at row 16 (t / 32) + (t % 32) / 4 + 8,  same columns.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory matrix descriptor for a K-major tile whose rows are exactly 128 bytes (64 x fp16) written by TMA
// with CU_TENSOR_MAP_SWIZZLE_128B: 8-row x 128 B swizzle atoms stacked every 1024 B (stride byte offset).  Bit layout:
// start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled K-major; 1), SBO>>4 [32,46), layout [62,64) (1 = SWIZZLE_128B).
// A k-step of 16 fp16 inside the 128 B row advances the start address by 32 B.
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// m64nNk16 with both operands in shared memory; N = 2 x (accumulator registers per thread) = 16 / 32 / 64 / 128
__device__ __forceinline__ void wgmma_ss(float (&d)[8], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7"
        "}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
        "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
        "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, "
        "%42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, "
        "%62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// A from registers (the m64k16 fp16 fragment: 4 x b32 per thread), B = 64 x 16 K-major tile in shared memory
__device__ __forceinline__ void wgmma_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
        "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}
#endif  // __CUDACC__

}  // namespace stb
