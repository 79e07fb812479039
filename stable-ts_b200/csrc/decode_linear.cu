// Linear layers of the KV-cached decode step for 17..128 sequences (stable_whisper/decode.py:40 -> whisper's
// TextDecoder on the newest token): out[s][n] = epilogue( sum_k x[s][k] * W[n][k] ), a few hundred MB of weights per
// step streamed once, ~120 sequences: HBM-bound on the weights, and -- with ~200 such GEMMs per step -- latency-bound
// on everything between them.  The legacy route runs each as a swapped split-K GEMM writing fp32 partials to L2 plus a
// second "finish" kernel (bias / GELU / residual): 12 dependent launches per decoder layer.
//
// This kernel does one Linear in ONE launch with no partials in global memory:
//   * SWAPPED: the 128 output features of a tile sit on the MMA's M side (every weight byte is read by exactly one CTA),
//     the sequences on the N side (BN = 32 / 64 / 128 >= B, rows past B are zero-filled by TMA);
//   * split-K across a THREAD-BLOCK CLUSTER: the CTAs of a cluster own the same feature tile and consecutive K ranges, so
//     tiles x split ~ 80-115 CTAs stream the weights concurrently;
//   * each CTA: TMA (SWIZZLE_128B, mbarrier ring) -> two consumer warpgroups of 64 features each, wgmma m64nBNk16
//     (hi*hi + hi*lo + lo*hi passes in parity mode) -> fp32 accumulator fragments in registers -> the CTA's OWN shared
//     memory as an fp32 [sequence][feature] tile;
//   * cluster barrier; CTA r then sums column slice r of all peers' tiles over distributed shared memory
//     (ld.shared::cluster, fixed summation order: bit-reproducible) and applies bias / GELU / residual, storing fp32 and/or
//     split-fp16 rows [sequence][feature] coalesced along the features;
//   * programmatic dependent launch: barrier init and the WEIGHT tiles of the first ring stages are issued
//     before griddepcontrol.wait (weights do not depend on the previous kernel); only the activation tiles wait.
#include <string.h>

#include "common.cuh"
#include "kernels.h"

namespace stb {

struct DLArgs {
    int n, B, kb_total;       // output features, sequences, 64-wide k blocks
    const float* bias;
    int act;
    const float* res;
    long long ld_res;
    float* out_f32;
    __half* out_hi;
    __half* out_lo;
    long long ld_out;
};

__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_size() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// exit barrier: nothing is published, the peers only need to know that this CTA has finished READING their tiles
__device__ __forceinline__ void cluster_sync_relaxed() {
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t dsmem_addr(uint32_t local_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
    return r;
}
// 16-byte load from a peer CTA's shared memory (volatile + memory clobber keep it behind the cluster barrier; the loads of
// one reduction step go to distinct registers, so they still issue back to back and their latencies overlap)
__device__ __forceinline__ float4 dsmem_ld4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

template <int BN, int PASSES>
struct DLCfg {
    static constexpr int NPL = PASSES == 3 ? 2 : 1;
    static constexpr uint32_t A_TILE = 128 * 128;             // 128 features x 64 fp16
    static constexpr uint32_t B_TILE = BN * 128;               // BN sequences x 64 fp16
    static constexpr uint32_t STAGE = NPL * (A_TILE + B_TILE);
    static constexpr uint32_t PART = BN * 128 * 4;             // fp32 [BN sequences][128 features], aliases the ring
    static constexpr int STAGES_RAW = (200 * 1024) / STAGE;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr uint32_t RING = STAGES * STAGE;
    static constexpr uint32_t SMEM = (RING > PART ? RING : PART) + 1024;
};

constexpr int DL_THREADS = 288;      // 2 consumer warpgroups + the producer warp

template <int BN, int PASSES>
__global__ void __launch_bounds__(DL_THREADS, 1)
decode_linear_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                     const __grid_constant__ CUtensorMap tmXh, const __grid_constant__ CUtensorMap tmXl, const DLArgs g) {
    using Cfg = DLCfg<BN, PASSES>;
    constexpr int NPL = Cfg::NPL;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int rank = (int)cluster_rank(), split = (int)cluster_size();
    const int m0 = (blockIdx.x / split) * 128;                 // first output feature of this cluster's tile
    const int kb0 = (int)((long long)rank * g.kb_total / split), kb1 = (int)((long long)(rank + 1) * g.kb_total / split);
    const int nk = kb1 - kb0;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmWh);
        tma_prefetch_desc(&tmXh);
        if (NPL == 2) {
            tma_prefetch_desc(&tmWl);
            tma_prefetch_desc(&tmXl);
        }
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);                        // one arrival per consumer warpgroup
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_trigger();

    if (warp == 8) {
        // ------------------------------------------------ TMA producer
        if (lane == 0) {
            const int pre = nk < STAGES ? nk : STAGES;
            // weights of the first ring stages: independent of the previous kernel, issued before the dependency wait
            for (int i = 0; i < pre; ++i) {
                uint8_t* s = tiles + (size_t)i * Cfg::STAGE;
                mbar_arrive_expect_tx(&full_bar[i], Cfg::STAGE);
                const int k0 = (kb0 + i) * 64;
                tma_load_4d(s, &tmWh, &full_bar[i], k0, m0, 0, 0);
                if (NPL == 2) tma_load_4d(s + Cfg::A_TILE, &tmWl, &full_bar[i], k0, m0, 0, 0);
            }
            pdl_wait();                                         // the activations are the previous kernel's output
            for (int i = 0; i < pre; ++i) {
                uint8_t* s = tiles + (size_t)i * Cfg::STAGE;
                const int k0 = (kb0 + i) * 64;
                tma_load_4d(s + NPL * Cfg::A_TILE, &tmXh, &full_bar[i], k0, 0, 0, 0);
                if (NPL == 2) tma_load_4d(s + NPL * Cfg::A_TILE + Cfg::B_TILE, &tmXl, &full_bar[i], k0, 0, 0, 0);
            }
            int stage = pre == STAGES ? 0 : pre;
            uint32_t phase = pre == STAGES ? 1 : 0;
            for (int i = pre; i < nk; ++i) {
                mbar_wait_mma(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE);
                uint8_t* s = tiles + (size_t)stage * Cfg::STAGE;
                const int k0 = (kb0 + i) * 64;
                tma_load_4d(s, &tmWh, &full_bar[stage], k0, m0, 0, 0);
                if (NPL == 2) tma_load_4d(s + Cfg::A_TILE, &tmWl, &full_bar[stage], k0, m0, 0, 0);
                tma_load_4d(s + NPL * Cfg::A_TILE, &tmXh, &full_bar[stage], k0, 0, 0, 0);
                if (NPL == 2) tma_load_4d(s + NPL * Cfg::A_TILE + Cfg::B_TILE, &tmXl, &full_bar[stage], k0, 0, 0, 0);
                if (++stage == STAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
    } else {
        // ------------------------------------------------ consumers: warpgroup wg owns features [64 wg, 64 wg + 64) of the tile
        const int wg = warp >> 2;
        const uint32_t a_row_off = (uint32_t)wg * 64u * 128u;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;         // an empty K range contributes zeros
        int stage = 0, prev_stage = -1;
        uint32_t phase = 0, accum = 0;
        for (int i = 0; i < nk; ++i) {
            mbar_wait_mma(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(tiles + (size_t)stage * Cfg::STAGE);
            const uint32_t a_hi = sa + a_row_off, a_lo = a_hi + Cfg::A_TILE;
            const uint32_t b_hi = sa + NPL * Cfg::A_TILE, b_lo = b_hi + Cfg::B_TILE;
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < PASSES; ++pass) {        // pass 0: hi*hi, 1: hi*lo, 2: lo*hi
                const uint32_t pa = (pass == 2) ? a_lo : a_hi;
                const uint32_t pb = (pass == 1) ? b_lo : b_hi;
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4) {
                    wgmma_ss(acc, wgmma_desc_k128(pa + k4 * 32), wgmma_desc_k128(pb + k4 * 32), accum);
                    accum = 1;
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                                    // the previous k-block's MMAs have retired: free its slot
            if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = stage;
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
        // accumulator fragments -> own shared memory, fp32 [sequence][feature].  The tile aliases the ring: both
        // warpgroups must have finished reading it
        asm volatile("bar.sync 1, 256;" ::: "memory");
        float* part = reinterpret_cast<float*>(tiles);
        const int t = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // feature row inside the tile
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);              // sequence
            part[c * 128 + t] = acc[4 * j];
            part[(c + 1) * 128 + t] = acc[4 * j + 1];
            part[c * 128 + t + 8] = acc[4 * j + 2];
            part[(c + 1) * 128 + t + 8] = acc[4 * j + 3];
        }
    }
    __syncwarp();
    cluster_sync_all();                                         // every peer's tile is complete and visible
    if (warp < 8) {
        // Reduce-scatter over distributed shared memory: rank r owns sequences [r BN / split, (r + 1) BN / split).  A warp
        // handles one sequence per iteration, a lane 4 consecutive features of it: it issues the 16-byte loads of ALL peers
        // first (independent, so their DSMEM latencies overlap), adds them in rank order (bit-reproducible), applies the
        // epilogue and stores 16 bytes.  The loop bounds are warp-uniform; lanes whose features lie past n skip their
        // global loads and stores.
        const int e = warp * 32 + lane;                        // 0 .. 255
        const int quad = e & 31;                               // features m0 + 4 quad .. + 3
        const int m = m0 + quad * 4;
        const int c0 = rank * BN / split, c1 = (rank + 1) * BN / split;
        const uint32_t local = smem_u32(tiles);
        uint32_t peer[8];
#pragma unroll
        for (int p = 0; p < 8; ++p) peer[p] = p < split ? dsmem_addr(local, (uint32_t)p) : 0u;
        pdl_wait();                                             // the residual is an earlier kernel's output
        const bool full = m + 3 < g.n;                          // all 4 features exist
        const bool vec = full && (g.ld_out & 3) == 0 && (g.res == nullptr || (g.ld_res & 3) == 0);
        auto load4 = [&](const float* p) -> float4 {            // 4 per-feature constants, zero past n
            float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p == nullptr) return r;
            if (full) return __ldg(reinterpret_cast<const float4*>(p + m));
            if (m < g.n) r.x = __ldg(p + m);
            if (m + 1 < g.n) r.y = __ldg(p + m + 1);
            if (m + 2 < g.n) r.z = __ldg(p + m + 2);
            return r;
        };
        const float4 bias = load4(g.bias);
        for (int c = c0 + (e >> 5); c < c1 && c < g.B; c += 8) {
            const uint32_t off = (uint32_t)((c * 128 + quad * 4) * 4);
            float4 v[8];
#pragma unroll
            for (int p = 0; p < 8; ++p)
                if (p < split) v[p] = dsmem_ld4(peer[p] + off);
            float4 a = v[0];
#pragma unroll
            for (int p = 1; p < 8; ++p)
                if (p < split) { a.x += v[p].x; a.y += v[p].y; a.z += v[p].z; a.w += v[p].w; }
            a.x += bias.x; a.y += bias.y; a.z += bias.z; a.w += bias.w;
            if (g.act == STB_ACT_GELU) { a.x = gelu_erf(a.x); a.y = gelu_erf(a.y); a.z = gelu_erf(a.z); a.w = gelu_erf(a.w); }
            if (g.res != nullptr) {
                const float* rp = g.res + (long long)c * g.ld_res + m;
                if (vec) {
                    const float4 r = *reinterpret_cast<const float4*>(rp);
                    a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w;
                } else {
                    if (m < g.n) a.x += rp[0];
                    if (m + 1 < g.n) a.y += rp[1];
                    if (m + 2 < g.n) a.z += rp[2];
                    if (m + 3 < g.n) a.w += rp[3];
                }
            }
            const long long off_o = (long long)c * g.ld_out + m;
            if (vec) {
                if (g.out_f32 != nullptr) *reinterpret_cast<float4*>(g.out_f32 + off_o) = a;
                if (g.out_hi != nullptr) {
                    __half h[4], l[4];
                    split_f16(a.x, h[0], l[0]); split_f16(a.y, h[1], l[1]);
                    split_f16(a.z, h[2], l[2]); split_f16(a.w, h[3], l[3]);
                    *reinterpret_cast<uint2*>(g.out_hi + off_o) = *reinterpret_cast<const uint2*>(h);
                    if (g.out_lo != nullptr) *reinterpret_cast<uint2*>(g.out_lo + off_o) = *reinterpret_cast<const uint2*>(l);
                }
            } else {
                const float vals[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (m + j >= g.n) break;
                    if (g.out_f32 != nullptr) g.out_f32[off_o + j] = vals[j];
                    if (g.out_hi != nullptr) {
                        __half hi, lo;
                        split_f16(vals[j], hi, lo);
                        g.out_hi[off_o + j] = hi;
                        if (g.out_lo != nullptr) g.out_lo[off_o + j] = lo;
                    }
                }
            }
        }
    }
    __syncwarp();
    cluster_sync_relaxed();                                     // nobody exits while a peer may still read its tile
}

// cluster size in 1..8 (every size up to 8 is portable) that puts the most CTAs on the machine: every rank gets at least
// one k block, and all clusters are co-resident with margin for GPC granularity (a cluster lives inside one GPC, whose
// SM count is not a multiple of every cluster size): 7/8 of the SMs, 115 CTAs on the 132 SMs of an H100
int decode_linear_split(int n, int k) {
    const int mt = cdiv(n, 128), nkb = k / 64;
    const int budget = (sm_count() * 7) / 8;
    int split = 1;
    for (int s = 2; s <= 8; ++s)
        if (s <= nkb && (long long)mt * s <= budget) split = s;
    return split;
}

template <int BN, int PASSES>
static int launch_dl(const TmapVal& wh, const TmapVal& wl, const TmapVal& xh, const TmapVal& xl, const DLArgs& g, int split,
                     cudaStream_t st) {
    using Cfg = DLCfg<BN, PASSES>;
    const int mt = cdiv(g.n, 128);
    const double wbytes = (double)g.n * g.kb_total * 64 * 2.0 * Cfg::NPL;
    ProfScope ps("decode_linear", st, wbytes + (double)g.B * g.kb_total * 64 * 2.0 * Cfg::NPL + (double)g.B * g.n * 4.0,
                 2.0 * g.n * (double)g.B * g.kb_total * 64);
    return launch(decode_linear_kernel<BN, PASSES>,
                  {dim3((unsigned)(mt * split)), dim3(DL_THREADS), Cfg::SMEM, st, /*pdl=*/true, /*cluster=*/(unsigned)split}, wh.map,
                  wl.map, xh.map, xl.map, g);
}

// out[B][n] = epilogue(x[B][k] . W[n][k]^T); x / W split-fp16 planes, K-major; B <= 128; k a multiple of 64.
int decode_linear(const void* x_hi, const void* x_lo, int B, int k, const void* w_hi, const void* w_lo, int n, const float* bias,
                  int act, const float* res, long long ld_res, float* out_f32, void* out_hi, void* out_lo, long long ld_out,
                  cudaStream_t st) {
    STB_REQUIRE(x_hi && w_hi && (out_f32 || out_hi), "decode_linear: null argument");
    STB_REQUIRE(B >= 1 && B <= 128 && k % 64 == 0 && n >= 1, "decode_linear: unsupported shape B=%d k=%d n=%d", B, k, n);
    STB_REQUIRE((x_lo != nullptr) == (w_lo != nullptr), "decode_linear: lo planes must be given for both operands or neither");
    const int BN = B <= 32 ? 32 : B <= 64 ? 64 : 128;
    DLArgs g;
    memset(&g, 0, sizeof(g));
    g.n = n; g.B = B; g.kb_total = k / 64;
    g.bias = bias; g.act = act; g.res = res; g.ld_res = ld_res;
    g.out_f32 = out_f32; g.out_hi = (__half*)out_hi; g.out_lo = (__half*)out_lo; g.ld_out = ld_out;
    const int split = decode_linear_split(n, k);
    TmapVal wh, wl, xh, xl;
    STB_TRY(make_tmap(w_hi, n, k, 1, 1, k, 0, 0, 128, &wh));
    STB_TRY(make_tmap(x_hi, B, k, 1, 1, k, 0, 0, BN, &xh));
    if (w_lo) {
        STB_TRY(make_tmap(w_lo, n, k, 1, 1, k, 0, 0, 128, &wl));
        STB_TRY(make_tmap(x_lo, B, k, 1, 1, k, 0, 0, BN, &xl));
    } else {
        wl = wh;
        xl = xh;
    }
#define STB_DL_CASE(bn)                                                                                   \
    case bn:                                                                                              \
        return w_lo ? launch_dl<bn, 3>(wh, wl, xh, xl, g, split, st) : launch_dl<bn, 1>(wh, wl, xh, xl, g, split, st);
    switch (BN) {
        STB_DL_CASE(32)
        STB_DL_CASE(64)
        STB_DL_CASE(128)
    }
#undef STB_DL_CASE
    return STB_ERR_UNSUPPORTED;
}

}  // namespace stb

static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

extern "C" int stb_decode_linear(const void* x_hi, const void* x_lo, int B, int K, const void* w_hi, const void* w_lo, int N,
                                 const float* bias, int act, const float* res, long long ld_res, float* out_f32, void* out_hi,
                                 void* out_lo, long long ld_out, void* stream) {
    STB_REQUIRE(B >= 1 && B <= 128, "stb_decode_linear: B=%d outside 1..128", B);
    STB_REQUIRE(K >= 64 && K % 64 == 0, "stb_decode_linear: K=%d must be a positive multiple of 64", K);
    STB_REQUIRE(N >= 1, "stb_decode_linear: N=%d must be positive", N);
    STB_REQUIRE(ld_out >= N && (res == nullptr || ld_res >= N), "stb_decode_linear: leading dimensions smaller than N");
    STB_REQUIRE(act == STB_ACT_NONE || act == STB_ACT_GELU, "stb_decode_linear: unknown activation %d", act);
    STB_REQUIRE(x_hi && w_hi && (out_f32 || out_hi) && (out_lo == nullptr || out_hi != nullptr), "stb_decode_linear: null argument");
    STB_REQUIRE((x_lo != nullptr) == (w_lo != nullptr), "stb_decode_linear: lo planes must be given for both operands or neither");
    // vector loads / stores: per-feature constants and fp32 rows as float4, fp16 rows as 4 halves
    STB_REQUIRE(aligned(bias, 16) && aligned(res, 16) && aligned(out_f32, 16) && aligned(out_hi, 8) && aligned(out_lo, 8),
                "stb_decode_linear: misaligned pointer");
    return stb::decode_linear(x_hi, x_lo, B, K, w_hi, w_lo, N, bias, act, res, ld_res, out_f32, out_hi, out_lo, ld_out,
                              (cudaStream_t)stream);
}

extern "C" int stb_decode_linear_split(int n, int k) {
    if (n < 1 || k < 64 || k % 64 != 0) {                      // 0: not a cluster size, so not mistaken for one
        stb::set_error("stb_decode_linear_split: bad shape n=%d k=%d", n, k);
        return 0;
    }
    return stb::decode_linear_split(n, k);
}
