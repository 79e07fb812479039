// K3: tensor-core GEMM core for sm_90a -- wgmma.mma_async (fp16 inputs, fp32 accumulators in registers) fed by TMA.
//
//   D[b,h][m][n] = epilogue( alpha * sum_k A[b,h][m][k] * B[b,h][n][k] )
//
// Replaces the cuBLAS calls under whisper.model.Linear / Conv1d / the q@k^T and w@v contractions of
// MultiHeadAttention.qkv_attention (reached from stable_whisper/timing.py:60-61, decode.py:29,40).
//
// Operands are K-major "split fp16" views: hi plane (+ optional lo plane, hi+lo == fp32 value to 2^-22).  With both
// lo planes present the kernel issues three MMA passes per k-block (hi*hi + hi*lo + lo*hi) into the same
// accumulator, which reproduces an fp32 GEMM to ~1e-6 relative on the fp16 tensor pipe (the reference's CPU/align
// path is fp32; SURVEY.md section 7 "precision vs the 1e-3 logits gate").  One pass = STB_PREC_FP16.
//
// Structure (PERSISTENT: one CTA per SM loops over 128 x BN output tiles; 288 threads):
//   warps 0..3, 4..7 : two consumer warpgroups, each owns 64 rows of the tile: wgmma m64nBNk16 from the swizzled shared-memory
//                      tiles (one group kept in flight across k-blocks), then the epilogue straight from the accumulator
//                      fragments: bias / GELU / residual / scale -> global (fp32 row-major, split-fp16 row-major, or either
//                      transposed)
//   warp 8           : TMA producer (cp.async.bulk.tensor.4d, SWIZZLE_128B tiles, mbarrier complete_tx); it runs ahead into the
//                      next tile's k-blocks while the consumers are in their epilogue
#include <mutex>
#include <string.h>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace stb {

struct GemmArgs {
    int M, N, K, H, Z;        // Z = n_batch * H independent (batch, head) problems
    int permA[3], permB[3];   // which of (row=0, head=1, batch=2) feeds TMA coordinate 1,2,3
    float* out_f32;
    __half* out_hi;
    __half* out_lo;
    long long ld_out, out_h, out_b;
    int transposed;
    const float* bias;
    int bias_per_row;
    const float* res;
    long long ld_res, res_h, res_b;
    float alpha;
    int act;
};

template <int BN, int PASSES>
struct GemmCfg {
    static constexpr int NPL = PASSES == 3 ? 2 : 1;                 // planes per operand
    static constexpr uint32_t A_TILE = 128 * 128;                   // 128 rows x 128 B
    static constexpr uint32_t B_TILE = BN * 128;
    static constexpr uint32_t STAGE = NPL * (A_TILE + B_TILE);
    static constexpr int STAGES_RAW = (200 * 1024) / STAGE;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr uint32_t SMEM = STAGES * STAGE + 1024;         // + slack for 1024 B alignment
};

constexpr int GEMM_THREADS = 288;    // 2 consumer warpgroups + the producer warp

__device__ __forceinline__ void pick_coords(const int (&perm)[3], int row, int h, int b, int& c1, int& c2, int& c3) {
    int v[4] = {row, h, b, 0};      // perm id 3 = broadcast dim (stride 0): coordinate pinned to 0
    c1 = v[perm[0]];
    c2 = v[perm[1]];
    c3 = v[perm[2]];
}

template <int BN, int PASSES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, const GemmArgs g) {
    using Cfg = GemmCfg<BN, PASSES>;
    constexpr int NPL = Cfg::NPL;
    constexpr int STAGES = Cfg::STAGES;

    extern __shared__ uint8_t smem_dyn[];
    uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int num_kb = (g.K + 63) >> 6;
    // persistent tile loop: tile id -> (z, m block, n block), n fastest so concurrently running CTAs share the A tile in L2
    const int tiles_n = (g.N + BN - 1) / BN;
    const int tiles_m = (g.M + 127) >> 7;
    const long long num_tiles = (long long)tiles_n * tiles_m * g.Z;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmAh);
        tma_prefetch_desc(&tmBh);
        if (NPL == 2) {
            tma_prefetch_desc(&tmAl);
            tma_prefetch_desc(&tmBl);
        }
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);                        // one arrival per consumer warpgroup
        }
        fence_mbar_init();
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlapped the tail of the
    // previous kernel in the stream; its outputs (our operands / residual) are visible after the wait.
    pdl_trigger();
    pdl_wait();

    if (warp == 8) {
        // ------------------------------------------------ TMA producer
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int nb = (int)(tile % tiles_n);
                const int mb = (int)((tile / tiles_n) % tiles_m);
                const int z = (int)(tile / ((long long)tiles_n * tiles_m));
                int a1, a2, a3, b1, b2, b3;
                pick_coords(g.permA, mb * 128, z % g.H, z / g.H, a1, a2, a3);
                pick_coords(g.permB, nb * BN, z % g.H, z / g.H, b1, b2, b3);
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait_mma(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE);
                    uint8_t* s = tiles + (size_t)stage * Cfg::STAGE;
                    const int k0 = kb * 64;
                    tma_load_4d(s, &tmAh, &full_bar[stage], k0, a1, a2, a3);
                    if (NPL == 2) tma_load_4d(s + Cfg::A_TILE, &tmAl, &full_bar[stage], k0, a1, a2, a3);
                    tma_load_4d(s + NPL * Cfg::A_TILE, &tmBh, &full_bar[stage], k0, b1, b2, b3);
                    if (NPL == 2) tma_load_4d(s + NPL * Cfg::A_TILE + Cfg::B_TILE, &tmBl, &full_bar[stage], k0, b1, b2, b3);
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        __syncwarp();
        return;
    }
    // ---------------------------------------------------- consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile
    const int wg = warp >> 2;
    const uint32_t a_row_off = (uint32_t)wg * 64u * 128u;      // 8 swizzle atoms of 1024 B
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int frag_col = 2 * (lane & 3);
    const bool out_vec = ((g.ld_out | g.out_h | g.out_b) & 1) == 0 && (reinterpret_cast<uintptr_t>(g.out_f32) & 7) == 0;
    const bool res_vec = ((g.ld_res | g.res_h | g.res_b) & 1) == 0 && (reinterpret_cast<uintptr_t>(g.res) & 7) == 0;
    const bool bias_vec = (reinterpret_cast<uintptr_t>(g.bias) & 7) == 0;
    int stage = 0;
    uint32_t phase = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev_stage = -1;
        uint32_t accum = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait_mma(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(tiles + (size_t)stage * Cfg::STAGE);
            const uint32_t a_hi = sa + a_row_off, a_lo = a_hi + Cfg::A_TILE;
            const uint32_t b_hi = sa + NPL * Cfg::A_TILE, b_lo = b_hi + Cfg::B_TILE;
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < PASSES; ++pass) {
                // pass 0: hi*hi, pass 1: hi*lo, pass 2: lo*hi
                const uint32_t pa = (pass == 2) ? a_lo : a_hi;
                const uint32_t pb = (pass == 1) ? b_lo : b_hi;
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4) {               // 4 x (K = 16 fp16 = 32 B) per 128 B swizzle row
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
        if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);

        // ------------------------------------------------ epilogue from the accumulator fragments
        const int nbk = (int)(tile % tiles_n);
        const int mbk = (int)((tile / tiles_n) % tiles_m);
        const int z = (int)(tile / ((long long)tiles_n * tiles_m));
        const int n0 = nbk * BN + frag_col, h = z % g.H, b = z / g.H;
        const long long zo = (long long)b * g.out_b + (long long)h * g.out_h;
        const long long zr = (long long)b * g.res_b + (long long)h * g.res_h;
#pragma unroll
        for (int half = 0; half < 2; ++half) {                 // fragment rows r and r + 8
            const int m = mbk * 128 + frag_row + half * 8;
            if (m >= g.M) continue;
            float bias_row = 0.f;
            if (g.bias != nullptr && g.bias_per_row) bias_row = __ldg(g.bias + m);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = n0 + 8 * j;
                if (n >= g.N) break;
                const bool two = n + 1 < g.N;
                float v0 = acc[4 * j + 2 * half] * g.alpha, v1 = acc[4 * j + 2 * half + 1] * g.alpha;
                if (g.bias != nullptr) {
                    if (g.bias_per_row) {
                        v0 += bias_row;
                        v1 += bias_row;
                    } else if (two && bias_vec) {
                        const float2 bv = __ldg(reinterpret_cast<const float2*>(g.bias + n));
                        v0 += bv.x;
                        v1 += bv.y;
                    } else {
                        v0 += __ldg(g.bias + n);
                        if (two) v1 += __ldg(g.bias + n + 1);
                    }
                }
                if (g.act == STB_ACT_GELU) {
                    v0 = gelu_erf(v0);
                    v1 = gelu_erf(v1);
                }
                if (g.res != nullptr) {
                    const float* rp = g.res + zr + (long long)m * g.ld_res + n;
                    if (two && res_vec) {
                        const float2 rv = *reinterpret_cast<const float2*>(rp);
                        v0 += rv.x;
                        v1 += rv.y;
                    } else {
                        v0 += rp[0];
                        if (two) v1 += rp[1];
                    }
                }
                __half h0, l0, h1, l1;
                if (g.out_hi != nullptr) {
                    split_f16(v0, h0, l0);
                    split_f16(v1, h1, l1);
                }
                if (!g.transposed) {
                    const long long off = zo + (long long)m * g.ld_out + n;
                    if (g.out_f32 != nullptr) {
                        if (two && out_vec) {
                            *reinterpret_cast<float2*>(g.out_f32 + off) = make_float2(v0, v1);
                        } else {
                            g.out_f32[off] = v0;
                            if (two) g.out_f32[off + 1] = v1;
                        }
                    }
                    if (g.out_hi != nullptr) {
                        g.out_hi[off] = h0;
                        if (two) g.out_hi[off + 1] = h1;
                        if (g.out_lo != nullptr) {
                            g.out_lo[off] = l0;
                            if (two) g.out_lo[off + 1] = l1;
                        }
                    }
                } else {
                    // transposed store: the 8 row-lanes of a fragment column hit 8 consecutive addresses
                    const long long off = zo + (long long)n * g.ld_out + m;
                    if (g.out_f32 != nullptr) {
                        g.out_f32[off] = v0;
                        if (two) g.out_f32[off + g.ld_out] = v1;
                    }
                    if (g.out_hi != nullptr) {
                        g.out_hi[off] = h0;
                        if (two) g.out_hi[off + g.ld_out] = h1;
                        if (g.out_lo != nullptr) {
                            g.out_lo[off] = l0;
                            if (two) g.out_lo[off + g.ld_out] = l1;
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// host side: tensor maps (cached) + launch
// ---------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

struct TmapKey {
    const void* base;
    int rows, k, H, B, box_rows;
    long long rs, hs, bs;
    bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        const uint64_t* p = reinterpret_cast<const uint64_t*>(&k);
        uint64_t h = 1469598103934665603ull;
        for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) h = (h ^ p[i]) * 1099511628211ull;
        return (size_t)h;
    }
};
static_assert(sizeof(TmapKey) % 8 == 0, "TmapKey must be a multiple of 8 bytes");

static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, TmapVal, TmapKeyHash> g_tmap_cache;

// 4-D fp16 tensor map over one plane: inner dim = k (contiguous), then (row, head, batch) ordered by increasing stride.
int make_tmap(const void* base, int rows, int k, int H, int B, long long rs, long long hs, long long bs, int box_rows,
              TmapVal* out) {
    TmapKey key;
    memset(&key, 0, sizeof(key));
    key.base = base; key.rows = rows; key.k = k; key.H = H; key.B = B; key.box_rows = box_rows;
    key.rs = rs; key.hs = hs; key.bs = bs;
    {
        std::lock_guard<std::mutex> lk(g_tmap_mu);
        auto it = g_tmap_cache.find(key);
        if (it != g_tmap_cache.end()) {
            *out = it->second;
            return STB_OK;
        }
    }
    EncodeTiledFn enc = get_encode_fn();
    STB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
    STB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer must be 16-byte aligned");
    struct D { unsigned long long size, stride; int id; };
    D d[3] = {{(unsigned long long)rows, (unsigned long long)rs * 2, 0},
              {(unsigned long long)H, (unsigned long long)hs * 2, 1},
              {(unsigned long long)B, (unsigned long long)bs * 2, 2}};
    for (int i = 1; i < 3; ++i)
        if (d[i].stride == 0 || d[i].size == 1) {   // broadcast (e.g. weights shared by every batch item) or degenerate
            d[i].size = 1;
            d[i].id = 3;
        }
    // sort by stride ascending; size-1 dims go last (their stride is irrelevant and is rewritten below)
    for (int i = 0; i < 3; ++i)
        for (int j = i + 1; j < 3; ++j) {
            const bool i_last = d[i].size == 1, j_last = d[j].size == 1;
            const bool swap = (i_last && !j_last) || (i_last == j_last && d[j].stride < d[i].stride);
            if (swap) { D t = d[i]; d[i] = d[j]; d[j] = t; }
        }
    unsigned long long prev = 128;   // harmless stride for degenerate dims
    for (int i = 0; i < 3; ++i) {
        if (d[i].size == 1) d[i].stride = prev;
        STB_REQUIRE(d[i].stride % 16 == 0 && d[i].stride > 0, "TMA stride %llu (dim %d) must be a positive multiple of 16 B",
                    d[i].stride, d[i].id);
        prev = d[i].stride * d[i].size;
        if (prev % 16) prev = (prev + 15) / 16 * 16;
    }
    cuuint64_t gdim[4] = {(cuuint64_t)k, d[0].size, d[1].size, d[2].size};
    cuuint64_t gstr[3] = {d[0].stride, d[1].stride, d[2].stride};
    cuuint32_t box[4] = {64, 1, 1, 1};
    for (int i = 0; i < 3; ++i)
        if (d[i].id == 0) box[1 + i] = (cuuint32_t)box_rows;
    cuuint32_t estr[4] = {1, 1, 1, 1};
    TmapVal v;
    CUresult r = enc(&v.map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    STB_REQUIRE(r == CUDA_SUCCESS,
                "cuTensorMapEncodeTiled failed (%d): dims {%llu,%llu,%llu,%llu} strides {%llu,%llu,%llu} box rows %d",
                (int)r, (unsigned long long)gdim[0], (unsigned long long)gdim[1], (unsigned long long)gdim[2],
                (unsigned long long)gdim[3], (unsigned long long)gstr[0], (unsigned long long)gstr[1],
                (unsigned long long)gstr[2], box_rows);
    for (int i = 0; i < 3; ++i) v.perm[i] = d[i].id;
    {
        std::lock_guard<std::mutex> lk(g_tmap_mu);
        // keyed by raw pointers: a long-lived process that keeps allocating new buffers would grow it without bound
        if (g_tmap_cache.size() >= 16384) g_tmap_cache.clear();
        g_tmap_cache.emplace(key, v);
    }
    *out = v;
    return STB_OK;
}

template <int BN, int PASSES>
static int launch_gemm(const TmapVal& ah, const TmapVal& al, const TmapVal& bh, const TmapVal& bl, GemmArgs& g,
                       int n_batch, cudaStream_t st) {
    using Cfg = GemmCfg<BN, PASSES>;
    for (int i = 0; i < 3; ++i) {
        g.permA[i] = ah.perm[i];
        g.permB[i] = bh.perm[i];
    }
    g.Z = n_batch * g.H;
    const long long num_tiles = (long long)cdiv(g.N, BN) * cdiv(g.M, 128) * g.Z;
    dim3 grid((unsigned)(num_tiles < sm_count() ? num_tiles : sm_count()));     // persistent: one CTA per SM
    // algorithmic FLOPs of ONE fp32-grade GEMM (not x PASSES); bytes: operands once + output once
    const double zz = (double)n_batch * g.H;
    ProfScope ps("gemm_tc", st, zz * ((double)g.M * g.K + (double)g.N * g.K) * 2.0 * Cfg::NPL + zz * (double)g.M * g.N * 4.0,
                 2.0 * g.M * (double)g.N * g.K * zz);
    return launch(gemm_tc_kernel<BN, PASSES>, {grid, dim3(GEMM_THREADS), (size_t)Cfg::SMEM, st, /*pdl=*/true}, ah.map, al.map,
                  bh.map, bl.map, g);
}

int gemm(const stb_operand& A, const stb_operand& B, int n_batch, int n_head, const stb_epilogue& ep, cudaStream_t st) {
    STB_REQUIRE(A.k == B.k, "gemm: K mismatch %d vs %d", A.k, B.k);
    STB_REQUIRE(A.hi && B.hi, "gemm: hi planes are required");
    STB_REQUIRE((A.lo != nullptr) == (B.lo != nullptr), "gemm: lo planes must be given for both operands or neither");
    STB_REQUIRE(ep.out_f32 || ep.out_hi, "gemm: no output");
    const int passes = A.lo ? 3 : 1;
    const int N = B.rows;
    // 128 x 128 is the widest tile: its accumulator is 64 registers per consumer thread, and three ring stages of the
    // four split-fp16 planes (64 KB each) fit the 227 KB of shared memory
    int BN = N <= 16 ? 16 : N <= 32 ? 32 : N <= 64 ? 64 : 128;
    if (A.rows <= 128 && n_batch * n_head == 1) {
        // decode-step shape (M = batch of sequences): HBM-bound on the weights; use narrow N tiles so that enough CTAs
        // (~80 % of the SMs or more) stream them concurrently
        while (BN > 16 && cdiv(N, BN) < (sm_count() * 4) / 5) BN >>= 1;
    }
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = A.rows; g.N = N; g.K = A.k; g.H = n_head;
    g.out_f32 = ep.out_f32; g.out_hi = (__half*)ep.out_hi; g.out_lo = (__half*)ep.out_lo;
    g.ld_out = ep.ld_out; g.out_h = ep.out_h_stride; g.out_b = ep.out_b_stride; g.transposed = ep.transposed;
    g.bias = ep.bias; g.bias_per_row = ep.bias_per_row;
    g.res = ep.residual; g.ld_res = ep.ld_res; g.res_h = ep.res_h_stride; g.res_b = ep.res_b_stride;
    g.alpha = ep.alpha; g.act = ep.act;
    TmapVal ah, al, bh, bl;
    STB_TRY(make_tmap(A.hi, A.rows, A.k, n_head, n_batch, A.row_stride, A.h_stride, A.b_stride, 128, &ah));
    STB_TRY(make_tmap(B.hi, B.rows, B.k, n_head, n_batch, B.row_stride, B.h_stride, B.b_stride, BN, &bh));
    if (passes == 3) {
        STB_TRY(make_tmap(A.lo, A.rows, A.k, n_head, n_batch, A.row_stride, A.h_stride, A.b_stride, 128, &al));
        STB_TRY(make_tmap(B.lo, B.rows, B.k, n_head, n_batch, B.row_stride, B.h_stride, B.b_stride, BN, &bl));
    } else {
        al = ah;
        bl = bh;
    }
#define STB_GEMM_CASE(bn)                                                                   \
    case bn:                                                                                \
        return passes == 3 ? launch_gemm<bn, 3>(ah, al, bh, bl, g, n_batch, st)             \
                           : launch_gemm<bn, 1>(ah, al, bh, bl, g, n_batch, st);
    switch (BN) {
        STB_GEMM_CASE(16)
        STB_GEMM_CASE(32)
        STB_GEMM_CASE(64)
        STB_GEMM_CASE(128)
    }
#undef STB_GEMM_CASE
    return STB_ERR_UNSUPPORTED;
}

}  // namespace stb

extern "C" int stb_gemm(const stb_operand* A, const stb_operand* B, int n_batch, int n_head, const stb_epilogue* ep,
                        void* stream) {
    STB_REQUIRE(A && B && ep, "stb_gemm: null argument");
    return stb::gemm(*A, *B, n_batch, n_head, *ep, (cudaStream_t)stream);
}
