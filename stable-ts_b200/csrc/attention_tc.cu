// K4: fused multi-head attention for sm_90a -- softmax(q k^T / 8) v with the scores and probabilities kept in registers;
// nothing but q, k, v^T and the output touches HBM.
//
// Replaces MultiHeadAttention.qkv_attention of whisper.model for the encoder's 1500 x 1500 self-attention
// (reached from stable_whisper/timing.py:60 / decode.py:29).
//
// One CTA = one (batch, head, 128-query tile); 9 warps:
//   warps 0..3, 4..7  two consumer warpgroups of 64 query rows each: wgmma for both products, softmax in between
//   warp 8            TMA producer: Q tile once, K tiles through a 2-stage ring (twice: pass 1 and pass 2), V^T tiles (pass 2)
//
// Exact two-pass softmax (same formula as the reference: exp(s - max) / sum), no accumulator rescaling:
//   pass 1   S_t = Q K_t^T  (wgmma m64n128k16, operands in swizzled shared memory)  ->  row max m
//   pass 2   S_t again      ->  p = exp(s - m)  ->  split fp16 (hi, lo): the accumulator fragment of 16 keys IS the A
//            fragment of the next product, so P never leaves the registers  ->  O += P_t V_t  (wgmma m64n64k16, A from
//            registers, V^T from shared memory), row sum l applied to O in the epilogue
// Split precision as in the GEMM core: every product is hi*hi + hi*lo + lo*hi (3 MMA passes), fp32 accumulation.
#include "common.cuh"
#include "kernels.h"

namespace stb {

constexpr int AT_BQ = 128;       // queries per CTA
constexpr int AT_BK = 128;       // keys per tile
constexpr int AT_THREADS = 288;

struct AttnArgs {
    int Mq, Mk, H;
    int permQ[3], permK[3], permV[3];
    __half* out_hi;
    __half* out_lo;
    long long ld_out, out_h, out_b;
};

template <int PASSES>
struct AttnCfg {
    static constexpr int NPL = PASSES == 3 ? 2 : 1;
    static constexpr uint32_t Q_TILE = AT_BQ * 128;                 // 16 KB: 128 rows x 128 B
    static constexpr uint32_t K_TILE = AT_BK * 128;                 // 16 KB
    static constexpr uint32_t V_CHUNK = 64 * 128;                   // 8 KB: 64 head dims x 64 keys
    static constexpr uint32_t OFF_Q = 0;
    static constexpr uint32_t OFF_K = OFF_Q + NPL * Q_TILE;         // 2 stages x NPL x K_TILE
    static constexpr uint32_t OFF_V = OFF_K + 2 * NPL * K_TILE;     // 2 stages x NPL x 2 chunks
    static constexpr uint32_t SMEM = OFF_V + 2 * NPL * 2 * V_CHUNK + 1024;
};

__device__ __forceinline__ void pick3(const int (&perm)[3], int row, int h, int b, int& c1, int& c2, int& c3) {
    int v[4] = {row, h, b, 0};
    c1 = v[perm[0]];
    c2 = v[perm[1]];
    c3 = v[perm[2]];
}

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

template <int PASSES>
__global__ void __launch_bounds__(AT_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
                    const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
                    const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl, const AttnArgs g) {
    using Cfg = AttnCfg<PASSES>;
    constexpr int NPL = Cfg::NPL;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t q_full, k_full[2], k_empty[2], v_full[2], v_empty[2];

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AT_BQ;
    const int h = blockIdx.y, b = blockIdx.z;
    const int NT = (g.Mk + AT_BK - 1) / AT_BK;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmQh); tma_prefetch_desc(&tmKh); tma_prefetch_desc(&tmVh);
        if (NPL == 2) { tma_prefetch_desc(&tmQl); tma_prefetch_desc(&tmKl); tma_prefetch_desc(&tmVl); }
        mbar_init(&q_full, 1);
        for (int i = 0; i < 2; ++i) {                            // "empty": one arrival per consumer warpgroup
            mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 2);
            mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 2);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        // =========================================================== TMA producer
        if (lane == 0) {
            int c1, c2, c3;
            pick3(g.permQ, q0, h, b, c1, c2, c3);
            mbar_arrive_expect_tx(&q_full, NPL * Cfg::Q_TILE);
            tma_load_4d(sm + Cfg::OFF_Q, &tmQh, &q_full, 0, c1, c2, c3);
            if (NPL == 2) tma_load_4d(sm + Cfg::OFF_Q + Cfg::Q_TILE, &tmQl, &q_full, 0, c1, c2, c3);
            for (int i = 0; i < 2 * NT; ++i) {
                const int t = i % NT, st = i & 1;
                const uint32_t ph = (i >> 1) & 1;
                mbar_wait_mma(&k_empty[st], ph ^ 1);
                mbar_arrive_expect_tx(&k_full[st], NPL * Cfg::K_TILE);
                pick3(g.permK, t * AT_BK, h, b, c1, c2, c3);
                uint8_t* kd = sm + Cfg::OFF_K + st * NPL * Cfg::K_TILE;
                tma_load_4d(kd, &tmKh, &k_full[st], 0, c1, c2, c3);
                if (NPL == 2) tma_load_4d(kd + Cfg::K_TILE, &tmKl, &k_full[st], 0, c1, c2, c3);
                if (i >= NT) {                                   // pass 2: the V^T tile of the same keys
                    const int vs = t & 1;
                    const uint32_t vph = (t >> 1) & 1;
                    mbar_wait_mma(&v_empty[vs], vph ^ 1);
                    mbar_arrive_expect_tx(&v_full[vs], NPL * 2 * Cfg::V_CHUNK);
                    pick3(g.permV, 0, h, b, c1, c2, c3);
                    uint8_t* vd = sm + Cfg::OFF_V + vs * NPL * 2 * Cfg::V_CHUNK;
                    tma_load_4d(vd, &tmVh, &v_full[vs], t * AT_BK, c1, c2, c3);
                    tma_load_4d(vd + Cfg::V_CHUNK, &tmVh, &v_full[vs], t * AT_BK + 64, c1, c2, c3);
                    if (NPL == 2) {
                        tma_load_4d(vd + 2 * Cfg::V_CHUNK, &tmVl, &v_full[vs], t * AT_BK, c1, c2, c3);
                        tma_load_4d(vd + 3 * Cfg::V_CHUNK, &tmVl, &v_full[vs], t * AT_BK + 64, c1, c2, c3);
                    }
                }
            }
        }
        return;
    }
    // =============================================================== consumers: warpgroup wg owns 64 query rows.  A thread
    // holds two rows of the score fragment (r and r + 8), each shared with the 3 other lanes of its quad.
    const int wg = warp >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment row r inside the CTA's query tile
    const int colq = 2 * (lane & 3);
    const uint32_t q_hi = smem_u32(sm + Cfg::OFF_Q) + (uint32_t)wg * 64u * 128u, q_lo = q_hi + Cfg::Q_TILE;
    constexpr float LOG2E = 1.4426950408889634f;
    const float sc = 0.125f * LOG2E;                           // scores in log2 units: exp(x) = exp2(x * log2e)
    mbar_wait_mma(&q_full, 0);

    float s[64];
    // S = Q K_t^T for K ring use i (64 x 128 per warpgroup), then the K slot is released
    auto scores = [&](int i) {
        const int st = i & 1;
        mbar_wait_mma(&k_full[st], (i >> 1) & 1);
        const uint32_t k_hi = smem_u32(sm + Cfg::OFF_K + st * NPL * Cfg::K_TILE), k_lo = k_hi + Cfg::K_TILE;
        uint32_t accum = 0;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < PASSES; ++pass) {
            const uint32_t pa = (pass == 2) ? q_lo : q_hi;
            const uint32_t pb = (pass == 1) ? k_lo : k_hi;
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
                wgmma_ss(s, wgmma_desc_k128(pa + k4 * 32), wgmma_desc_k128(pb + k4 * 32), accum);
                accum = 1;
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (leader) mbar_arrive(&k_empty[st]);
    };

    // ---------------- pass 1: row max only (the sum is accumulated in pass 2 and applied to O in the epilogue:
    // softmax(s) v == (sum_j exp(s_j - m) v_j) / (sum_j exp(s_j - m)))
    float m0 = -INFINITY, m1 = -INFINITY;
    for (int t = 0; t < NT; ++t) {
        scores(t);
        const int kbase = t * AT_BK + colq;
        const bool full_tile = (t + 1) * AT_BK <= g.Mk;        // warp-uniform: no per-element key masking needed
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (full_tile || kbase + 8 * j + e < g.Mk) {
                    m0 = fmaxf(m0, s[4 * j + e]);
                    m1 = fmaxf(m1, s[4 * j + 2 + e]);
                }
            }
        }
    }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2)) * sc;  // row max in log2 units
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2)) * sc;

    // ---------------- pass 2: S again -> p = exp(s - m) -> split fp16 (hi, lo) A fragments in registers -> O += P_t V_t
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float l0 = 0.f, l1 = 0.f;
    uint32_t o_accum = 0;
    for (int t = 0; t < NT; ++t) {
        scores(NT + t);
        const int kbase = t * AT_BK + colq;
        const bool full_tile = (t + 1) * AT_BK <= g.Mk;
        // the score fragment of 16 keys (two 8-column groups) is exactly the m64k16 A fragment of the same rows
        uint32_t p_hi[8][4], p_lo[8][4];
#pragma unroll
        for (int kc = 0; kc < 8; ++kc) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {                        // q = 2 (column group within the chunk) + (row r + 8 ?)
                const int j = 2 * kc + (q >> 1);
                float pv[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float mrow = (q & 1) ? m1 : m0;
                    float pe = exp2f(fmaf(s[4 * j + 2 * (q & 1) + e], sc, -mrow));
                    if (!full_tile && kbase + 8 * j + e >= g.Mk) pe = 0.f;
                    pv[e] = pe;
                }
                if (q & 1) l1 += pv[0] + pv[1]; else l0 += pv[0] + pv[1];
                __half h0, lo0, h1, lo1;
                split_f16(pv[0], h0, lo0);
                split_f16(pv[1], h1, lo1);
                p_hi[kc][q] = pack_h2(h0, h1);
                p_lo[kc][q] = pack_h2(lo0, lo1);
            }
        }
        const int vs = t & 1;
        mbar_wait_mma(&v_full[vs], (t >> 1) & 1);
        const uint32_t v_base = smem_u32(sm + Cfg::OFF_V + vs * NPL * 2 * Cfg::V_CHUNK);
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < PASSES; ++pass) {
            const uint32_t pb = v_base + ((pass == 1) ? 2 * Cfg::V_CHUNK : 0);
#pragma unroll
            for (int kc = 0; kc < 8; ++kc) {                     // 128 keys = 2 chunks x 4 k-steps of 16
                const uint64_t vd = wgmma_desc_k128(pb + (kc >> 2) * Cfg::V_CHUNK + (kc & 3) * 32);
                if (pass == 2) wgmma_rs(o, p_lo[kc], vd, o_accum); else wgmma_rs(o, p_hi[kc], vd, o_accum);
                o_accum = 1;
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (leader) mbar_arrive(&v_empty[vs]);
    }
    // ---------------- epilogue: O / l -> split fp16 -> attention output
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int qrow = q0 + row + half * 8;
        if (qrow >= g.Mq) continue;
        const float inv_l = 1.0f / (half ? l1 : l0);
        const long long off = (long long)b * g.out_b + (long long)h * g.out_h + (long long)qrow * g.ld_out + colq;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            __half h0, lo0, h1, lo1;
            split_f16(o[4 * j + 2 * half] * inv_l, h0, lo0);
            split_f16(o[4 * j + 2 * half + 1] * inv_l, h1, lo1);
            *reinterpret_cast<uint32_t*>(g.out_hi + off + 8 * j) = pack_h2(h0, h1);
            if (g.out_lo != nullptr) *reinterpret_cast<uint32_t*>(g.out_lo + off + 8 * j) = pack_h2(lo0, lo1);
        }
    }
}

template <int PASSES>
static int launch_attention(const TmapVal (&tm)[6], AttnArgs& g, int n_batch, cudaStream_t st) {
    using Cfg = AttnCfg<PASSES>;
    dim3 grid(cdiv(g.Mq, AT_BQ), g.H, n_batch);
    const double zz = (double)n_batch * g.H;
    ProfScope ps("attention_tc", st, zz * ((double)g.Mq * 64 + 2.0 * g.Mk * 64) * 2.0 * Cfg::NPL + zz * g.Mq * 64.0 * 2.0 * Cfg::NPL,
                 zz * 4.0 * g.Mq * (double)g.Mk * 64);
    return launch(attention_tc_kernel<PASSES>, {grid, AT_THREADS, Cfg::SMEM, st}, tm[0].map, tm[1].map, tm[2].map, tm[3].map,
                  tm[4].map, tm[5].map, g);
}

// q: rows Mq, k = 64; k: rows Mk, k = 64; vT: rows 64, k = keys (>= Mk, zero padded); out split [..][ld_out].
int fused_attention(const stb_operand& q, const stb_operand& k, const stb_operand& vT, int n_batch, int n_head, int Mq, int Mk,
                    void* out_hi, void* out_lo, long long ld_out, long long out_h, long long out_b, cudaStream_t st) {
    STB_REQUIRE(q.k == 64 && k.k == 64 && vT.rows == 64, "fused_attention: head_dim must be 64");
    STB_REQUIRE((q.lo != nullptr) == (k.lo != nullptr) && (q.lo != nullptr) == (vT.lo != nullptr),
                "fused_attention: lo planes must be given for all operands or none");
    STB_REQUIRE((ld_out & 7) == 0, "fused_attention: ld_out must be a multiple of 8");
    const bool lo = q.lo != nullptr;
    TmapVal tm[6];
    STB_TRY(make_tmap(q.hi, Mq, 64, n_head, n_batch, q.row_stride, q.h_stride, q.b_stride, AT_BQ, &tm[0]));
    STB_TRY(make_tmap(k.hi, Mk, 64, n_head, n_batch, k.row_stride, k.h_stride, k.b_stride, AT_BK, &tm[2]));
    STB_TRY(make_tmap(vT.hi, 64, vT.k, n_head, n_batch, vT.row_stride, vT.h_stride, vT.b_stride, 64, &tm[4]));
    if (lo) {
        STB_TRY(make_tmap(q.lo, Mq, 64, n_head, n_batch, q.row_stride, q.h_stride, q.b_stride, AT_BQ, &tm[1]));
        STB_TRY(make_tmap(k.lo, Mk, 64, n_head, n_batch, k.row_stride, k.h_stride, k.b_stride, AT_BK, &tm[3]));
        STB_TRY(make_tmap(vT.lo, 64, vT.k, n_head, n_batch, vT.row_stride, vT.h_stride, vT.b_stride, 64, &tm[5]));
    } else {
        tm[1] = tm[0]; tm[3] = tm[2]; tm[5] = tm[4];
    }
    AttnArgs g;
    g.Mq = Mq; g.Mk = Mk; g.H = n_head;
    for (int i = 0; i < 3; ++i) { g.permQ[i] = tm[0].perm[i]; g.permK[i] = tm[2].perm[i]; g.permV[i] = tm[4].perm[i]; }
    g.out_hi = (__half*)out_hi; g.out_lo = (__half*)out_lo; g.ld_out = ld_out; g.out_h = out_h; g.out_b = out_b;
    return lo ? launch_attention<3>(tm, g, n_batch, st) : launch_attention<1>(tm, g, n_batch, st);
}

}  // namespace stb

extern "C" int stb_attention(const stb_operand* q, const stb_operand* k, const stb_operand* vT, int n_batch, int n_head, int Mq,
                             int Mk, void* out_hi, void* out_lo, long long ld_out, long long out_h_stride,
                             long long out_b_stride, void* stream) {
    STB_REQUIRE(q && k && vT && out_hi && n_batch >= 1 && n_head >= 1 && Mq >= 1 && Mk >= 1, "stb_attention: bad arguments");
    return stb::fused_attention(*q, *k, *vT, n_batch, n_head, Mq, Mk, out_hi, out_lo, ld_out, out_h_stride, out_b_stride,
                                (cudaStream_t)stream);
}
