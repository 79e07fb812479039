// K4: fused multi-head attention for sm_90a -- softmax(q k^T / 8) v with the scores and probabilities kept in registers;
// nothing but q, k, v^T and the output touches HBM.
//
// Replaces MultiHeadAttention.qkv_attention of whisper.model for the encoder's 1500 x 1500 self-attention
// (reached from stable_whisper/timing.py:60 / decode.py:29) and for the teacher-forced decoder's cross-attention
// (engine.cu).  Scores a caller captures come from a GEMM of their own.
//
// One CTA = one (batch, head, 128-query tile); 9 warps:
//   warps 0..3, 4..7  two consumer warpgroups of 64 query rows each: wgmma for both products, softmax in between
//   warp 8            TMA producer: Q tile once, then every 64-key K tile and V^T tile once, through a 4-stage K ring and
//                     a 4-stage V^T ring that advance together
// Registers bound the key tile: a consumer thread holds S_t, P_{t-1} (hi and lo), O and the Q fragments at once.  Under
// __launch_bounds__(288, 1) ptxas gives this kernel at most 168 registers per thread (65536 / 384, as if the producer warp
// were a whole warpgroup); so did a 384-thread variant whose producer warpgroup handed registers over by setmaxnreg.  At
// that limit 128-key tiles use 168 registers, spill 240 bytes and serialise the wgmma; 64-key tiles take 154 registers
// (122 with PASSES = 1) and do not spill.
//
// One pass with an online softmax, in base-2 units (the 1/8 log2(e) scale folded into the exponent):
//   S_t = Q K_t^T  (wgmma m64n64k16, Q from registers, K from swizzled shared memory)
//   m' = max(m, rowmax S_t);  p = exp2(s - m');  l = l exp2(m - m') + rowsum p;  O = O exp2(m - m') + P_t V_t
//   P_t is split fp16 (hi, lo): the accumulator fragment of 16 keys IS the A fragment of the next product, so P never leaves
//   the registers (wgmma m64n64k16, A from registers, V^T from shared memory); O / l in the epilogue.
// Overlap: a warpgroup issues S_t = Q K_t^T and O += P_{t-1} V_{t-1} together and computes the softmax of S_t while P.V
// still runs; the two warpgroups take turns to issue (named barriers), so one's softmax runs under the other's MMAs.
// Split precision as in the GEMM core: every product is hi*hi + hi*lo + lo*hi (3 MMA passes), fp32 accumulation.
#include "common.cuh"
#include "kernels.h"

namespace stb {

constexpr int AT_BQ = 128;       // queries per CTA
constexpr int AT_BK = 64;        // keys per tile
constexpr int AT_STAGES = 4;     // K and V^T ring depth
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
    static constexpr uint32_t K_TILE = AT_BK * 128;                 // 8 KB: 64 keys x 64 head dims
    static constexpr uint32_t V_TILE = 64 * AT_BK * 2;              // 8 KB: 64 head dims x 64 keys
    static constexpr uint32_t OFF_Q = 0;
    static constexpr uint32_t OFF_K = OFF_Q + NPL * Q_TILE;         // stages x NPL x K_TILE
    static constexpr uint32_t OFF_V = OFF_K + AT_STAGES * NPL * K_TILE;
    static constexpr uint32_t SMEM = OFF_V + AT_STAGES * NPL * V_TILE + 1024;
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

// named barriers 1 and 2 (0 is __syncthreads) between the two consumer warpgroups
template <int ID>
__device__ __forceinline__ void named_bar_sync() { asm volatile("bar.sync %0, 256;" ::"n"(ID) : "memory"); }
template <int ID>
__device__ __forceinline__ void named_bar_arrive() { asm volatile("bar.arrive %0, 256;" ::"n"(ID) : "memory"); }

// keeps the compiler from moving reads or writes of a wgmma accumulator across the wgmma_wait that makes it valid
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
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
    __shared__ __align__(8) uint64_t q_full, k_full[AT_STAGES], k_empty[AT_STAGES], v_full[AT_STAGES], v_empty[AT_STAGES];

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AT_BQ;
    const int h = blockIdx.y, b = blockIdx.z;
    const int NT = (g.Mk + AT_BK - 1) / AT_BK;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmQh); tma_prefetch_desc(&tmKh); tma_prefetch_desc(&tmVh);
        if (NPL == 2) { tma_prefetch_desc(&tmQl); tma_prefetch_desc(&tmKl); tma_prefetch_desc(&tmVl); }
        mbar_init(&q_full, 1);
        for (int i = 0; i < AT_STAGES; ++i) {                    // "empty": one arrival per consumer warpgroup
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
            for (int t = 0; t < NT; ++t) {
                const int st = t % AT_STAGES;
                const uint32_t ph = (t / AT_STAGES) & 1;
                mbar_wait_mma(&k_empty[st], ph ^ 1);
                mbar_arrive_expect_tx(&k_full[st], NPL * Cfg::K_TILE);
                pick3(g.permK, t * AT_BK, h, b, c1, c2, c3);
                uint8_t* kd = sm + Cfg::OFF_K + st * NPL * Cfg::K_TILE;
                tma_load_4d(kd, &tmKh, &k_full[st], 0, c1, c2, c3);
                if (NPL == 2) tma_load_4d(kd + Cfg::K_TILE, &tmKl, &k_full[st], 0, c1, c2, c3);
                mbar_wait_mma(&v_empty[st], ph ^ 1);                 // the V^T tile of the same keys
                mbar_arrive_expect_tx(&v_full[st], NPL * Cfg::V_TILE);
                pick3(g.permV, 0, h, b, c1, c2, c3);
                uint8_t* vd = sm + Cfg::OFF_V + st * NPL * Cfg::V_TILE;
                tma_load_4d(vd, &tmVh, &v_full[st], t * AT_BK, c1, c2, c3);
                if (NPL == 2) tma_load_4d(vd + Cfg::V_TILE, &tmVl, &v_full[st], t * AT_BK, c1, c2, c3);
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
    constexpr float LOG2E = 1.4426950408889634f;
    const float sc = 0.125f * LOG2E;                           // scores in log2 units: exp(x) = exp2(x * log2e)

    // Issue turns alternate between the warpgroups, warpgroup 0 first: a warpgroup waits on its own barrier before it
    // issues and arrives on the other's after.  Both make NT + 1 turns; warpgroup 1's initial arrival stands in for its
    // last one, so every barrier phase is completed.
    if (wg == 1) named_bar_arrive<1>();
    int turn = 0;
    auto turn_begin = [&] {
        if (wg == 0) named_bar_sync<1>(); else named_bar_sync<2>();
        wgmma_fence();
    };
    auto turn_end = [&] {
        if (wg == 0) named_bar_arrive<2>(); else if (++turn <= NT) named_bar_arrive<1>();
    };

    float s[32];                                               // S_t, then exp2(s - m) in place
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    uint32_t p_hi[4][4], p_lo[4][4];                           // P_{t-1}: the A fragments of the P.V product in flight
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    mbar_wait_mma(&q_full, 0);
    // Q as m64k16 A fragments in registers (loaded once from the swizzled tile), so that Q K^T reads only K from shared
    // memory: with both operands there, a 64-key product would need all of the SM's shared-memory bandwidth
    uint32_t qa[NPL][4][4];
#pragma unroll
    for (int pl = 0; pl < NPL; ++pl)
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4)
#pragma unroll
            for (int i = 0; i < 4; ++i) {                        // i = 2 (k + 8 ?) + (row r + 8 ?)
                const int rr = row + 8 * (i & 1), cb = 2 * (16 * k4 + 8 * (i >> 1) + colq);   // byte column in the row
                qa[pl][k4][i] = *reinterpret_cast<const uint32_t*>(sm + Cfg::OFF_Q + pl * Cfg::Q_TILE + rr * 128 +
                                                                    ((((cb >> 4) ^ (rr & 7))) << 4) + (cb & 15));
            }
    auto issue_scores = [&](int t) {                           // S = Q K_t^T (64 x 64 per warpgroup)
        const uint32_t k_hi = smem_u32(sm + Cfg::OFF_K + (t % AT_STAGES) * NPL * Cfg::K_TILE), k_lo = k_hi + Cfg::K_TILE;
#pragma unroll
        for (int pass = 0; pass < PASSES; ++pass) {
            const uint32_t pb = (pass == 1) ? k_lo : k_hi;
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4)
                wgmma_rs(s, qa[pass == 2 ? NPL - 1 : 0][k4], wgmma_desc_k128(pb + k4 * 32), pass + k4 > 0);
        }
        wgmma_commit();
    };
    auto issue_pv = [&](int t) {                               // O += P_t V_t
        const uint32_t v_base = smem_u32(sm + Cfg::OFF_V + (t % AT_STAGES) * NPL * Cfg::V_TILE);
#pragma unroll
        for (int pass = 0; pass < PASSES; ++pass) {
            const uint32_t pb = v_base + ((pass == 1) ? Cfg::V_TILE : 0);
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) {                     // 64 keys = 4 k-steps of 16
                const uint64_t vd = wgmma_desc_k128(pb + kc * 32);
                if (pass == 2) wgmma_rs(o, p_lo[kc], vd, 1); else wgmma_rs(o, p_hi[kc], vd, 1);
            }
        }
        wgmma_commit();
    };
    // the new row maxima from S_t, p = exp2(s - m) in place, l rescaled and summed; returns the O rescale factors
    auto softmax = [&](int t, float& a0, float& a1) {
        fence_regs(s);
        if ((t + 1) * AT_BK > g.Mk) {                          // the partial last tile: keys past Mk do not exist
            const int kbase = t * AT_BK + colq;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (kbase + 8 * j + e >= g.Mk) s[4 * j + e] = s[4 * j + 2 + e] = -INFINITY;
        }
        float x0 = -INFINITY, x1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            x0 = fmaxf(x0, fmaxf(s[4 * j], s[4 * j + 1]));
            x1 = fmaxf(x1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
        }
        x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1));
        x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
        const float n0 = fmaxf(m0, x0 * sc), n1 = fmaxf(m1, x1 * sc);   // finite: every tile has a key
        a0 = exp2f(m0 - n0);                                   // 0 on the first tile (m = -inf)
        a1 = exp2f(m1 - n1);
        m0 = n0;
        m1 = n1;
        float r0 = 0.f, r1 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                s[4 * j + e] = exp2f(fmaf(s[4 * j + e], sc, -n0));
                s[4 * j + 2 + e] = exp2f(fmaf(s[4 * j + 2 + e], sc, -n1));
                r0 += s[4 * j + e];
                r1 += s[4 * j + 2 + e];
            }
        }
        l0 = fmaf(l0, a0, r0);
        l1 = fmaf(l1, a1, r1);
    };
    // P_t = split fp16 of s: the score fragment of 16 keys (two 8-column groups) is exactly the m64k16 A fragment
    auto split_p = [&] {
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {                        // q = 2 (column group within the chunk) + (row r + 8 ?)
                const int i = 4 * (2 * kc + (q >> 1)) + 2 * (q & 1);
                __half h0, lo0, h1, lo1;
                split_f16(s[i], h0, lo0);
                split_f16(s[i + 1], h1, lo1);
                p_hi[kc][q] = pack_h2(h0, h1);
                p_lo[kc][q] = pack_h2(lo0, lo1);
            }
        }
    };
    auto rescale_o = [&](float a0, float a1) {
        fence_regs(o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[4 * j] *= a0; o[4 * j + 1] *= a0;
            o[4 * j + 2] *= a1; o[4 * j + 3] *= a1;
        }
    };

    float a0, a1;
    auto full = [&](uint64_t* bars, int t) { mbar_wait_mma(&bars[t % AT_STAGES], (t / AT_STAGES) & 1); };
    auto release = [&](uint64_t* bars, int t) { if (leader) mbar_arrive(&bars[t % AT_STAGES]); };
    full(k_full, 0);
    turn_begin();
    issue_scores(0);
    turn_end();
    wgmma_wait<0>();
    release(k_empty, 0);
    softmax(0, a0, a1);                                        // O is still zero: no rescale
    split_p();
    for (int t = 1; t < NT; ++t) {
        full(k_full, t);
        full(v_full, t - 1);
        turn_begin();
        issue_scores(t);
        issue_pv(t - 1);
        turn_end();
        wgmma_wait<1>();                                       // S_t is ready; P_{t-1} V_{t-1} may still run
        release(k_empty, t);
        softmax(t, a0, a1);
        wgmma_wait<0>();
        release(v_empty, t - 1);
        rescale_o(a0, a1);
        split_p();
    }
    full(v_full, NT - 1);
    turn_begin();
    issue_pv(NT - 1);
    turn_end();
    wgmma_wait<0>();
    fence_regs(o);

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
