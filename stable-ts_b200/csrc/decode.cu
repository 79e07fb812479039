// a9 / K10: KV-cached autoregressive decode step (stable_whisper/decode.py:33-65 -> whisper PyTorchInference.logits with
// kv-cache hooks, the logit filters, GreedyDecoder.update).
//
//   stb_decode_step     one decoder forward for the newest token of B sequences (engine.cu: decode_step).  Linear layers:
//                       mma.sync batched GEMV (gemv.cu) up to 16 sequences, the cluster split-K wgmma kernel of
//                       decode_linear.cu up to 128.  Attention over the caches is in this file, flash-decoding style: the
//                       cross-attention (HBM-bound by the fp16 cross K/V, the largest stream of a step) on ldmatrix +
//                       mma.sync over TMA-swizzled tiles, the self-attention over the fp32 cache on scalar lanes.
//   stb_sample          SuppressBlank / SuppressTokens / ApplyTimestampRules / silent-timestamp mask / argmax or inverse-CDF
//                       draw / log-prob accumulation / EOT latching fused into one kernel per step, state kept on the device.
//
// Everything position-dependent is read from a DEVICE counter (`pos`), so one captured CUDA graph replays every step.
#include <float.h>

#include "common.cuh"
#include "kernels.h"

namespace stb {

// softmax in base 2: exp(x) = 2^(x log2 e); q is pre-scaled by log2 e, so every exponential of the attention kernels is one
// exp2f (MUFU.EX2 + range fix-up) instead of expf's multiply + range reduction, executed per key by all 8 lanes of a group
constexpr float LOG2E_F = 1.4426950408889634f;

// ---------------------------------------------------------------------------------------------------------
// self-attention over the fp32 K/V cache.  grid (H, B), 128 threads.
//   qkv [B][3d] fp32 (q | k | v of the newest token); caches Kc, Vc [B][ctx][d] fp32; out split [B][d].
// (With an fp16 cache the step logits against the fp32 oracle move from 2e-5 to 2e-4 -- few keys, peaky weights: V's
//  rounding reaches the output unaveraged -- so the cache stays fp32.)
__global__ void __launch_bounds__(128)
decode_self_attn_kernel(const float* __restrict__ qkv, float* __restrict__ Kc, float* __restrict__ Vc, int d, int ctx,
                        const int32_t* __restrict__ pos_ptr, const int32_t* __restrict__ seq_off, __half* __restrict__ out_hi,
                        __half* __restrict__ out_lo, float* __restrict__ out_f32) {
    __shared__ float s_m[4][4], s_l[4][4];
    __shared__ float s_acc[4][4][64];
    const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int w = tid >> 5, lane = tid & 31;
    const int sub = lane & 7, grp = lane >> 3;
    pdl_trigger();
    pdl_wait();
    const int pos = *pos_ptr;
    const int n = pos + 1;
    // ragged initial tokens (prompts of different lengths in one batch) are RIGHT-aligned on the shared position counter:
    // sequence b's own tokens occupy cache rows [seq_off[b], pos]; earlier rows hold idle steps and are never attended
    const int first_row = seq_off != nullptr ? min(seq_off[b], pos) : 0;
    const float* row = qkv + (long long)b * 3 * d;
    float* kc = Kc + (long long)b * ctx * d + h * 64;
    float* vc = Vc + (long long)b * ctx * d + h * 64;
    if (tid < 64) kc[(long long)pos * d + tid] = row[d + h * 64 + tid];
    else vc[(long long)pos * d + (tid - 64)] = row[2 * d + h * 64 + (tid - 64)];
    float qr[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) qr[e] = row[h * 64 + sub * 8 + e] * (0.125f * LOG2E_F);   // scores in log2 units: exp2f below
    __syncthreads();                                         // the newest K / V row is visible to the whole CTA
    float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int base = first_row; base < n; base += 64) {       // block-uniform trip count: 64 keys per CTA iteration
        const int j0 = base + w * 4 + grp;
        float4 ka[4], kb[4], va[4], vb[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int j = j0 + u * 16;
            ka[u] = kb[u] = va[u] = vb[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j < n) {
                const float4* kr = reinterpret_cast<const float4*>(kc + (long long)j * d + sub * 8);
                const float4* vr = reinterpret_cast<const float4*>(vc + (long long)j * d + sub * 8);
                ka[u] = kr[0]; kb[u] = kr[1];
                va[u] = vr[0]; vb[u] = vr[1];
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int j = j0 + u * 16;
            float s = qr[0] * ka[u].x;
            s = fmaf(qr[1], ka[u].y, s); s = fmaf(qr[2], ka[u].z, s); s = fmaf(qr[3], ka[u].w, s);
            s = fmaf(qr[4], kb[u].x, s); s = fmaf(qr[5], kb[u].y, s); s = fmaf(qr[6], kb[u].z, s); s = fmaf(qr[7], kb[u].w, s);
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            if (j < n) {                                      // uniform within the 8-lane group
                const float mn = fmaxf(m, s);
                const float corr = exp2f(m - mn);              // exp(-inf) = 0 on the first key
                const float p = exp2f(s - mn);
                l = l * corr + p;
                acc[0] = fmaf(p, va[u].x, acc[0] * corr); acc[1] = fmaf(p, va[u].y, acc[1] * corr);
                acc[2] = fmaf(p, va[u].z, acc[2] * corr); acc[3] = fmaf(p, va[u].w, acc[3] * corr);
                acc[4] = fmaf(p, vb[u].x, acc[4] * corr); acc[5] = fmaf(p, vb[u].y, acc[5] * corr);
                acc[6] = fmaf(p, vb[u].z, acc[6] * corr); acc[7] = fmaf(p, vb[u].w, acc[7] * corr);
                m = mn;
            }
        }
    }
    // ---- merge the 16 lane groups ----
    if (sub == 0) { s_m[w][grp] = m; s_l[w][grp] = l; }
#pragma unroll
    for (int e = 0; e < 8; ++e) s_acc[w][grp][sub * 8 + e] = acc[e];
    __syncthreads();
    if (tid < 64) {
        float M = -INFINITY;
#pragma unroll
        for (int i = 0; i < 16; ++i) M = fmaxf(M, s_m[i >> 2][i & 3]);
        float Lsum = 0.f, o = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float mi = s_m[i >> 2][i & 3];
            const float sc = (mi == -INFINITY) ? 0.f : exp2f(mi - M);
            Lsum += s_l[i >> 2][i & 3] * sc;
            o += s_acc[i >> 2][i & 3][tid] * sc;
        }
        o /= Lsum;
        if (out_f32) out_f32[(long long)b * d + h * 64 + tid] = o;
        if (out_hi) {
            __half hi, lo;
            split_f16(o, hi, lo);
            out_hi[(long long)b * d + h * 64 + tid] = hi;
            if (out_lo) out_lo[(long long)b * d + h * 64 + tid] = lo;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// cross-attention of one new token per sequence over the per-window K and V, head-major fp16 [B][H][T][64]: every
// (sequence, head) is a pair of contiguous 192 KB streams.  HBM-bound: 2 x 1500 x 128 B = 384 KB per (sequence, head) per
// step.  The decode step reads the fp16 `hi` plane only -- K is the GEMM plane itself, V a head-major copy written once
// per window batch.  Measured at 32 layers against the fp32 oracle (tests/test_gpu_depth.py): worst step-logit error
// 2.15e-5 with fp16 K/V vs 2.07e-5 with a 3-byte hi + int8-residual format (gate 1e-3), greedy tokens bit-exact -- the
// residual bought nothing measurable, so its 35 % of extra bytes were dropped.
//
// Flash-decoding layout: grid (XS, H, B); the keys of one (b,h) are cut into XS splits of XT_CHUNKS x XT_KEYS = 192 keys
// (8 x 192 = 1536 >= 1500).  One CTA (4 warps) owns one split: an elected thread issues the split's K and V tiles as TMA
// copies BEFORE waiting on the producer of q (programmatic dependent launch: the K/V stream does not depend on it).  Each
// CTA writes its partial (m, l, acc[64]) -- 66 floats at partial[((b H + h) XS + split) 66] -- and the last CTA of a (b,h)
// to finish (atomic ticket on tickets[b H + h], re-armed to 0 for the next launch) merges the XS partials and writes the
// output.  The arithmetic runs on the warp-level tensor cores; one query row costs ~150 warp instructions per 192 keys:
//   * K and V tiles [96 keys][64] fp16 land through 2-D TMA copies with SWIZZLE_128B (zero fill past the last key), so
//     ldmatrix reads them without bank conflicts;
//   * scores: mma.sync m16n8k16, A = the query in rows 0 / 1 (fp16 hi / lo of q * log2(e) / 8: the fp32 query is
//     represented to 2^-22), B = 8 keys per tile straight from ldmatrix; row 0 + row 1 = the fp32-grade score;
//   * one exact softmax per CTA (max over its 192 keys through shared memory);
//   * P.V: mma.sync m16n8k8 per 8-key tile, A = p in rows 0 / 1 (hi / lo), B = V through ldmatrix.trans.
// Warp w owns tiles w, w + 4, w + 8 of each 12-tile chunk.
// (Not a persistent, double-buffered kernel: a per-item fence + ticket + barriers serialise inside a CTA, whereas 4
//  short-lived CTAs per SM overlap each other's tails.)
// ---------------------------------------------------------------------------------------------------------
constexpr int XS = 8;                        // key splits per (sequence, head)
constexpr int XT_KEYS = 96;                  // keys per chunk
constexpr int XT_CHUNKS = 2;                 // chunks per split: 8 x 192 = 1536 >= 1500
constexpr int XT_TILES = XT_KEYS / 8 / 4;    // 8-key tiles per warp per chunk
constexpr int XT_SMEM = XT_CHUNKS * 2 * XT_KEYS * 128 + 1024;

struct XPerm { int p[3]; };

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void mma_16816(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_1688(float (&c)[4], uint32_t a0, uint32_t b0) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(0u), "r"(b0));
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    __half2 h = __halves2half2(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(128, 4)
decode_cross_attn_tc_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, const XPerm perm,
                            const float* __restrict__ q, int d, int T, float* __restrict__ partial, int* __restrict__ tickets,
                            __half* __restrict__ out_hi, __half* __restrict__ out_lo, float* __restrict__ out_f32) {
    extern __shared__ uint8_t xt_dyn[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(xt_dyn) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t s_bar[XT_CHUNKS];
    __shared__ float s_m[4], s_l[4];
    __shared__ float s_acc[4][64];
    __shared__ int s_last;
    const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z, H = gridDim.y;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int key0 = split * (XT_CHUNKS * XT_KEYS);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
#pragma unroll
        for (int c = 0; c < XT_CHUNKS; ++c) mbar_init(&s_bar[c], 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int c = 0; c < XT_CHUNKS; ++c) {
            int v[4] = {key0 + c * XT_KEYS, h, b, 0};
            uint8_t* dst = sm + (size_t)c * 2 * XT_KEYS * 128;
            mbar_arrive_expect_tx(&s_bar[c], 2u * XT_KEYS * 128u);       // the box is always transferred whole (zero fill past T)
            tma_load_4d(dst, &tmK, &s_bar[c], 0, v[perm.p[0]], v[perm.p[1]], v[perm.p[2]]);
            tma_load_4d(dst + XT_KEYS * 128, &tmV, &s_bar[c], 0, v[perm.p[0]], v[perm.p[1]], v[perm.p[2]]);
        }
    }
    pdl_trigger();
    pdl_wait();                                              // q comes from the preceding linear
    // ---- query fragments: rows 0 / 1 of A hold the fp16 hi / lo parts of q * log2(e) / 8, every other row is zero
    uint32_t qa0[4], qa2[4];
    {
        const float* qp = q + (long long)b * d + h * 64;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            __half hv[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int idx = ks * 16 + 2 * t + (e & 1) + (e >> 1) * 8;
                const float x = qp[idx] * (0.125f * LOG2E_F);
                __half hi, lo;
                split_f16(x, hi, lo);
                hv[e] = g == 0 ? hi : (g == 1 ? lo : __float2half(0.f));
            }
            qa0[ks] = pack_h2(hv[0], hv[1]);
            qa2[ks] = pack_h2(hv[2], hv[3]);
        }
    }
    const uint32_t sm_base = smem_u32(sm);
    const int mrow = lane & 7, mat = lane >> 3;              // ldmatrix: this lane addresses row `mrow` of matrix `mat`
    // ---- scores of this warp's 6 tiles (lanes 0..3 end up with the two keys 2t, 2t + 1 of each tile)
    float sc[XT_CHUNKS * XT_TILES][2];
#pragma unroll
    for (int c = 0; c < XT_CHUNKS; ++c) {
        mbar_wait(&s_bar[c], 0, 40 + c);
        const uint32_t kbase = sm_base + (uint32_t)(c * 2 * XT_KEYS * 128);
#pragma unroll
        for (int i = 0; i < XT_TILES; ++i) {
            const int r0 = (w + 4 * i) * 8;
            const int row = r0 + mrow;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int half = 0; half < 2; ++half) {            // dims 0..31, 32..63: four 16-byte chunks each
                uint32_t r[4];
                ldsm_x4(r, kbase + (uint32_t)(row * 128) + (uint32_t)((((half * 4 + mat) ^ (row & 7)) << 4)));
                mma_16816(acc, qa0[half * 2], qa2[half * 2], r[0], r[1]);
                mma_16816(acc, qa0[half * 2 + 1], qa2[half * 2 + 1], r[2], r[3]);
            }
            // row 0 (lanes 0..3) + row 1 (lanes 4..7): hi and lo parts of the query
            const float s0 = acc[0] + __shfl_down_sync(0xffffffffu, acc[0], 4);
            const float s1 = acc[1] + __shfl_down_sync(0xffffffffu, acc[1], 4);
            const int key = key0 + c * XT_KEYS + r0 + 2 * t;
            sc[c * XT_TILES + i][0] = (g == 0 && key < T) ? s0 : -INFINITY;
            sc[c * XT_TILES + i][1] = (g == 0 && key + 1 < T) ? s1 : -INFINITY;
        }
    }
    // ---- exact softmax over the CTA's keys
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < XT_CHUNKS * XT_TILES; ++i) m = fmaxf(m, fmaxf(sc[i][0], sc[i][1]));
    m = warp_max(m);
    if (lane == 0) s_m[w] = m;
    __syncthreads();
    const float M = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
    float l = 0.f;
    float oacc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) { oacc[nt][0] = oacc[nt][1] = oacc[nt][2] = oacc[nt][3] = 0.f; }
#pragma unroll
    for (int c = 0; c < XT_CHUNKS; ++c) {
        const uint32_t vbase = sm_base + (uint32_t)(c * 2 * XT_KEYS * 128 + XT_KEYS * 128);
#pragma unroll
        for (int i = 0; i < XT_TILES; ++i) {
            const float p0 = (M == -INFINITY) ? 0.f : exp2f(sc[c * XT_TILES + i][0] - M);   // 0 for lanes / keys without a score
            const float p1 = (M == -INFINITY) ? 0.f : exp2f(sc[c * XT_TILES + i][1] - M);
            l += p0 + p1;
            __half h0, l0, h1, l1;
            split_f16(p0, h0, l0);
            split_f16(p1, h1, l1);
            const uint32_t hi = pack_h2(h0, h1), lo = pack_h2(l0, l1);
            const uint32_t lo_up = __shfl_up_sync(0xffffffffu, lo, 4);   // row 1 (lanes 4..7) carries the lo parts
            const uint32_t a0 = g == 0 ? hi : (g == 1 ? lo_up : 0u);
            const int r0 = (w + 4 * i) * 8;
            const int row = r0 + mrow;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                uint32_t r[4];
                ldsm_x4_t(r, vbase + (uint32_t)(row * 128) + (uint32_t)((((half * 4 + mat) ^ (row & 7)) << 4)));
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_1688(oacc[half * 4 + j], a0, r[j]);
            }
        }
    }
    // ---- per warp: row 0 + row 1 of every n-tile -> 64 output dims in lanes 0..3; then the 4 warps through shared memory
    l = warp_sum(l);
    if (lane == 0) s_l[w] = l;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        const float o0 = oacc[nt][0] + __shfl_down_sync(0xffffffffu, oacc[nt][0], 4);
        const float o1 = oacc[nt][1] + __shfl_down_sync(0xffffffffu, oacc[nt][1], 4);
        if (g == 0) {
            s_acc[w][nt * 8 + 2 * t] = o0;
            s_acc[w][nt * 8 + 2 * t + 1] = o1;
        }
    }
    __syncthreads();
    float* part = partial + (((long long)b * H + h) * XS + split) * 66;
    if (threadIdx.x < 64) {
        part[2 + threadIdx.x] = (s_acc[0][threadIdx.x] + s_acc[1][threadIdx.x]) + (s_acc[2][threadIdx.x] + s_acc[3][threadIdx.x]);
        if (threadIdx.x == 0) { part[0] = M; part[1] = (s_l[0] + s_l[1]) + (s_l[2] + s_l[3]); }
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int tk = atomicAdd(tickets + b * H + h, 1);
        s_last = (tk == XS - 1);
        if (s_last) tickets[b * H + h] = 0;                  // re-arm for the next launch
    }
    __syncthreads();
    if (s_last && threadIdx.x < 64) {
        __threadfence();
        const float* p0 = partial + ((long long)b * H + h) * XS * 66;
        float Mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < XS; ++i) Mx = fmaxf(Mx, __ldcg(p0 + i * 66));
        float Lsum = 0.f, o = 0.f;
#pragma unroll
        for (int i = 0; i < XS; ++i) {
            const float mi = __ldcg(p0 + i * 66);
            const float scl = (mi == -INFINITY) ? 0.f : exp2f(mi - Mx);
            Lsum += __ldcg(p0 + i * 66 + 1) * scl;
            o += __ldcg(p0 + i * 66 + 2 + threadIdx.x) * scl;
        }
        o /= Lsum;
        const long long oo = (long long)b * d + h * 64 + threadIdx.x;
        if (out_f32) out_f32[oo] = o;
        if (out_hi) {
            __half hi, lo;
            split_f16(o, hi, lo);
            out_hi[oo] = hi;
            if (out_lo) out_lo[oo] = lo;
        }
    }
}

// V^T plane [B][H][64][Tp] fp16 -> V head-major [B][H][T][64] (decode-step layout).  64 x 64 smem tile transpose.
__global__ void __launch_bounds__(256) v_headmajor_kernel(const __half* __restrict__ vT_hi, int T, int Tp,
                                                          __half* __restrict__ v_hi) {
    __shared__ __half tile[64][72];
    const long long bh = blockIdx.y;
    const int t0 = blockIdx.x * 64;
    for (int i = threadIdx.x; i < 64 * 64; i += 256) {
        const int c = i >> 6, t = i & 63;
        tile[c][t] = (t0 + t < T) ? vT_hi[(bh * 64 + c) * Tp + t0 + t] : __float2half(0.f);
    }
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int t = w; t < 64; t += 8) {                        // one warp per key row, two channels per lane
        if (t0 + t >= T) break;
        const long long row = bh * T + t0 + t;
        reinterpret_cast<__half2*>(v_hi + row * 64)[lane] = __halves2half2(tile[2 * lane][t], tile[2 * lane + 1][t]);
    }
}

__global__ void embed_step_kernel(const int32_t* __restrict__ tokens, const int32_t* __restrict__ pos_ptr,
                                  const int32_t* __restrict__ seq_off, int n_pos, int d, const float* __restrict__ emb,
                                  const float* __restrict__ posemb, float* __restrict__ x) {
    const int b = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    int pos = *pos_ptr;
    if (seq_off != nullptr) pos = max(pos - seq_off[b], 0);  // the sequence's own position (idle steps before it: row 0)
    pos = min(pos, n_pos - 1);                               // a sequence past its n_ctx stop idles on the last row
    const float4* e = reinterpret_cast<const float4*>(emb + (long long)tokens[b] * d);
    const float4* p = reinterpret_cast<const float4*>(posemb + (long long)pos * d);
    float4* o = reinterpret_cast<float4*>(x + (long long)b * d);
    for (int i = threadIdx.x; i < (d >> 2); i += blockDim.x) {
        const float4 a = __ldg(e + i), c = __ldg(p + i);
        o[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
    }
}

// ---------------------------------------------------------------------------------------------------------
// fused logit filters + greedy pick.  One CTA (1024 threads) per sequence.
// ---------------------------------------------------------------------------------------------------------
struct BlockRed {
    float f[32];
    int i[32];
};

__device__ __forceinline__ float block_max(float v, BlockRed& r) {
    v = warp_max(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) r.f[threadIdx.x >> 5] = v;
    __syncthreads();
    float m = r.f[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fmaxf(m, r.f[k]);
    return m;
}
__device__ __forceinline__ float block_sum(float v, BlockRed& r) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) r.f[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += r.f[k];
    return s;
}

__global__ void __launch_bounds__(1024)
sample_greedy_kernel(float* __restrict__ logits, long long ld, int V, int eot, int ts_begin, int no_timestamps,
                     const uint8_t* __restrict__ suppress, const uint8_t* __restrict__ first_mask,
                     const uint8_t* __restrict__ ts_mask, long long ts_mask_stride, int max_initial_ts, int apply_ts_rules,
                     const int32_t* __restrict__ forced_table, stb_seq_state* __restrict__ states,
                     int32_t* __restrict__ next_out, int32_t* __restrict__ token_table, int32_t* __restrict__ argmax_table,
                     int table_rows, float temperature, const float* __restrict__ uniform_table,
                     const int32_t* __restrict__ sample_cap) {
    __shared__ BlockRed red;
    const int b = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    float* l = logits + (long long)b * ld;
    if (ts_mask) ts_mask += (long long)b * ts_mask_stride;   // stride 0: one mask for the batch; else one row per sequence
    stb_seq_state st = states[b];
    const bool first = st.n_sampled == 0;
    const bool last_ts = st.n_sampled >= 1 && st.last_tok >= ts_begin;
    const bool penult_ts = st.n_sampled < 2 || st.prev_tok >= ts_begin;
    int ts_floor = -1;                                      // timestamps below this id are forbidden
    if (apply_ts_rules && st.last_ts >= 0) ts_floor = (last_ts && !penult_ts) ? st.last_ts : st.last_ts + 1;
    // ---- pass 1: SuppressBlank / SuppressTokens / ApplyTimestampRules masks; max over text / timestamp ranges
    float mx_text = -INFINITY, mx_ts = -INFINITY;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        float v = l[i];
        bool kill = (suppress && suppress[i]) || (first && first_mask && first_mask[i]);
        if (apply_ts_rules) {
            if (i == no_timestamps) kill = true;
            if (last_ts) {
                if (penult_ts) { if (i >= ts_begin) kill = true; }      // pair complete -> text next
                else { if (i < eot) kill = true; }                      // open pair -> timestamp / EOT next
            }
            if (i >= ts_begin && i < ts_floor) kill = true;
            if (first) {
                if (i < ts_begin) kill = true;
                if (max_initial_ts >= 0 && i > ts_begin + max_initial_ts) kill = true;
            }
        }
        if (kill) v = -INFINITY;
        l[i] = v;
        if (i < ts_begin) mx_text = fmaxf(mx_text, v); else mx_ts = fmaxf(mx_ts, v);
    }
    mx_text = block_max(mx_text, red);
    mx_ts = block_max(mx_ts, red);
    bool kill_text = false;
    if (apply_ts_rules && mx_ts > -INFINITY) {              // logsumexp over timestamps vs best text logit
        float s = 0.f;                                      // (evaluated BEFORE the silent-timestamp mask, as the
        for (int i = ts_begin + threadIdx.x; i < V; i += blockDim.x) s += expf(l[i] - mx_ts);   //  reference does)
        s = block_sum(s, red);
        kill_text = (mx_ts + logf(s)) > mx_text;
    }
    __syncthreads();
    // ---- pass 2: timestamp-vs-text rule, silent-timestamp mask (decode.py:14-16,53), nan_to_num_(-inf); final max
    float gmax = -INFINITY;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        float v = l[i];
        if (kill_text && i < ts_begin) v = -INFINITY;
        if (ts_mask && i >= ts_begin && ts_mask[i - ts_begin]) v = -INFINITY;
        // logits.nan_to_num_(-inf) (decode.py:55): NaN -> -inf, while -inf / +inf become the lowest / greatest finite
        // float -- so a fully masked row degenerates to a uniform distribution (argmax = index 0), not to NaN
        if (v != v) v = -INFINITY;
        else v = fminf(fmaxf(v, -FLT_MAX), FLT_MAX);
        l[i] = v;
        gmax = fmaxf(gmax, v);
    }
    gmax = block_max(gmax, red);
    __syncthreads();
    // ---- pass 3: argmax (first index on ties) + logsumexp of the final logits
    float s = 0.f;
    int arg = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        const float v = l[i];
        s += expf(v - gmax);
        if (v == gmax && i < arg) arg = i;
    }
    s = block_sum(s, red);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) arg = min(arg, __shfl_xor_sync(0xffffffffu, arg, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red.i[threadIdx.x >> 5] = arg;
    __syncthreads();
    // ---- temperature > 0 (GreedyDecoder.update: Categorical(logits / T).sample()): inverse-CDF draw from
    // p_i ~ exp((l_i - max) / T) with the caller's uniform u in [0, 1) for this (step, sequence): the first index whose
    // running sum exceeds u * total.  Every thread owns a CONTIGUOUS index range, so the block scan follows index order.
    int pick = 0x7fffffff;
    if (temperature > 0.f && uniform_table != nullptr && st.n_sampled < table_rows) {
        // running sums in fp64: a token's share (~1e-5 of the total for flat distributions) must stay far above the
        // rounding of the sum, or the draw would depend on the summation order
        __shared__ double dsum[32];
        const float inv_t = 1.f / temperature;
        const int chunk = (V + (int)blockDim.x - 1) / (int)blockDim.x;
        const int i0 = min((int)threadIdx.x * chunk, V), i1 = min(i0 + chunk, V);
        double cs = 0.0;
        for (int i = i0; i < i1; ++i) cs += (double)expf((l[i] - gmax) * inv_t);
        double inc = cs;                                      // inclusive scan inside the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double v = __shfl_up_sync(0xffffffffu, inc, o);
            if ((int)(threadIdx.x & 31) >= o) inc += v;
        }
        if ((threadIdx.x & 31) == 31) dsum[threadIdx.x >> 5] = inc;
        __syncthreads();
        double before = 0.0, total = 0.0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
            if (k < (int)(threadIdx.x >> 5)) before += dsum[k];
            total += dsum[k];
        }
        const double target = (double)uniform_table[(long long)st.n_sampled * gridDim.x + b] * total;
        double run = before + (inc - cs);                     // sum of everything before this thread's range
        if (target < run + cs) {
            for (int i = i0; i < i1; ++i) {
                run += (double)expf((l[i] - gmax) * inv_t);
                if (run > target) { pick = i; break; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) pick = min(pick, __shfl_xor_sync(0xffffffffu, pick, o));
        __syncthreads();
        if ((threadIdx.x & 31) == 0) red.f[threadIdx.x >> 5] = __int_as_float(pick);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int a = red.i[0];
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) a = min(a, red.i[k]);
        int drawn = a;                                        // temperature 0: the argmax
        if (temperature > 0.f && uniform_table != nullptr && st.n_sampled < table_rows) {
            int pk = 0x7fffffff;
            for (int k = 0; k < (int)(blockDim.x >> 5); ++k) pk = min(pk, __float_as_int(red.f[k]));
            if (pk < V) drawn = pk;                           // (rounding left u * total >= every running sum: keep the argmax)
        }
        const float log_s = logf(s);                          // lse = gmax + log_s; kept apart: gmax may be -FLT_MAX
        // ended: EOT sampled earlier, or the per-sequence cap reached (the reference's `tokens.shape[-1] > n_ctx` stop for a
        // sequence whose initial tokens are longer than its neighbours')
        const bool was_done = (st.n_sampled >= 1 && st.last_tok == eot) || (sample_cap != nullptr && st.n_sampled >= sample_cap[b]);
        int next = drawn;
        const int B = gridDim.x;
        const bool in_table = st.n_sampled < table_rows;
        if (argmax_table && in_table) argmax_table[(long long)st.n_sampled * B + b] = a;
        // GreedyDecoder.update accumulates the log-prob (log_softmax of the UNSCALED logits) of ITS pick (the argmax, or the
        // draw at temperature > 0); a forced script (benchmarks, tests) only replaces the token that is appended afterwards,
        // exactly as oracle/stable_path.py:decode_window does
        const float lp = (l[drawn] - gmax) - log_s;
        if (forced_table && in_table) next = forced_table[(long long)st.n_sampled * B + b];
        if (!was_done) st.sum_logprob += lp;
        if (was_done) next = eot;                           // finished rows keep emitting EOT
        if (token_table && in_table) token_table[(long long)st.n_sampled * B + b] = next;
        st.prev_tok = st.last_tok;
        st.last_tok = next;
        if (next >= ts_begin) st.last_ts = next;
        st.n_sampled += 1;
        st.done = next == eot;
        states[b] = st;
        next_out[b] = next;
    }
}

__global__ void bump_pos_kernel(int32_t* pos) {
    pdl_trigger();
    pdl_wait();
    *pos += 1;
}

}  // namespace stb

extern "C" int stb_sample(float* logits, long long ld, int B, int V, int eot, int ts_begin, int no_timestamps,
                          const uint8_t* suppress_mask, const uint8_t* first_step_mask, const uint8_t* ts_mask,
                          long long ts_mask_stride, int max_initial_ts, int apply_ts_rules, const int32_t* forced_table,
                          stb_seq_state* states, int32_t* next_out, int32_t* token_table, int32_t* argmax_table, int table_rows,
                          float temperature, const float* uniform_table, const int32_t* sample_cap, void* stream) {
    STB_REQUIRE(logits && states && next_out && B >= 1 && V >= 1 && ld >= V, "stb_sample: bad arguments");
    STB_REQUIRE(ts_mask_stride == 0 || ts_mask_stride >= 1501, "stb_sample: ts_mask_stride must be 0 (shared) or >= 1501");
    STB_REQUIRE(temperature >= 0.f && (temperature == 0.f || uniform_table != nullptr),
                "stb_sample: temperature > 0 needs the table of uniform draws [table_rows][B]");
    stb::ProfScope ps("sample_greedy", (cudaStream_t)stream, (double)B * V * 4.0 * 3);
    return stb::launch(stb::sample_greedy_kernel, {dim3(B), dim3(1024), 0, (cudaStream_t)stream, /*pdl=*/true}, logits, ld, V, eot,
                       ts_begin, no_timestamps, suppress_mask, first_step_mask, ts_mask, ts_mask_stride, max_initial_ts, apply_ts_rules,
                       forced_table, states, next_out, token_table, argmax_table, table_rows, temperature, uniform_table, sample_cap);
}

extern "C" int stb_sample_greedy(float* logits, long long ld, int B, int V, int eot, int ts_begin, int no_timestamps,
                                 const uint8_t* suppress_mask, const uint8_t* first_step_mask, const uint8_t* ts_mask,
                                 long long ts_mask_stride, int max_initial_ts, int apply_ts_rules, const int32_t* forced_table, stb_seq_state* states,
                                 int32_t* next_out, int32_t* token_table, int32_t* argmax_table, int table_rows, void* stream) {
    return stb_sample(logits, ld, B, V, eot, ts_begin, no_timestamps, suppress_mask, first_step_mask, ts_mask, ts_mask_stride,
                      max_initial_ts, apply_ts_rules, forced_table, states, next_out, token_table, argmax_table, table_rows, 0.f,
                      nullptr, nullptr, stream);
}

namespace stb {
int decode_attn_self(const float* qkv, float* Kc, float* Vc, int B, int H, int d, int ctx, const int32_t* pos,
                     const int32_t* seq_off, __half* oh, __half* ol, float* of, cudaStream_t st) {
    ProfScope ps("decode_self_attn", st);
    return launch(decode_self_attn_kernel, {dim3(H, B), dim3(128), 0, st, /*pdl=*/true}, qkv, Kc, Vc, d, ctx, pos, seq_off, oh, ol, of);
}
int decode_attn_cross(const float* q, const CrossDecodeKV& kv, int B, int H, int d, float* partial, int* tickets, __half* oh,
                      __half* ol, float* of, cudaStream_t st) {
    ProfScope ps("decode_cross_attn", st, (double)B * H * 2.0 * STB_N_AUDIO_CTX * 64 * 2.0);
    const int T = (int)STB_N_AUDIO_CTX;
    TmapVal tk, tv;
    STB_TRY(make_tmap(kv.k_hi, T, 64, H, B, 64, (long long)T * 64, (long long)H * T * 64, XT_KEYS, &tk));
    STB_TRY(make_tmap(kv.v_hi, T, 64, H, B, 64, (long long)T * 64, (long long)H * T * 64, XT_KEYS, &tv));
    XPerm perm;
    for (int i = 0; i < 3; ++i) {
        STB_REQUIRE(tk.perm[i] == tv.perm[i], "decode_attn_cross: K / V tensor maps disagree");
        perm.p[i] = tk.perm[i];
    }
    return launch(decode_cross_attn_tc_kernel,
                  {dim3(XS, H, B), dim3(128), (size_t)XT_SMEM, st, /*pdl=*/true, /*cluster=*/0, /*max_carveout=*/true}, tk.map, tv.map,
                  perm, q, d, T, partial, tickets, oh, ol, of);
}
int decode_cross_splits() { return XS; }
int v_headmajor(const __half* vT_hi, int BH, int T, int Tp, __half* v_hi, cudaStream_t st) {
    ProfScope ps("v_headmajor", st, (double)BH * T * 64 * 4.0);
    return launch(v_headmajor_kernel, {dim3(cdiv(T, 64), BH), 256, 0, st}, vT_hi, T, Tp, v_hi);
}
int embed_step(const int32_t* tokens, const int32_t* pos, const int32_t* seq_off, int n_pos, int B, int d, const float* emb,
               const float* posemb, float* x, cudaStream_t st) {
    return launch(embed_step_kernel, {dim3(B), dim3(128), 0, st, /*pdl=*/true}, tokens, pos, seq_off, n_pos, d, emb, posemb, x);
}
int bump_pos(int32_t* pos, cudaStream_t st) {
    return launch(bump_pos_kernel, {dim3(1), dim3(1), 0, st, /*pdl=*/true}, pos);
}
}  // namespace stb

// ---------------------------------------------------------------------------------------------------------
// test entry points: the two attention kernels of the decode step on their own (include/stablets_b200.h)
// ---------------------------------------------------------------------------------------------------------
static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

extern "C" int stb_decode_self_attn(const float* qkv, float* k_cache, float* v_cache, int B, int H, int cache_rows, const int32_t* pos,
                                    const int32_t* seq_off, float* out_f32, void* out_hi, void* out_lo, void* stream) {
    // grid (H, B): B is grid.y
    STB_REQUIRE(B >= 1 && B <= 65535, "stb_decode_self_attn: B=%d outside 1..65535", B);
    STB_REQUIRE(H >= 1 && H <= 65535, "stb_decode_self_attn: H=%d outside 1..65535", H);
    STB_REQUIRE(cache_rows >= 1, "stb_decode_self_attn: cache_rows=%d must be positive", cache_rows);
    STB_REQUIRE(qkv && k_cache && v_cache && pos, "stb_decode_self_attn: null qkv, cache or pos");
    STB_REQUIRE(out_f32 || out_hi, "stb_decode_self_attn: no output (out_f32 and out_hi are both null)");
    STB_REQUIRE(out_lo == nullptr || out_hi != nullptr, "stb_decode_self_attn: out_lo needs out_hi");
    // qkv and the caches are read as float4
    STB_REQUIRE(aligned(qkv, 16) && aligned(k_cache, 16) && aligned(v_cache, 16),
                "stb_decode_self_attn: qkv, k_cache and v_cache must be 16-byte aligned");
    STB_REQUIRE(aligned(pos, 4) && aligned(seq_off, 4) && aligned(out_f32, 4) && aligned(out_hi, 2) && aligned(out_lo, 2),
                "stb_decode_self_attn: misaligned pos, seq_off or output");
    return stb::decode_attn_self(qkv, k_cache, v_cache, B, H, 64 * H, cache_rows, pos, seq_off, (__half*)out_hi, (__half*)out_lo,
                                 out_f32, (cudaStream_t)stream);
}

extern "C" int stb_decode_cross_attn(const float* q, const void* k_hi, const void* v_hi, int B, int H, float* partial, int32_t* tickets,
                                     float* out_f32, void* out_hi, void* out_lo, void* stream) {
    // grid (splits, H, B); tickets are indexed b * H + h in int
    STB_REQUIRE(B >= 1 && B <= 65535, "stb_decode_cross_attn: B=%d outside 1..65535", B);
    STB_REQUIRE(H >= 1 && H <= 65535 && (long long)B * H <= 0x7fffffffLL, "stb_decode_cross_attn: H=%d outside 1..65535 or B*H too large", H);
    STB_REQUIRE(q && k_hi && v_hi && partial && tickets, "stb_decode_cross_attn: null q, K / V plane, partial or tickets");
    STB_REQUIRE(out_f32 || out_hi, "stb_decode_cross_attn: no output (out_f32 and out_hi are both null)");
    STB_REQUIRE(out_lo == nullptr || out_hi != nullptr, "stb_decode_cross_attn: out_lo needs out_hi");
    // the K / V planes are TMA sources
    STB_REQUIRE(aligned(k_hi, 16) && aligned(v_hi, 16), "stb_decode_cross_attn: k_hi and v_hi must be 16-byte aligned");
    STB_REQUIRE(aligned(q, 4) && aligned(partial, 4) && aligned(tickets, 4) && aligned(out_f32, 4) && aligned(out_hi, 2) &&
                    aligned(out_lo, 2),
                "stb_decode_cross_attn: misaligned q, partial, tickets or output");
    stb::CrossDecodeKV kv = {(const __half*)k_hi, (const __half*)v_hi};
    return stb::decode_attn_cross(q, kv, B, H, 64 * H, partial, (int*)tickets, (__half*)out_hi, (__half*)out_lo, out_f32,
                                  (cudaStream_t)stream);
}

extern "C" int stb_decode_cross_splits(void) { return stb::decode_cross_splits(); }
