// Decode-step linear layers, small batches (the engine uses this kernel for B <= 16 sequences; up to 4 groups of 16 rows per
// CTA share the register-resident weights, so B <= 64 works): out[b][n] = epi( sum_k W[n][k] * x[b][k] ).
// Larger batches run on the cluster split-K wgmma kernel of decode_linear.cu.
//
// With M = B <= 16 rows every weight byte is used once: the op is a batched GEMV bound by HBM (d*d*4 B of weights in
// parity mode), and its enemy is LATENCY, not FLOPs: a 6.5 MB matrix is 1 us of HBM time.  Design:
//   * one CTA = 8 output features, 8 warps splitting K: at kernel start every lane issues ALL its weight loads
//     (128-bit, hi and lo planes) -- the whole weight tile of the CTA is in flight after one issue slot;
//   * meanwhile the 16 x K activation tile (split fp16, L2-resident) is staged into padded shared memory with
//     cp.async (all pieces in flight at once, zero-fill for absent rows);
//   * the products run on the warp-level tensor path, mma.sync m16n8k16 (fp16 x fp16 -> fp32): M = 16 is exactly the
//     batch, N = 8 the CTA's features.  wgmma (M = 64 atoms, B operand via smem descriptors) has no shape for this;
//     three MMAs per k-step (hi*hi + hi*lo + lo*hi) keep the fp32-grade accuracy of the parity mode;
//   * weights are consumed straight from registers: the k index inside each 32-wide block is permuted identically for
//     A and B so that a lane's 16-byte load IS its fragment (no shuffles, no smem for W);
//   * cross-warp reduction of the 16 x 8 partial tiles through 4 KB of shared memory, fused epilogue.
#include <mma.h>

#include "common.cuh"
#include "kernels.h"

namespace stb {

constexpr int GM_WARPS = 8;
constexpr int GM_KC = 1280;                 // K chunk staged per pass (40 blocks of 32 -> 5 per warp)
constexpr int GM_MAXBLK = GM_KC / 32 / GM_WARPS;

__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

constexpr int GM_MAXGRP = 4;                // up to 64 sequences: 4 groups of 16 rows share the register-resident weights

__global__ void __launch_bounds__(GM_WARPS * 32, 2)
gemv_mma_kernel(const __half* __restrict__ x_hi, const __half* __restrict__ x_lo, int B, int K,
                const __half* __restrict__ w_hi, const __half* __restrict__ w_lo, int N, const float* __restrict__ bias,
                int act, const float* __restrict__ res, long long ld_res, float* __restrict__ out_f32,
                __half* __restrict__ out_hi, __half* __restrict__ out_lo, long long ld_out) {
    extern __shared__ __align__(16) uint8_t gsm[];
    const int kc_max = K < GM_KC ? K : GM_KC;
    const int pitch = kc_max * 2 + 64;                       // bytes; == 64 mod 128 -> conflict-free fragment reads
    uint8_t* xs_hi = gsm;                                    // [16][pitch]
    uint8_t* xs_lo = gsm + 16 * pitch;
    float* red = reinterpret_cast<float*>(gsm + 32 * pitch); // [GM_WARPS][16][8]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    const int n0 = blockIdx.x * 8;
    const int n = n0 + g;
    const bool n_ok = n < N;
    const bool has_lo = w_lo != nullptr;
    const int ngrp = (B + 15) >> 4;
    float c[GM_MAXGRP][4];
#pragma unroll
    for (int gi = 0; gi < GM_MAXGRP; ++gi) c[gi][0] = c[gi][1] = c[gi][2] = c[gi][3] = 0.f;
    pdl_trigger();                                           // the next kernel may start its own weight prefetch

    for (int kc0 = 0; kc0 < K; kc0 += GM_KC) {
        const int kc = min(GM_KC, K - kc0);
        const int nblk = kc >> 5;
        // ---- 1. all weight loads of this chunk in flight (block index = warp + i * GM_WARPS); they stay in registers
        //         and are reused by every group of 16 sequences ----
        uint4 wh[GM_MAXBLK], wl[GM_MAXBLK];
#pragma unroll
        for (int i = 0; i < GM_MAXBLK; ++i) {
            const int blk = warp + i * GM_WARPS;
            wh[i] = make_uint4(0, 0, 0, 0);
            wl[i] = make_uint4(0, 0, 0, 0);
            if (blk < nblk && n_ok) {
                const long long off = (long long)n * K + kc0 + blk * 32 + q * 8;
                wh[i] = __ldg(reinterpret_cast<const uint4*>(w_hi + off));
                if (has_lo) wl[i] = __ldg(reinterpret_cast<const uint4*>(w_lo + off));
            }
        }
        if (kc0 == 0) pdl_wait();                            // weights are constants; x / res / out belong to predecessors
        const int vec_per_row = kc >> 3;                     // 16-byte pieces per row
#pragma unroll
        for (int gi = 0; gi < GM_MAXGRP; ++gi) {
            if (gi < ngrp) {
                const int row0 = gi * 16;
                const int rows = min(16, B - row0);
                // ---- 2. stage x[row0 : row0+16, kc0 : kc0+kc] with cp.async (zero-fill for absent rows) ----
                if (kc0 > 0 || gi > 0) __syncthreads();      // the previous tile's fragment reads are done
                for (int i = threadIdx.x; i < 16 * vec_per_row; i += blockDim.x) {
                    const int r = i / vec_per_row, v = i - r * vec_per_row;
                    const bool ok = r < rows;
                    const long long off = (long long)(row0 + (ok ? r : 0)) * K + kc0 + v * 8;
                    const uint32_t dh = smem_u32(xs_hi + r * pitch + v * 16);
                    const uint32_t dl = smem_u32(xs_lo + r * pitch + v * 16);
                    const int nbytes_h = ok ? 16 : 0;
                    const int nbytes_l = (ok && x_lo != nullptr) ? 16 : 0;
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dh), "l"(x_hi + off), "r"(nbytes_h) : "memory");
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dl),
                                 "l"((x_lo != nullptr ? x_lo : x_hi) + off), "r"(nbytes_l)
                                 : "memory");
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 0;" ::: "memory");
                __syncthreads();
                // ---- 3. MMAs: k inside a 32-block is permuted so that uint4 {x,y | z,w} are the two k16 steps ----
#pragma unroll
                for (int i = 0; i < GM_MAXBLK; ++i) {
                    const int blk = warp + i * GM_WARPS;
                    if (blk < nblk) {
                        const int col = (blk * 32 + q * 8) * 2;      // byte offset inside the row
                        const uint4 ah0 = *reinterpret_cast<const uint4*>(xs_hi + g * pitch + col);
                        const uint4 ah1 = *reinterpret_cast<const uint4*>(xs_hi + (g + 8) * pitch + col);
                        mma16816(c[gi], ah0.x, ah1.x, ah0.y, ah1.y, wh[i].x, wh[i].y);
                        mma16816(c[gi], ah0.z, ah1.z, ah0.w, ah1.w, wh[i].z, wh[i].w);
                        if (has_lo) {
                            mma16816(c[gi], ah0.x, ah1.x, ah0.y, ah1.y, wl[i].x, wl[i].y);
                            mma16816(c[gi], ah0.z, ah1.z, ah0.w, ah1.w, wl[i].z, wl[i].w);
                            const uint4 al0 = *reinterpret_cast<const uint4*>(xs_lo + g * pitch + col);
                            const uint4 al1 = *reinterpret_cast<const uint4*>(xs_lo + (g + 8) * pitch + col);
                            mma16816(c[gi], al0.x, al1.x, al0.y, al1.y, wh[i].x, wh[i].y);
                            mma16816(c[gi], al0.z, al1.z, al0.w, al1.w, wh[i].z, wh[i].w);
                        }
                    }
                }
            }
        }
    }
    // ---- 4. cross-warp reduction per group: lane holds D[g][2q,2q+1] (c0,c1) and D[g+8][2q,2q+1] (c2,c3) ----
#pragma unroll
    for (int gi = 0; gi < GM_MAXGRP; ++gi) {
        if (gi < ngrp) {
            __syncthreads();
            float* rw = red + warp * 128;
            rw[g * 8 + 2 * q] = c[gi][0];
            rw[g * 8 + 2 * q + 1] = c[gi][1];
            rw[(g + 8) * 8 + 2 * q] = c[gi][2];
            rw[(g + 8) * 8 + 2 * q + 1] = c[gi][3];
            __syncthreads();
            if (threadIdx.x < 128) {
                const int row = gi * 16 + (threadIdx.x >> 3), col = threadIdx.x & 7;
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < GM_WARPS; ++w) v += red[w * 128 + threadIdx.x];
                const int nn = n0 + col;
                if (row < B && nn < N) {
                    if (bias != nullptr) v += __ldg(bias + nn);
                    if (act == STB_ACT_GELU) v = gelu_erf(v);
                    if (res != nullptr) v += res[(long long)row * ld_res + nn];
                    const long long o = (long long)row * ld_out + nn;
                    if (out_f32 != nullptr) out_f32[o] = v;
                    if (out_hi != nullptr) {
                        __half hi, lo;
                        split_f16(v, hi, lo);
                        out_hi[o] = hi;
                        if (out_lo != nullptr) out_lo[o] = lo;
                    }
                }
            }
        }
    }
}

// x split [B][K] (row pitch K), W split [N][K]; out = act(W x + bias) + res as fp32 and/or split planes.
int gemv(const void* x_hi, const void* x_lo, int B, int K, const void* w_hi, const void* w_lo, int N, const float* bias,
         int act, const float* res, long long ld_res, float* out_f32, void* out_hi, void* out_lo, long long ld_out,
         cudaStream_t st) {
    STB_REQUIRE(B >= 1 && B <= 64 && K % 32 == 0 && K >= 32, "gemv: unsupported shape B=%d K=%d", B, K);
    const int kc = K < GM_KC ? K : GM_KC;
    const size_t smem = (size_t)32 * (kc * 2 + 64) + GM_WARPS * 128 * sizeof(float);
    ProfScope ps("gemv_mma", st, (double)N * K * 2.0 * (w_lo ? 2 : 1) + (double)B * K * 4.0 + (double)B * N * 4.0, 2.0 * B * (double)N * K);
    return launch(gemv_mma_kernel, {dim3(cdiv(N, 8)), dim3(GM_WARPS * 32), smem, st, /*pdl=*/true}, (const __half*)x_hi,
                  (const __half*)x_lo, B, K, (const __half*)w_hi, (const __half*)w_lo, N, bias, act, res, ld_res, out_f32,
                  (__half*)out_hi, (__half*)out_lo, ld_out);
}

}  // namespace stb

extern "C" int stb_gemv(const void* x_hi, const void* x_lo, int B, int K, const void* w_hi, const void* w_lo, int N,
                        const float* bias, int act, const float* res, long long ld_res, float* out_f32, void* out_hi,
                        void* out_lo, long long ld_out, void* stream) {
    STB_REQUIRE(x_hi && w_hi && (out_f32 || out_hi) && N >= 1, "stb_gemv: bad arguments");
    STB_REQUIRE(ld_out >= N && (res == nullptr || ld_res >= N), "stb_gemv: leading dimensions smaller than N");
    return stb::gemv(x_hi, x_lo, B, K, w_hi, w_lo, N, bias, act, res, ld_res, out_f32, out_hi, out_lo, ld_out,
                     (cudaStream_t)stream);
}
