// a5 / K6+K8: cross-attention post-processing of the legacy alignment-head path
// (stable_whisper/timing.py:105-110 + the head mean of :194; median = whisper.timing.median_filter):
//
//   qk[b][a][S..M-2][0..F)  --softmax(x*qk_scale) over frames-->  --z-norm over the R token rows of every frame
//   (biased std)-->  --median filter (width 7, reflect) along frames-->  --mean over the A heads--> matrix[b][R][F]
//
// Three small kernels over an L2-resident working set (A*R*F*4 B, ~6 MB at A=10,R=101,F=1500):
//   1. row softmax           one warp per (b,a,r) row, values kept in registers, written once to W
//   2. column z-norm         one thread per (b,a,column), coalesced across columns, two-pass mean/var, in place on W
//   3. median-7 + head mean  one thread per (b,r,column): 7-tap sorting network per head, accumulate over heads
#include "common.cuh"

namespace stb {

constexpr int QK_MAXV = 47;

__global__ void __launch_bounds__(256) qk_softmax_kernel(const float* __restrict__ qk, long long n_rows, int M,
                                                         long long ldq, int S, int R, int F, float scale,
                                                         float* __restrict__ W, int Fp) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // over B*A*R
    if (row >= n_rows) return;
    const int lane = threadIdx.x & 31;
    const long long ba = row / R;
    const int r = (int)(row - ba * R);
    const float* src = qk + (ba * M + (S + r)) * ldq;
    float v[QK_MAXV];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < QK_MAXV; ++i) {
        const int c = i * 32 + lane;
        v[i] = (c < F) ? src[c] * scale : -INFINITY;
        mx = fmaxf(mx, v[i]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < QK_MAXV; ++i) {
        const int c = i * 32 + lane;
        v[i] = (c < F) ? expf(v[i] - mx) : 0.f;
        sum += v[i];
    }
    sum = warp_sum(sum);
    float* dst = W + row * Fp;
#pragma unroll
    for (int i = 0; i < QK_MAXV; ++i) {
        const int c = i * 32 + lane;
        if (c < F) dst[c] = v[i] / sum;
    }
}

__global__ void __launch_bounds__(128) qk_znorm_kernel(float* __restrict__ W, int R, int F, int Fp) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= F) return;
    float* base = W + (long long)blockIdx.y * R * Fp + c;       // blockIdx.y over B*A
    float s = 0.f;
    for (int r = 0; r < R; ++r) s += base[(long long)r * Fp];
    const float mean = s / (float)R;
    float q = 0.f;
    for (int r = 0; r < R; ++r) {
        const float d = base[(long long)r * Fp] - mean;
        q += d * d;
    }
    const float sd = sqrtf(q / (float)R);
    for (int r = 0; r < R; ++r) base[(long long)r * Fp] = (base[(long long)r * Fp] - mean) / sd;
}

__device__ __forceinline__ void cswap(float& a, float& b) {
    const float lo = fminf(a, b), hi = fmaxf(a, b);
    a = lo;
    b = hi;
}
// median of 7 via a 16-comparator sorting network (only element 3 is needed)
__device__ __forceinline__ float median7(float a0, float a1, float a2, float a3, float a4, float a5, float a6) {
    cswap(a0, a5); cswap(a0, a3); cswap(a1, a6); cswap(a2, a4); cswap(a0, a1); cswap(a3, a5); cswap(a2, a6);
    cswap(a2, a3); cswap(a3, a6); cswap(a4, a5); cswap(a1, a4); cswap(a1, a3); cswap(a3, a4);
    return a3;
}

__device__ __forceinline__ int reflect(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * (n - 1) - i;
    return i;
}

__global__ void __launch_bounds__(128) qk_median_mean_kernel(const float* __restrict__ W, int A, int R, int F, int Fp,
                                                             int width, float* __restrict__ out, long long ldm) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= F) return;
    const int r = blockIdx.y, b = blockIdx.z;
    float acc = 0.f;
    const bool filt = (width == 7) && (F > 3);
    for (int a = 0; a < A; ++a) {
        const float* row = W + (((long long)b * A + a) * R + r) * Fp;
        float v;
        if (filt) {
            v = median7(row[reflect(c - 3, F)], row[reflect(c - 2, F)], row[reflect(c - 1, F)], row[c],
                        row[reflect(c + 1, F)], row[reflect(c + 2, F)], row[reflect(c + 3, F)]);
        } else {
            v = row[c];
        }
        acc += v;
    }
    out[((long long)b * R + r) * ldm + c] = acc / (float)A;
}

}  // namespace stb

extern "C" size_t stb_qkpost_ws_bytes(int B, int A, int R, int F) {
    const int Fp = (F + 3) & ~3;
    return (size_t)B * A * R * Fp * sizeof(float);
}

extern "C" int stb_qk_postprocess(const float* qk, int B, int A, int M, long long ldq, int S, int R, int F, float qk_scale,
                                  int medfilt_width, float* matrix, long long ldm, void* ws, size_t ws_bytes, void* stream) {
    STB_REQUIRE(S >= 0 && S + R <= M, "stb_qk_postprocess: rows S=%d R=%d exceed M=%d", S, R, M);
    STB_REQUIRE(qk && matrix && ws, "stb_qk_postprocess: null pointer");
    STB_REQUIRE(R >= 1 && F >= 1 && F <= 1504 && A >= 1 && B >= 1, "stb_qk_postprocess: bad shape R=%d F=%d A=%d B=%d", R, F, A, B);
    STB_REQUIRE(medfilt_width == 7 || medfilt_width == 1, "stb_qk_postprocess: medfilt_width %d unsupported (7 or 1)", medfilt_width);
    STB_REQUIRE(ws_bytes >= stb_qkpost_ws_bytes(B, A, R, F), "stb_qk_postprocess: workspace too small");
    const int Fp = (F + 3) & ~3;
    float* W = (float*)ws;
    cudaStream_t st = (cudaStream_t)stream;
    const long long n_rows = (long long)B * A * R;
    stb::ProfScope ps("qk_postprocess(3 kernels)", st, (double)B * A * R * F * 4.0 + (double)B * R * F * 4.0);
    STB_TRY(stb::launch(stb::qk_softmax_kernel, {stb::cdiv(n_rows, 8), 256, 0, st}, qk, n_rows, M, ldq, S, R, F, qk_scale, W, Fp));
    STB_TRY(stb::launch(stb::qk_znorm_kernel, {dim3(stb::cdiv(F, 128), B * A), 128, 0, st}, W, R, F, Fp));
    return stb::launch(stb::qk_median_mean_kernel, {dim3(stb::cdiv(F, 128), R, B), 128, 0, st}, W, A, R, F, Fp, medfilt_width, matrix,
                       ldm);
}

// =========================================================================================================
// a5 variants: per-token dynamic head selection (stable_whisper/timing.py:85-103) and the "new" aligner
// (stable_whisper/timing.py:115-163, arXiv 2509.09987).  Both start from the scores of ALL L*H cross-attention heads
// (stb_decoder_forward with n_sel < 0) and end in the same [R][F] matrix that feeds the DTW.
// =========================================================================================================
namespace stb {

// scores[head][row] = sum_f |peak - f| / 1500 * W[head][row][f]; peak = argmax_f W (first iteration) or the midpoint
// of the previous jump interval of that row.  One warp per (b, head, row).
__global__ void __launch_bounds__(256) dyn_score_kernel(const float* __restrict__ W, long long n_rows, int LH, int R, int F,
                                                        int Fp, const int32_t* __restrict__ prev_jumps,
                                                        float* __restrict__ scores) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // over B*LH*R
    if (row >= n_rows) return;
    const int lane = threadIdx.x & 31;
    const int r = (int)(row % R);
    const long long bh = row / R;
    const int b = (int)(bh / LH);
    const float* w = W + row * Fp;
    float peak;
    if (prev_jumps != nullptr) {
        const int j0 = prev_jumps[(long long)b * R + r];
        const int j1 = (r + 1 < R) ? prev_jumps[(long long)b * R + r + 1] : F;
        peak = (float)j0 + (float)(j1 - j0) * 0.5f;
    } else {
        float best = -INFINITY;
        int arg = 0x7fffffff;
        for (int f = lane; f < F; f += 32) {
            const float v = w[f];
            if (v > best) { best = v; arg = f; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
        }
        peak = (float)arg;
    }
    float s = 0.f;
    for (int f = lane; f < F; f += 32) s += fabsf(peak - (float)f) / 1500.0f * w[f];
    s = warp_sum(s);
    if (lane == 0) scores[row] = s;
}

// per (b, row): the `count` heads with the smallest score.  One warp per (b, row); table[b][a][row] = head index.
__global__ void __launch_bounds__(32) dyn_select_kernel(const float* __restrict__ scores, int LH, int R, int count,
                                                       int32_t* __restrict__ table) {
    const int r = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
    unsigned long long taken[20];                               // bitmask over <= 1280 heads
#pragma unroll
    for (int i = 0; i < 20; ++i) taken[i] = 0ull;
    for (int a = 0; a < count; ++a) {
        float best = INFINITY;
        int arg = 0x7fffffff;
        for (int hd = lane; hd < LH; hd += 32) {
            if ((taken[hd >> 6] >> (hd & 63)) & 1ull) continue;
            const float v = scores[((long long)b * LH + hd) * R + r];
            if (v < best) { best = v; arg = hd; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (ob < best || (ob == best && oa < arg)) { best = ob; arg = oa; }
        }
        taken[arg >> 6] |= 1ull << (arg & 63);                  // every lane tracks the same set
        if (lane == 0) table[((long long)b * count + a) * R + r] = arg;
    }
}

// Wsel[b][a][r][:] = W[b][table[b][a][r]][r][:]
__global__ void __launch_bounds__(128) dyn_gather_kernel(const float* __restrict__ W, int LH, int R, int Fp, int count,
                                                        const int32_t* __restrict__ table, float* __restrict__ Wsel) {
    const int r = blockIdx.x, a = blockIdx.y, b = blockIdx.z;
    const int hd = table[((long long)b * count + a) * R + r];
    const float4* src = reinterpret_cast<const float4*>(W + (((long long)b * LH + hd) * R + r) * Fp);
    float4* dst = reinterpret_cast<float4*>(Wsel + (((long long)b * count + a) * R + r) * Fp);
    for (int i = threadIdx.x; i < (Fp >> 2); i += blockDim.x) dst[i] = src[i];
}

// ---- "new" aligner ----
// one warp per (b, head, m) row of the RAW scores: median-7 (reflect) along frames, then softmax over frames -> W
__global__ void __launch_bounds__(256) new_median_softmax_kernel(const float* __restrict__ qk, long long n_rows, long long ldq,
                                                                 int F, float scale, int width, float* __restrict__ W, int Fp) {
    __shared__ float s_row[8][STB_KPAD];
    const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * 8 + wp;
    if (row >= n_rows) return;
    const float* src = qk + row * ldq;
    for (int f = lane; f < F; f += 32) s_row[wp][f] = src[f];
    __syncwarp();
    const bool filt = (width == 7) && (F > 3);
    float v[QK_MAXV];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < QK_MAXV; ++i) {
        const int c = i * 32 + lane;
        float x = -INFINITY;
        if (c < F) {
            const float* rw = s_row[wp];
            x = filt ? median7(rw[reflect(c - 3, F)], rw[reflect(c - 2, F)], rw[reflect(c - 1, F)], rw[c], rw[reflect(c + 1, F)],
                               rw[reflect(c + 2, F)], rw[reflect(c + 3, F)])
                     : rw[c];
            x *= scale;
        }
        v[i] = x;
        mx = fmaxf(mx, x);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < QK_MAXV; ++i) {
        const int c = i * 32 + lane;
        v[i] = (c < F) ? expf(v[i] - mx) : 0.f;
        sum += v[i];
    }
    sum = warp_sum(sum);
    float* dst = W + row * Fp;
#pragma unroll
    for (int i = 0; i < QK_MAXV; ++i) {
        const int c = i * 32 + lane;
        if (c < F) dst[c] = v[i] / sum;
    }
}

// colnorm[b][hd][f] = sqrt(sum_m W^2), coverage[b][hd][f] = sum_m W (thread per column; blockIdx.y over B*LH)
__global__ void __launch_bounds__(128) new_colstats_kernel(const float* __restrict__ W, int M, int F, int Fp,
                                                          float* __restrict__ colnorm, float* __restrict__ cover) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= F) return;
    const float* base = W + (long long)blockIdx.y * M * Fp + c;
    float q = 0.f, s = 0.f;
    for (int r = 0; r < M; ++r) {
        const float v = base[(long long)r * Fp];
        q += v * v;
        s += v;
    }
    colnorm[(long long)blockIdx.y * Fp + c] = sqrtf(q);
    cover[(long long)blockIdx.y * Fp + c] = s;
}

// score[b][hd] = w_col * sum_f colnorm + w_row * sum_m ||W[m,:]|| - w_cov * (sum_f max(cover, .5) - .5 F).  One CTA per (b,hd).
__global__ void __launch_bounds__(256) new_score_kernel(const float* __restrict__ W, const float* __restrict__ colnorm,
                                                        const float* __restrict__ cover, int M, int F, int Fp, float w_col,
                                                        float w_row, float w_cov, float* __restrict__ score) {
    __shared__ float s_red[8];
    const long long bh = blockIdx.x;
    const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc = 0.f;
    if (w_row > 0.f) {
        for (int r = wp; r < M; r += 8) {
            const float* rw = W + (bh * M + r) * Fp;
            float q = 0.f;
            for (int f = lane; f < F; f += 32) q += rw[f] * rw[f];
            q = warp_sum(q);
            if (lane == 0) acc += w_row * sqrtf(q);
        }
    }
    float part = 0.f;
    for (int f = threadIdx.x; f < F; f += 256) {
        if (w_col > 0.f) part += w_col * colnorm[bh * Fp + f];
        if (w_cov > 0.f) part -= w_cov * (fmaxf(cover[bh * Fp + f], 0.5f) - 0.5f);
    }
    part = warp_sum(part);
    if (lane == 0) s_red[wp] = part + acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += s_red[i];
        score[bh] = t;
    }
}

// top-k heads by score (largest), one warp per batch item
__global__ void __launch_bounds__(32) new_topk_kernel(const float* __restrict__ score, int LH, int topk, int32_t* __restrict__ top) {
    const int b = blockIdx.x, lane = threadIdx.x;
    unsigned long long taken[20];
#pragma unroll
    for (int i = 0; i < 20; ++i) taken[i] = 0ull;
    for (int a = 0; a < topk; ++a) {
        float best = -INFINITY;
        int arg = 0x7fffffff;
        for (int hd = lane; hd < LH; hd += 32) {
            if ((taken[hd >> 6] >> (hd & 63)) & 1ull) continue;
            const float v = score[(long long)b * LH + hd];
            if (v > best) { best = v; arg = hd; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
        }
        taken[arg >> 6] |= 1ull << (arg & 63);
        if (lane == 0) top[(long long)b * topk + a] = arg;
    }
}

// matrix[b][r][f] = mean_k W[top_k][S + r][f] / colnorm[top_k][f]
__global__ void __launch_bounds__(128) new_matrix_kernel(const float* __restrict__ W, const float* __restrict__ colnorm,
                                                        const int32_t* __restrict__ top, int LH, int M, int S, int F, int Fp,
                                                        int topk, float* __restrict__ out, long long ldm, int R) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= F) return;
    const int r = blockIdx.y, b = blockIdx.z;
    float acc = 0.f;
    for (int k = 0; k < topk; ++k) {
        const long long bh = (long long)b * LH + top[(long long)b * topk + k];
        acc += W[(bh * M + S + r) * Fp + c] / colnorm[bh * Fp + c];
    }
    out[((long long)b * R + r) * ldm + c] = acc / (float)topk;
}

}  // namespace stb

extern "C" size_t stb_qkpost_dynamic_ws_bytes(int B, int LH, int R, int F, int count) {
    const size_t Fp = (F + 3) & ~3;
    return ((size_t)B * LH * R * Fp + (size_t)B * count * R * Fp + (size_t)B * LH * R) * sizeof(float) +
           (size_t)B * count * R * sizeof(int32_t) + 1024;
}

extern "C" int stb_qk_postprocess_dynamic(const float* qk, int B, int LH, int M, long long ldq, int S, int R, int F, float qk_scale,
                                          int medfilt_width, int count, const int32_t* prev_jumps, int reuse_softmax,
                                          float* matrix, long long ldm, void* ws, size_t ws_bytes, void* stream) {
    STB_REQUIRE(qk && matrix && ws, "stb_qk_postprocess_dynamic: null pointer");
    STB_REQUIRE(S >= 0 && S + R <= M && R >= 1 && F >= 1 && F <= 1504 && B >= 1, "stb_qk_postprocess_dynamic: bad shape");
    STB_REQUIRE(count >= 1 && count <= LH && LH <= 1280, "stb_qk_postprocess_dynamic: count=%d LH=%d unsupported", count, LH);
    STB_REQUIRE(medfilt_width == 7 || medfilt_width == 1, "stb_qk_postprocess_dynamic: medfilt_width %d unsupported", medfilt_width);
    STB_REQUIRE(ws_bytes >= stb_qkpost_dynamic_ws_bytes(B, LH, R, F, count), "stb_qk_postprocess_dynamic: workspace too small");
    const int Fp = (F + 3) & ~3;
    cudaStream_t st = (cudaStream_t)stream;
    float* W = (float*)ws;                                      // [B][LH][R][Fp] softmaxed scores (kept for reuse)
    float* Wsel = W + (size_t)B * LH * R * Fp;                  // [B][count][R][Fp]
    float* scores = Wsel + (size_t)B * count * R * Fp;          // [B][LH][R]
    int32_t* table = (int32_t*)(scores + (size_t)B * LH * R);   // [B][count][R]
    const long long n_rows = (long long)B * LH * R;
    stb::ProfScope ps("qk_postprocess_dynamic", st, (double)n_rows * F * 4.0 * 2);
    if (!reuse_softmax)
        STB_TRY(stb::launch(stb::qk_softmax_kernel, {stb::cdiv(n_rows, 8), 256, 0, st}, qk, n_rows, M, ldq, S, R, F, qk_scale, W, Fp));
    STB_TRY(stb::launch(stb::dyn_score_kernel, {stb::cdiv(n_rows, 8), 256, 0, st}, W, n_rows, LH, R, F, Fp, prev_jumps, scores));
    STB_TRY(stb::launch(stb::dyn_select_kernel, {dim3(R, B), 32, 0, st}, scores, LH, R, count, table));
    STB_TRY(stb::launch(stb::dyn_gather_kernel, {dim3(R, count, B), 128, 0, st}, W, LH, R, Fp, count, table, Wsel));
    STB_TRY(stb::launch(stb::qk_znorm_kernel, {dim3(stb::cdiv(F, 128), B * count), 128, 0, st}, Wsel, R, F, Fp));
    return stb::launch(stb::qk_median_mean_kernel, {dim3(stb::cdiv(F, 128), R, B), 128, 0, st}, Wsel, count, R, F, Fp, medfilt_width,
                       matrix, ldm);
}

extern "C" size_t stb_qkpost_new_ws_bytes(int B, int LH, int M, int F, int topk) {
    const size_t Fp = (F + 3) & ~3;
    return ((size_t)B * LH * M * Fp + 2 * (size_t)B * LH * Fp + (size_t)B * LH) * sizeof(float) + (size_t)B * topk * sizeof(int32_t) + 1024;
}

extern "C" int stb_qk_postprocess_new(const float* qk, int B, int LH, int M, long long ldq, int S, int R, int F, float qk_scale,
                                      int medfilt_width, int topk, float w_colnorm, float w_rownorm, float w_coverage,
                                      float* matrix, long long ldm, void* ws, size_t ws_bytes, void* stream) {
    STB_REQUIRE(qk && matrix && ws, "stb_qk_postprocess_new: null pointer");
    STB_REQUIRE(S >= 0 && S + R <= M && R >= 1 && F >= 1 && F <= 1504 && B >= 1, "stb_qk_postprocess_new: bad shape");
    STB_REQUIRE(topk >= 1 && topk <= LH && LH <= 1280, "stb_qk_postprocess_new: topk=%d LH=%d unsupported", topk, LH);
    STB_REQUIRE(medfilt_width == 7 || medfilt_width == 1, "stb_qk_postprocess_new: medfilt_width %d unsupported", medfilt_width);
    STB_REQUIRE(ws_bytes >= stb_qkpost_new_ws_bytes(B, LH, M, F, topk), "stb_qk_postprocess_new: workspace too small");
    const int Fp = (F + 3) & ~3;
    cudaStream_t st = (cudaStream_t)stream;
    float* W = (float*)ws;                                      // [B][LH][M][Fp]
    float* colnorm = W + (size_t)B * LH * M * Fp;               // [B][LH][Fp]
    float* cover = colnorm + (size_t)B * LH * Fp;
    float* score = cover + (size_t)B * LH * Fp;                 // [B][LH]
    int32_t* top = (int32_t*)(score + (size_t)B * LH);
    const long long n_rows = (long long)B * LH * M;
    stb::ProfScope ps("qk_postprocess_new", st, (double)n_rows * F * 4.0 * 2);
    STB_TRY(stb::launch(stb::new_median_softmax_kernel, {stb::cdiv(n_rows, 8), 256, 0, st}, qk, n_rows, ldq, F, qk_scale, medfilt_width,
                        W, Fp));
    STB_TRY(stb::launch(stb::new_colstats_kernel, {dim3(stb::cdiv(F, 128), B * LH), 128, 0, st}, W, M, F, Fp, colnorm, cover));
    STB_TRY(stb::launch(stb::new_score_kernel, {B * LH, 256, 0, st}, W, colnorm, cover, M, F, Fp, w_colnorm, w_rownorm, w_coverage,
                        score));
    STB_TRY(stb::launch(stb::new_topk_kernel, {B, 32, 0, st}, score, LH, topk, top));
    return stb::launch(stb::new_matrix_kernel, {dim3(stb::cdiv(F, 128), R, B), 128, 0, st}, W, colnorm, top, LH, M, S, F, Fp, topk,
                       matrix, ldm, R);
}
