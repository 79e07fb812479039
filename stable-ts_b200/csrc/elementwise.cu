// K5 / K9: bandwidth-bound row kernels around the GEMMs -- LayerNorm, softmax (plain / causal), token embedding,
// mel repack for conv-as-GEMM, cross-attention capture copy, token probability + rank.
// All use one warp per row with 128-bit global accesses and warp-shuffle reductions; outputs that feed a GEMM are
// written directly as split-fp16 planes so no separate conversion pass touches HBM.
#include "common.cuh"
#include "kernels.h"

namespace stb {

// ---------------------------------------------------------------------------------------------------------
// LayerNorm (whisper.model.LayerNorm: fp32 statistics, eps 1e-5, biased variance).  d % 128 == 0, d <= 1280.
// x fp32 [rows][d] -> split planes [rows][d] (+ optional fp32 copy).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, long long rows, int d,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        __half* __restrict__ hi, __half* __restrict__ lo,
                                                        float* __restrict__ out_f32) {
    pdl_trigger();
    pdl_wait();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const int nv = d >> 7;                                   // float4 per lane
    const float4* xr = reinterpret_cast<const float4*>(x + row * d);
    float4 v[10];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i)
        if (i < nv) {
            v[i] = xr[i * 32 + lane];
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i)
        if (i < nv) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
            q += (a * a + b * b) + (c * c + e * e);
        }
    const float var = warp_sum(q) / (float)d;
    const float rstd = 1.0f / sqrtf(var + 1e-5f);
#pragma unroll
    for (int i = 0; i < 10; ++i)
        if (i < nv) {
            const int c4 = i * 32 + lane;
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
            const float4 bb = __ldg(reinterpret_cast<const float4*>(beta) + c4);
            float4 y;
            y.x = (v[i].x - mean) * rstd * g.x + bb.x;
            y.y = (v[i].y - mean) * rstd * g.y + bb.y;
            y.z = (v[i].z - mean) * rstd * g.z + bb.z;
            y.w = (v[i].w - mean) * rstd * g.w + bb.w;
            if (out_f32) reinterpret_cast<float4*>(out_f32 + row * d)[c4] = y;
            if (hi) {
                __half h[4], l[4];
                split_f16(y.x, h[0], l[0]); split_f16(y.y, h[1], l[1]);
                split_f16(y.z, h[2], l[2]); split_f16(y.w, h[3], l[3]);
                reinterpret_cast<uint2*>(hi + row * d)[c4] = *reinterpret_cast<uint2*>(h);
                if (lo) reinterpret_cast<uint2*>(lo + row * d)[c4] = *reinterpret_cast<uint2*>(l);
            }
        }
}

int layernorm(const float* x, long long rows, int d, const float* gamma, const float* beta, __half* hi, __half* lo,
              float* out_f32, cudaStream_t st) {
    STB_REQUIRE(d % 128 == 0 && d <= 1280, "layernorm: d=%d must be a multiple of 128 and <= 1280", d);
    if (rows == 0) return STB_OK;
    ProfScope ps("layernorm", st, (double)rows * d * (4.0 + (hi ? 2.0 : 0.0) + (lo ? 2.0 : 0.0) + (out_f32 ? 4.0 : 0.0)));
    return launch(layernorm_kernel, {dim3(cdiv(rows, 8)), dim3(256), 0, st, /*pdl=*/true}, x, rows, d, gamma, beta, hi, lo, out_f32);
}

// ---------------------------------------------------------------------------------------------------------
// Row softmax of attention scores (F.softmax(qk.float(), -1) in MultiHeadAttention.qkv_attention).
// S fp32 [n_rows][ld_s] -> P split [n_rows][ld_p]; columns >= n_valid(row) are written as 0 up to ld_p.
// causal: n_valid = (row % rows_per_slice) + 1 (the -inf upper triangle of the decoder mask), else n_cols.
// ---------------------------------------------------------------------------------------------------------
constexpr int SM_MAXV = 47;   // 47*32 = 1504 columns

__global__ void __launch_bounds__(256) softmax_kernel(const float* __restrict__ S, long long n_rows, int n_cols,
                                                      long long ld_s, int rows_per_slice, int causal,
                                                      __half* __restrict__ hi, __half* __restrict__ lo, long long ld_p) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int lane = threadIdx.x & 31;
    const int nvalid = causal ? min(n_cols, (int)(row % rows_per_slice) + 1) : n_cols;
    const float* s = S + row * ld_s;
    float v[SM_MAXV];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < SM_MAXV; ++i) {
        const int c = i * 32 + lane;
        v[i] = (c < nvalid) ? s[c] : -INFINITY;
        mx = fmaxf(mx, v[i]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < SM_MAXV; ++i) {
        const int c = i * 32 + lane;
        v[i] = (c < nvalid) ? expf(v[i] - mx) : 0.f;
        sum += v[i];
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < SM_MAXV; ++i) {
        const int c = i * 32 + lane;
        if (c < ld_p) {
            __half h, l;
            split_f16(v[i] * inv, h, l);
            hi[row * ld_p + c] = h;
            if (lo) lo[row * ld_p + c] = l;
        }
    }
}

int softmax_rows(const float* S, long long n_rows, int n_cols, long long ld_s, int rows_per_slice, int causal, __half* hi,
                 __half* lo, long long ld_p, cudaStream_t st) {
    STB_REQUIRE(n_cols <= SM_MAXV * 32 && ld_p <= SM_MAXV * 32, "softmax: n_cols=%d ld_p=%lld exceed %d", n_cols, ld_p,
                SM_MAXV * 32);
    if (n_rows == 0) return STB_OK;
    ProfScope ps("softmax", st, (double)n_rows * n_cols * 4.0 + (double)n_rows * ld_p * 2.0 * (lo ? 2 : 1));
    return launch(softmax_kernel, {cdiv(n_rows, 8), 256, 0, st}, S, n_rows, n_cols, ld_s, rows_per_slice, causal, hi, lo, ld_p);
}

// ---------------------------------------------------------------------------------------------------------
// Token embedding + learned positions (TextDecoder.forward): x[b][t] = E[tok[b][t]] + pos[offset + t].
// ---------------------------------------------------------------------------------------------------------
__global__ void embed_kernel(const int32_t* __restrict__ tokens, long long n_tok, int M, int offset, int d,
                             const float* __restrict__ emb, const float* __restrict__ pos, float* __restrict__ x) {
    const long long row = blockIdx.x;
    const int tok = tokens[row];
    const int t = (int)(row % M) + offset;
    const float4* e = reinterpret_cast<const float4*>(emb + (long long)tok * d);
    const float4* p = reinterpret_cast<const float4*>(pos + (long long)t * d);
    float4* o = reinterpret_cast<float4*>(x + row * d);
    for (int i = threadIdx.x; i < (d >> 2); i += blockDim.x) {
        const float4 a = __ldg(e + i), b = __ldg(p + i);
        o[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
}

int embed_tokens(const int32_t* tokens, long long n_tok, int M, int offset, int d, const float* emb, const float* pos,
                 float* x, cudaStream_t st) {
    if (n_tok == 0) return STB_OK;
    return launch(embed_kernel, {(unsigned)n_tok, 128, 0, st}, tokens, n_tok, M, offset, d, emb, pos, x);
}

// ---------------------------------------------------------------------------------------------------------
// mel fp32 [B][C][3000] -> time-major split planes [B][3002][C] with zero rows 0 and 3001 (conv padding=1), the
// layout whose overlapping 3*C-wide rows ARE the im2col matrix of conv1 (k index = tap*C + c).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mel_repack_kernel(const float* __restrict__ mel, int C, int T,
                                                         __half* __restrict__ hi, __half* __restrict__ lo) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 8 rows of 32
    const float* src = mel + (long long)b * C * T;
    for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, t = t0 + tx;
        tile[i][tx] = (c < C && t < T) ? src[(long long)c * T + t] : 0.f;
    }
    __syncthreads();
    const long long plane = (long long)(T + 2) * C;
    for (int i = ty; i < 32; i += 8) {
        const int t = t0 + i, c = c0 + tx;
        if (t < T && c < C) {
            __half h, l;
            split_f16(tile[tx][i], h, l);
            const long long off = (long long)b * plane + (long long)(t + 1) * C + c;
            hi[off] = h;
            if (lo) lo[off] = l;
        }
    }
    if (blockIdx.x == 0 && blockIdx.y == 0) {                    // zero the two padding rows of this batch item
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            const long long o0 = (long long)b * plane + c, o1 = (long long)b * plane + (long long)(T + 1) * C + c;
            hi[o0] = __float2half(0.f); hi[o1] = __float2half(0.f);
            if (lo) { lo[o0] = __float2half(0.f); lo[o1] = __float2half(0.f); }
        }
    }
}

int mel_repack(const float* mel, int B, int C, int T, __half* hi, __half* lo, cudaStream_t st) {
    dim3 grid(cdiv(T, 32), cdiv(C, 32), B);
    return launch(mel_repack_kernel, {grid, 256, 0, st}, mel, C, T, hi, lo);
}

// zero the padding rows (0 and T+1) of a time-major [B][T+2][C] split buffer
__global__ void zero_pad_rows_kernel(__half* hi, __half* lo, int C, int T) {
    const long long plane = (long long)(T + 2) * C;
    const int b = blockIdx.x;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const long long o0 = (long long)b * plane + c, o1 = (long long)b * plane + (long long)(T + 1) * C + c;
        hi[o0] = __float2half(0.f); hi[o1] = __float2half(0.f);
        if (lo) { lo[o0] = __float2half(0.f); lo[o1] = __float2half(0.f); }
    }
}
int zero_pad_rows(__half* hi, __half* lo, int B, int C, int T, cudaStream_t st) {
    return launch(zero_pad_rows_kernel, {B, 256, 0, st}, hi, lo, C, T);
}

// ---------------------------------------------------------------------------------------------------------
// Token probability (+ rank): p = softmax(logits[r][:n_classes])[target[r]]; rank = #classes with logit < target's.
// One CTA per row (n_classes ~ 50k fp32 = 200 KB: a streaming read, two passes served by L2).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) token_prob_kernel(const float* __restrict__ logits, long long ld, int n_classes,
                                                         const int32_t* __restrict__ targets, float* __restrict__ prob,
                                                         int32_t* __restrict__ rank) {
    __shared__ float red[16];
    __shared__ int redi[16];
    const int r = blockIdx.x;
    const float* l = logits + (long long)r * ld;
    const int tgt = targets[r];
    const float lt = l[tgt];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n_classes; i += blockDim.x) mx = fmaxf(mx, l[i]);
    mx = warp_max(mx);
    if (lane == 0) red[w] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int i = 1; i < 16; ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float s = 0.f;
    int cnt = 0;
    for (int i = threadIdx.x; i < n_classes; i += blockDim.x) {
        const float v = l[i];
        s += expf(v - mx);
        cnt += (v < lt) ? 1 : 0;
    }
    s = warp_sum(s);
    cnt = warp_sum_i(cnt);
    if (lane == 0) { red[w] = s; redi[w] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        int c = 0;
        for (int i = 0; i < 16; ++i) { tot += red[i]; c += redi[i]; }
        prob[r] = expf(lt - mx) / tot;
        if (rank) rank[r] = c;
    }
}

// Full probability rows (the 3-D form of the refine plugin, stable_whisper/alignment.py:669-671): out[r][c] =
// softmax(logits[r][:n_classes])[c].  One CTA per row; the row (200 KB) is re-read from L2 for the second and third pass.
__global__ void __launch_bounds__(512) softmax_probs_kernel(const float* __restrict__ logits, long long ld, int n_classes,
                                                            float* __restrict__ out, long long ld_out) {
    __shared__ float red[16];
    const int r = blockIdx.x;
    const float* l = logits + (long long)r * ld;
    float* o = out + (long long)r * ld_out;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n_classes; i += blockDim.x) mx = fmaxf(mx, l[i]);
    mx = warp_max(mx);
    if (lane == 0) red[w] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int i = 1; i < 16; ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float s = 0.f;
    for (int i = threadIdx.x; i < n_classes; i += blockDim.x) s += expf(l[i] - mx);
    s = warp_sum(s);
    if (lane == 0) red[w] = s;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) tot += red[i];
    for (int i = threadIdx.x; i < n_classes; i += blockDim.x) o[i] = expf(l[i] - mx) / tot;
}

}  // namespace stb

extern "C" int stb_softmax_probs(const float* logits, long long ld, int n_rows, int n_classes, float* out, long long ld_out,
                                 void* stream) {
    STB_REQUIRE(logits && out && n_classes > 0 && ld >= n_classes && ld_out >= n_classes, "stb_softmax_probs: bad arguments");
    if (n_rows == 0) return STB_OK;
    stb::ProfScope ps("softmax_probs", (cudaStream_t)stream, (double)n_rows * n_classes * 8.0);
    return stb::launch(stb::softmax_probs_kernel, {n_rows, 512, 0, (cudaStream_t)stream}, logits, ld, n_classes, out, ld_out);
}

extern "C" int stb_token_probs(const float* logits, long long ld, int n_rows, int n_classes, const int32_t* targets,
                               float* prob_out, int32_t* rank_out, void* stream) {
    STB_REQUIRE(logits && targets && prob_out && n_classes > 0 && ld >= n_classes, "stb_token_probs: bad arguments");
    if (n_rows == 0) return STB_OK;
    stb::ProfScope ps("token_prob", (cudaStream_t)stream, (double)n_rows * n_classes * 4.0);
    return stb::launch(stb::token_prob_kernel, {n_rows, 512, 0, (cudaStream_t)stream}, logits, ld, n_classes, targets, prob_out,
                       rank_out);
}

// ---------------------------------------------------------------------------------------------------------
// test entry points: the LayerNorm and softmax row kernels on their own (include/stablets_b200.h)
// ---------------------------------------------------------------------------------------------------------
static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

extern "C" int stb_layernorm(const float* x, long long rows, int d, const float* gamma, const float* beta, void* out_hi,
                             void* out_lo, float* out_f32, void* stream) {
    // one warp per row, d / 128 float4 per lane held in registers (at most 10)
    STB_REQUIRE(d % 128 == 0 && d >= 128 && d <= 1280, "stb_layernorm: d=%d must be a multiple of 128 in 128..1280", d);
    STB_REQUIRE(rows >= 0, "stb_layernorm: rows=%lld is negative", rows);
    STB_REQUIRE(x && gamma && beta, "stb_layernorm: null x, gamma or beta");
    STB_REQUIRE(out_f32 || out_hi, "stb_layernorm: no output (out_f32 and out_hi are both null)");
    STB_REQUIRE(out_lo == nullptr || out_hi != nullptr, "stb_layernorm: out_lo needs out_hi");
    // x, gamma, beta and out_f32 are accessed as float4, the planes as uint2
    STB_REQUIRE(aligned(x, 16) && aligned(gamma, 16) && aligned(beta, 16) && aligned(out_f32, 16),
                "stb_layernorm: x, gamma, beta and out_f32 must be 16-byte aligned");
    STB_REQUIRE(aligned(out_hi, 8) && aligned(out_lo, 8), "stb_layernorm: out_hi and out_lo must be 8-byte aligned");
    return stb::layernorm(x, rows, d, gamma, beta, (__half*)out_hi, (__half*)out_lo, out_f32, (cudaStream_t)stream);
}

extern "C" int stb_softmax_rows(const float* S, long long n_rows, int n_cols, long long ld_s, int rows_per_slice, int causal,
                                void* p_hi, void* p_lo, long long ld_p, void* stream) {
    // one warp per row, 47 columns per lane held in registers: at most 1504 columns
    STB_REQUIRE(n_cols >= 1 && n_cols <= stb::SM_MAXV * 32, "stb_softmax_rows: n_cols=%d outside 1..%d", n_cols, stb::SM_MAXV * 32);
    STB_REQUIRE(ld_s >= n_cols, "stb_softmax_rows: ld_s=%lld < n_cols=%d", ld_s, n_cols);
    STB_REQUIRE(ld_p >= n_cols && ld_p <= stb::SM_MAXV * 32, "stb_softmax_rows: ld_p=%lld outside n_cols..%d", ld_p,
                stb::SM_MAXV * 32);
    STB_REQUIRE(n_rows >= 0, "stb_softmax_rows: n_rows=%lld is negative", n_rows);
    STB_REQUIRE(!causal || rows_per_slice >= 1, "stb_softmax_rows: rows_per_slice=%d must be positive when causal", rows_per_slice);
    STB_REQUIRE(S && p_hi, "stb_softmax_rows: null S or p_hi");
    return stb::softmax_rows(S, n_rows, n_cols, ld_s, rows_per_slice, causal, (__half*)p_hi, (__half*)p_lo, ld_p,
                             (cudaStream_t)stream);
}
