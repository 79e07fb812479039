// Section 8(f) row 1: non-VAD silence detection of a batch of windows, device part.
//
// Replaces stable_whisper/stabilization/nonvad.py:16-41 (audio2loudness: |x|, k-th largest magnitude as the loudness
// reference, linear down-sampling to one value per 20 ms token) and :58-76 of wav2mask (reflect-padded moving average,
// quantisation to q_levels, -> bool "sound" mask).  The run-length logic that follows (mask2timing / timing2mask on <= 1501
// booleans, nonvad.py:76-88) stays on the host (stable-ts_b200/silence.py), as the reference keeps it in numpy.
//
// One CTA (1024 threads) per window:
//   1. k-th largest |x| by a 3-pass radix select on the float bits (11 + 11 + 10 bits, shared-memory histograms); the
//      window (<= 1.9 MB) is read from HBM once and from L2 twice;
//   2. loudness[i] = fma(l0, |x[i0]| / d, rn(l1 * |x[i1]| / d)): exactly the arithmetic of F.interpolate(mode='linear',
//      align_corners=False) as the reference's CPU path evaluates it (pinned in oracle/silence.py) -- round-to-nearest
//      intrinsics keep the compiler from contracting or reordering anything;
//   3. moving average over the reflect-padded loudness: sequential fp32 sum, then one division (avg_pool1d's order).
// Results are bit-identical to the CPU oracle, so the masks are identical (tests/test_gpu_silence.py).
#include "common.cuh"

namespace stb {

constexpr int SIL_THREADS = 1024;
constexpr int SIL_MAX_TOKENS = 1501;

// Finds, scanning the histogram from its top bin down, the bin that holds the k-th largest element; returns the bin and
// the rank of that element inside the bin (1 = largest of the bin).  Warp 0 only; nbins = 2048 (64 per lane).
__device__ __forceinline__ void select_bin(const uint32_t* hist, uint32_t k, uint32_t& bin_out, uint32_t& k_out) {
    const int lane = threadIdx.x & 31;
    uint32_t mine = 0;
    for (int j = 0; j < 64; ++j) mine += hist[lane * 64 + j];
    // above = number of elements in bins of higher lanes
    uint32_t above = 0;
    for (int l = 31; l >= 0; --l) {
        const uint32_t c = __shfl_sync(0xffffffffu, mine, l);
        if (l > lane) above += c;
    }
    const bool here = above < k && k <= above + mine;
    const uint32_t ballot = __ballot_sync(0xffffffffu, here);
    const int src = __ffs(ballot) - 1;                        // exactly one lane when 1 <= k <= total
    uint32_t bin = 0, kk = 0;
    if (lane == src) {
        uint32_t acc = above;
        for (int j = 63; j >= 0; --j) {
            const uint32_t c = hist[lane * 64 + j];
            if (acc + c >= k) {
                bin = (uint32_t)(lane * 64 + j);
                kk = k - acc;
                break;
            }
            acc += c;
        }
    }
    bin_out = __shfl_sync(0xffffffffu, bin, src < 0 ? 0 : src);
    k_out = __shfl_sync(0xffffffffu, kk, src < 0 ? 0 : src);
}

__global__ void __launch_bounds__(SIL_THREADS)
silence_mask_kernel(const float* __restrict__ audio, long long stride, int n, int k, int token_count, int q_levels, int k_size,
                    const float* __restrict__ thr_in, float* __restrict__ loud_out, uint8_t* __restrict__ mask_out,
                    float* __restrict__ thr_out) {
    __shared__ uint32_t hist[2048];
    __shared__ float L[SIL_MAX_TOKENS + 3];
    __shared__ uint32_t s_bin, s_k;
    const int b = blockIdx.x, tid = threadIdx.x;
    const float* x = audio + (long long)b * stride;

    float thr;
    if (thr_in != nullptr) {
        thr = thr_in[b];
    } else {
        uint32_t prefix = 0, kk = (uint32_t)k;
        // pass 0: bits 31..21, pass 1: bits 20..10, pass 2: bits 9..0 (restricted to the prefix found so far)
        for (int pass = 0; pass < 3; ++pass) {
            for (int i = tid; i < 2048; i += SIL_THREADS) hist[i] = 0;
            __syncthreads();
            for (int i = tid; i < n; i += SIL_THREADS) {
                const uint32_t u = __float_as_uint(fabsf(x[i]));
                if (pass == 0) atomicAdd(&hist[u >> 21], 1u);
                else if (pass == 1) { if ((u >> 21) == prefix) atomicAdd(&hist[(u >> 10) & 0x7FFu], 1u); }
                else { if ((u >> 10) == prefix) atomicAdd(&hist[u & 0x3FFu], 1u); }
            }
            __syncthreads();
            if (tid < 32) {
                uint32_t bin, k2;
                select_bin(hist, kk, bin, k2);
                if (tid == 0) { s_bin = bin; s_k = k2; }
            }
            __syncthreads();
            prefix = (pass == 2) ? ((prefix << 10) | s_bin) : ((prefix << 11) | s_bin);
            kk = s_k;
            __syncthreads();
        }
        thr = __uint_as_float(prefix);
    }
    if (thr_out != nullptr && tid == 0) thr_out[b] = thr;

    const bool silent = thr < 1e-5f;                          // nonvad.py:31-32: loudness = zeros
    const float t175 = __fmul_rn(thr, 1.75f);
    const float denom = (1.0f < t175) ? 1.0f : t175;          // min(1., threshold * 1.75)
    const float scale = __fdiv_rn((float)n, (float)token_count);
    for (int i = tid; i < token_count; i += SIL_THREADS) {
        float v = 0.f;
        if (!silent) {
            const float src = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)i, 0.5f)), 0.5f), 0.f);
            const int i0 = (int)src;
            const int i1 = i0 + (i0 < n - 1 ? 1 : 0);
            const float l1 = __fsub_rn(src, (float)i0);
            const float l0 = __fsub_rn(1.0f, l1);
            const float a0 = __fdiv_rn(fabsf(x[i0]), denom);
            const float a1 = __fdiv_rn(fabsf(x[i1]), denom);
            v = __fmaf_rn(l0, a0, __fmul_rn(l1, a1));
        }
        L[i] = v;
        if (loud_out != nullptr) loud_out[(long long)b * SIL_MAX_TOKENS + i] = v;
    }
    __syncthreads();
    const int p = k_size > 0 ? k_size / 2 : 0;
    const bool pool = p > 0 && p < token_count;
    for (int i = tid; i < token_count; i += SIL_THREADS) {
        float m;
        if (pool) {
            float s = 0.f;
            for (int j = -p; j <= p; ++j) {
                int idx = i + j;
                if (idx < 0) idx = -idx;                                   // reflect (no edge repeat)
                if (idx >= token_count) idx = 2 * (token_count - 1) - idx;
                s = __fadd_rn(s, L[idx]);
            }
            m = __fdiv_rn(s, (float)k_size);
        } else {
            m = L[i];
        }
        if (q_levels > 0) m = rintf(__fmul_rn(m, (float)q_levels));     // torch.round: half to even
        mask_out[(long long)b * SIL_MAX_TOKENS + i] = (m != 0.f) ? 1 : 0;
    }
}

}  // namespace stb

extern "C" int stb_silence_mask(const float* audio, int B, int n_samples, long long stride, int k, int token_count, int q_levels,
                                int k_size, const float* thr_in, float* loudness_out, uint8_t* mask_out, float* thr_out,
                                void* stream) {
    STB_REQUIRE(audio && mask_out && B >= 1, "stb_silence_mask: null pointer");
    STB_REQUIRE(n_samples >= 1 && stride >= n_samples, "stb_silence_mask: bad sample count / stride");
    STB_REQUIRE(token_count > 2 && token_count <= stb::SIL_MAX_TOKENS, "stb_silence_mask: token_count %d outside (2, %d]", token_count,
                stb::SIL_MAX_TOKENS);
    STB_REQUIRE(thr_in != nullptr || (k >= 1 && k <= n_samples), "stb_silence_mask: k = %d must be in [1, n] (or pass thresholds)", k);
    STB_REQUIRE(k_size == 0 || (k_size % 2 == 1 && k_size <= 31), "stb_silence_mask: kernel size must be odd");
    cudaStream_t st = (cudaStream_t)stream;
    stb::ProfScope ps("silence_mask", st, (double)B * n_samples * 4.0);
    return stb::launch(stb::silence_mask_kernel, {B, stb::SIL_THREADS, 0, st}, audio, stride, n_samples, k, token_count, q_levels,
                       k_size, thr_in, loudness_out, mask_out, thr_out);
}
