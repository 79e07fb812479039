// a1 / K1: log-mel front-end.  Replaces whisper.audio.log_mel_spectrogram (+ pad_or_trim to 3000 frames):
//   zero-pad to `padded` samples -> STFT(n_fft 400, hop 160, periodic Hann, center/reflect) -> drop last frame ->
//   |.|^2 -> mel filterbank [n_mels x 201] -> log10(max(.,1e-10)) -> max(x, max(x) - 8) -> (x + 4) / 4.
// Call sites: stable_whisper/alignment.py:411-413 (align, padded = 480000), :660-661 (refine: padded = n, max over the
// whole batch), original_whisper.py:528-530.
//
// Kernel 1: one CTA per (window, 8 frames).  Windowed samples -> smem; thread k computes DFT bin k for the 8 frames
// from a 400-entry twiddle table in smem (index (k*n) mod 400 walked incrementally, exact fp32 table from the host);
// power -> smem; mel projection; log10; per-CTA max to the workspace.
// Kernel 2: reduce the maxima (per window or over the batch), apply the 8 dB floor + affine, zero frames >= n_frames.
#include "common.cuh"

namespace stb {

constexpr int LM_FR = 8;        // frames per CTA
constexpr int LM_NFFT = 400;
constexpr int LM_BINS = 201;
constexpr int LM_THREADS = 256;

__global__ void __launch_bounds__(LM_THREADS)
logmel_kernel(const float* __restrict__ audio, int n_samples, int padded, int n_frames, int n_mels,
              const float* __restrict__ filters, const float* __restrict__ window, const float* __restrict__ dft,
              float* __restrict__ mel_out, float* __restrict__ blockmax) {
    __shared__ float s_x[LM_FR][LM_NFFT];
    __shared__ float2 s_tw[LM_NFFT];
    __shared__ float s_pw[LM_FR][LM_BINS + 3];
    __shared__ float s_red[LM_THREADS / 32];
    const int b = blockIdx.y;
    const int f0 = blockIdx.x * LM_FR;
    const float* a = audio + (long long)b * n_samples;

    for (int i = threadIdx.x; i < LM_NFFT; i += LM_THREADS) s_tw[i] = reinterpret_cast<const float2*>(dft)[i];
    for (int i = threadIdx.x; i < LM_FR * LM_NFFT; i += LM_THREADS) {
        const int f = i / LM_NFFT, n = i - f * LM_NFFT;
        int idx = (f0 + f) * 160 + n - 200;                 // center=True: frame f starts at f*hop - n_fft/2
        if (idx < 0) idx = -idx;                            // reflect (no edge repeat)
        if (idx >= padded) idx = 2 * (padded - 1) - idx;
        float v = 0.f;
        if (f0 + f < n_frames && idx >= 0 && idx < n_samples) v = a[idx];
        s_x[f][n] = v * __ldg(window + n);
    }
    __syncthreads();

    const int k = threadIdx.x;
    if (k < LM_BINS) {
        float re[LM_FR], im[LM_FR];
#pragma unroll
        for (int f = 0; f < LM_FR; ++f) re[f] = im[f] = 0.f;
        int idx = 0;
        for (int n = 0; n < LM_NFFT; ++n) {
            const float2 tw = s_tw[idx];                    // (cos, sin)(2 pi k n / 400)
#pragma unroll
            for (int f = 0; f < LM_FR; ++f) {
                const float xv = s_x[f][n];
                re[f] = fmaf(xv, tw.x, re[f]);
                im[f] = fmaf(xv, tw.y, im[f]);
            }
            idx += k;
            if (idx >= LM_NFFT) idx -= LM_NFFT;
        }
#pragma unroll
        for (int f = 0; f < LM_FR; ++f) s_pw[f][k] = re[f] * re[f] + im[f] * im[f];
    }
    __syncthreads();

    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n_mels * LM_FR; i += LM_THREADS) {
        const int m = i / LM_FR, f = i - m * LM_FR;
        if (f0 + f < n_frames) {
            const float* w = filters + (long long)m * LM_BINS;
            float acc = 0.f;
            for (int kk = 0; kk < LM_BINS; ++kk) acc = fmaf(__ldg(w + kk), s_pw[f][kk], acc);
            const float lv = log10f(fmaxf(acc, 1e-10f));
            mel_out[((long long)b * n_mels + m) * STB_N_FRAMES + f0 + f] = lv;
            mx = fmaxf(mx, lv);
        }
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m2 = s_red[0];
        for (int i = 1; i < LM_THREADS / 32; ++i) m2 = fmaxf(m2, s_red[i]);
        blockmax[(long long)b * gridDim.x + blockIdx.x] = m2;
    }
}

__global__ void __launch_bounds__(256)
logmel_finalize_kernel(float* __restrict__ mel, int n_mels, int n_frames, const float* __restrict__ blockmax,
                       int blocks_per_item, int B, int batch_global) {
    __shared__ float s_red[8];
    __shared__ float s_max;
    const int b = blockIdx.y;
    const float* bm = batch_global ? blockmax : blockmax + (long long)b * blocks_per_item;
    const int nb = batch_global ? blocks_per_item * B : blocks_per_item;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < nb; i += blockDim.x) mx = fmaxf(mx, bm[i]);
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m2 = s_red[0];
        for (int i = 1; i < 8; ++i) m2 = fmaxf(m2, s_red[i]);
        s_max = m2;
    }
    __syncthreads();
    const float floorv = s_max - 8.0f;
    float* base = mel + (long long)b * n_mels * STB_N_FRAMES;
    const long long total = (long long)n_mels * STB_N_FRAMES;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int f = (int)(i % STB_N_FRAMES);
        base[i] = (f < n_frames) ? (fmaxf(base[i], floorv) + 4.0f) / 4.0f : 0.0f;
    }
}

}  // namespace stb

extern "C" int stb_logmel(const float* audio, int B, int n_samples, int padded_samples, int n_mels, const float* filters,
                          const float* window, const float* dft_table, int batch_global_max, float* mel_out, void* ws,
                          size_t ws_bytes, void* stream) {
    STB_REQUIRE(audio && filters && window && dft_table && mel_out && ws, "stb_logmel: null pointer");
    STB_REQUIRE(B >= 1 && n_samples >= 1 && padded_samples >= n_samples && padded_samples <= 480000 + 160,
                "stb_logmel: bad sample counts n=%d padded=%d", n_samples, padded_samples);
    STB_REQUIRE(padded_samples > 200, "stb_logmel: reflect padding needs more than 200 samples");
    STB_REQUIRE(n_mels == 80 || n_mels == 128, "stb_logmel: n_mels must be 80 or 128");
    int n_frames = padded_samples / 160;                     // 1 + n/160 STFT frames, last one dropped
    if (n_frames > STB_N_FRAMES) n_frames = STB_N_FRAMES;    // pad_or_trim
    const int blocks = stb::cdiv(STB_N_FRAMES, stb::LM_FR);
    STB_REQUIRE(ws_bytes >= (size_t)B * blocks * sizeof(float), "stb_logmel: workspace too small (%zu < %zu)", ws_bytes,
                (size_t)B * blocks * sizeof(float));
    cudaStream_t st = (cudaStream_t)stream;
    // every CTA writes its max (-inf when it holds no valid frame) so the workspace needs no initialisation
    stb::ProfScope ps("logmel(2 kernels)", st, (double)B * (n_samples * 4.0 + n_mels * 3000 * 4.0));
    STB_TRY(stb::launch(stb::logmel_kernel, {dim3(blocks, B), stb::LM_THREADS, 0, st}, audio, n_samples, padded_samples, n_frames,
                        n_mels, filters, window, dft_table, mel_out, (float*)ws));
    return stb::launch(stb::logmel_finalize_kernel, {dim3(64, B), 256, 0, st}, mel_out, n_mels, n_frames, (const float*)ws, blocks,
                       B, batch_global_max);
}
