// Section 8(f) row 3 -- audio ingest on the device: interleaved PCM of a decoded WAV (any rate, 1..8 channels, s16 / s32 / f32)
// -> mono 16 kHz fp32, the waveform the hot path (stb_logmel, stb_silence_mask) starts from.  Replaces the reference's
// ffmpeg pipe (stable_whisper/audio/utils.py:96-125: `ffmpeg -ac 1 -ar 16000 -f s16le` then int16 -> float32 / 32768).
//
// One pass: sample-format conversion, down-mix (equal-weight mean of the channels, ffmpeg's default stereo -> mono),
// polyphase FIR resampling by L / M, optional re-quantisation to the s16 grid (what the reference's s16le pipe does).
//   y[m] = sum_j tab[(m M) mod L][j] * x[(m M) div L - half + j],     tab = Kaiser-windowed sinc, [L][taps] fp32, host-built
// HBM-bound: every input sample is read ~taps * L / M times, but consecutive outputs share their taps' inputs, so the reads
// are served by L1/L2; algorithmic bytes = n_in * channels * sample_bytes + n_out * 4.
#include "common.cuh"

namespace stb {

template <int FMT>   // 0: s16, 1: s32, 2: f32
__device__ __forceinline__ float pcm_at(const void* pcm, long long i) {
    if (FMT == 0) return (float)__ldg(reinterpret_cast<const short*>(pcm) + i) * (1.0f / 32768.0f);
    if (FMT == 1) return (float)((double)__ldg(reinterpret_cast<const int*>(pcm) + i) * (1.0 / 2147483648.0));
    return __ldg(reinterpret_cast<const float*>(pcm) + i);
}

template <int FMT>
__global__ void __launch_bounds__(256)
resample_mono_kernel(const void* __restrict__ pcm, int channels, long long n_in, int L, int M, const float* __restrict__ tab,
                     int taps, float* __restrict__ out, long long n_out, int quantize_s16) {
    const int half = taps / 2;
    const float inv_c = 1.0f / (float)channels;
    for (long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x; m < n_out; m += (long long)gridDim.x * blockDim.x) {
        const long long pos = m * M;
        const long long n0 = pos / L;
        const int phase = (int)(pos - n0 * L);
        const float* t = tab + (long long)phase * taps;
        float acc = 0.f;
        for (int j = 0; j < taps; ++j) {
            const long long n = n0 - half + j;
            if (n < 0 || n >= n_in) continue;
            float x = 0.f;
            for (int c = 0; c < channels; ++c) x += pcm_at<FMT>(pcm, n * channels + c);
            acc = fmaf(__ldg(t + j), x * inv_c, acc);
        }
        if (quantize_s16) {                                  // the s16le pipe: round to nearest, saturate, back to float
            float q = rintf(acc * 32768.0f);
            q = fminf(fmaxf(q, -32768.0f), 32767.0f);
            acc = q * (1.0f / 32768.0f);
        }
        out[m] = acc;
    }
}

}  // namespace stb

extern "C" int stb_resample_mono(const void* pcm, int sample_format, int channels, long long n_frames_in, int L, int M,
                                 const float* table, int taps, float* out, long long n_out, int quantize_s16, void* stream) {
    STB_REQUIRE(pcm && table && out, "stb_resample_mono: null pointer");
    STB_REQUIRE(sample_format >= 0 && sample_format <= 2, "stb_resample_mono: sample_format must be 0 (s16), 1 (s32) or 2 (f32)");
    STB_REQUIRE(channels >= 1 && channels <= 8 && n_frames_in >= 0 && n_out >= 0, "stb_resample_mono: bad sizes");
    STB_REQUIRE(L >= 1 && M >= 1 && taps >= 1 && (taps & 1), "stb_resample_mono: L, M >= 1 and an odd tap count are required");
    if (n_out == 0) return STB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int sb = sample_format == 0 ? 2 : 4;
    stb::ProfScope ps("resample_mono", st, (double)n_frames_in * channels * sb + (double)n_out * 4.0);
    long long blocks = (n_out + 255) / 256;
    const long long cap = (long long)stb::sm_count() * 16;
    if (blocks > cap) blocks = cap;
    const auto kernel = sample_format == 0 ? stb::resample_mono_kernel<0>
                        : sample_format == 1 ? stb::resample_mono_kernel<1>
                                             : stb::resample_mono_kernel<2>;
    return stb::launch(kernel, {(unsigned)blocks, 256, 0, st}, pcm, channels, n_frames_in, L, M, table, taps, out, n_out, quantize_s16);
}
