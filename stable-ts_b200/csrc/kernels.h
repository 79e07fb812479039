// Internal (non-ABI) declarations shared between the translation units of libstablets_b200.so.
#pragma once
#include "common.cuh"

namespace stb {

// cached 4-D fp16 TMA tensor map over one plane of a K-major operand view (gemm_tc.cu); perm[i] tells which of
// (row=0, head=1, batch=2, zero=3) feeds TMA coordinate 1+i
struct TmapVal {
    CUtensorMap map;
    int perm[3];
};
int make_tmap(const void* base, int rows, int k, int H, int B, long long rs, long long hs, long long bs, int box_rows,
              TmapVal* out);
int fused_attention(const stb_operand& q, const stb_operand& k, const stb_operand& vT, int n_batch, int n_head, int Mq, int Mk,
                    void* out_hi, void* out_lo, long long ld_out, long long out_h, long long out_b, cudaStream_t st);

int gemm(const stb_operand& A, const stb_operand& B, int n_batch, int n_head, const stb_epilogue& ep, cudaStream_t st);

int layernorm(const float* x, long long rows, int d, const float* gamma, const float* beta, __half* hi, __half* lo,
              float* out_f32, cudaStream_t st);
int softmax_rows(const float* S, long long n_rows, int n_cols, long long ld_s, int rows_per_slice, int causal, __half* hi,
                 __half* lo, long long ld_p, cudaStream_t st);
int embed_tokens(const int32_t* tokens, long long n_tok, int M, int offset, int d, const float* emb, const float* pos,
                 float* x, cudaStream_t st);
int mel_repack(const float* mel, int B, int C, int T, __half* hi, __half* lo, cudaStream_t st);
int zero_pad_rows(__half* hi, __half* lo, int B, int C, int T, cudaStream_t st);

// seq_off (nullable) [B]: first cache row of each sequence (ragged initial tokens right-aligned on the shared counter)
int decode_attn_self(const float* qkv, float* Kc, float* Vc, int B, int H, int d, int ctx, const int32_t* pos,
                     const int32_t* seq_off, __half* oh, __half* ol, float* of, cudaStream_t st);
// decode-step view of one layer's cross K / V: fp16 planes, head-major [B][H][T][64] (K is the GEMM hi plane itself)
struct CrossDecodeKV {
    const __half* k_hi;
    const __half* v_hi;
};
int decode_attn_cross(const float* q, const CrossDecodeKV& kv, int B, int H, int d, float* partial, int* tickets, __half* oh,
                      __half* ol, float* of, cudaStream_t st);
int decode_cross_splits();
int v_headmajor(const __half* vT_hi, int BH, int T, int Tp, __half* v_hi, cudaStream_t st);
int gemv(const void* x_hi, const void* x_lo, int B, int K, const void* w_hi, const void* w_lo, int N, const float* bias,
         int act, const float* res, long long ld_res, float* out_f32, void* out_hi, void* out_lo, long long ld_out,
         cudaStream_t st);
// one Linear of the decode step in one launch: swapped wgmma GEMM, split-K across a thread-block cluster, partial tiles
// reduced over distributed shared memory, fused bias / GELU / residual epilogue (decode_linear.cu)
int decode_linear(const void* x_hi, const void* x_lo, int B, int k, const void* w_hi, const void* w_lo, int n, const float* bias,
                  int act, const float* res, long long ld_res, float* out_f32, void* out_hi, void* out_lo, long long ld_out,
                  cudaStream_t st);
int decode_linear_split(int n, int k);
int embed_step(const int32_t* tokens, const int32_t* pos, const int32_t* seq_off, int n_pos, int B, int d, const float* emb,
               const float* posemb, float* x, cudaStream_t st);
int bump_pos(int32_t* pos, cudaStream_t st);

}  // namespace stb
