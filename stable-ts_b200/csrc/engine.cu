// Model handle and the per-window forward passes as launch sequences over the sm_90a kernels.
//
//   stb_encoder_forward   a2: whisper.model.AudioEncoder.forward          (reference call site stable_whisper/timing.py:60)
//   stb_cross_kv          cross-attention K / V^T of every decoder layer  (whisper's kv_cache for cross_attn.key/value)
//   stb_decoder_forward   a3: TextDecoder.forward with the cross-attention `qk` of selected heads captured
//                             (stable_whisper/timing.py:50-61 under disable_sdpa)
//
// Data layout in HBM (all caller-owned):
//   residual stream          fp32  [rows][d]
//   GEMM inputs              split fp16 planes written by the producing kernel's epilogue (LayerNorm, GELU, softmax...)
//   self-attention scores    fp32  [B][H][Mq][ldk]  (decoder, causal; ldk = keys rounded up to 8); probabilities split,
//                            same shape.  The encoder and the cross-attention keep them in registers (attention_tc.cu)
//   V                        stored transposed [B][H][64][ldk] so P.V is a K-major GEMM
//   conv inputs              time-major [B][T+2][C] with zero pad rows: overlapping TMA rows (stride C or 2C, width 3C)
//                            are the im2col matrix, no copy
#include <string.h>
#include <vector>

#include "common.cuh"
#include "kernels.h"

struct stb_model {
    stb_dims dims;
    int prec;
    const void* t[STB_T_LAYER_BASE][2];
    struct Layer { const void* p[STB_L_COUNT][2]; };
    std::vector<Layer> enc, dec;
};

namespace stb {

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

struct Carver {               // bump allocator over a caller-provided workspace
    char* base;
    size_t off = 0;
    explicit Carver(void* p) : base((char*)p) {}
    template <typename T> T* take(size_t n) {
        T* r = reinterpret_cast<T*>(base ? base + off : nullptr);
        off = align_up(off + n * sizeof(T));
        return r;
    }
};

struct Split {                // a split-fp16 matrix in the workspace
    __half* hi;
    __half* lo;
};
static Split take_split(Carver& c, size_t n, bool lo) {
    Split s;
    s.hi = c.take<__half>(n);
    s.lo = lo ? c.take<__half>(n) : nullptr;
    return s;
}

static stb_operand opnd(const void* hi, const void* lo, int rows, int k, long long rs, long long hs = 0, long long bs = 0) {
    stb_operand o;
    o.hi = hi; o.lo = lo; o.rows = rows; o.k = k; o.row_stride = rs; o.h_stride = hs; o.b_stride = bs;
    return o;
}
static const __half* offs(const void* p, long long elems) { return p ? (const __half*)p + elems : nullptr; }
static __half* offs(__half* p, long long elems) { return p ? p + elems : nullptr; }

static stb_epilogue ep_split(Split out, long long ld, const float* bias, int act, long long out_h = 0, long long out_b = 0) {
    stb_epilogue e;
    memset(&e, 0, sizeof(e));
    e.out_hi = out.hi; e.out_lo = out.lo; e.ld_out = ld; e.out_h_stride = out_h; e.out_b_stride = out_b;
    e.bias = bias; e.act = act; e.alpha = 1.0f;
    return e;
}
static stb_epilogue ep_f32(float* out, long long ld, const float* bias, const float* res, long long ld_res, float alpha = 1.0f) {
    stb_epilogue e;
    memset(&e, 0, sizeof(e));
    e.out_f32 = out; e.ld_out = ld; e.bias = bias; e.residual = res; e.ld_res = ld_res; e.alpha = alpha;
    return e;
}

#define W_HI(layer, id) ((layer).p[id][0])
#define W_LO(layer, id) (m->prec == STB_PREC_FP16X3 ? (layer).p[id][1] : nullptr)
#define W_F32(layer, id) ((const float*)(layer).p[id][0])

// ---- one causal multi-head attention: scores, softmax, P.V.  q / k are split views with (row, head, batch) strides. ----
struct AttnBufs {
    float* S;          // [B][H][Mq][ldk]
    Split P;           // same shape
    Split vT;          // [B][H][64][ldk]
    Split out;         // [B*Mq][d]
};

static int attention(const stb_model* m, int B, int H, int d, int Mq, int Mk, int ldk, const stb_operand& q,
                     const stb_operand& k, const AttnBufs& bufs, cudaStream_t st) {
    // S = (q k^T) / 8  (whisper scales q and k by 64^-0.25 each; head_dim is 64 for every released model)
    stb_epilogue e = ep_f32(bufs.S, ldk, nullptr, nullptr, 0, 0.125f);
    e.out_h_stride = (long long)Mq * ldk;
    e.out_b_stride = (long long)H * Mq * ldk;
    STB_TRY(gemm(q, k, B, H, e, st));
    STB_TRY(softmax_rows(bufs.S, (long long)B * H * Mq, Mk, ldk, Mq, 1, bufs.P.hi, bufs.P.lo, ldk, st));
    stb_operand p = opnd(bufs.P.hi, bufs.P.lo, Mq, ldk, ldk, (long long)Mq * ldk, (long long)H * Mq * ldk);
    stb_operand v = opnd(bufs.vT.hi, bufs.vT.lo, 64, ldk, ldk, 64LL * ldk, (long long)d * ldk);
    stb_epilogue eo = ep_split(bufs.out, d, nullptr, STB_ACT_NONE, 64, (long long)Mq * d);
    STB_TRY(gemm(p, v, B, H, eo, st));
    return STB_OK;
}

// V^T projection: rows of `x` (per batch item) times W_v^T, stored transposed into vT [B][H*64][ldk]
static int project_vT(const stb_model* m, const Split& x, int B, int rows, int d, const void* w_hi, const void* w_lo,
                      const float* bias, Split vT, int ldk, cudaStream_t st) {
    const bool lo = m->prec == STB_PREC_FP16X3;
    STB_CUDA_OK(cudaMemsetAsync(vT.hi, 0, (size_t)B * d * ldk * sizeof(__half), st));
    if (lo) STB_CUDA_OK(cudaMemsetAsync(vT.lo, 0, (size_t)B * d * ldk * sizeof(__half), st));
    stb_operand a = opnd(x.hi, x.lo, rows, d, d, 0, (long long)rows * d);
    stb_operand w = opnd(w_hi, w_lo, d, d, d);
    stb_epilogue e = ep_split(vT, ldk, bias, STB_ACT_NONE, 0, (long long)d * ldk);
    e.transposed = 1;
    return gemm(a, w, B, 1, e, st);
}

static int linear(const stb_model* m, const Split& x, long long rows, int k, const void* w_hi, const void* w_lo, int n,
                  const stb_epilogue& e, cudaStream_t st) {
    STB_REQUIRE(rows < (1LL << 31), "linear: too many rows");
    stb_operand a = opnd(x.hi, x.lo, (int)rows, k, k);
    stb_operand w = opnd(w_hi, w_lo, n, k, k);
    return gemm(a, w, 1, 1, e, st);
}

// ---------------------------------------------------------------------------------------------------------
// encoder
// ---------------------------------------------------------------------------------------------------------
struct EncWs {
    Split melT, h1, ln, qk, vT, attn, hid;
    float* x;
    size_t bytes;
};
static EncWs carve_encoder(const stb_model* m, int B, void* ws) {
    const stb_dims& D = m->dims;
    const bool lo = m->prec == STB_PREC_FP16X3;
    const size_t T = D.n_audio_ctx, Tp = STB_KPAD, d = D.n_audio_state, C = D.n_mels;
    Carver c(ws);
    EncWs w;
    w.melT = take_split(c, (size_t)B * (STB_N_FRAMES + 2) * C, lo);
    w.h1 = take_split(c, (size_t)B * (STB_N_FRAMES + 2) * d, lo);
    w.x = c.take<float>((size_t)B * T * d);
    w.ln = take_split(c, (size_t)B * T * d, lo);
    w.qk = take_split(c, (size_t)B * T * 2 * d, lo);
    w.vT = take_split(c, (size_t)B * d * Tp, lo);
    w.attn = take_split(c, (size_t)B * T * d, lo);
    w.hid = take_split(c, (size_t)B * T * 4 * d, lo);
    w.bytes = c.off;
    return w;
}

static int encoder_forward(stb_model* m, const float* mel, int B, float* xa_f32, __half* xa_hi, __half* xa_lo, void* ws,
                           cudaStream_t st) {
    const stb_dims& D = m->dims;
    const bool lo = m->prec == STB_PREC_FP16X3;
    const int T = D.n_audio_ctx, Tp = STB_KPAD, d = D.n_audio_state, H = D.n_audio_head, C = D.n_mels, F = STB_N_FRAMES;
    EncWs w = carve_encoder(m, B, ws);
    const void* const(*t)[2] = m->t;

    // conv1 (k=3, pad 1) + GELU as a GEMM over the overlapping-row view of the time-major mel
    STB_TRY(mel_repack(mel, B, C, F, w.melT.hi, w.melT.lo, st));
    STB_TRY(zero_pad_rows(w.h1.hi, w.h1.lo, B, d, F, st));
    {
        Split out = {offs(w.h1.hi, d), offs(w.h1.lo, d)};                       // skip the leading pad row
        stb_epilogue e = ep_split(out, d, (const float*)t[STB_T_ENC_CONV1_B][0], STB_ACT_GELU, 0, (long long)(F + 2) * d);
        stb_operand wt = opnd(t[STB_T_ENC_CONV1_W][0], lo ? t[STB_T_ENC_CONV1_W][1] : nullptr, d, 3 * C, 3 * C);
        stb_operand a = opnd(w.melT.hi, w.melT.lo, F, 3 * C, C, 0, (long long)(F + 2) * C);
        STB_TRY(gemm(a, wt, B, 1, e, st));
    }
    // conv2 (k=3, stride 2, pad 1) + GELU + sinusoidal positions -> residual stream x [B][1500][d]
    {
        stb_epilogue e = ep_f32(w.x, d, (const float*)t[STB_T_ENC_CONV2_B][0], (const float*)t[STB_T_ENC_POS][0], d);
        e.act = STB_ACT_GELU;
        e.out_b_stride = (long long)T * d;
        e.res_b_stride = 0;
        stb_operand wt = opnd(t[STB_T_ENC_CONV2_W][0], lo ? t[STB_T_ENC_CONV2_W][1] : nullptr, d, 3 * d, 3 * d);
        stb_operand a = opnd(w.h1.hi, w.h1.lo, T, 3 * d, 2 * d, 0, (long long)(F + 2) * d);
        STB_TRY(gemm(a, wt, B, 1, e, st));
    }
    const long long rows = (long long)B * T;
    for (int l = 0; l < D.n_audio_layer; ++l) {
        const stb_model::Layer& L = m->enc[l];
        STB_TRY(layernorm(w.x, rows, d, W_F32(L, STB_L_ATTN_LN_G), W_F32(L, STB_L_ATTN_LN_B), w.ln.hi, w.ln.lo, nullptr, st));
        // q,k projection (2d columns) row-major; v projection transposed
        STB_TRY(linear(m, w.ln, rows, d, W_HI(L, STB_L_QKV_W), W_LO(L, STB_L_QKV_W), 2 * d,
                       ep_split(w.qk, 2 * d, W_F32(L, STB_L_QKV_B), STB_ACT_NONE), st));
        STB_TRY(project_vT(m, w.ln, B, T, d, offs(W_HI(L, STB_L_QKV_W), 2LL * d * d), offs(W_LO(L, STB_L_QKV_W), 2LL * d * d),
                           W_F32(L, STB_L_QKV_B) + 2 * d, w.vT, Tp, st));
        stb_operand q = opnd(w.qk.hi, w.qk.lo, T, 64, 2 * d, 64, (long long)T * 2 * d);
        stb_operand k = opnd(offs(w.qk.hi, d), offs(w.qk.lo, d), T, 64, 2 * d, 64, (long long)T * 2 * d);
        stb_operand v = opnd(w.vT.hi, w.vT.lo, 64, Tp, Tp, 64LL * Tp, (long long)d * Tp);
        // fused wgmma attention: scores never leave the SM
        STB_TRY(fused_attention(q, k, v, B, H, T, T, w.attn.hi, w.attn.lo, d, 64, (long long)T * d, st));
        STB_TRY(linear(m, w.attn, rows, d, W_HI(L, STB_L_OUT_W), W_LO(L, STB_L_OUT_W), d,
                       ep_f32(w.x, d, W_F32(L, STB_L_OUT_B), w.x, d), st));
        STB_TRY(layernorm(w.x, rows, d, W_F32(L, STB_L_MLP_LN_G), W_F32(L, STB_L_MLP_LN_B), w.ln.hi, w.ln.lo, nullptr, st));
        STB_TRY(linear(m, w.ln, rows, d, W_HI(L, STB_L_FC1_W), W_LO(L, STB_L_FC1_W), 4 * d,
                       ep_split(w.hid, 4 * d, W_F32(L, STB_L_FC1_B), STB_ACT_GELU), st));
        STB_TRY(linear(m, w.hid, rows, 4 * d, W_HI(L, STB_L_FC2_W), W_LO(L, STB_L_FC2_W), d,
                       ep_f32(w.x, d, W_F32(L, STB_L_FC2_B), w.x, d), st));
    }
    STB_TRY(layernorm(w.x, rows, d, (const float*)t[STB_T_ENC_LNPOST_G][0], (const float*)t[STB_T_ENC_LNPOST_B][0], xa_hi,
                      lo ? xa_lo : nullptr, xa_f32, st));
    return STB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// cross K / V^T for all decoder layers
// ---------------------------------------------------------------------------------------------------------
struct CrossKV {             // per layer: K split head-major [B][H][T][64], vT split [B][H][64][Tp], V hi head-major
    size_t k_elems, v_elems, layer_halfs;
};
static CrossKV cross_layout(const stb_model* m, int B) {
    CrossKV c;
    c.k_elems = (size_t)B * m->dims.n_audio_ctx * m->dims.n_text_state;
    c.v_elems = (size_t)B * m->dims.n_text_state * STB_KPAD;
    // per layer: K hi | K lo | V^T hi | V^T lo | V hi head-major (k_elems halfs; the decode step's fp16 V, decode.cu)
    c.layer_halfs = 2 * (2 * c.k_elems + c.v_elems) + c.k_elems;
    return c;
}
static void cross_ptrs(const stb_model* m, int B, const void* base, int l, Split& K, Split& vT, CrossDecodeKV* Vd = nullptr) {
    CrossKV c = cross_layout(m, B);
    __half* p = (__half*)base + (size_t)l * c.layer_halfs;
    const bool lo = m->prec == STB_PREC_FP16X3;
    K.hi = p; K.lo = lo ? p + c.k_elems : nullptr;
    vT.hi = p + 2 * c.k_elems; vT.lo = lo ? p + 2 * c.k_elems + c.v_elems : nullptr;
    if (Vd) {
        Vd->k_hi = K.hi;
        Vd->v_hi = p + 2 * c.k_elems + 2 * c.v_elems;
    }
}

static int cross_kv(stb_model* m, const __half* xa_hi, const __half* xa_lo, int B, void* out, bool decode_layout, cudaStream_t st) {
    const stb_dims& D = m->dims;
    const int T = D.n_audio_ctx, d = D.n_text_state;
    STB_REQUIRE(D.n_audio_state == D.n_text_state, "cross_kv: audio/text widths differ");
    Split xa = {(__half*)xa_hi, m->prec == STB_PREC_FP16X3 ? (__half*)xa_lo : nullptr};
    for (int l = 0; l < D.n_text_layer; ++l) {
        const stb_model::Layer& L = m->dec[l];
        Split K, vT;
        CrossDecodeKV Vd;
        cross_ptrs(m, B, out, l, K, vT, &Vd);
        {   // K head-major [B][H][T][64] (sequential 192 KB streams per (sequence, head) for the decode-step kernel):
            // per-head batched GEMM, A = xa broadcast over heads, B = rows h*64..h*64+63 of W_k; whisper's key has no bias
            const int H = D.n_text_head;
            stb_operand a = opnd(xa.hi, xa.lo, T, d, d, 0, (long long)T * d);
            stb_operand wk = opnd(W_HI(L, STB_L_CKV_W), W_LO(L, STB_L_CKV_W), 64, d, d, 64LL * d, 0);
            stb_epilogue e = ep_split(K, 64, nullptr, STB_ACT_NONE, (long long)T * 64, (long long)H * T * 64);
            STB_TRY(gemm(a, wk, B, H, e, st));
        }
        STB_TRY(project_vT(m, xa, B, T, d, offs(W_HI(L, STB_L_CKV_W), (long long)d * d), offs(W_LO(L, STB_L_CKV_W), (long long)d * d),
                           W_F32(L, STB_L_CKV_B) + d, vT, STB_KPAD, st));
        if (decode_layout)     // head-major fp16 copy of V for the decode-step kernel (contiguous per (sequence, head), like K)
            STB_TRY(v_headmajor(vT.hi, B * D.n_text_head, T, STB_KPAD, const_cast<__half*>(Vd.v_hi), st));
    }
    return STB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// teacher-forced decoder with cross-attention capture
// ---------------------------------------------------------------------------------------------------------
struct DecWs {
    float* x;
    Split ln, qk, vT, Ps, attn, q, hid;
    float* Ss;
    size_t bytes;
};
static DecWs carve_decoder(const stb_model* m, int B, int M, void* ws) {
    const stb_dims& D = m->dims;
    const bool lo = m->prec == STB_PREC_FP16X3;
    const size_t d = D.n_text_state, H = D.n_text_head, Mp = (M + 7) & ~7;
    Carver c(ws);
    DecWs w;
    w.x = c.take<float>((size_t)B * M * d);
    w.ln = take_split(c, (size_t)B * M * d, lo);
    w.qk = take_split(c, (size_t)B * M * 2 * d, lo);
    w.vT = take_split(c, (size_t)B * d * Mp, lo);
    w.Ss = c.take<float>((size_t)B * H * M * Mp);
    w.Ps = take_split(c, (size_t)B * H * M * Mp, lo);
    w.attn = take_split(c, (size_t)B * M * d, lo);
    w.q = take_split(c, (size_t)B * M * d, lo);
    w.hid = take_split(c, (size_t)B * M * 4 * d, lo);
    w.bytes = c.off;
    return w;
}

static int decoder_forward(stb_model* m, const int32_t* tokens, int B, int M, const void* ckv, float* logits,
                           long long ld_logits, float* qk_out, const int32_t* sel, int n_sel, void* ws, cudaStream_t st) {
    const stb_dims& D = m->dims;
    const int d = D.n_text_state, H = D.n_text_head, T = D.n_audio_ctx, Tp = STB_KPAD, Mp = (M + 7) & ~7;
    const void* const(*t)[2] = m->t;
    DecWs w = carve_decoder(m, B, M, ws);
    const long long rows = (long long)B * M;
    const int n_sel_total = n_sel < 0 ? D.n_text_layer * H : n_sel;

    STB_TRY(embed_tokens(tokens, rows, M, 0, d, (const float*)t[STB_T_DEC_TOKEMB_F32][0], (const float*)t[STB_T_DEC_POS][0], w.x, st));
    for (int l = 0; l < D.n_text_layer; ++l) {
        const stb_model::Layer& L = m->dec[l];
        // ---- causal self-attention ----
        STB_TRY(layernorm(w.x, rows, d, W_F32(L, STB_L_ATTN_LN_G), W_F32(L, STB_L_ATTN_LN_B), w.ln.hi, w.ln.lo, nullptr, st));
        STB_TRY(linear(m, w.ln, rows, d, W_HI(L, STB_L_QKV_W), W_LO(L, STB_L_QKV_W), 2 * d,
                       ep_split(w.qk, 2 * d, W_F32(L, STB_L_QKV_B), STB_ACT_NONE), st));
        STB_TRY(project_vT(m, w.ln, B, M, d, offs(W_HI(L, STB_L_QKV_W), 2LL * d * d), offs(W_LO(L, STB_L_QKV_W), 2LL * d * d),
                           W_F32(L, STB_L_QKV_B) + 2 * d, w.vT, Mp, st));
        {
            stb_operand q = opnd(w.qk.hi, w.qk.lo, M, 64, 2 * d, 64, (long long)M * 2 * d);
            stb_operand k = opnd(offs(w.qk.hi, d), offs(w.qk.lo, d), M, 64, 2 * d, 64, (long long)M * 2 * d);
            AttnBufs ab = {w.Ss, w.Ps, w.vT, w.attn};
            STB_TRY(attention(m, B, H, d, M, M, Mp, q, k, ab, st));
        }
        STB_TRY(linear(m, w.attn, rows, d, W_HI(L, STB_L_OUT_W), W_LO(L, STB_L_OUT_W), d,
                       ep_f32(w.x, d, W_F32(L, STB_L_OUT_B), w.x, d), st));
        // ---- cross-attention (scores = the `qk` the reference's hooks capture) ----
        STB_TRY(layernorm(w.x, rows, d, W_F32(L, STB_L_CROSS_LN_G), W_F32(L, STB_L_CROSS_LN_B), w.ln.hi, w.ln.lo, nullptr, st));
        STB_TRY(linear(m, w.ln, rows, d, W_HI(L, STB_L_CQ_W), W_LO(L, STB_L_CQ_W), d,
                       ep_split(w.q, d, W_F32(L, STB_L_CQ_B), STB_ACT_NONE), st));
        Split Kx, vTx;
        cross_ptrs(m, B, ckv, l, Kx, vTx);
        stb_operand q = opnd(w.q.hi, w.q.lo, M, 64, d, 64, (long long)M * d);
        stb_operand k = opnd(Kx.hi, Kx.lo, T, 64, 64, (long long)T * 64, (long long)H * T * 64);   // head-major K
        stb_operand v = opnd(vTx.hi, vTx.lo, 64, Tp, Tp, 64LL * Tp, (long long)d * Tp);
        // The attention output never depends on what is captured, so the logits are the same with or without a capture.
        STB_TRY(fused_attention(q, k, v, B, H, M, T, w.attn.hi, w.attn.lo, d, 64, (long long)M * d, st));
        // The captured scores are their own GEMM, (q k^T) / 8 straight into qk_out; columns T..Tp-1 are not written.
        if (qk_out != nullptr && n_sel < 0) {
            stb_epilogue e = ep_f32(qk_out + (long long)l * H * M * Tp, Tp, nullptr, nullptr, 0, 0.125f);
            e.out_h_stride = (long long)M * Tp;
            e.out_b_stride = (long long)n_sel_total * M * Tp;
            STB_TRY(gemm(q, k, B, H, e, st));
        }
        for (int i = 0; qk_out != nullptr && i < n_sel; ++i) {
            if (sel[2 * i] != l) continue;
            const int h = sel[2 * i + 1];
            stb_operand qh = opnd(offs(w.q.hi, 64 * h), offs(w.q.lo, 64 * h), M, 64, d, 0, (long long)M * d);
            stb_operand kh = opnd(offs(Kx.hi, (long long)h * T * 64), offs(Kx.lo, (long long)h * T * 64), T, 64, 64, 0,
                                  (long long)H * T * 64);
            stb_epilogue e = ep_f32(qk_out + (long long)i * M * Tp, Tp, nullptr, nullptr, 0, 0.125f);
            e.out_b_stride = (long long)n_sel * M * Tp;
            STB_TRY(gemm(qh, kh, B, 1, e, st));
        }
        STB_TRY(linear(m, w.attn, rows, d, W_HI(L, STB_L_COUT_W), W_LO(L, STB_L_COUT_W), d,
                       ep_f32(w.x, d, W_F32(L, STB_L_COUT_B), w.x, d), st));
        // ---- MLP ----
        STB_TRY(layernorm(w.x, rows, d, W_F32(L, STB_L_MLP_LN_G), W_F32(L, STB_L_MLP_LN_B), w.ln.hi, w.ln.lo, nullptr, st));
        STB_TRY(linear(m, w.ln, rows, d, W_HI(L, STB_L_FC1_W), W_LO(L, STB_L_FC1_W), 4 * d,
                       ep_split(w.hid, 4 * d, W_F32(L, STB_L_FC1_B), STB_ACT_GELU), st));
        STB_TRY(linear(m, w.hid, rows, 4 * d, W_HI(L, STB_L_FC2_W), W_LO(L, STB_L_FC2_W), d,
                       ep_f32(w.x, d, W_F32(L, STB_L_FC2_B), w.x, d), st));
    }
    if (logits != nullptr) {
        STB_TRY(layernorm(w.x, rows, d, (const float*)t[STB_T_DEC_LN_G][0], (const float*)t[STB_T_DEC_LN_B][0], w.ln.hi, w.ln.lo,
                          nullptr, st));
        STB_TRY(linear(m, w.ln, rows, d, t[STB_T_DEC_TOKEMB][0], m->prec == STB_PREC_FP16X3 ? t[STB_T_DEC_TOKEMB][1] : nullptr,
                       D.n_vocab, ep_f32(logits, ld_logits, nullptr, nullptr, 0), st));
    }
    return STB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// KV-cached decode step
// ---------------------------------------------------------------------------------------------------------
struct StepWs {
    float* x;
    float* qkv;
    float* q;
    float* xpart;      // cross-attention split partials + tickets
    int* tickets;
    Split ln, attn, hid;
    size_t bytes;
};
constexpr int STEP_GEMV_MAX_B = 16;      // <= : mma.sync batched GEMV; above: the cluster split-K wgmma kernel
constexpr int STEP_SPLITK_MAX_B = 128;    // sequences on the N side of one wgmma tile (BN = 16 / 32 / 64 / 128)
static StepWs carve_step(const stb_model* m, int B, void* ws) {
    const bool lo = m->prec == STB_PREC_FP16X3;
    const size_t d = m->dims.n_text_state;
    Carver c(ws);
    StepWs w;
    w.x = c.take<float>((size_t)B * d);
    w.qkv = c.take<float>((size_t)B * 3 * d);
    w.q = c.take<float>((size_t)B * d);
    w.xpart = c.take<float>((size_t)B * m->dims.n_text_head * decode_cross_splits() * 66);
    w.tickets = c.take<int>((size_t)B * m->dims.n_text_head);
    w.ln = take_split(c, (size_t)B * d, lo);
    w.attn = take_split(c, (size_t)B * d, lo);
    w.hid = take_split(c, (size_t)B * 4 * d, lo);
    w.bytes = c.off;
    return w;
}
static size_t decode_state_bytes(const stb_model* m, int B, int cache_rows) {
    return (size_t)m->dims.n_text_layer * 2 * B * cache_rows * m->dims.n_text_state * sizeof(float);
}

// seq_off (nullable) [B]: first cache row of each sequence; cache_rows: rows per sequence of the K/V caches (>= n_text_ctx
// when ragged initial tokens are right-aligned, so that the shortest sequence still reaches its own n_text_ctx positions)
static int decode_step(stb_model* m, const int32_t* tokens, int B, int32_t* pos, const int32_t* seq_off, int cache_rows,
                       const void* ckv, void* state, float* logits, long long ld_logits, void* ws, cudaStream_t st) {
    const stb_dims& D = m->dims;
    const int d = D.n_text_state, H = D.n_text_head, ctx = cache_rows;
    const void* const(*t)[2] = m->t;
    StepWs w = carve_step(m, B, ws);
    const size_t cache = (size_t)B * ctx * d;
    const void* emb_hi = t[STB_T_DEC_TOKEMB][0];
    const void* emb_lo = m->prec == STB_PREC_FP16X3 ? t[STB_T_DEC_TOKEMB][1] : nullptr;
    // Linear layers of the step, by shape:
    //   B <= 16      : latency-optimised batched GEMV (mma.sync, gemv.cu) -- one launch, weights straight into fragments
    //   17 .. 128    : SWAPPED wgmma GEMM (decode_linear.cu): the features take the 128-row M side (every weight byte is
    //                  read by exactly one CTA), the sequences the N side (BN = 32/64/128); split-K across a thread-block
    //                  cluster, partial tiles reduced over distributed shared memory, fused epilogue, ONE launch.  Needs
    //                  k % 64 == 0 and n >= 128
    //   otherwise    : the plain wgmma GEMM (sequences on the M side); with n_text_state % 128 == 0 the only shape the
    //                  cluster kernel refuses is a vocabulary below 128
    const bool use_gemv = B <= STEP_GEMV_MAX_B, use_splitk = !use_gemv && B <= STEP_SPLITK_MAX_B;
    const Split none = {nullptr, nullptr};
    // ln_g != nullptr: also produce LayerNorm(out)*ln_g+ln_b into w.ln (only with a residual, out_f32 = w.x)
    int least = 0, lin_priority = 0;                           // the linears launch at the device's greatest priority (e.g. -5)
    if (cudaDeviceGetStreamPriorityRange(&least, &lin_priority) != cudaSuccess) lin_priority = 0;
    struct PriorityScope {                                     // the linears (and their LayerNorm) only
        int saved;
        explicit PriorityScope(int p) : saved(launch_priority()) { launch_priority() = p; }
        ~PriorityScope() { launch_priority() = saved; }
    };
    STB_TRY(embed_step(tokens, pos, seq_off, D.n_text_ctx, B, d, (const float*)t[STB_T_DEC_TOKEMB_F32][0],
                       (const float*)t[STB_T_DEC_POS][0], w.x, st));
    auto lin = [&](const Split& x, int k, const void* w_hi, const void* w_lo, int n, const float* bias, int act,
                   const float* res, float* out_f32, Split out_split, long long ld, const float* ln_g,
                   const float* ln_b) -> int {
        PriorityScope prio(lin_priority);
        if (use_gemv) {
            STB_TRY(gemv(x.hi, x.lo, B, k, w_hi, w_lo, n, bias, act, res, ld, out_f32, out_split.hi, out_split.lo, ld, st));
        } else if (use_splitk && k % 64 == 0 && n >= 128) {
            STB_TRY(decode_linear(x.hi, x.lo, B, k, w_hi, w_lo, n, bias, act, res, ld, out_f32, out_split.hi, out_split.lo, ld, st));
        } else {
            stb_epilogue e;
            memset(&e, 0, sizeof(e));
            e.out_f32 = out_f32; e.out_hi = out_split.hi; e.out_lo = out_split.lo; e.ld_out = ld;
            e.bias = bias; e.act = act; e.residual = res; e.ld_res = ld; e.alpha = 1.0f;
            STB_TRY(linear(m, x, B, k, w_hi, w_lo, n, e, st));
        }
        if (ln_g != nullptr)
            STB_TRY(layernorm(out_f32, B, n, ln_g, ln_b, w.ln.hi, w.ln.lo, nullptr, st));
        return STB_OK;
    };
    const float* final_g = (const float*)t[STB_T_DEC_LN_G][0];
    const float* final_b = (const float*)t[STB_T_DEC_LN_B][0];
    if (D.n_text_layer > 0)
        STB_TRY(layernorm(w.x, B, d, W_F32(m->dec[0], STB_L_ATTN_LN_G), W_F32(m->dec[0], STB_L_ATTN_LN_B), w.ln.hi, w.ln.lo, nullptr, st));
    else
        STB_TRY(layernorm(w.x, B, d, final_g, final_b, w.ln.hi, w.ln.lo, nullptr, st));
    for (int l = 0; l < D.n_text_layer; ++l) {
        const stb_model::Layer& L = m->dec[l];
        const bool last = l + 1 == D.n_text_layer;
        const float* next_g = last ? final_g : W_F32(m->dec[l + 1], STB_L_ATTN_LN_G);
        const float* next_b = last ? final_b : W_F32(m->dec[l + 1], STB_L_ATTN_LN_B);
        float* Kc = (float*)state + (size_t)l * 2 * cache;
        float* Vc = Kc + cache;
        // w.ln holds attn_ln(x) here (previous layer's fc2 finish, or the standalone LayerNorm above)
        STB_TRY(lin(w.ln, d, W_HI(L, STB_L_QKV_W), W_LO(L, STB_L_QKV_W), 3 * d, W_F32(L, STB_L_QKV_B), STB_ACT_NONE, nullptr,
                    w.qkv, none, 3 * d, nullptr, nullptr));
        STB_TRY(decode_attn_self(w.qkv, Kc, Vc, B, H, d, ctx, pos, seq_off, w.attn.hi, w.attn.lo, nullptr, st));
        STB_TRY(lin(w.attn, d, W_HI(L, STB_L_OUT_W), W_LO(L, STB_L_OUT_W), d, W_F32(L, STB_L_OUT_B), STB_ACT_NONE, w.x, w.x,
                    none, d, W_F32(L, STB_L_CROSS_LN_G), W_F32(L, STB_L_CROSS_LN_B)));
        STB_TRY(lin(w.ln, d, W_HI(L, STB_L_CQ_W), W_LO(L, STB_L_CQ_W), d, W_F32(L, STB_L_CQ_B), STB_ACT_NONE, nullptr, w.q,
                    none, d, nullptr, nullptr));
        Split Kx, vTx;
        CrossDecodeKV Vd;
        cross_ptrs(m, B, ckv, l, Kx, vTx, &Vd);
        STB_TRY(decode_attn_cross(w.q, Vd, B, H, d, w.xpart, w.tickets, w.attn.hi, w.attn.lo, nullptr, st));
        STB_TRY(lin(w.attn, d, W_HI(L, STB_L_COUT_W), W_LO(L, STB_L_COUT_W), d, W_F32(L, STB_L_COUT_B), STB_ACT_NONE, w.x,
                    w.x, none, d, W_F32(L, STB_L_MLP_LN_G), W_F32(L, STB_L_MLP_LN_B)));
        STB_TRY(lin(w.ln, d, W_HI(L, STB_L_FC1_W), W_LO(L, STB_L_FC1_W), 4 * d, W_F32(L, STB_L_FC1_B), STB_ACT_GELU, nullptr,
                    nullptr, w.hid, 4 * d, nullptr, nullptr));
        STB_TRY(lin(w.hid, 4 * d, W_HI(L, STB_L_FC2_W), W_LO(L, STB_L_FC2_W), d, W_F32(L, STB_L_FC2_B), STB_ACT_NONE, w.x, w.x,
                    none, d, next_g, next_b));
    }
    STB_TRY(lin(w.ln, d, emb_hi, emb_lo, D.n_vocab, nullptr, STB_ACT_NONE, nullptr, logits, none, ld_logits, nullptr, nullptr));
    STB_TRY(bump_pos(pos, st));
    return STB_OK;
}

}  // namespace stb

// ---------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------
extern "C" int stb_model_create(const stb_dims* dims, int precision, stb_model** out) {
    STB_REQUIRE(dims && out, "stb_model_create: null argument");
    STB_REQUIRE(precision == STB_PREC_FP16 || precision == STB_PREC_FP16X3, "stb_model_create: unknown precision %d", precision);
    STB_REQUIRE(dims->n_audio_state % 128 == 0 && dims->n_text_state % 128 == 0 && dims->n_audio_state <= 1280 &&
                    dims->n_text_state <= 1280,
                "stb_model_create: widths must be multiples of 128 and <= 1280");
    STB_REQUIRE(dims->n_audio_state == 64 * dims->n_audio_head && dims->n_text_state == 64 * dims->n_text_head,
                "stb_model_create: head_dim must be 64");
    STB_REQUIRE(dims->n_audio_ctx == STB_N_AUDIO_CTX, "stb_model_create: n_audio_ctx must be 1500");
    stb_model* m = new stb_model();
    m->dims = *dims;
    m->prec = precision;
    memset(m->t, 0, sizeof(m->t));
    m->enc.resize(dims->n_audio_layer);
    m->dec.resize(dims->n_text_layer);
    for (auto& l : m->enc) memset(&l, 0, sizeof(l));
    for (auto& l : m->dec) memset(&l, 0, sizeof(l));
    *out = m;
    return STB_OK;
}

extern "C" void stb_model_destroy(stb_model* m) { delete m; }

extern "C" int stb_model_set_tensor(stb_model* m, int tensor_id, int is_decoder, int layer, const void* p0, const void* p1) {
    STB_REQUIRE(m, "stb_model_set_tensor: null model");
    if (tensor_id < STB_T_LAYER_BASE) {
        STB_REQUIRE(tensor_id >= 0, "stb_model_set_tensor: bad id %d", tensor_id);
        m->t[tensor_id][0] = p0;
        m->t[tensor_id][1] = p1;
        return STB_OK;
    }
    const int id = tensor_id - STB_T_LAYER_BASE;
    STB_REQUIRE(id < STB_L_COUNT, "stb_model_set_tensor: bad layer tensor id %d", tensor_id);
    auto& tab = is_decoder ? m->dec : m->enc;
    STB_REQUIRE(layer >= 0 && layer < (int)tab.size(), "stb_model_set_tensor: layer %d out of range", layer);
    tab[layer].p[id][0] = p0;
    tab[layer].p[id][1] = p1;
    return STB_OK;
}

static int check_weights(const stb_model* m, bool enc, bool dec) {
    const bool lo = m->prec == STB_PREC_FP16X3;
    auto need = [&](const void* const p[2], bool split, const char* what, int l) -> int {
        STB_REQUIRE(p[0] != nullptr && (!split || !lo || p[1] != nullptr), "model tensor %s (layer %d) is not set", what, l);
        return STB_OK;
    };
    static const int enc_ids[] = {STB_L_ATTN_LN_G, STB_L_ATTN_LN_B, STB_L_QKV_W, STB_L_QKV_B, STB_L_OUT_W, STB_L_OUT_B,
                                  STB_L_MLP_LN_G, STB_L_MLP_LN_B, STB_L_FC1_W, STB_L_FC1_B, STB_L_FC2_W, STB_L_FC2_B};
    auto is_split = [](int id) {
        return id == STB_L_QKV_W || id == STB_L_OUT_W || id == STB_L_FC1_W || id == STB_L_FC2_W || id == STB_L_CQ_W ||
               id == STB_L_CKV_W || id == STB_L_COUT_W;
    };
    if (enc) {
        STB_TRY(need(m->t[STB_T_ENC_CONV1_W], true, "enc.conv1.w", -1));
        STB_TRY(need(m->t[STB_T_ENC_CONV1_B], false, "enc.conv1.b", -1));
        STB_TRY(need(m->t[STB_T_ENC_CONV2_W], true, "enc.conv2.w", -1));
        STB_TRY(need(m->t[STB_T_ENC_CONV2_B], false, "enc.conv2.b", -1));
        STB_TRY(need(m->t[STB_T_ENC_POS], false, "enc.pos", -1));
        STB_TRY(need(m->t[STB_T_ENC_LNPOST_G], false, "enc.ln_post.g", -1));
        STB_TRY(need(m->t[STB_T_ENC_LNPOST_B], false, "enc.ln_post.b", -1));
        for (size_t l = 0; l < m->enc.size(); ++l)
            for (int id : enc_ids) STB_TRY(need(m->enc[l].p[id], is_split(id), "enc.layer", (int)l));
    }
    if (dec) {
        STB_TRY(need(m->t[STB_T_DEC_TOKEMB_F32], false, "dec.tok_emb.f32", -1));
        STB_TRY(need(m->t[STB_T_DEC_TOKEMB], true, "dec.tok_emb", -1));
        STB_TRY(need(m->t[STB_T_DEC_POS], false, "dec.pos", -1));
        STB_TRY(need(m->t[STB_T_DEC_LN_G], false, "dec.ln.g", -1));
        STB_TRY(need(m->t[STB_T_DEC_LN_B], false, "dec.ln.b", -1));
        for (size_t l = 0; l < m->dec.size(); ++l)
            for (int id = 0; id < STB_L_COUNT; ++id) STB_TRY(need(m->dec[l].p[id], is_split(id), "dec.layer", (int)l));   // a decoder layer uses every id
    }
    return STB_OK;
}

extern "C" size_t stb_encoder_ws_bytes(const stb_model* m, int B) { return m ? stb::carve_encoder(m, B, nullptr).bytes : 0; }

extern "C" int stb_encoder_forward(stb_model* m, const float* mel, int B, float* xa_f32, void* xa_hi, void* xa_lo, void* ws,
                                   size_t ws_bytes, void* stream) {
    STB_REQUIRE(m && mel && ws && B >= 1 && (xa_f32 || xa_hi), "stb_encoder_forward: bad arguments");
    STB_TRY(check_weights(m, true, false));
    STB_REQUIRE(ws_bytes >= stb_encoder_ws_bytes(m, B), "stb_encoder_forward: workspace %zu < %zu", ws_bytes, stb_encoder_ws_bytes(m, B));
    STB_REQUIRE(m->prec != STB_PREC_FP16X3 || !xa_hi || xa_lo, "stb_encoder_forward: xa_lo required in FP16X3 mode");
    return stb::encoder_forward(m, mel, B, xa_f32, (__half*)xa_hi, (__half*)xa_lo, ws, (cudaStream_t)stream);
}

extern "C" size_t stb_cross_kv_bytes(const stb_model* m, int B) {
    return m ? stb::cross_layout(m, B).layer_halfs * sizeof(__half) * m->dims.n_text_layer : 0;
}

extern "C" int stb_cross_kv(stb_model* m, const void* xa_hi, const void* xa_lo, int B, int decode_layout, void* cross_kv,
                            void* stream) {
    STB_REQUIRE(m && xa_hi && cross_kv && B >= 1, "stb_cross_kv: bad arguments");
    STB_REQUIRE(m->prec != STB_PREC_FP16X3 || xa_lo, "stb_cross_kv: xa_lo required in FP16X3 mode");
    STB_TRY(check_weights(m, false, true));
    return stb::cross_kv(m, (const __half*)xa_hi, (const __half*)xa_lo, B, cross_kv, decode_layout != 0, (cudaStream_t)stream);
}

extern "C" size_t stb_decoder_ws_bytes(const stb_model* m, int B, int M) { return m ? stb::carve_decoder(m, B, M, nullptr).bytes : 0; }

extern "C" int stb_decoder_forward(stb_model* m, const int32_t* tokens, int B, int M, const void* cross_kv, float* logits,
                                   long long ld_logits, float* qk_out, const int32_t* sel_pairs_host, int n_sel, void* ws,
                                   size_t ws_bytes, void* stream) {
    STB_REQUIRE(m && tokens && cross_kv && ws && B >= 1 && M >= 1, "stb_decoder_forward: bad arguments");
    STB_REQUIRE(M <= m->dims.n_text_ctx, "stb_decoder_forward: M=%d exceeds n_text_ctx=%d", M, m->dims.n_text_ctx);
    STB_REQUIRE(!logits || (ld_logits >= m->dims.n_vocab && ld_logits % 4 == 0), "stb_decoder_forward: ld_logits must be >= n_vocab and a multiple of 4");
    STB_REQUIRE(!qk_out || n_sel < 0 || sel_pairs_host, "stb_decoder_forward: sel_pairs_host missing");
    if (qk_out && n_sel >= 0)
        for (int i = 0; i < n_sel; ++i)
            STB_REQUIRE(sel_pairs_host[2 * i] >= 0 && sel_pairs_host[2 * i] < m->dims.n_text_layer && sel_pairs_host[2 * i + 1] >= 0 &&
                            sel_pairs_host[2 * i + 1] < m->dims.n_text_head,
                        "stb_decoder_forward: head pair %d out of range", i);
    STB_TRY(check_weights(m, false, true));
    STB_REQUIRE(ws_bytes >= stb_decoder_ws_bytes(m, B, M), "stb_decoder_forward: workspace %zu < %zu", ws_bytes, stb_decoder_ws_bytes(m, B, M));
    return stb::decoder_forward(m, tokens, B, M, cross_kv, logits, ld_logits, qk_out, sel_pairs_host, n_sel, ws, (cudaStream_t)stream);
}

extern "C" size_t stb_decode_state_bytes(const stb_model* m, int B) { return m ? stb::decode_state_bytes(m, B, m->dims.n_text_ctx) : 0; }
extern "C" size_t stb_decode_state_bytes_rows(const stb_model* m, int B, int cache_rows) {
    return m && cache_rows >= 1 ? stb::decode_state_bytes(m, B, cache_rows) : 0;
}
extern "C" size_t stb_decode_ws_bytes(const stb_model* m, int B) { return m ? stb::carve_step(m, B, nullptr).bytes : 0; }

extern "C" int stb_decode_step_ragged(stb_model* m, const int32_t* tokens_in, int B, int32_t* pos, const int32_t* seq_off,
                                      int cache_rows, const void* cross_kv, void* state, float* logits_out, long long ld_logits,
                                      void* ws, size_t ws_bytes, void* stream) {
    STB_REQUIRE(m && tokens_in && pos && cross_kv && state && logits_out && ws && B >= 1, "stb_decode_step: bad arguments");
    STB_REQUIRE(ld_logits >= m->dims.n_vocab && ld_logits % 4 == 0, "stb_decode_step: ld_logits must be >= n_vocab and a multiple of 4");
    STB_REQUIRE(m->dims.n_text_ctx <= 448, "stb_decode_step: n_text_ctx > 448 unsupported");
    STB_REQUIRE(cache_rows >= m->dims.n_text_ctx && cache_rows <= 2 * m->dims.n_text_ctx,
                "stb_decode_step: cache_rows must be in [n_text_ctx, 2 n_text_ctx]");
    STB_TRY(check_weights(m, false, true));
    STB_REQUIRE(ws_bytes >= stb_decode_ws_bytes(m, B), "stb_decode_step: workspace too small");
    return stb::decode_step(m, tokens_in, B, pos, seq_off, cache_rows, cross_kv, state, logits_out, ld_logits, ws,
                            (cudaStream_t)stream);
}

extern "C" int stb_decode_step(stb_model* m, const int32_t* tokens_in, int B, int32_t* pos, const void* cross_kv, void* state,
                               float* logits_out, long long ld_logits, void* ws, size_t ws_bytes, void* stream) {
    STB_REQUIRE(m, "stb_decode_step: bad arguments");
    return stb_decode_step_ragged(m, tokens_in, B, pos, nullptr, m->dims.n_text_ctx, cross_kv, state, logits_out, ld_logits, ws,
                                  ws_bytes, stream);
}
