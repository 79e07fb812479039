// a6 / K7: monotone DTW + backtrack + jump extraction, one CTA per 30 s window.
//
// Replaces whisper.timing.dtw (CPU semantics: numba dtw_cpu + backtrace) and the jump extraction of
// stable_whisper/timing.py:195-198.  Bit-exact contract: fp32 cost, strict '<' tie rule
// (diag iff c0<c1 && c0<c2; up iff c1<c0 && c1<c2; else left), +inf borders, cost[0][0] = 0.
//
// Parallelisation (R <= 480 rows x F <= 1500 frames):
//   * lane l of warp w owns row r = 32 w + l and walks its row left to right; within a warp the anti-diagonal
//     wavefront is kept with ONE shuffle per step (up = lane-1's previous value, diag = the up of the previous step);
//   * warps are software-pipelined: warp w+1 consumes the last row of warp w through a small shared-memory ring
//     (256 columns) guarded by two monotone progress counters -- no block-wide barrier in the sweep;
//   * x is pre-transposed and pre-skewed (xs[t][r] = x[r][t - r%32], dtw_skew_kernel) so every step of a warp is ONE
//     coalesced 128-byte load, prefetched one 32-step block ahead into registers (static register index);
//   * the sweep body is branch-free (~15 instructions per step): out-of-matrix cells are computed on zero-padded x and
//     ignored, flow control sits at compile-time positions of the 32-step unrolled block;
//   * the trace is 2 bits per cell, packed 16 STEPS per word (static bit position) in shared memory (<= 187 KB), and the
//     backtrack runs in the same kernel on one thread with the current trace word cached in a register.
#include <math.h>

#include "common.cuh"

namespace stb {

constexpr int DTW_RING = 256;                 // columns per inter-warp boundary ring
constexpr int DTW_RING_CHUNKS = DTW_RING / 32;
constexpr int DTW_MAX_ROWS = 480;             // 15 warps

// Trace words per row: 16 steps per word over (Fpad/32 + 1) blocks of 32 steps, +1 to make the row pitch odd
// (lanes store to the same word index of 32 consecutive rows: an odd pitch is conflict-free).
__host__ __device__ __forceinline__ int dtw_trace_words(int F) { return (((F + 31) >> 5) + 1) * 2 + 1; }

__device__ __forceinline__ int vload(const volatile int* p) { return *p; }
// bounded spin on a monotone shared-memory progress counter (a protocol bug traps instead of hanging the box)
__device__ __forceinline__ void wait_ge(const volatile int* p, int need) {
    if (vload(p) >= need) return;
    const long long t0 = clock64();
    while (vload(p) < need) {
        if (clock64() - t0 > 4000000000LL) {
            printf("stb: dtw progress timeout block=%d thread=%d need=%d have=%d\n", blockIdx.x, threadIdx.x, need, vload(p));
            __trap();
        }
    }
}

__global__ void __launch_bounds__(DTW_MAX_ROWS, 1)
dtw_kernel(const float* __restrict__ xs, int R, int F, int Rpad, int32_t* __restrict__ jumps, int32_t* __restrict__ path,
           int32_t* __restrict__ path_len) {
    extern __shared__ uint32_t dsm[];
    const int TW = dtw_trace_words(F);                         // trace words per row (indexed by step t = j + lane)
    const int NW = (R + 31) >> 5;
    uint32_t* trace = dsm;                                     // [R][TW]
    volatile float* ring = reinterpret_cast<volatile float*>(trace + (size_t)R * TW);   // [NW-1][DTW_RING]
    volatile int* prod = reinterpret_cast<volatile int*>(const_cast<float*>(ring) + (size_t)(NW > 1 ? NW - 1 : 0) * DTW_RING);  // [NW]
    volatile int* cons = prod + NW;                            // [NW]

    const int b = blockIdx.x;
    const int w = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int r = w * 32 + lane;
    const bool row_ok = r < R;
    // xs [B][F+32][Rpad]: xs[t][r] = cost[r][t - (r & 31)] (0 outside): lane l of a warp reads ONE coalesced 128-byte
    // row per step instead of 32 scattered sectors (the skew of the wavefront is baked into the layout by dtw_skew_kernel)
    const float* xcol = xs + (long long)b * (F + 32) * Rpad + r;
    const float INF = INFINITY;

    if (threadIdx.x < NW) {
        prod[threadIdx.x] = 0;
        cons[threadIdx.x] = 0;
    }
    __syncthreads();

    if (w < NW) {
        const bool is_prod = w < NW - 1;
        const bool is_cons = w > 0;
        const volatile float* ring_in = ring + (size_t)(w - 1) * DTW_RING;     // valid if is_cons
        volatile float* ring_out = ring + (size_t)w * DTW_RING;                // valid if is_prod
        // Borders without per-step special cases: `own` (left) and `diag` start at +inf, which IS the j = 0 border
        // (cost[i][0] = inf); only global row 0 sees cost[0][0] = 0 as its first diagonal.
        float own = INF;                       // cost[r][j-1] (left)
        float diag = (r == 0) ? 0.f : INF;     // cost[r-1][j-1]
        uint32_t tacc = 0;
        const int Fpad = (F + 31) & ~31;                              // flow control works on whole 32-column chunks
        const int n_blocks = (Fpad >> 5) + 1;                         // lane 31 reaches column Fpad - 1
        const bool l0c = is_cons && lane == 0;                        // reads the ring
        const bool l31p = is_prod && lane == 31;                      // writes the ring
        uint32_t* trow = trace + (size_t)r * TW;
        float xc[32], xn[32];
#pragma unroll
        for (int s = 0; s < 32; ++s) xc[s] = xcol[(long long)s * Rpad];
#pragma unroll 1
        for (int kb = 0; kb < n_blocks; ++kb) {
            // prefetch the next block: one coalesced 128-byte row per step, lands while the 32 dependent steps run
#pragma unroll
            for (int s = 0; s < 32; ++s) {
                const int t2 = (kb + 1) * 32 + s;
                xn[s] = (t2 < F + 32) ? xcol[(long long)t2 * Rpad] : 0.f;
            }
            const volatile float* rin_blk = ring_in + (kb & (DTW_RING_CHUNKS - 1)) * 32;
            volatile float* rout_cur = ring_out + (kb & (DTW_RING_CHUNKS - 1)) * 32;
            volatile float* rout_prev = ring_out + ((kb - 1) & (DTW_RING_CHUNKS - 1)) * 32;
            // The step body is branch-free.  Cells outside the matrix (j < 0, j >= F, r >= R) are computed too: their x
            // is 0 in the skewed buffer, so a lane that has not started keeps own = inf + 0, garbage past the right edge
            // only flows to lanes that are past it as well, and their trace bits are never read by the backtrack.
#pragma unroll
            for (int s = 0; s < 32; ++s) {                            // s is a compile-time constant in every copy
                const int t = kb * 32 + s;                            // warp-uniform step
                const int j = t - lane;                               // this lane's column
                // ---- flow control, only at chunk edges (compile-time positions) ----
                if (s == 0) {
                    if (is_cons && t < Fpad) wait_ge(&prod[w - 1], (t >> 5) + 1);   // lane 0 reads ring chunk t/32 next
                }
                if (s == 31) {
                    const int jp = t - 31;                            // lane 31's column: start of its chunk jp/32
                    if (is_prod && jp < Fpad) wait_ge(&cons[w + 1], (jp >> 5) - (DTW_RING_CHUNKS - 1));
                }
                float rv = INF;
                if (l0c && t < F) rv = rin_blk[s];                    // == ring_in[t & (DTW_RING - 1)]
                const float sh = __shfl_up_sync(0xffffffffu, own, 1);
                const float up = (lane == 0) ? rv : sh;
                // 3-way strict-'<' selection + trace bits in one PTX block (keeps the two predicates next to their uses;
                // left to the compiler, the 32 predicate pairs get parked in a register and unpacked 16 steps later).
                // trace bits = (p0, p1): 1 diagonal, 2 up, 0 left; indexed by STEP, so the bit position is static.
                float c;
                asm volatile(
                    "{\n\t.reg .pred p0, p1;\n\t.reg .f32 m;\n\t"
                    "setp.lt.f32 p0, %2, %4;\n\t"
                    "setp.lt.and.f32 p0, %2, %3, p0;\n\t"          // diagonal: c0 < c2 && c0 < c1
                    "setp.lt.f32 p1, %3, %4;\n\t"
                    "setp.lt.and.f32 p1, %3, %2, p1;\n\t"          // up: c1 < c2 && c1 < c0
                    "selp.f32 m, %3, %4, p1;\n\t"
                    "selp.f32 %0, %2, m, p0;\n\t"
                    "@p0 add.u32 %1, %1, %5;\n\t"
                    "@p1 add.u32 %1, %1, %6;\n\t}"
                    : "=f"(c), "+r"(tacc)
                    : "f"(diag), "f"(up), "f"(own), "r"(1u << ((s & 15) * 2)), "r"(2u << ((s & 15) * 2)));
                own = xc[s] + c;
                if (l31p && (unsigned)j < (unsigned)F) {              // lane 31: j = t - 31 -> ring_out[j & (DTW_RING - 1)]
                    if (s == 31) rout_cur[0] = own; else rout_prev[s + 1] = own;
                }
                diag = up;
                if ((s & 15) == 15) {
                    if (row_ok) trow[t >> 4] = tacc;
                    tacc = 0;
                }
                // ---- publish progress at chunk ends ----
                if (s == 30) {
                    const int jp = t - 31;                            // lane 31 just finished column jp, jp & 31 == 31
                    if (is_prod && jp >= 0 && jp < Fpad) {
                        __threadfence_block();
                        if (lane == 31) prod[w] = (jp >> 5) + 1;
                    }
                }
                if (s == 31) {
                    if (is_cons && t < Fpad) {
                        __threadfence_block();
                        if (lane == 0) cons[w] = (t >> 5) + 1;
                    }
                }
            }
#pragma unroll
            for (int s = 0; s < 32; ++s) xc[s] = xn[s];
        }
    }
    __syncthreads();

    // ---- backtrack (whisper.timing.backtrace): padded coords (i, j), emit (i-1, j-1) until (0, 0) ----
    int32_t* pt = path ? path + (long long)b * 2 * (R + F) : nullptr;
    int32_t* pj = pt ? pt + (R + F) : nullptr;
    __shared__ int s_len;
    if (threadIdx.x == 0) {
        int i = R, j = F, n = 0;
        int cached_row = -1, cached_word = -1;
        uint32_t word = 0;
        int32_t* jb = jumps + (long long)b * R;
        while (i > 0 || j > 0) {
            if (pt) { pt[n] = i - 1; pj[n] = j - 1; }
            if (i >= 1) jb[i - 1] = (j - 1) < 0 ? 0 : (j - 1);
            ++n;
            uint32_t code;
            if (i == 0) code = 2u;                             // trace[0, :] = 2
            else if (j == 0) code = 1u;                        // trace[:, 0] = 1
            else {
                const int rr = i - 1, tt = j - 1 + ((i - 1) & 31);      // cell (rr, cc) was computed at step cc + lane
                if (rr != cached_row || (tt >> 4) != cached_word) {
                    cached_row = rr;
                    cached_word = tt >> 4;
                    word = trace[(size_t)rr * TW + cached_word];
                }
                const uint32_t bits = (word >> ((tt & 15) * 2)) & 3u;   // (p0, p1) of the sweep
                code = bits == 1u ? 0u : (bits == 2u ? 1u : 2u);
            }
            if (code == 0u) { --i; --j; }
            else if (code == 1u) { --i; }
            else { --j; }
        }
        s_len = n;
        if (path_len) path_len[b] = n;
    }
    __syncthreads();
    if (pt) {                                                  // reverse into forward order
        const int n = s_len;
        for (int k = threadIdx.x; k < n / 2; k += blockDim.x) {
            int32_t a = pt[k]; pt[k] = pt[n - 1 - k]; pt[n - 1 - k] = a;
            a = pj[k]; pj[k] = pj[n - 1 - k]; pj[n - 1 - k] = a;
        }
    }
}

// xs[b][t][r] = (+-) x[b][r][t - (r & 31)], zero outside [0, F) and for r >= R.  Tile transpose through shared memory:
// coalesced reads along frames, coalesced writes along rows.
__global__ void __launch_bounds__(256) dtw_skew_kernel(const float* __restrict__ x, int R, int F, long long ldx, int Rpad,
                                                       int negate, float* __restrict__ xs) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;     // source tile: rows r0.., columns c0..
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const float* src = x + (long long)b * R * ldx;
    for (int i = ty; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + tx;
        float v = 0.f;
        if (r < R && c < F) v = src[(long long)r * ldx + c];
        tile[i][tx] = negate ? -v : v;
    }
    __syncthreads();
    float* dst = xs + (long long)b * (F + 32) * Rpad;
    for (int i = ty; i < 32; i += 8) {                       // i = source column offset, tx = row offset (lane index)
        const int c = c0 + i;
        if (c < F) dst[(long long)(c + tx) * Rpad + r0 + tx] = tile[tx][i];    // t = c + (r & 31), r & 31 == tx
    }
}

static size_t dtw_smem(int R, int F) {
    const int TW = dtw_trace_words(F), NW = (R + 31) >> 5;
    return (size_t)R * TW * 4 + (size_t)(NW > 1 ? NW - 1 : 0) * DTW_RING * 4 + (size_t)NW * 2 * 4 + 16;
}

}  // namespace stb

extern "C" size_t stb_dtw_smem_bytes(int R, int F) { return stb::dtw_smem(R, F); }

extern "C" size_t stb_dtw_ws_bytes(int B, int R, int F) {
    const size_t Rpad = (size_t)((R + 31) / 32) * 32;
    return (size_t)B * (F + 32) * Rpad * sizeof(float);
}

extern "C" int stb_dtw(const float* x, int B, int R, int F, long long ldx, int negate, int32_t* jumps, int32_t* path,
                       int32_t* path_len, void* ws, size_t ws_bytes, void* stream) {
    STB_REQUIRE(x && jumps && ws, "stb_dtw: null pointer");
    STB_REQUIRE(ws_bytes >= stb_dtw_ws_bytes(B, R, F), "stb_dtw: workspace too small");
    STB_REQUIRE(B >= 1 && R >= 1 && F >= 1 && R <= stb::DTW_MAX_ROWS && F <= 1504 && ldx >= F,
                "stb_dtw: unsupported shape B=%d R=%d F=%d ld=%lld (R<=%d, F<=1504)", B, R, F, ldx, stb::DTW_MAX_ROWS);
    const size_t smem = stb::dtw_smem(R, F);
    size_t max_dyn = 0;
    STB_TRY(stb::max_dynamic_smem((const void*)stb::dtw_kernel, &max_dyn));
    STB_REQUIRE(smem <= max_dyn, "stb_dtw: trace needs %zu B of shared memory (limit %zu)", smem, max_dyn);
    const int NW = (R + 31) / 32;
    const int Rpad = NW * 32;
    cudaStream_t st = (cudaStream_t)stream;
    stb::ProfScope ps("dtw(+skew)", st, (double)B * R * F * 4.0 * 3, (double)B * R * F);
    STB_CUDA_OK(cudaMemsetAsync(ws, 0, stb_dtw_ws_bytes(B, R, F), st));      // zero border (t - (r&31) outside [0,F))
    STB_TRY(stb::launch(stb::dtw_skew_kernel, {dim3(stb::cdiv(F, 32), NW, B), 256, 0, st}, x, R, F, ldx, Rpad, negate, (float*)ws));
    return stb::launch(stb::dtw_kernel, {B, NW * 32, smem, st}, (const float*)ws, R, F, Rpad, jumps, path, path_len);
}
