// forward.cu — the neural forward at the informative (supported) positions only.
//
// Contract being replaced: src/inference.rs:147-175 — bases i32 [B,L,31], quals f32 [B,L,31]
// (u8 * fl(2/93) - fl(66/93+1), two fp32 ops, H11), lens, indices ->
// info_logits [sum lens], bases_logits [sum lens, 5].  The reference's TorchScript graph
// evaluates its stem over every row of the padded batch tensor and then gathers `indices`;
// because everything after the stem is local to one position (read-axis attention,
// per-token FFN, read-axis collapse, heads), only the rows within the stem's receptive field
// of a supported row are ever consumed.  This file therefore gathers FIRST: one work item per
// supported row, reading the 2*(K/2)+1 neighbouring rows of the [L',32] token/quality matrix
// straight from HBM, with the reference's batch-padding rows (token 11, qual byte 126 up to
// the Lmax of the reference batch, zero beyond; H10) reproduced arithmetically.
//
// This is the fp32 SIMT implementation (bit-for-bit order-insensitive to ~1e-6 vs torch fp32).
#include <cstdlib>

#include "common.cuh"
#include "forward.h"

namespace hb {

constexpr int TOK_PER_POS = 32;  // 31 reads + 1 zero pad token, so that 4 positions = 128 rows

// ---- stem: Embedding(12,6) ++ qual -> Conv(7->C, k=(K,1)) + bias + ReLU, + read_pos ---------
// grid = positions, block = C threads (one output channel each).
__global__ void k_stem(BatchView b, FwdWeights wt, uint32_t n0, uint32_t npos, float* __restrict__ X) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const int K = wt.stem_k, C = wt.C;
    uint8_t* s_tok = smem_raw;                          // [K][32]; 0xff = contributes nothing
    float* s_q = (float*)(smem_raw + ((K * 32 + 15) & ~15));  // [K][32]
    const uint32_t n = blockIdx.x;
    if (n >= npos) return;
    const uint32_t w = b.fwd_win[n0 + n], r = b.fwd_row[n0 + n];
    const uint32_t L = b.w_L[w], Lref = b.w_reflmax[w];
    const uint64_t rowbase = b.w_rowbase[w];
    const float QS = (float)(2.0 / 93.0), QO = (float)(2.0 * 33.0 / 93.0 + 1.0);  // src/inference.rs:19-21
    for (int i = threadIdx.x; i < K * 32; i += blockDim.x) {
        const int j = i >> 5, c = i & 31;
        const int64_t row = (int64_t)r + j - K / 2;
        uint8_t tok = 0xff;
        float q = 0.f;
        if (c < R_COLS && row >= 0 && row < (int64_t)Lref) {
            uint8_t qb;
            if (row < (int64_t)L) {
                tok = b.mat_bases[(rowbase + row) * ROW_BYTES + c];
                qb = b.mat_quals[(rowbase + row) * ROW_BYTES + c];
            } else {  // batch padding row of the reference's collate (src/inference.rs:86-97)
                tok = (uint8_t)TOK_PAD;
                qb = QUAL_PAD;
            }
            q = __fsub_rn(__fmul_rn((float)qb, QS), QO);
        }
        s_tok[i] = tok;
        s_q[i] = q;
    }
    __syncthreads();
    const int c = threadIdx.x;
    if (c >= C) return;
    const float bias = wt.stem_b[c];
    float* xo = X + (size_t)n * TOK_PER_POS * C;
    for (int rd = 0; rd < R_COLS; rd++) {
        float acc = bias;
        for (int j = 0; j < K; j++) {
            const uint8_t tok = s_tok[j * 32 + rd];
            if (tok != 0xff) {
                acc += wt.stem_tab[((size_t)j * 12 + tok) * C + c];
                acc = fmaf(s_q[j * 32 + rd], wt.stem_wq[(size_t)j * C + c], acc);
            }
        }
        xo[(size_t)rd * C + c] = fmaxf(acc, 0.f) + wt.read_pos[(size_t)rd * C + c];
    }
    xo[(size_t)31 * C + c] = 0.f;
}

// ---- LayerNorm over C (eps 1e-5), one warp per token row; output as split bf16 (hi + lo), the
//      A-operand format of the wgmma contractions (gemm_tc.cu) --------------------------------
__device__ __forceinline__ uint32_t pack_bf2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
__device__ __forceinline__ void split2f(float a, float b, uint32_t& hi, uint32_t& lo) {  // 2-wide converts (F2FP.PACK_AB)
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void split4(const float (&y)[4], uint2& hi, uint2& lo) {
    split2f(y[0], y[1], hi.x, lo.x);
    split2f(y[2], y[3], hi.y, lo.y);
}
__global__ void k_layernorm(const float* __restrict__ X, __nv_bfloat16* __restrict__ Yhi, __nv_bfloat16* __restrict__ Ylo,
                            const float* __restrict__ g, const float* __restrict__ be, uint32_t rows, int C) {
    const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* x = X + (size_t)row * C;
    float s = 0.f;
    for (int i = lane * 4; i < C; i += 128) { const float4 v = *(const float4*)(x + i); s += (v.x + v.y) + (v.z + v.w); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(HB_FULL, s, o);
    const float mean = s / (float)C;
    float v2 = 0.f;
    for (int i = lane * 4; i < C; i += 128) {
        const float4 v = *(const float4*)(x + i);
        const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
        v2 = fmaf(a, a, v2); v2 = fmaf(b, b, v2); v2 = fmaf(c, c, v2); v2 = fmaf(d, d, v2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v2 += __shfl_xor_sync(HB_FULL, v2, o);
    const float rstd = rsqrtf(v2 / (float)C + 1e-5f);
    for (int i = lane * 4; i < C; i += 128) {
        const float4 v = *(const float4*)(x + i), gv = *(const float4*)(g + i), bv = *(const float4*)(be + i);
        const float y[4] = {(v.x - mean) * rstd * gv.x + bv.x, (v.y - mean) * rstd * gv.y + bv.y,
                            (v.z - mean) * rstd * gv.z + bv.z, (v.w - mean) * rstd * gv.w + bv.w};
        uint2 hi, lo;
        split4(y, hi, lo);
        *(uint2*)(Yhi + (size_t)row * C + i) = hi;
        *(uint2*)(Ylo + (size_t)row * C + i) = lo;
    }
}

// ---- fp32 GEMM  Cout[M,N] = act(A[M,K] * Wt[N,K]^T + bias) (+ Res) -----------------------------
// 128x64 tile, BK 16, 256 threads, 8x4 micro-tile.  M is padded by the caller to a multiple of 128
// (buffers are allocated padded), N % 64 == 0, K % 16 == 0.
template <int ACT, int RES>
__global__ void __launch_bounds__(256) k_gemm(const float* __restrict__ A, int lda, const float* __restrict__ Wt,
                                              const float* __restrict__ bias, float* Cout, int ldc,
                                              const float* Res, int K) {
    __shared__ __align__(16) float As[16][128 + 4];
    __shared__ __align__(16) float Ws[16][64 + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * 64;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
    // load mapping: A tile 128 rows x 16 k = 512 float4: thread -> (row = tid/4 + 64*h, k4 = tid%4)
    const int ar = tid >> 2, ak = (tid & 3) * 4;
    const int wr = tid >> 2, wk = (tid & 3) * 4;  // W tile 64 rows x 16 k = 256 float4
    for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const float4 v = *(const float4*)(A + (size_t)(m0 + ar + 64 * h) * lda + k0 + ak);
            As[ak + 0][ar + 64 * h] = v.x; As[ak + 1][ar + 64 * h] = v.y;
            As[ak + 2][ar + 64 * h] = v.z; As[ak + 3][ar + 64 * h] = v.w;
        }
        {
            const float4 v = *(const float4*)(Wt + (size_t)(n0 + wr) * K + k0 + wk);
            Ws[wk + 0][wr] = v.x; Ws[wk + 1][wr] = v.y; Ws[wk + 2][wr] = v.z; Ws[wk + 3][wr] = v.w;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; kk++) {
            float a[8], wv[4];
            const float4 a0 = *(const float4*)&As[kk][ty * 8], a1 = *(const float4*)&As[kk][ty * 8 + 4];
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            const float4 w0 = *(const float4*)&Ws[kk][tx * 4];
            wv[0] = w0.x; wv[1] = w0.y; wv[2] = w0.z; wv[3] = w0.w;
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], wv[j], acc[i][j]);
        }
        __syncthreads();
    }
    const float4 bv = *(const float4*)(bias + n0 + tx * 4);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const size_t o = (size_t)(m0 + ty * 8 + i) * ldc + n0 + tx * 4;
        float4 v = make_float4(acc[i][0] + bv.x, acc[i][1] + bv.y, acc[i][2] + bv.z, acc[i][3] + bv.w);
        if (ACT) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (RES) { const float4 r = *(const float4*)(Res + o); v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
        *(float4*)(Cout + o) = v;
    }
}

// ---- read-axis multi-head attention: S = 31 tokens per position ----------------------------
// one warp per (position, head); lane = query token; online softmax, all in registers.
template <int DH>
__global__ void __launch_bounds__(128) k_attention(const float* __restrict__ QKV, __nv_bfloat16* __restrict__ Ohi,
                                                   __nv_bfloat16* __restrict__ Olo, uint32_t npos, int C, int H) {
    __shared__ __align__(16) float sK[4][32][DH + 4], sV[4][32][DH + 4];
    __shared__ __align__(16) uint32_t s_out[4][32 * (DH / 2)];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t item = blockIdx.x * 4 + warp;
    if (item >= npos * (uint32_t)H) return;
    const uint32_t n = item / H, h = item % H;
    const float* base = QKV + (size_t)n * TOK_PER_POS * 3 * C;
    // stage K and V of this head: 32 tokens x DH, 16-byte loads (a row of a head is DH*4 contiguous bytes)
    constexpr int V4 = DH / 4;
    for (int i = lane; i < 32 * V4; i += 32) {
        const int t = i / V4, d4 = (i % V4) * 4;
        *(float4*)&sK[warp][t][d4] = *(const float4*)(base + (size_t)t * 3 * C + C + h * DH + d4);
        *(float4*)&sV[warp][t][d4] = *(const float4*)(base + (size_t)t * 3 * C + 2 * C + h * DH + d4);
    }
    float q[DH], o[DH];
#pragma unroll
    for (int d = 0; d < DH; d++) o[d] = 0.f;
    if constexpr (DH == 32) {
        // the lane's own query row, loaded with whole 64-byte row segments per instruction and transposed through s_out
        float* stq = (float*)s_out[warp];
#pragma unroll
        for (int half = 0; half < 2; half++) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
                const int rr = jj * 8 + (lane >> 2), cq = lane & 3;
                *(float4*)(stq + rr * 16 + ((cq ^ ((rr >> 1) & 3)) << 2)) =
                    *(const float4*)(base + (size_t)rr * 3 * C + h * DH + half * 16 + cq * 4);
            }
            __syncwarp();
#pragma unroll
            for (int cq = 0; cq < 4; cq++) {
                const float4 v = *(const float4*)(stq + lane * 16 + ((cq ^ ((lane >> 1) & 3)) << 2));
                q[half * 16 + cq * 4] = v.x; q[half * 16 + cq * 4 + 1] = v.y; q[half * 16 + cq * 4 + 2] = v.z; q[half * 16 + cq * 4 + 3] = v.w;
            }
            __syncwarp();
        }
    } else {
#pragma unroll
        for (int d = 0; d < DH; d += 4) {
            const float4 v = *(const float4*)(base + (size_t)lane * 3 * C + h * DH + d);
            q[d] = v.x; q[d + 1] = v.y; q[d + 2] = v.z; q[d + 3] = v.w;
        }
    }
    __syncwarp();
    // two passes: all 31 scores first (registers), then softmax weights and the weighted sum of V.  exp via ex2.approx
    // (2 ulp) on log2e-prescaled scores: far inside the 1e-3 logit tolerance, and ~35 % fewer instructions than the
    // online-softmax form (no running-max rescale of the accumulator).
    const float scale_l2 = rsqrtf((float)DH) * 1.4426950408889634f;
    float sc[R_COLS];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < R_COLS; j++) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int d = 0; d < DH; d += 4) {
            const float4 k = *(const float4*)&sK[warp][j][d];
            s0 = fmaf(q[d], k.x, s0); s1 = fmaf(q[d + 1], k.y, s1); s2 = fmaf(q[d + 2], k.z, s2); s3 = fmaf(q[d + 3], k.w, s3);
        }
        sc[j] = ((s0 + s1) + (s2 + s3)) * scale_l2;
        m = fmaxf(m, sc[j]);
    }
    float l = 0.f;
#pragma unroll
    for (int j = 0; j < R_COLS; j++) {
        const float p = exp2f(sc[j] - m);
        l += p;
#pragma unroll
        for (int d = 0; d < DH; d += 4) {
            const float4 v = *(const float4*)&sV[warp][j][d];
            o[d] = fmaf(p, v.x, o[d]); o[d + 1] = fmaf(p, v.y, o[d + 1]); o[d + 2] = fmaf(p, v.z, o[d + 2]); o[d + 3] = fmaf(p, v.w, o[d + 3]);
        }
    }
    const float inv = (lane < R_COLS) ? 1.f / l : 0.f;  // the pad token row is written as zeros
    // split bf16 output.  A lane owns a token row (DH values = DH*2 bytes of hi and of lo); rows are transposed through a
    // per-warp buffer so that each global store instruction covers whole 64-byte row segments instead of 32 scattered pieces.
    uint32_t* stg = s_out[warp];
    constexpr int WPR = DH / 2;  // packed words per row and array
    uint32_t hiw[WPR], low[WPR];
#pragma unroll
    for (int d = 0; d < DH; d += 2) split2f(o[d] * inv, o[d + 1] * inv, hiw[d >> 1], low[d >> 1]);
    const size_t ob = (size_t)n * TOK_PER_POS * C + h * DH;  // row 0 of this position, this head's columns
#pragma unroll
    for (int arr = 0; arr < 2; arr++) {
        const uint32_t* w = arr ? low : hiw;
        __nv_bfloat16* gb = (arr ? Olo : Ohi) + ob;
#pragma unroll
        for (int cq = 0; cq < WPR / 4; cq++)
            *(uint4*)(stg + lane * WPR + ((cq ^ ((lane >> 1) & (WPR / 4 - 1))) << 2)) = make_uint4(w[cq * 4], w[cq * 4 + 1], w[cq * 4 + 2], w[cq * 4 + 3]);
        __syncwarp();
        constexpr int LPR = WPR / 4;        // lanes per row (16-byte chunks per row)
        constexpr int RPI = 32 / LPR;       // rows per instruction
#pragma unroll
        for (int jj = 0; jj < 32 / RPI; jj++) {
            const int rr = jj * RPI + lane / LPR, cq = lane % LPR;
            *(uint4*)(gb + (size_t)rr * C + cq * 8) = *(const uint4*)(stg + rr * WPR + ((cq ^ ((rr >> 1) & (LPR - 1))) << 2));
        }
        __syncwarp();
    }
}

// ---- heads: base logits (5) + info logit (1), argmax (last maximal index wins, NaN greatest:
//      Rust max_by_key over OrderedFloat, src/consensus.rs:136-141; of_less in common.cuh) written into row_emit. -----
__global__ void k_heads(BatchView b, FwdWeights wt, uint32_t n0, uint32_t npos, const float* __restrict__ Z,
                        float* __restrict__ logits, float* __restrict__ info) {
    const uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (n >= npos) return;
    const int D = wt.D;
    const float* z = Z + (size_t)n * D;
    float acc[6] = {0, 0, 0, 0, 0, 0};
    for (int i = lane; i < D; i += 32) {
        const float zv = z[i];
#pragma unroll
        for (int k = 0; k < 5; k++) acc[k] = fmaf(zv, wt.wb[(size_t)k * D + i], acc[k]);
        acc[5] = fmaf(zv, wt.wi[i], acc[5]);
    }
#pragma unroll
    for (int k = 0; k < 6; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(HB_FULL, acc[k], o);
    if (lane == 0) {
        float lg[5];
#pragma unroll
        for (int k = 0; k < 5; k++) { lg[k] = acc[k] + wt.bb[k]; logits[(size_t)(n0 + n) * 5 + k] = lg[k]; }
        info[n0 + n] = acc[5] + wt.bi[0];
        int am = 0;
#pragma unroll
        for (int k = 1; k < 5; k++) if (!of_less(lg[k], lg[am])) am = k;
        const uint32_t w = b.fwd_win[n0 + n], r = b.fwd_row[n0 + n];
        if (b.w_nsel[w] >= 2) b.row_emit[b.w_rowbase[w] + r] = (uint8_t)(am | 0x80);
    }
}

// ------------------------------------------------------------------------------------------
struct FwdWs {
    float *X, *QKV, *Z;
    __nv_bfloat16 *Hhi, *Hlo, *Fhi, *Flo;
    // position-axis stage (only carved when the model has one): its QKV, LayerNorm / attention output and hidden layer
    float* Pqkv = nullptr;
    __nv_bfloat16 *Phi = nullptr, *Plo = nullptr, *PFhi = nullptr, *PFlo = nullptr;
    size_t bytes;
};
static bool ffn_is_fused(const FwdWeights& wt) { return wt.C == 128 && wt.F == 512 && !wt.no_fuse_ln && !wt.no_fuse_ffn; }
// the attention out-projection (+ residual + ln2) runs inside the fused FFN kernel
static bool oproj_in_ffn(const FwdWeights& wt) { return ffn_is_fused(wt) && !wt.no_fuse_oproj; }
static FwdWs carve(const FwdWeights& wt, size_t npos, uint8_t* base) {
    const size_t np = (npos + 127) / 128 * 128;  // positions padded to a GEMM tile
    const size_t T = np * TOK_PER_POS;
    FwdWs w;
    size_t o = 0;
    w.X = (float*)(base + o); o += al256(T * wt.C * 4);
    w.QKV = (float*)(base + o); o += al256(T * 3 * wt.C * 4);
    w.Z = (float*)(base + o); o += al256(np * wt.D * 4);
    w.Hhi = (__nv_bfloat16*)(base + o); o += al256(T * wt.C * 2);
    w.Hlo = (__nv_bfloat16*)(base + o); o += al256(T * wt.C * 2);
    // the [T,F] hidden activations exist in memory only on the unfused FFN path
    const size_t TF = ffn_is_fused(wt) ? 0 : T;
    w.Fhi = (__nv_bfloat16*)(base + o); o += al256(TF * wt.F * 2);
    w.Flo = (__nv_bfloat16*)(base + o); o += al256(TF * wt.F * 2);
    if (wt.pos_layers) {
        w.Pqkv = (float*)(base + o); o += al256(np * 3 * wt.D * 4);
        w.Phi = (__nv_bfloat16*)(base + o); o += al256(np * wt.D * 2);
        w.Plo = (__nv_bfloat16*)(base + o); o += al256(np * wt.D * 2);
        w.PFhi = (__nv_bfloat16*)(base + o); o += al256(np * wt.pos_ffn * 2);
        w.PFlo = (__nv_bfloat16*)(base + o); o += al256(np * wt.pos_ffn * 2);
    }
    w.bytes = o;
    return w;
}
size_t fwd_workspace_bytes(const FwdWeights& wt, uint32_t chunk_pos) { return carve(wt, chunk_pos, nullptr).bytes; }

void gemm_simt(int act, int res, const float* A, int lda, const float* Wt, const float* bias, float* Cout, int ldc,
               const float* Res, size_t M, int N, int K, cudaStream_t st) {
    dim3 grid((unsigned)((M + 127) / 128), (unsigned)(N / 64));
    if (act == 0 && res == 0) k_gemm<0, 0><<<grid, 256, 0, st>>>(A, lda, Wt, bias, Cout, ldc, Res, K);
    else if (act == 1 && res == 0) k_gemm<1, 0><<<grid, 256, 0, st>>>(A, lda, Wt, bias, Cout, ldc, Res, K);
    else k_gemm<0, 1><<<grid, 256, 0, st>>>(A, lda, Wt, bias, Cout, ldc, Res, K);
}

static void gemm(const FwdWeights& wt, int mode, const __nv_bfloat16* Ahi, const __nv_bfloat16* Alo, size_t lda, const SplitW& sw,
                 const float* bias, float* out, const float* res, size_t ldc, __nv_bfloat16* ohi, __nv_bfloat16* olo, size_t ldo,
                 size_t M, int N, int K, cudaStream_t st, KTimer& kt) {
    GemmArgs a{};
    a.Ahi = Ahi; a.Alo = Alo; a.lda = lda;
    a.Whi = (const __nv_bfloat16*)sw.hi; a.Wlo = (const __nv_bfloat16*)sw.lo; a.K = (uint32_t)K;
    a.bias = bias; a.out = out; a.res = res; a.ldc = ldc; a.out_hi = ohi; a.out_lo = olo; a.ldo = ldo;
    a.m_tiles = (uint32_t)(M / 128); a.n_chunks = (uint32_t)(N / 128); a.k_blocks = (uint32_t)(K / 64);
    a.mode = mode;
    kt.begin(K_GEMM);
    gemm_tc(a, wt.num_sms, st);
    kt.end();
}

// residual-stream contraction with N == C == 128 and the following LayerNorm fused in the epilogue
static void gemm_ln(const FwdWeights& wt, const __nv_bfloat16* Ahi, const __nv_bfloat16* Alo, size_t lda, const SplitW& sw,
                    const float* bias, float* X, const float* ln_g, const float* ln_b, __nv_bfloat16* ohi, __nv_bfloat16* olo,
                    size_t M, int K, cudaStream_t st, KTimer& kt) {
    GemmArgs a{};
    a.Ahi = Ahi; a.Alo = Alo; a.lda = lda;
    a.Whi = (const __nv_bfloat16*)sw.hi; a.Wlo = (const __nv_bfloat16*)sw.lo; a.K = (uint32_t)K;
    a.bias = bias; a.out = X; a.res = X; a.ldc = 128; a.out_hi = ohi; a.out_lo = olo; a.ldo = 128;
    a.ln_g = ln_g; a.ln_b = ln_b;
    a.m_tiles = (uint32_t)(M / 128); a.n_chunks = 1; a.k_blocks = (uint32_t)(K / 64);
    a.mode = GEMM_OUT_F32_RES_LN;
    kt.begin(K_GEMM);
    gemm_tc(a, wt.num_sms, st);
    kt.end();
}

// contractions of the position-axis stage per supported position: QKV, out-projection, FFN1, FFN2
static uint64_t pos_gemm_flops_per_pos(const FwdWeights& wt) {
    const uint64_t D = wt.D, P = wt.pos_ffn;
    return (uint64_t)wt.pos_layers * 2 * (D * 3 * D + D * D + 2 * D * P);
}
uint64_t pos_attn_flops(const FwdWeights& wt, const uint32_t* nsup, size_t nwin) {
    uint64_t s2 = 0;
    for (size_t w = 0; w < nwin; w++) s2 += (uint64_t)nsup[w] * nsup[w];
    return 4 * (uint64_t)wt.D * wt.pos_layers * s2;  // per layer and head: QK^T and PV, 2 * n^2 * head_dim each
}

// algorithmic FLOPs per supported position (2 * MACs), and the part that is dense contractions
uint64_t forward_flops_per_pos(const FwdWeights& wt, uint64_t* gemm_flops) {
    const uint64_t C = wt.C, F = wt.F, D = wt.D, K = wt.stem_k, S = R_COLS, dh = wt.C / wt.H;
    const uint64_t stem = S * K * 7 * C * 2;
    const uint64_t per_layer_gemm = S * 2 * (C * 3 * C + C * C + 2 * C * F);
    const uint64_t per_layer_attn = (uint64_t)wt.H * 2 * 2 * S * S * dh;
    const uint64_t collapse = 2 * S * C * D;
    const uint64_t heads = 2 * D * 6;
    const uint64_t g = (uint64_t)wt.layers * per_layer_gemm + collapse + pos_gemm_flops_per_pos(wt);
    if (gemm_flops) *gemm_flops = g;
    return stem + g + (uint64_t)wt.layers * per_layer_attn + heads;
}

static bool attn_is_fused(const FwdWeights& wt) { return wt.layer[0].bqkvp && !wt.no_fuse_attn; }
void forward_class_flops_per_pos(const FwdWeights& wt, uint64_t (&out)[16]) {
    const uint64_t C = wt.C, F = wt.F, D = wt.D, K = wt.stem_k, S = R_COLS, dh = wt.C / wt.H, L = wt.layers;
    for (auto& o : out) o = 0;
    out[K_STEM] = S * K * 7 * C * 2;
    const uint64_t qkv = S * 2 * C * 3 * C, attn = (uint64_t)wt.H * 2 * 2 * S * S * dh, oproj = S * 2 * C * C, ffn = S * 2 * 2 * C * F;
    if (attn_is_fused(wt)) out[K_QKV_ATTN] = L * (qkv + attn);
    else { out[K_GEMM] += L * qkv; out[K_ATTENTION] = L * attn; }
    out[K_GEMM] += 2 * S * C * D;
    if (oproj_in_ffn(wt)) out[K_FFN] += L * oproj; else out[K_GEMM] += L * oproj;
    if (ffn_is_fused(wt)) out[K_FFN] += L * ffn; else out[K_GEMM] += L * ffn;
    out[K_GEMM] += pos_gemm_flops_per_pos(wt);
    out[K_HEADS] = 2 * D * 6;
}

// The position-axis encoder stage on Z [np_pad][D] (the collapse output), in place: Z += pe, then per layer
// Z += Wo·Attn(LN1(Z)) and Z += W2·relu(W1·LN2(Z)).  The chunk holds whole windows [w0, w0+nwin); each is one sequence.
static int pos_stage(const BatchView& b, const FwdWeights& wt, const FwdWs& ws, uint32_t n0, uint32_t npos, uint32_t w0,
                     uint32_t nwin, size_t np_pad, cudaStream_t st, KTimer& kt) {
    const int D = wt.D, P = wt.pos_ffn;
    const unsigned ln_blocks = (unsigned)((np_pad * 32 + 255) / 256);
    int nl = 0;
    kt.begin(K_LAYERNORM);
    launch_pos_embed(b, n0, npos, D, ws.Z, st);
    k_layernorm<<<ln_blocks, 256, 0, st>>>(ws.Z, ws.Phi, ws.Plo, wt.pos[0].ln1_g, wt.pos[0].ln1_b, (uint32_t)np_pad, D);
    kt.end(); nl += 2;
    for (int l = 0; l < wt.pos_layers; l++) {
        const PosLayer& ly = wt.pos[l];
        gemm(wt, GEMM_OUT_F32, ws.Phi, ws.Plo, D, ly.s_qkv, ly.bqkv, ws.Pqkv, nullptr, 3 * D, nullptr, nullptr, 0, np_pad, 3 * D, D, st, kt); nl++;
        // the attention output goes over the LN buffers, which the QKV contraction has consumed (stream order); the rows of
        // the last tile's pad positions are in no window and keep their finite LayerNorm values
        PosAttnArgs pa{ws.Pqkv, (size_t)3 * D, b.w_supbase + w0, b.w_nsup + w0, n0, nwin, D, wt.pos_heads, ws.Phi, ws.Plo, (size_t)D};
        kt.begin(K_POS_ATTN); pos_attention(pa, st); kt.end(); nl++;
        gemm(wt, GEMM_OUT_F32_RES, ws.Phi, ws.Plo, D, ly.s_o, ly.bo, ws.Z, ws.Z, D, nullptr, nullptr, 0, np_pad, D, D, st, kt); nl++;
        kt.begin(K_LAYERNORM); k_layernorm<<<ln_blocks, 256, 0, st>>>(ws.Z, ws.Phi, ws.Plo, ly.ln2_g, ly.ln2_b, (uint32_t)np_pad, D); kt.end(); nl++;
        gemm(wt, GEMM_OUT_SPLIT_RELU, ws.Phi, ws.Plo, D, ly.s_1, ly.b1, nullptr, nullptr, 0, ws.PFhi, ws.PFlo, P, np_pad, P, D, st, kt); nl++;
        gemm(wt, GEMM_OUT_F32_RES, ws.PFhi, ws.PFlo, P, ly.s_2, ly.b2, ws.Z, ws.Z, D, nullptr, nullptr, 0, np_pad, D, P, st, kt); nl++;
        if (l + 1 < wt.pos_layers) {
            kt.begin(K_LAYERNORM);
            k_layernorm<<<ln_blocks, 256, 0, st>>>(ws.Z, ws.Phi, ws.Plo, wt.pos[l + 1].ln1_g, wt.pos[l + 1].ln1_b, (uint32_t)np_pad, D);
            kt.end(); nl++;
        }
    }
    return nl;
}

// Runs positions [n0, n0+npos) of the work list, the whole windows [w0, w0+nwin).  Returns the number of kernel launches.
int launch_forward_chunk(const BatchView& b, const FwdWeights& wt, uint32_t n0, uint32_t npos, uint32_t w0, uint32_t nwin,
                         uint8_t* wsb, float* logits, float* info, cudaStream_t st, KTimer& kt) {
    const int C = wt.C, F = wt.F, D = wt.D, H = wt.H;
    const size_t np_pad = (size_t)(npos + 127) / 128 * 128;
    const size_t T = np_pad * TOK_PER_POS;
    const FwdWs ws = carve(wt, npos, wsb);
    int nl = 0;
    // tokens of the pad positions of the last tile must be finite
    if (T > (size_t)npos * TOK_PER_POS)
        cudaMemsetAsync(ws.X + (size_t)npos * TOK_PER_POS * C, 0, (T - (size_t)npos * TOK_PER_POS) * C * sizeof(float), st);
    const size_t stem_smem = ((wt.stem_k * 32 + 15) & ~15) + (size_t)wt.stem_k * 32 * 4;
    const unsigned ln_blocks = (unsigned)((T * 32 + 255) / 256);
    // With C == 128 a kernel that writes the residual stream owns whole rows in its epilogue, so the LayerNorm that
    // follows is computed there (stem epilogue, GEMM_OUT_F32_RES_LN, fused FFN); k_layernorm is the fallback.
    const bool no_fuse = wt.no_fuse_ln != 0;  // debugging aid / A-B parity test
    const bool fuse_ln = (C == 128) && !no_fuse;
    const bool stem_ln = fuse_ln && wt.stem_kblocks;
    if (stem_ln && T > (size_t)npos * TOK_PER_POS) {  // rows of the pad positions: defined operands for the contractions
        const size_t off = (size_t)npos * TOK_PER_POS * C, n = (T - (size_t)npos * TOK_PER_POS) * C;
        cudaMemsetAsync(ws.Hhi + off, 0, n * sizeof(__nv_bfloat16), st);
        cudaMemsetAsync(ws.Hlo + off, 0, n * sizeof(__nv_bfloat16), st);
    }
    kt.begin(K_STEM);
    if (wt.stem_kblocks) {
        StemArgs sa{(const __nv_bfloat16*)wt.s_stem.hi, (const __nv_bfloat16*)wt.s_stem.lo, (uint32_t)wt.stem_kblocks * 64,
                    (uint32_t)wt.stem_kblocks, (uint32_t)wt.stem_k, wt.stem_b, wt.read_pos, ws.X, n0, npos};
        if (stem_ln) { sa.ln_g = wt.layer[0].ln1_g; sa.ln_b = wt.layer[0].ln1_b; sa.out_hi = ws.Hhi; sa.out_lo = ws.Hlo; }
        stem_tc(b, sa, wt.num_sms, st);
    } else {
        k_stem<<<npos, (C + 31) / 32 * 32, stem_smem, st>>>(b, wt, n0, npos, ws.X);
    }
    kt.end(); nl++;
    if (!stem_ln) {
        kt.begin(K_LAYERNORM);
        k_layernorm<<<ln_blocks, 256, 0, st>>>(ws.X, ws.Hhi, ws.Hlo, wt.layer[0].ln1_g, wt.layer[0].ln1_b, (uint32_t)T, C);
        kt.end(); nl++;
    }
    for (int l = 0; l < wt.layers; l++) {
        const FwdLayer& ly = wt.layer[l];
        if (attn_is_fused(wt)) {  // HERRO_B200_NO_FUSE_ATTN: debugging aid / A-B parity test
            // QKV projection + attention in one kernel (q, k, v stay on chip); output over the LN buffers, tile-local in-place
            QkvAttnArgs qa{ws.Hhi, ws.Hlo, (const __nv_bfloat16*)ly.s_qkvp.hi, (const __nv_bfloat16*)ly.s_qkvp.lo, ly.bqkvp, ws.Hhi, ws.Hlo,
                           (uint32_t)(T / 128)};
            kt.begin(K_QKV_ATTN); qkv_attn_tc(qa, wt.num_sms, st); kt.end(); nl++;
        } else {
            gemm(wt, GEMM_OUT_F32, ws.Hhi, ws.Hlo, C, ly.s_qkv, ly.bqkv, ws.QKV, nullptr, 3 * C, nullptr, nullptr, 0, T, 3 * C, C, st, kt); nl++;
            // attention writes its (split) output over the LN buffers: the QKV contraction has consumed them (stream order)
            const unsigned ab = (unsigned)(((size_t)np_pad * H + 3) / 4);
            kt.begin(K_ATTENTION);
            if (C / H == 16) k_attention<16><<<ab, 128, 0, st>>>(ws.QKV, ws.Hhi, ws.Hlo, (uint32_t)np_pad, C, H);
            else k_attention<32><<<ab, 128, 0, st>>>(ws.QKV, ws.Hhi, ws.Hlo, (uint32_t)np_pad, C, H);  // head_dim validated at load
            kt.end(); nl++;
        }
        // out-proj + residual (+ LN2 -> split H).  In-place on H is safe: a row's outputs are written by the
        // thread that owns the row only after every MMA that reads the tile has completed (tfull barrier).
        if (oproj_in_ffn(wt)) {
            // nothing here: k_ffn_ws<true> applies Wo, the residual and ln2 to the attention output itself
        } else if (fuse_ln) {
            gemm_ln(wt, ws.Hhi, ws.Hlo, C, ly.s_o, ly.bo, ws.X, ly.ln2_g, ly.ln2_b, ws.Hhi, ws.Hlo, T, C, st, kt); nl++;
        } else {
            gemm(wt, GEMM_OUT_F32_RES, ws.Hhi, ws.Hlo, C, ly.s_o, ly.bo, ws.X, ws.X, C, nullptr, nullptr, 0, T, C, C, st, kt); nl++;
            kt.begin(K_LAYERNORM); k_layernorm<<<ln_blocks, 256, 0, st>>>(ws.X, ws.Hhi, ws.Hlo, ly.ln2_g, ly.ln2_b, (uint32_t)T, C); kt.end(); nl++;
        }
        const float* ng = (l + 1 < wt.layers) ? wt.layer[l + 1].ln1_g : wt.lnf_g;
        const float* nb = (l + 1 < wt.layers) ? wt.layer[l + 1].ln1_b : wt.lnf_b;
        if (ffn_is_fused(wt)) {
            // FFN1 -> ReLU -> FFN2 + residual + next LayerNorm in one kernel; the hidden activations stay on chip.
            // In-place on H is safe: the tile's H rows are only overwritten after all of its MMAs have completed.
            FfnArgs fa{ws.Hhi, ws.Hlo, (const __nv_bfloat16*)ly.s_1.hi, (const __nv_bfloat16*)ly.s_1.lo,
                       (const __nv_bfloat16*)ly.s_2.hi, (const __nv_bfloat16*)ly.s_2.lo, ly.b1, ly.b2, ws.X, ng, nb, ws.Hhi, ws.Hlo,
                       (uint32_t)F, (uint32_t)(T / 128)};
            fa.store_x = (l + 1 < wt.layers) ? 1 : 0;
            if (oproj_in_ffn(wt)) {
                fa.Wohi = (const __nv_bfloat16*)ly.s_o.hi; fa.Wolo = (const __nv_bfloat16*)ly.s_o.lo;
                fa.bo = ly.bo; fa.ln2_g = ly.ln2_g; fa.ln2_b = ly.ln2_b;
            }
            kt.begin(K_FFN); ffn_tc(fa, wt.num_sms, st); kt.end(); nl++;
            continue;
        }
        gemm(wt, GEMM_OUT_SPLIT_RELU, ws.Hhi, ws.Hlo, C, ly.s_1, ly.b1, nullptr, nullptr, 0, ws.Fhi, ws.Flo, F, T, F, C, st, kt); nl++;
        if (fuse_ln) {
            gemm_ln(wt, ws.Fhi, ws.Flo, F, ly.s_2, ly.b2, ws.X, ng, nb, ws.Hhi, ws.Hlo, T, F, st, kt); nl++;
        } else {
            gemm(wt, GEMM_OUT_F32_RES, ws.Fhi, ws.Flo, F, ly.s_2, ly.b2, ws.X, ws.X, C, nullptr, nullptr, 0, T, C, F, st, kt); nl++;
            kt.begin(K_LAYERNORM); k_layernorm<<<ln_blocks, 256, 0, st>>>(ws.X, ws.Hhi, ws.Hlo, ng, nb, (uint32_t)T, C); kt.end(); nl++;
        }
    }
    // read-axis collapse: row n = the 31*C contiguous values of position n (token 31 excluded)
    gemm(wt, GEMM_OUT_F32_RELU, ws.Hhi, ws.Hlo, (size_t)TOK_PER_POS * C, wt.s_c, wt.bc, ws.Z, nullptr, D, nullptr, nullptr, 0, np_pad, D,
         R_COLS * C, st, kt); nl++;
    if (wt.pos_layers) nl += pos_stage(b, wt, ws, n0, npos, w0, nwin, np_pad, st, kt);
    kt.begin(K_HEADS);
    k_heads<<<(unsigned)(((size_t)npos * 32 + 127) / 128), 128, 0, st>>>(b, wt, n0, npos, ws.Z, logits, info);
    kt.end(); nl++;
    return nl;
}

}  // namespace hb
