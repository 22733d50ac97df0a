// pos_attn.cu — the position-axis encoder stage's device pieces: the sinusoidal position encoding, and multi-head attention
// over variable-length sequences (each window's supported positions) with the keys past a sequence's length masked out.
//
// Attention layout: one CTA of 4 warps per (sequence, head).  The CTA walks the sequence in 64-query blocks, 16 queries per
// warp, and for each block walks 64-key blocks staged in shared memory as split bf16 (K row-major, V transposed, so both
// B fragments are 32-bit shared loads).  QK^T and PV are mma.sync.m16n8k16 in three passes (hi*hi + lo*hi + hi*lo) with
// fp32 accumulation, like every other contraction of the forward (DESIGN.md §4.3); the softmax is the online (running max)
// form in fp32 on log2e-prescaled scores.  The probabilities are split into bf16 hi/lo in registers: the S accumulator
// layout of two adjacent 8-key tiles is the A fragment layout of one 16-key step.
#include <cuda_bf16.h>

#include "common.cuh"
#include "forward.h"

namespace hb {

namespace {

constexpr int PA_Q = 64, PA_K = 64, PA_THREADS = 128;

__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int DH>
__global__ void __launch_bounds__(PA_THREADS) k_pos_attn(PosAttnArgs a) {
    constexpr int KS = DH + 8;    // K row stride (bf16): 8 rows x 4 words of a fragment load hit 32 distinct banks
    constexpr int VS = PA_K + 8;  // V^T row stride (bf16)
    __shared__ __align__(16) __nv_bfloat16 sKhi[PA_K][KS], sKlo[PA_K][KS], sVhi[DH][VS], sVlo[DH][VS];
    const uint32_t len = a.seq_len[blockIdx.x];
    if (len == 0) return;
    const int h = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const size_t row0 = (size_t)(a.seq_base[blockIdx.x] - a.base_sub);
    const float* Qg = a.qkv + row0 * a.ld_qkv + (size_t)h * DH;
    const float* Kg = Qg + a.D;
    const float* Vg = Qg + 2 * a.D;
    const float scale_l2 = rsqrtf((float)DH) * 1.4426950408889634f;
    for (uint32_t q0 = 0; q0 < len; q0 += PA_Q) {
        const uint32_t qr = q0 + warp * 16;  // this warp's first query
        const bool active = qr < len;
        // Q fragments of the warp's 16 queries, split: [k-step][4] (rows g / g+8, columns 2t / 2t+8 of the step)
        uint32_t qh[DH / 16][4], ql[DH / 16][4];
#pragma unroll
        for (int ks = 0; ks < DH / 16; ks++)
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const uint32_t qi = qr + g + (r & 1) * 8;
                float2 v = make_float2(0.f, 0.f);
                if (qi < len) v = *(const float2*)(Qg + (size_t)qi * a.ld_qkv + ks * 16 + (r >> 1) * 8 + 2 * t);
                split2(v.x, v.y, qh[ks][r], ql[ks][r]);
            }
        float o[DH / 8][4];
#pragma unroll
        for (int i = 0; i < DH / 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows g and g+8 (l: this thread's partial sums)
        for (uint32_t k0 = 0; k0 < len; k0 += PA_K) {
            __syncthreads();  // the previous key block has been consumed
            for (int i = threadIdx.x; i < PA_K * DH / 4; i += PA_THREADS) {
                const int kr = i / (DH / 4), d = (i % (DH / 4)) * 4;
                float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;  // keys past the end: zeros (masked, and 0 * V stays 0)
                if (k0 + kr < len) {
                    kv = *(const float4*)(Kg + (size_t)(k0 + kr) * a.ld_qkv + d);
                    vv = *(const float4*)(Vg + (size_t)(k0 + kr) * a.ld_qkv + d);
                }
                uint2 hi, lo;
                split2(kv.x, kv.y, hi.x, lo.x);
                split2(kv.z, kv.w, hi.y, lo.y);
                *(uint2*)&sKhi[kr][d] = hi;
                *(uint2*)&sKlo[kr][d] = lo;
                split2(vv.x, vv.y, hi.x, lo.x);
                split2(vv.z, vv.w, hi.y, lo.y);
                const __nv_bfloat16* ph = (const __nv_bfloat16*)&hi;
                const __nv_bfloat16* pl = (const __nv_bfloat16*)&lo;
#pragma unroll
                for (int j = 0; j < 4; j++) { sVhi[d + j][kr] = ph[j]; sVlo[d + j][kr] = pl[j]; }
            }
            __syncthreads();
            if (!active) continue;
            // S = Q K^T for 64 keys: 8 tiles of 8 keys
            float s[PA_K / 8][4];
#pragma unroll
            for (int j = 0; j < PA_K / 8; j++) {
                s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
                for (int ks = 0; ks < DH / 16; ks++) {
                    const uint32_t bh0 = *(const uint32_t*)&sKhi[j * 8 + g][ks * 16 + 2 * t];
                    const uint32_t bh1 = *(const uint32_t*)&sKhi[j * 8 + g][ks * 16 + 2 * t + 8];
                    const uint32_t bl0 = *(const uint32_t*)&sKlo[j * 8 + g][ks * 16 + 2 * t];
                    const uint32_t bl1 = *(const uint32_t*)&sKlo[j * 8 + g][ks * 16 + 2 * t + 8];
                    mma_bf16(s[j], qh[ks], bh0, bh1);
                    mma_bf16(s[j], ql[ks], bh0, bh1);
                    mma_bf16(s[j], qh[ks], bl0, bl1);
                }
            }
            // mask, scale, running max of rows g (elements 0,1) and g+8 (elements 2,3)
            float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
            for (int j = 0; j < PA_K / 8; j++)
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const uint32_t key = k0 + j * 8 + 2 * t + (e & 1);
                    s[j][e] = key < len ? s[j][e] * scale_l2 : -INFINITY;
                    if (e < 2) bm0 = fmaxf(bm0, s[j][e]); else bm1 = fmaxf(bm1, s[j][e]);
                }
#pragma unroll
            for (int x = 1; x <= 2; x <<= 1) {
                bm0 = fmaxf(bm0, __shfl_xor_sync(HB_FULL, bm0, x));
                bm1 = fmaxf(bm1, __shfl_xor_sync(HB_FULL, bm1, x));
            }
            const float mn0 = fmaxf(m0, bm0), mn1 = fmaxf(m1, bm1);  // finite: key k0 < len is in every block
            const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
            m0 = mn0; m1 = mn1;
            l0 *= c0; l1 *= c1;
#pragma unroll
            for (int i = 0; i < DH / 8; i++) { o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1; }
#pragma unroll
            for (int j = 0; j < PA_K / 8; j++) {
                s[j][0] = exp2f(s[j][0] - mn0); s[j][1] = exp2f(s[j][1] - mn0);
                s[j][2] = exp2f(s[j][2] - mn1); s[j][3] = exp2f(s[j][3] - mn1);
                l0 += s[j][0] + s[j][1];
                l1 += s[j][2] + s[j][3];
            }
            // O += P V: 4 steps of 16 keys; P's A fragment of step kk is tiles 2kk (columns 2t) and 2kk+1 (columns 2t+8)
#pragma unroll
            for (int kk = 0; kk < PA_K / 16; kk++) {
                uint32_t ph[4], pl[4];
                split2(s[2 * kk][0], s[2 * kk][1], ph[0], pl[0]);
                split2(s[2 * kk][2], s[2 * kk][3], ph[1], pl[1]);
                split2(s[2 * kk + 1][0], s[2 * kk + 1][1], ph[2], pl[2]);
                split2(s[2 * kk + 1][2], s[2 * kk + 1][3], ph[3], pl[3]);
#pragma unroll
                for (int nd = 0; nd < DH / 8; nd++) {
                    const uint32_t bh0 = *(const uint32_t*)&sVhi[nd * 8 + g][kk * 16 + 2 * t];
                    const uint32_t bh1 = *(const uint32_t*)&sVhi[nd * 8 + g][kk * 16 + 2 * t + 8];
                    const uint32_t bl0 = *(const uint32_t*)&sVlo[nd * 8 + g][kk * 16 + 2 * t];
                    const uint32_t bl1 = *(const uint32_t*)&sVlo[nd * 8 + g][kk * 16 + 2 * t + 8];
                    mma_bf16(o[nd], ph, bh0, bh1);
                    mma_bf16(o[nd], pl, bh0, bh1);
                    mma_bf16(o[nd], ph, bl0, bl1);
                }
            }
        }
        if (!active) continue;
#pragma unroll
        for (int x = 1; x <= 2; x <<= 1) {
            l0 += __shfl_xor_sync(HB_FULL, l0, x);
            l1 += __shfl_xor_sync(HB_FULL, l1, x);
        }
        const float i0 = 1.f / l0, i1 = 1.f / l1;
        const uint32_t r0 = qr + g, r1 = qr + g + 8;
#pragma unroll
        for (int nd = 0; nd < DH / 8; nd++) {
            const size_t col = (size_t)h * DH + nd * 8 + 2 * t;
            uint32_t hi, lo;
            if (r0 < len) {
                split2(o[nd][0] * i0, o[nd][1] * i0, hi, lo);
                *(uint32_t*)(a.out_hi + (row0 + r0) * a.ldo + col) = hi;
                *(uint32_t*)(a.out_lo + (row0 + r0) * a.ldo + col) = lo;
            }
            if (r1 < len) {
                split2(o[nd][2] * i1, o[nd][3] * i1, hi, lo);
                *(uint32_t*)(a.out_hi + (row0 + r1) * a.ldo + col) = hi;
                *(uint32_t*)(a.out_lo + (row0 + r1) * a.ldo + col) = lo;
            }
        }
    }
}

// Z[n] += pe(k) for the chunk's positions, k = the position's index in its window's supported list.  pe is evaluated in
// float64 and rounded to float32, so the host reference gets the same value from a different libm.  One warp per row.
__global__ void k_pos_embed(BatchView b, uint32_t n0, uint32_t npos, int D, float* __restrict__ Z) {
    const uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (n >= npos) return;
    const uint32_t w = b.fwd_win[n0 + n];
    const double k = (double)(n0 + n - b.w_supbase[w]);
    float* z = Z + (size_t)n * D;
    for (int i = lane * 2; i < D; i += 64) {
        double sv, cv;
        sincos(k * pow(10000.0, -((double)i / (double)D)), &sv, &cv);
        z[i] += (float)sv;
        z[i + 1] += (float)cv;
    }
}

}  // namespace

cudaError_t pos_attention(const PosAttnArgs& a, cudaStream_t st) {
    if (a.n_seq == 0) return cudaSuccess;
    const dim3 grid(a.n_seq, (unsigned)a.heads);
    const int dh = a.D / a.heads;
    if (dh == 32) k_pos_attn<32><<<grid, PA_THREADS, 0, st>>>(a);
    else if (dh == 64) k_pos_attn<64><<<grid, PA_THREADS, 0, st>>>(a);
    else return cudaErrorInvalidValue;  // head_dim is validated when the model is loaded
    return cudaGetLastError();
}

void launch_pos_embed(const BatchView& b, uint32_t n0, uint32_t npos, int D, float* Z, cudaStream_t st) {
    k_pos_embed<<<(unsigned)(((size_t)npos * 32 + 255) / 256), 256, 0, st>>>(b, n0, npos, D, Z);
}

}  // namespace hb
