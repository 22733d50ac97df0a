// gemm_tc.cu — the dense contractions of the forward on the Hopper tensor cores (wgmma).
//
//   D[M,N] = A[M,K] · W[N,K]^T  (+ bias, ReLU, residual, per the epilogue mode)      fp32 accumulate
//
// Precision: the north_star bound is 1e-3 absolute on fp32 logits, which a single bf16 pass
// (2^-9 operand rounding over ~9 chained contractions) does not meet.  Every fp32 operand x is
// carried as two bf16 terms x = hi + lo (lo = bf16(x - hi)); three wgmma passes accumulate
// hi·hi + lo·hi + hi·lo in the fp32 register accumulator (the dropped lo·lo term is 2^-18 relative).
// Weights are split once at load; activations are produced already split by the kernel that
// writes them (LayerNorm, attention, the FFN1 epilogue), so operand staging is pure copying.
//
// Kernels (all persistent, warp-specialised, one CTA per SM; operands as K-major SWIZZLE_128B shared-memory tiles):
//   k_gemm_ws      D = A·W^T with bias / ReLU / residual / LayerNorm epilogues (out-proj, read-axis collapse, fallbacks)
//   k_ffn_ws       FFN1 -> ReLU -> FFN2 + residual + LayerNorm, hidden activations kept on chip
//   k_qkv_attn_ws  QKV projection (wgmma) + per-position attention (mma.sync)
//   k_stem_tc      embedding + conv stem as a contraction, A tile synthesised from the pileup matrix, + first LayerNorm
// Common skeleton: two consumer warpgroups (warps 0-7) and one producer warp (warp 8; k_ffn_ws: producer warpgroup, warps 8-11),
// one lane of which issues TMA into a ring of k-block stages guarded by full / empty mbarriers.  A work item is a tile of 128
// rows; consumer warpgroup wg issues
// wgmma.m64nNk16 for rows [64 wg, 64 wg + 64) and runs the epilogue on its own accumulator fragments:
// thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 and that + 8, columns 8 j + 2 (t % 4) + {0, 1}
// (acc[4 j], acc[4 j + 1] for the first row, acc[4 j + 2], acc[4 j + 3] for the second).  A row's 128 columns live in
// the 4 lanes of a quad, so a LayerNorm reduces with two shuffles.
#include <cstdio>
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "forward.h"

namespace hb {

namespace {

constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3;
constexpr int STAGE_BYTES = (2 * BM + 2 * BN) * 128;  // A hi/lo + W hi/lo tiles of one k-block: 64 KB
constexpr int C_THREADS = 256, G_THREADS = 288, G_PROD_WARP = 8;  // consumers: warps 0-7 (two warpgroups); producer: warp 8

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA: one thread copies a [rows x 64 bf16] box of a 2-D tensor into a SWIZZLE_128B shared-memory tile
// (the layout the wgmma descriptors expect) and completes `bytes` on the mbarrier
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c_inner, int c_row) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
                 "l"((uint64_t)tm), "r"(smem_u32(bar)), "r"(c_inner), "r"(c_row)
                 : "memory");
}
// named barrier over `n` threads (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// generic-proxy shared-memory writes -> visible to the tensor core (async proxy)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma layout): start address, LBO (unused for a swizzled
// K-major operand that is one atom wide along K), SBO = 8 rows * 128 B, layout type 1 = SWIZZLE_128B.  Tiles are
// 1024-byte aligned, so the base offset is 0; a step of 16 along K inside the atom adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3ffffu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024u >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across an in-flight wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&a)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(a[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] · B[128 x 16]^T, both operands K-major in shared memory (descriptors), fp32 accumulator in registers
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// D[64 x 128] += A[64 x 16] · B[128 x 16]^T, A from registers, B K-major in shared memory.  The A fragment of the warpgroup's
// thread t is the accumulator layout above restricted to 16 columns: a0 = row r, columns 2 (t % 4) + {0, 1}; a1 = row r + 8;
// a2, a3 = the same rows 8 columns on (bf16 pairs, lower column in the low half)
__device__ __forceinline__ void wgmma_n128_ra(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t bdesc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc)
        : "memory");
}
// D[64 x 96] (+)= A[64 x 16] · B[96 x 16]^T, both operands K-major in shared memory (descriptors), fp32 accumulator in registers
__device__ __forceinline__ void wgmma_n96(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// one 64-wide k-block of split operands: hi·hi + lo·hi + hi·lo (4 k-steps of 16), committed as one wgmma group
__device__ __forceinline__ void mma_kblock(float (&acc)[64], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, bool zero) {
    const uint64_t dAh = make_desc(a_hi), dAl = make_desc(a_lo), dBh = make_desc(b_hi), dBl = make_desc(b_lo);
    wg_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; k++) {
        const uint64_t adv = (uint64_t)(k * 2);  // +32 bytes along K inside the swizzle atom
        wgmma_n128(acc, dAh + adv, dBh + adv, (zero && k == 0) ? 0u : 1u);
        wgmma_n128(acc, dAl + adv, dBh + adv, 1u);
        wgmma_n128(acc, dAh + adv, dBl + adv, 1u);
    }
    wg_commit();
}
// the same with A from registers: ah / al hold a 128-wide k range as 8 k-slices of 4 fragment registers; k-block kb is
// slices 4 kb .. 4 kb + 3.  Same pass order as mma_kblock.
__device__ __forceinline__ void mma_kblock_ra(float (&acc)[64], const uint32_t (&ah)[32], const uint32_t (&al)[32], int kb, uint32_t b_hi,
                                              uint32_t b_lo) {
    const uint64_t dBh = make_desc(b_hi), dBl = make_desc(b_lo);
    wg_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; k++) {
        const uint64_t adv = (uint64_t)(k * 2);
        const int s = 4 * (4 * kb + k);
        wgmma_n128_ra(acc, ah[s], ah[s + 1], ah[s + 2], ah[s + 3], dBh + adv);
        wgmma_n128_ra(acc, al[s], al[s + 1], al[s + 2], al[s + 3], dBh + adv);
        wgmma_n128_ra(acc, ah[s], ah[s + 1], ah[s + 2], ah[s + 3], dBl + adv);
    }
    wg_commit();
}
// keeps the compiler from reusing A fragment registers that an in-flight wgmma still reads
template <int R>
__device__ __forceinline__ void reg_fence(uint32_t (&a)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+r"(a[i])::"memory");
}

__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    // hi = bf16(x), lo = bf16(x - hi), two values per 2-wide convert
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    const float ah = __uint_as_float(hi << 16), bh = __uint_as_float(hi & 0xffff0000u);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - ah, b - bh);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ---- epilogue helpers on a [64 x 128] accumulator fragment (see the layout above) ------------------------------------
// LayerNorm statistics (eps 1e-5) of the thread's two rows: mean and 1/std, the row sums completed across the lane quad
__device__ __forceinline__ void frag_ln_stats(const float (&a)[64], float& m0, float& r0, float& m1, float& r1) {
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; j++) { s0 += a[4 * j] + a[4 * j + 1]; s1 += a[4 * j + 2] + a[4 * j + 3]; }
    s0 += __shfl_xor_sync(HB_FULL, s0, 1); s0 += __shfl_xor_sync(HB_FULL, s0, 2);
    s1 += __shfl_xor_sync(HB_FULL, s1, 1); s1 += __shfl_xor_sync(HB_FULL, s1, 2);
    m0 = s0 * (1.f / BN); m1 = s1 * (1.f / BN);
    float v0 = 0.f, v1 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; j++) {
        float d = a[4 * j] - m0; v0 = fmaf(d, d, v0);
        d = a[4 * j + 1] - m0; v0 = fmaf(d, d, v0);
        d = a[4 * j + 2] - m1; v1 = fmaf(d, d, v1);
        d = a[4 * j + 3] - m1; v1 = fmaf(d, d, v1);
    }
    v0 += __shfl_xor_sync(HB_FULL, v0, 1); v0 += __shfl_xor_sync(HB_FULL, v0, 2);
    v1 += __shfl_xor_sync(HB_FULL, v1, 1); v1 += __shfl_xor_sync(HB_FULL, v1, 2);
    r0 = rsqrtf(v0 * (1.f / BN) + 1e-5f); r1 = rsqrtf(v1 * (1.f / BN) + 1e-5f);
}
// LayerNorm of the thread's two rows, in place
__device__ __forceinline__ void frag_layernorm(float (&a)[64], const float* gam, const float* bet, int fc) {
    float m0, r0, m1, r1;
    frag_ln_stats(a, m0, r0, m1, r1);
#pragma unroll
    for (int j = 0; j < 16; j++) {
        const int c = 8 * j + fc;
        const float g0 = gam[c], g1 = gam[c + 1], b0 = bet[c], b1 = bet[c + 1];
        a[4 * j] = (a[4 * j] - m0) * r0 * g0 + b0;
        a[4 * j + 1] = (a[4 * j + 1] - m0) * r0 * g1 + b1;
        a[4 * j + 2] = (a[4 * j + 2] - m1) * r1 * g0 + b0;
        a[4 * j + 3] = (a[4 * j + 3] - m1) * r1 * g1 + b1;
    }
}
// fp32 rows -> row-major global [.., ld] at column c0 (a quad writes 32 contiguous bytes of a row)
__device__ __forceinline__ void frag_store_f32(const float (&a)[64], float* base, size_t ld, size_t row0, int c0, int fc) {
#pragma unroll
    for (int j = 0; j < 16; j++) {
        *(float2*)(base + row0 * ld + c0 + 8 * j + fc) = make_float2(a[4 * j], a[4 * j + 1]);
        *(float2*)(base + (row0 + 8) * ld + c0 + 8 * j + fc) = make_float2(a[4 * j + 2], a[4 * j + 3]);
    }
}
// fp32 rows -> split bf16 row-major global arrays
__device__ __forceinline__ void frag_store_split(const float (&a)[64], __nv_bfloat16* hi, __nv_bfloat16* lo, size_t ld, size_t row0, int c0,
                                                 int fc) {
#pragma unroll
    for (int j = 0; j < 16; j++) {
        uint32_t h, l;
        const size_t o0 = row0 * ld + c0 + 8 * j + fc, o1 = (row0 + 8) * ld + c0 + 8 * j + fc;
        split2(a[4 * j], a[4 * j + 1], h, l);
        *(uint32_t*)(hi + o0) = h; *(uint32_t*)(lo + o0) = l;
        split2(a[4 * j + 2], a[4 * j + 3], h, l);
        *(uint32_t*)(hi + o1) = h; *(uint32_t*)(lo + o1) = l;
    }
}
// fp32 rows -> split bf16 into an operand tile in shared memory ([kb][hi|lo][128 rows x 128 B], SWIZZLE_128B), row r = tile row.
// With `gam`, the rows are written LayerNorm-ed with the statistics ln = {mean0, rstd0, mean1, rstd1} (a is left as it is).
__device__ __forceinline__ void frag_store_tile(const float (&a)[64], uint8_t* tile, int r, int fc, const float* gam = nullptr,
                                                const float* bet = nullptr, const float* ln = nullptr) {
#pragma unroll
    for (int j = 0; j < 16; j++)
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int rr = r + 8 * hf, c = 8 * j + fc;
            float x = a[4 * j + 2 * hf], y = a[4 * j + 2 * hf + 1];
            if (gam) {
                x = (x - ln[2 * hf]) * ln[2 * hf + 1] * gam[c] + bet[c];
                y = (y - ln[2 * hf]) * ln[2 * hf + 1] * gam[c + 1] + bet[c + 1];
            }
            uint32_t h, l;
            split2(x, y, h, l);
            const uint32_t off = (uint32_t)(j >> 3) * (2 * BM * 128) + (uint32_t)rr * 128u + (uint32_t)((((j & 7) ^ (rr & 7)) << 4) + fc * 2);
            *(uint32_t*)(tile + off) = h;
            *(uint32_t*)(tile + off + BM * 128) = l;
        }
}

}  // namespace

__global__ void __launch_bounds__(G_THREADS, 1) k_gemm_ws(GemmArgs g, const __grid_constant__ CUtensorMap tmAhi,
                                                         const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmWhi,
                                                         const __grid_constant__ CUtensorMap tmWlo) {
    extern __shared__ uint8_t smem_dyn[];
    // SWIZZLE_128B operands need 1024-byte alignment; the dynamic segment starts after the static one
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    __shared__ __align__(16) float s_lng[BN], s_lnb[BN];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], C_THREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (g.mode == GEMM_OUT_F32_RES_LN && tid < BN) { s_lng[tid] = g.ln_g[tid]; s_lnb[tid] = g.ln_b[tid]; }
    __syncthreads();

    const uint32_t n_items = g.m_tiles * g.n_chunks;
    const uint32_t kbs = g.k_blocks;

    if (warp == G_PROD_WARP) {
        // =============================== producer: one lane issues the TMA copies ===============================
        if (lane == 0) {
            uint32_t it_stage = 0;  // running k-block counter -> ring stage / parity
            for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x) {
                const int m0 = (int)((item / g.n_chunks) * BM), n0 = (int)((item % g.n_chunks) * BN);
                for (uint32_t kb = 0; kb < kbs; kb++, it_stage++) {
                    const uint32_t s = it_stage % STAGES, ph = (it_stage / STAGES) & 1;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    const uint32_t sb = smem_u32(smem + (size_t)s * STAGE_BYTES);
                    const int k0 = (int)(kb * BK);
                    mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
                    tma_load_2d(sb, &tmAhi, &full_bar[s], k0, m0);
                    tma_load_2d(sb + BM * 128, &tmAlo, &full_bar[s], k0, m0);
                    tma_load_2d(sb + 2 * BM * 128, &tmWhi, &full_bar[s], k0, n0);
                    tma_load_2d(sb + 2 * BM * 128 + BN * 128, &tmWlo, &full_bar[s], k0, n0);
                }
            }
        }
        return;
    }
    // =============================== consumers: wgmma over this warpgroup's 64 rows, then the epilogue ===============
    const int wg = warp >> 2;
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2), fc = (lane & 3) * 2;  // fragment row (tile-local) / column offset
    uint32_t it_stage = 0;
    float acc[64];
    for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const uint32_t m0 = (item / g.n_chunks) * BM, n0 = (item % g.n_chunks) * BN;
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < kbs; kb++, it_stage++) {
            const uint32_t s = it_stage % STAGES, ph = (it_stage / STAGES) & 1;
            mbar_wait(&full_bar[s], ph);
            const uint32_t sb = smem_u32(smem + (size_t)s * STAGE_BYTES);
            mma_kblock(acc, sb + wg * 64 * 128, sb + BM * 128 + wg * 64 * 128, sb + 2 * BM * 128, sb + 2 * BM * 128 + BN * 128, kb == 0);
            if (kb > 0) {  // the previous k-block's group has completed: its stage may be refilled
                wg_wait<1>();
                mbar_arrive(&empty_bar[prev]);
            }
            prev = s;
        }
        wg_wait<0>();
        acc_fence(acc);
        mbar_arrive(&empty_bar[prev]);
        const size_t row0 = (size_t)m0 + fr;
        if (g.mode == GEMM_OUT_F32_RES_LN) {
            // residual add + fp32 store, then LayerNorm of the row -> split bf16 (N == 128: the whole row is in the quad)
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int c = 8 * j + fc;
                const float2 bv = *(const float2*)(g.bias + c);
                const float2 x0 = *(const float2*)(g.res + row0 * g.ldc + c), x1 = *(const float2*)(g.res + (row0 + 8) * g.ldc + c);
                acc[4 * j] = acc[4 * j] + bv.x + x0.x; acc[4 * j + 1] = acc[4 * j + 1] + bv.y + x0.y;
                acc[4 * j + 2] = acc[4 * j + 2] + bv.x + x1.x; acc[4 * j + 3] = acc[4 * j + 3] + bv.y + x1.y;
            }
            frag_store_f32(acc, g.out, g.ldc, row0, 0, fc);
            frag_layernorm(acc, s_lng, s_lnb, fc);
            frag_store_split(acc, g.out_hi, g.out_lo, g.ldo, row0, 0, fc);
            continue;
        }
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int c = (int)n0 + 8 * j + fc;
            const float2 bv = *(const float2*)(g.bias + c);
            acc[4 * j] += bv.x; acc[4 * j + 1] += bv.y; acc[4 * j + 2] += bv.x; acc[4 * j + 3] += bv.y;
            if (g.mode == GEMM_OUT_F32_RES) {
                const float2 x0 = *(const float2*)(g.res + row0 * g.ldc + c), x1 = *(const float2*)(g.res + (row0 + 8) * g.ldc + c);
                acc[4 * j] += x0.x; acc[4 * j + 1] += x0.y; acc[4 * j + 2] += x1.x; acc[4 * j + 3] += x1.y;
            } else if (g.mode == GEMM_OUT_F32_RELU || g.mode == GEMM_OUT_SPLIT_RELU) {
#pragma unroll
                for (int e = 0; e < 4; e++) acc[4 * j + e] = fmaxf(acc[4 * j + e], 0.f);
            }
        }
        if (g.mode == GEMM_OUT_SPLIT_RELU) frag_store_split(acc, g.out_hi, g.out_lo, g.ldo, row0, (int)n0, fc);
        else frag_store_f32(acc, g.out, g.ldc, row0, (int)n0, fc);
    }
}

// ------------------------------------------------------------------------------------------------
// Fused FFN for C == 128:   X += W2 · relu(W1 · H + b1) + b2 ;  H' = LayerNorm(X) (split bf16)
// The hidden activations never leave the SM: per 128-token tile and per 128-wide hidden chunk c, each consumer warpgroup
// (64 rows) runs
//   F1(c): accF = H · W1[c]^T           (H tile resident in shared memory)
//   E1(c): relu(accF + b1[c]) -> split bf16 -> A fragments in registers: the accumulator layout is the A fragment layout of
//          the next contraction, k-slice s being (accF[8s], accF[8s+1]), (accF[8s+2], accF[8s+3]), ..., (accF[8s+6], accF[8s+7])
//   F2(c): accO += A · W2[:, c]^T       (wgmma with A from registers)
// accO starts as X + b2, so after F2(3) it holds the new residual row: one final epilogue stores it and its LayerNorm.
// Issue order per warpgroup: F1(0) E1(0) [F2(0) F1(1)] E1(1) ... [F2(2) F1(3)] E1(3) F2(3).  F2(c) and F1(c+1) are issued
// back to back; F2(c) was issued first, so once F1(c+1) has completed the A fragments may be overwritten.  Live registers:
// accO 64 + accF 64 + A fragments 64, within the 240 that setmaxnreg gives each consumer thread.
// W k-block tiles stream through the TMA ring in issue order F1(0) F2(0) F1(1) F2(1) ... F2(3).  Every k-block is one wgmma
// group and its stage is freed as soon as that group has completed, so the producer runs up to FFN_STAGES k-blocks ahead,
// across contractions and tiles.  Saves writing and re-reading the [T, F] hidden tensor (4 KB per token and layer).
// FUSE_O: the attention out-projection, its residual add and LayerNorm (ln2) run in front of the FFN inside this kernel:
//   P0   : accO = O · Wo^T                       (O = attention output tile, loaded where H used to be)
//   E0   : accO = accO + bo + X (= X'), H = LN2(X') -> split bf16 -> written over the warpgroup's rows of the O tile
//          (the A operand of FFN1); accO += b2 and the FFN accumulates on top of it.
// This removes the HBM-bound out-projection kernel (it re-read and re-wrote the fp32 residual stream).
// ------------------------------------------------------------------------------------------------
constexpr int FFN_RING_BYTES = 2 * BN * 128;        // one W k-block tile, hi + lo: 32 KB
constexpr int FFN_A_BYTES = 2 * 2 * BM * 128;       // a [128 x 128] operand as 2 k-blocks x (hi, lo): 64 KB
constexpr int FFN_STAGES = 4;                       // 64 KB operand tile + 4 x 32 KB ring = 192 KB
// consumers: warps 0-7 (two warpgroups); producer: warpgroup 2 (warps 8-11), one lane of which issues the TMA.  setmaxnreg
// moves registers from the producer to the consumers: 24 x 128 + 240 x 256 <= 65 536.  The producer loop fits in 24; with
// 232 per consumer, FUSE_O spills loop state.
constexpr int FFN_THREADS = 384, FFN_PROD_WARP = 8, FFN_PROD_REGS = 24, FFN_CONS_REGS = 240;

// waits for the in-flight k-block groups oldest first and frees each one's ring stage as soon as it has completed;
// it_stage counts the k-blocks issued so far
template <int N>
__device__ __forceinline__ void ffn_retire(uint64_t* empty_bar, uint32_t it_stage) {
    wg_wait<N>();
    mbar_arrive(&empty_bar[(it_stage - 1 - N) % FFN_STAGES]);
    if constexpr (N > 0) ffn_retire<N - 1>(empty_bar, it_stage);
}

template <bool FUSE_O>
__global__ void __launch_bounds__(FFN_THREADS, 1) k_ffn_ws(FfnArgs g, const __grid_constant__ CUtensorMap tmHhi,
                                                        const __grid_constant__ CUtensorMap tmHlo, const __grid_constant__ CUtensorMap tmW1hi,
                                                        const __grid_constant__ CUtensorMap tmW1lo, const __grid_constant__ CUtensorMap tmW2hi,
                                                        const __grid_constant__ CUtensorMap tmW2lo, const __grid_constant__ CUtensorMap tmWohi,
                                                        const __grid_constant__ CUtensorMap tmWolo) {
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t* sA1 = smem;                            // H tile: [kb][hi|lo][128 x 128 B]
    uint8_t* ring = sA1 + FFN_A_BYTES;              // FFN_STAGES x FFN_RING_BYTES
    __shared__ uint64_t full_bar[FFN_STAGES], empty_bar[FFN_STAGES], a1_full, a1_empty;
    __shared__ __align__(16) float s_b1[512], s_b2[BN], s_lng[BN], s_lnb[BN], s_bo[BN], s_ln2g[BN], s_ln2b[BN];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < FFN_STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], C_THREADS); }
        mbar_init(&a1_full, 1); mbar_init(&a1_empty, C_THREADS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < 512; i += FFN_THREADS) s_b1[i] = g.b1[i];
    if (tid < BN) { s_b2[tid] = g.b2[tid]; s_lng[tid] = g.ln_g[tid]; s_lnb[tid] = g.ln_b[tid]; }
    if (FUSE_O && tid < BN) { s_bo[tid] = g.bo[tid]; s_ln2g[tid] = g.ln2_g[tid]; s_ln2b[tid] = g.ln2_b[tid]; }
    __syncthreads();

    if (warp >= FFN_PROD_WARP) {
        // =============================== producer: one lane issues the TMA copies ===============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FFN_PROD_REGS));
        if (warp == FFN_PROD_WARP && lane == 0) {
            uint32_t it_stage = 0, n_done = 0;
            auto load_w = [&](const CUtensorMap* hi, const CUtensorMap* lo, int col, int row) {
                const uint32_t s = it_stage % FFN_STAGES, ph = (it_stage / FFN_STAGES) & 1;
                mbar_wait(&empty_bar[s], ph ^ 1);
                const uint32_t sb = smem_u32(ring + (size_t)s * FFN_RING_BYTES);
                mbar_arrive_expect_tx(&full_bar[s], FFN_RING_BYTES);
                tma_load_2d(sb, hi, &full_bar[s], col, row);
                tma_load_2d(sb + BN * 128, lo, &full_bar[s], col, row);
                it_stage++;
            };
            for (uint32_t tile = blockIdx.x; tile < g.m_tiles; tile += gridDim.x, n_done++) {
                // H (or O) tile, resident for the whole tile: 2 k-blocks x (hi, lo); free once F1(3) of the previous tile is done
                mbar_wait(&a1_empty, (n_done & 1) ^ 1);
                mbar_arrive_expect_tx(&a1_full, FFN_A_BYTES);
                for (int kb = 0; kb < 2; kb++) {
                    tma_load_2d(smem_u32(sA1) + kb * (2 * BM * 128), &tmHhi, &a1_full, kb * BK, (int)(tile * BM));
                    tma_load_2d(smem_u32(sA1) + kb * (2 * BM * 128) + BM * 128, &tmHlo, &a1_full, kb * BK, (int)(tile * BM));
                }
                if (FUSE_O)
                    for (int kb = 0; kb < 2; kb++) load_w(&tmWohi, &tmWolo, kb * BK, 0);
                for (int c = 0; c < 4; c++) {
                    // F1(c): rows = hidden units c*128.., K = C;   F2(c): rows = outputs, K-columns = hidden units c*128..
                    for (int kb = 0; kb < 2; kb++) load_w(&tmW1hi, &tmW1lo, kb * BK, c * 128);
                    for (int kb = 0; kb < 2; kb++) load_w(&tmW2hi, &tmW2lo, c * 128 + kb * BK, 0);
                }
            }
        }
        return;
    }
    // =============================== consumers ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FFN_CONS_REGS));
    const int wg = warp >> 2;
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2), fc = (lane & 3) * 2;
    const uint32_t a1b = smem_u32(sA1) + wg * 64 * 128;  // this warpgroup's rows of the resident tile
    uint32_t it_stage = 0, n_done = 0;
    float accO[64], accF[64];
    uint32_t ahi[32], alo[32];  // relu(hidden chunk) as split bf16 A fragments of F2
    // k-block kb of the resident tile against the next ring stage, one wgmma group
    auto issue = [&](float (&acc)[64], int kb, bool zero) {
        const uint32_t s = it_stage % FFN_STAGES, ph = (it_stage / FFN_STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t sb = smem_u32(ring + (size_t)s * FFN_RING_BYTES), a = a1b + kb * (2 * BM * 128);
        mma_kblock(acc, a, a + BM * 128, sb, sb + BN * 128, zero && kb == 0);
        it_stage++;
    };
    // F2(c): k-blocks 0, 1 of the A fragments against the next two ring stages
    auto issue_f2 = [&]() {
#pragma unroll
        for (int kb = 0; kb < 2; kb++, it_stage++) {
            const uint32_t s = it_stage % FFN_STAGES, ph = (it_stage / FFN_STAGES) & 1;
            mbar_wait(&full_bar[s], ph);
            const uint32_t sb = smem_u32(ring + (size_t)s * FFN_RING_BYTES);
            mma_kblock_ra(accO, ahi, alo, kb, sb, sb + BN * 128);
        }
    };
    // E1(c): relu(accF + b1[c]) -> split bf16 A fragments
    auto e1 = [&](int c) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const float b0 = s_b1[c * 128 + 8 * j + fc], b1 = s_b1[c * 128 + 8 * j + fc + 1];
            split2(fmaxf(accF[4 * j] + b0, 0.f), fmaxf(accF[4 * j + 1] + b1, 0.f), ahi[2 * j], alo[2 * j]);
            split2(fmaxf(accF[4 * j + 2] + b0, 0.f), fmaxf(accF[4 * j + 3] + b1, 0.f), ahi[2 * j + 1], alo[2 * j + 1]);
        }
    };
    for (uint32_t tile = blockIdx.x; tile < g.m_tiles; tile += gridDim.x, n_done++) {
        const size_t row0 = (size_t)tile * BM + fr;
        // the residual rows X, loaded before the first wait so that their latency hides behind the tile's TMA (and P0)
        float2 xr[32];
#pragma unroll
        for (int j = 0; j < 16; j++) {
            xr[2 * j] = *(const float2*)(g.X + row0 * BN + 8 * j + fc);
            xr[2 * j + 1] = *(const float2*)(g.X + (row0 + 8) * BN + 8 * j + fc);
        }
        if (!FUSE_O) {  // accO = X + b2: the FFN2 contractions accumulate on top of the residual row
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int c = 8 * j + fc;
                const float2 x0 = xr[2 * j], x1 = xr[2 * j + 1];
                accO[4 * j] = x0.x + s_b2[c]; accO[4 * j + 1] = x0.y + s_b2[c + 1];
                accO[4 * j + 2] = x1.x + s_b2[c]; accO[4 * j + 3] = x1.y + s_b2[c + 1];
            }
        }
        mbar_wait(&a1_full, n_done & 1);
        if (FUSE_O) {
            // ---- P0 + E0: X' = O · Wo^T + bo + X;  H = LN2(X') over this warpgroup's rows of the O tile
            issue(accO, 0, true);
            issue(accO, 1, true);
            ffn_retire<1>(empty_bar, it_stage);
            acc_fence(accO);
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int c = 8 * j + fc;
                const float2 x0 = xr[2 * j], x1 = xr[2 * j + 1];
                accO[4 * j] = accO[4 * j] + s_bo[c] + x0.x; accO[4 * j + 1] = accO[4 * j + 1] + s_bo[c + 1] + x0.y;
                accO[4 * j + 2] = accO[4 * j + 2] + s_bo[c] + x1.x; accO[4 * j + 3] = accO[4 * j + 3] + s_bo[c + 1] + x1.y;
            }
            float ln[4];
            frag_ln_stats(accO, ln[0], ln[1], ln[2], ln[3]);
            bar_sync(1 + wg, 128);  // every warp of the warpgroup is past P0 before its O rows are overwritten
            frag_store_tile(accO, sA1, fr, fc, s_ln2g, s_ln2b, ln);
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int c = 8 * j + fc;
                accO[4 * j] += s_b2[c]; accO[4 * j + 1] += s_b2[c + 1]; accO[4 * j + 2] += s_b2[c]; accO[4 * j + 3] += s_b2[c + 1];
            }
            fence_async_smem();
            bar_sync(1 + wg, 128);  // the warpgroup's H rows are complete before its FFN1 reads them
        }
        issue(accF, 0, true);                                          // F1(0)
        issue(accF, 1, true);
        ffn_retire<1>(empty_bar, it_stage);
        acc_fence(accF);
        e1(0);
        for (int c = 0; c < 3; c++) {
            issue_f2();                                                // F2(c)
            issue(accF, 0, true);                                      // F1(c+1)
            issue(accF, 1, true);
            ffn_retire<3>(empty_bar, it_stage);
            acc_fence(accF);
            reg_fence(ahi);
            reg_fence(alo);
            if (c == 2) mbar_arrive(&a1_empty);                        // the H tile is no longer needed
            e1(c + 1);
        }
        issue_f2();                                                    // F2(3)
        ffn_retire<1>(empty_bar, it_stage);
        acc_fence(accO);
        reg_fence(ahi);
        reg_fence(alo);
        // ---- final epilogue: X = accO (residual already in); LayerNorm -> split bf16
        if (g.store_x) frag_store_f32(accO, g.X, BN, row0, 0, fc);
        frag_layernorm(accO, s_lng, s_lnb, fc);
        frag_store_split(accO, g.out_hi, g.out_lo, BN, row0, 0, fc);
    }
}

// ------------------------------------------------------------------------------------------------
// Fused QKV projection + read-axis attention for C == 128, 4 heads of 32:
//   per 128-token tile (4 positions x 32 read tokens) and head h, consumer warpgroup wg (positions 2 wg, 2 wg + 1):
//     MMA(h):  acc[64 x 96] = H rows · Wp[h]^T      Wp[h] = [Wq_h ; Wk_h ; Wv_h] (rows permuted at load), wgmma
//     ATT(h):  the warps write q|k|v (+ bias, q scaled) of their rows as split bf16 into the position's shared-memory arrays;
//              the two warps of a position then take 16 queries each: S = q·k^T and O = P·v as warp-level
//              mma.sync.m16n8k16 (operands by ldmatrix, bf16x3 like every other contraction here), softmax on the
//              accumulator fragments in registers.
//   wgmma cannot take the attention itself: every 32-token position has its own K and V, so a 64-row tile would be a
//   block-diagonal product.  q, k, v never reach HBM: saves writing and re-reading the fp32 [T, 3C] tensor.
// ------------------------------------------------------------------------------------------------
constexpr int QA_HROWS = 96;                        // q|k|v rows of one head
constexpr int QA_RING_BYTES = 2 * QA_HROWS * 128;   // one k-block of a head's weights, hi + lo: 24 KB
constexpr int QA_STAGES = 3;
constexpr int QA_POS_BYTES = 6 * 2048;              // per position: q, k, v as swizzled [32 rows][64 B] hi and lo arrays

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// [32 rows][32 bf16] array with 64-byte rows; the 16-byte chunk c of row r lives at chunk c ^ ((r >> 1) & 3), which keeps the
// ldmatrix row fetches (8 rows, same chunk) and the staged output rows bank-conflict free
__device__ __forceinline__ uint32_t qa_off(int row, int chunk) { return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4)); }

__global__ void __launch_bounds__(G_THREADS, 1) k_qkv_attn_ws(QkvAttnArgs g, const __grid_constant__ CUtensorMap tmHhi,
                                                             const __grid_constant__ CUtensorMap tmHlo, const __grid_constant__ CUtensorMap tmWhi,
                                                             const __grid_constant__ CUtensorMap tmWlo) {
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t* sA = smem;                                   // H tile: [kb][hi|lo][128 x 128 B]
    uint8_t* ring = sA + FFN_A_BYTES;                     // QA_STAGES x QA_RING_BYTES
    uint8_t* sP = ring + QA_STAGES * QA_RING_BYTES;       // [4 positions][QA_POS_BYTES]
    __shared__ uint64_t full_bar[QA_STAGES], empty_bar[QA_STAGES], a_full, a_empty;
    __shared__ __align__(16) float s_bias[4 * QA_HROWS];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < QA_STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], C_THREADS); }
        mbar_init(&a_full, 1); mbar_init(&a_empty, C_THREADS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < 4 * QA_HROWS; i += G_THREADS) s_bias[i] = g.bias[i];
    __syncthreads();

    if (warp == G_PROD_WARP) {
        if (lane == 0) {
            uint32_t it_stage = 0, n_done = 0;
            for (uint32_t tile = blockIdx.x; tile < g.m_tiles; tile += gridDim.x, n_done++) {
                const int m0 = (int)(tile * BM);
                mbar_wait(&a_empty, (n_done & 1) ^ 1);
                mbar_arrive_expect_tx(&a_full, FFN_A_BYTES);
                for (int kb = 0; kb < 2; kb++) {
                    tma_load_2d(smem_u32(sA) + kb * (2 * BM * 128), &tmHhi, &a_full, kb * BK, m0);
                    tma_load_2d(smem_u32(sA) + kb * (2 * BM * 128) + BM * 128, &tmHlo, &a_full, kb * BK, m0);
                }
                for (int h = 0; h < 4; h++)
                    for (int kb = 0; kb < 2; kb++, it_stage++) {
                        const uint32_t s = it_stage % QA_STAGES, ph = (it_stage / QA_STAGES) & 1;
                        mbar_wait(&empty_bar[s], ph ^ 1);
                        const uint32_t sb = smem_u32(ring + (size_t)s * QA_RING_BYTES);
                        mbar_arrive_expect_tx(&full_bar[s], QA_RING_BYTES);
                        tma_load_2d(sb, &tmWhi, &full_bar[s], kb * BK, h * QA_HROWS);
                        tma_load_2d(sb + QA_HROWS * 128, &tmWlo, &full_bar[s], kb * BK, h * QA_HROWS);
                    }
            }
        }
        return;
    }
    // =============================== consumers ===============================
    const int wg = warp >> 2;
    const int pos = wg * 2 + ((warp & 3) >> 1);     // position of the tile whose rows this warp holds
    const int mt = warp & 1;                        // this warp's 16 tokens of the position: rows mt*16 .. mt*16+15
    const int gq = lane >> 2, tq = lane & 3;        // mma fragment coordinates: row group, column pair
    uint8_t* pb = sP + (size_t)pos * QA_POS_BYTES;
    uint8_t *aQh = pb, *aQl = pb + 2048, *aKh = pb + 4096, *aKl = pb + 6144, *aVh = pb + 8192, *aVl = pb + 10240;
    const uint32_t uQh = smem_u32(aQh), uQl = smem_u32(aQl), uKh = smem_u32(aKh), uKl = smem_u32(aKl), uVh = smem_u32(aVh),
                   uVl = smem_u32(aVl);
    const float scale_l2 = rsqrtf(32.f) * 1.4426950408889634f;  // 1/sqrt(dh) and log2(e): scores come out in the exp2 domain
    const uint32_t ab = smem_u32(sA) + wg * 64 * 128;
    uint32_t it_stage = 0, n_done = 0;
    for (uint32_t tile = blockIdx.x; tile < g.m_tiles; tile += gridDim.x, n_done++) {
        mbar_wait(&a_full, n_done & 1);
        for (int h = 0; h < 4; h++) {
            float acc[48];
            for (int kb = 0; kb < 2; kb++, it_stage++) {
                const uint32_t s = it_stage % QA_STAGES, ph = (it_stage / QA_STAGES) & 1;
                mbar_wait(&full_bar[s], ph);
                const uint32_t sb = smem_u32(ring + (size_t)s * QA_RING_BYTES);
                const uint32_t a = ab + kb * (2 * BM * 128);
                const uint64_t dAh = make_desc(a), dAl = make_desc(a + BM * 128), dBh = make_desc(sb), dBl = make_desc(sb + QA_HROWS * 128);
                wg_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; k++) {
                    const uint64_t adv = (uint64_t)(k * 2);
                    wgmma_n96(acc, dAh + adv, dBh + adv, (kb | k) ? 1u : 0u);
                    wgmma_n96(acc, dAl + adv, dBh + adv, 1u);
                    wgmma_n96(acc, dAh + adv, dBl + adv, 1u);
                }
                wg_commit();
            }
            wg_wait<0>();
            acc_fence(acc);
            mbar_arrive(&empty_bar[(it_stage - 2) % QA_STAGES]);
            mbar_arrive(&empty_bar[(it_stage - 1) % QA_STAGES]);
            if (h == 3) mbar_arrive(&a_empty);  // H tile no longer needed
            // ---- q|k|v of this warp's rows -> split bf16 -> the position's arrays (the partner warp is done with head h-1's)
            bar_sync(3 + pos, 64);
            const float* bb = s_bias + h * QA_HROWS;
#pragma unroll
            for (int j = 0; j < 12; j++) {
                const int c = 8 * j + 2 * tq;                  // column of q|k|v
                const float sc = j < 4 ? scale_l2 : 1.f;
                uint8_t* hi_arr = j < 4 ? aQh : (j < 8 ? aKh : aVh);
                const int cc = c & 31;
#pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const int row = mt * 16 + hf * 8 + gq;     // token of the position
                    uint32_t hw, lw;
                    split2((acc[4 * j + 2 * hf] + bb[c]) * sc, (acc[4 * j + 2 * hf + 1] + bb[c + 1]) * sc, hw, lw);
                    const uint32_t off = qa_off(row, cc >> 3) + (cc & 7) * 2;
                    *(uint32_t*)(hi_arr + off) = hw;
                    *(uint32_t*)(hi_arr + 2048 + off) = lw;
                }
            }
            bar_sync(3 + pos, 64);
            // ---- S = q·k^T: [16 queries][32 keys] as 4 accumulator tiles of m16n8
            float sacc[4][4];
#pragma unroll
            for (int nt = 0; nt < 4; nt++)
#pragma unroll
                for (int e = 0; e < 4; e++) sacc[nt][e] = 0.f;
            {
                uint32_t qh[2][4], ql[2][4];
#pragma unroll
                for (int ks = 0; ks < 2; ks++) {
                    const uint32_t off = qa_off(mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, ks * 2 + (lane >> 4));
                    ldsm_x4(uQh + off, qh[ks]);
                    ldsm_x4(uQl + off, ql[ks]);
                }
#pragma unroll
                for (int ntp = 0; ntp < 2; ntp++)
#pragma unroll
                    for (int ks = 0; ks < 2; ks++) {
                        uint32_t kh[4], kl[4];
                        const uint32_t off = qa_off(ntp * 16 + (lane & 7) + (lane >> 4) * 8, ks * 2 + ((lane >> 3) & 1));
                        ldsm_x4(uKh + off, kh);
                        ldsm_x4(uKl + off, kl);
#pragma unroll
                        for (int j = 0; j < 2; j++) {
                            mma16816(sacc[ntp * 2 + j], qh[ks], kh[2 * j], kh[2 * j + 1]);
                            mma16816(sacc[ntp * 2 + j], ql[ks], kh[2 * j], kh[2 * j + 1]);
                            mma16816(sacc[ntp * 2 + j], qh[ks], kl[2 * j], kl[2 * j + 1]);
                        }
                    }
            }
            // ---- softmax over the 31 real keys (key 31 is the pad token).  A lane holds, for each of its 2 query rows
            //      (gq + 8*hf), the 8 keys {8*nt + 2*tq, +1}; the other 24 keys of a row are in the 3 neighbouring lanes.
            float inv[2];
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                if (tq == 3) sacc[3][2 * hf + 1] = -INFINITY;
                float m = -INFINITY;
#pragma unroll
                for (int nt = 0; nt < 4; nt++) m = fmaxf(m, fmaxf(sacc[nt][2 * hf], sacc[nt][2 * hf + 1]));
                m = fmaxf(m, __shfl_xor_sync(HB_FULL, m, 1));
                m = fmaxf(m, __shfl_xor_sync(HB_FULL, m, 2));
                float l = 0.f;
#pragma unroll
                for (int nt = 0; nt < 4; nt++) {
                    const float p0 = exp2f(sacc[nt][2 * hf] - m), p1 = exp2f(sacc[nt][2 * hf + 1] - m);
                    sacc[nt][2 * hf] = p0; sacc[nt][2 * hf + 1] = p1;
                    l += p0 + p1;
                }
                l += __shfl_xor_sync(HB_FULL, l, 1);
                l += __shfl_xor_sync(HB_FULL, l, 2);
                const int row = mt * 16 + hf * 8 + gq;
                inv[hf] = (row < R_COLS) ? 1.f / l : 0.f;  // the pad token's output row is written as zeros
            }
            // ---- O = P·v: P fragments come straight from the S accumulator layout (two n-tiles = one k16 A fragment)
            float oacc[4][4];
#pragma unroll
            for (int dt = 0; dt < 4; dt++)
#pragma unroll
                for (int e = 0; e < 4; e++) oacc[dt][e] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 2; ks++) {
                uint32_t ph[4], pl[4];
                split2(sacc[2 * ks][0], sacc[2 * ks][1], ph[0], pl[0]);
                split2(sacc[2 * ks][2], sacc[2 * ks][3], ph[1], pl[1]);
                split2(sacc[2 * ks + 1][0], sacc[2 * ks + 1][1], ph[2], pl[2]);
                split2(sacc[2 * ks + 1][2], sacc[2 * ks + 1][3], ph[3], pl[3]);
#pragma unroll
                for (int dp = 0; dp < 2; dp++) {
                    uint32_t vh[4], vl[4];
                    const uint32_t off = qa_off(ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dp * 2 + (lane >> 4));
                    ldsm_x4_trans(uVh + off, vh);
                    ldsm_x4_trans(uVl + off, vl);
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        mma16816(oacc[dp * 2 + j], ph, vh[2 * j], vh[2 * j + 1]);
                        mma16816(oacc[dp * 2 + j], pl, vh[2 * j], vh[2 * j + 1]);
                        mma16816(oacc[dp * 2 + j], ph, vl[2 * j], vl[2 * j + 1]);
                    }
                }
            }
            // ---- normalise, split, stage the warp's 16 output rows in its own q rows (only this warp reads them), store coalesced
            uint32_t* sth = (uint32_t*)aQh;
            uint32_t* stl = (uint32_t*)aQl;
            __syncwarp();
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                const int row = mt * 16 + hf * 8 + gq;
#pragma unroll
                for (int dt = 0; dt < 4; dt++) {
                    uint32_t hi, lo;
                    split2(oacc[dt][2 * hf] * inv[hf], oacc[dt][2 * hf + 1] * inv[hf], hi, lo);
                    const int w = row * 16 + ((dt ^ ((row >> 1) & 3)) << 2) + tq;
                    sth[w] = hi;
                    stl[w] = lo;
                }
            }
            __syncwarp();
            const size_t rb = ((size_t)tile * BM + pos * 32) * BN + h * 32;  // row 0 of this position, this head's columns
#pragma unroll
            for (int jj = 0; jj < 2; jj++) {
                const int rr = mt * 16 + jj * 8 + (lane >> 2), cq = lane & 3;
                const int w = rr * 16 + ((cq ^ ((rr >> 1) & 3)) << 2);
                *(uint4*)(g.out_hi + rb + (size_t)rr * BN + cq * 8) = *(const uint4*)(sth + w);
                *(uint4*)(g.out_lo + rb + (size_t)rr * BN + cq * 8) = *(const uint4*)(stl + w);
            }
            __syncwarp();
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Stem on the tensor cores: Embedding(12,6) ++ qual -> Conv(7->C, k=(K,1)) is linear in the one-hot
// token and in the quality value, so per read token it is a contraction over K' = taps x 16 features
// (one-hot token slots 0..10, q_hi, q_lo, a one-hot slot for the pad token 11, 2 zero) with
// W'[c][j*16+f] = tab[j][f][c] (f < 11), wq[j][c] (f = 11, 12), tab[j][11][c] (f = 13).  The A
// operand is exact in bf16 (one-hot entries, and the normalised quality carried as two bf16 columns),
// so two passes (A.W_hi + A.W_lo) reproduce the fp32 result.  Producers synthesise the swizzled A tile
// straight from the [L',32] token/quality matrix (pad/zero rows of the reference batch as in k_stem).
// One work item = 4 supported positions = 128 read tokens.
// ------------------------------------------------------------------------------------------------
constexpr int STEM_STAGE_BYTES = (BM + 2 * BN) * 128;  // A (hi only) + W' hi/lo tiles of one k-block: 48 KB
constexpr int STEM_MAXK = 64;                           // taps supported by the staging buffers
constexpr int STEM_RP_LD = 132;                         // row stride (floats) of the read_pos copy
// warps 0-7 consumers (two warpgroups), 8-11 producers (thread p synthesises row p of the A tile; one of them issues the
// TMA of W'), 12-13 gather (token/quality neighbourhoods from the pileup matrix, one item ahead)
constexpr int S_PROD = 128, S_GATHER = 64, S_THREADS = 448, S_GATHER_WARP = 12;

__global__ void __launch_bounds__(S_THREADS, 1) k_stem_tc(BatchView b, StemArgs g, const __grid_constant__ CUtensorMap tmWhi,
                                                         const __grid_constant__ CUtensorMap tmWlo) {
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t* tokbuf = smem + STAGES * STEM_STAGE_BYTES;          // [2][4 positions][STEM_MAXK taps][32] tokens
    uint8_t* qbuf = tokbuf + 2 * 4 * STEM_MAXK * 32;             // same shape, raw quality bytes
    float* s_rp = (float*)(qbuf + 2 * 4 * STEM_MAXK * 32);       // read_pos [32][STEM_RP_LD] (row 31 = zeros)
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES], buf_full[2], buf_empty[2];
    __shared__ __align__(16) float s_bias[BN], s_lng[BN], s_lnb[BN];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < BN) {
        s_bias[tid] = g.bias[tid];
        s_lng[tid] = g.out_hi ? g.ln_g[tid] : 1.f;
        s_lnb[tid] = g.out_hi ? g.ln_b[tid] : 0.f;
    }
    for (int i = tid; i < 32 * BN; i += S_THREADS) {
        const int r = i >> 7, c = i & 127;
        s_rp[r * STEM_RP_LD + c] = r < R_COLS ? g.read_pos[i] : 0.f;
    }
    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(&full_bar[s], S_PROD + 1); mbar_init(&empty_bar[s], C_THREADS); }
        for (int a = 0; a < 2; a++) { mbar_init(&buf_full[a], S_GATHER); mbar_init(&buf_empty[a], S_PROD); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t n_items = (g.npos + 3) / 4;
    const uint32_t kbs = g.k_blocks;
    const int K = g.taps;

    if (warp >= 8 && warp < S_GATHER_WARP) {
        // =============================== producers: thread p synthesises row p of the A tile ===============================
        const int p = tid - C_THREADS;
        const int pos = p >> 5, rd = p & 31;
        uint32_t it_stage = 0, n_done = 0;
        for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x, n_done++) {
            const uint8_t* tb = tokbuf + (n_done & 1) * 4 * STEM_MAXK * 32;
            const uint8_t* qb = qbuf + (n_done & 1) * 4 * STEM_MAXK * 32;
            mbar_wait(&buf_full[n_done & 1], (n_done >> 1) & 1);  // the gather warps have staged this item's neighbourhood
            const uint8_t* trow = tb + pos * STEM_MAXK * 32 + rd;  // this row's token of tap j at trow[j * 32]
            const uint8_t* qrow = qb + pos * STEM_MAXK * 32 + rd;
            for (uint32_t kb = 0; kb < kbs; kb++, it_stage++) {
                const uint32_t s = it_stage % STAGES, ph = (it_stage / STAGES) & 1;
                mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* sA = smem + (size_t)s * STEM_STAGE_BYTES;
                if (p == 0) {  // W' k-block (hi, lo) by TMA
                    mbar_arrive_expect_tx(&full_bar[s], 2 * BN * 128);
                    tma_load_2d(smem_u32(sA) + BM * 128, &tmWhi, &full_bar[s], (int)(kb * BK), 0);
                    tma_load_2d(smem_u32(sA) + BM * 128 + BN * 128, &tmWlo, &full_bar[s], (int)(kb * BK), 0);
                }
                // ---- A k-block: 4 taps x 16 features of this row, synthesised arithmetically: bf16 1.0 in the token's one-hot slot
                //      (features 0..10; '.' has a slot), the normalised quality as (q_hi, q_lo) in features 11, 12, and the pad
                //      token 11 of the reference's batch-padding rows as its own one-hot feature 13.  Rows outside the reference
                //      batch (0xff) are all zero.
                uint32_t tk[4], qq[4];
#pragma unroll
                for (int tl = 0; tl < 4; tl++) {
                    const int j = (int)kb * 4 + tl;
                    const bool in = (j < K) && (rd < R_COLS);
                    tk[tl] = in ? (uint32_t)trow[j * 32] : 0xffu;
                    qq[tl] = in ? (uint32_t)qrow[j * 32] : 0u;
                }
#pragma unroll
                for (int tl = 0; tl < 4; tl++) {
                    const uint32_t tok = tk[tl];
                    const bool live = tok < 12u;                       // 0xff: contributes nothing (not even its quality)
                    const uint32_t one = (tok & 1u) ? 0x3f800000u : 0x00003f80u;
                    const uint32_t slot = tok < 11u ? (tok >> 1) : 8u;  // word holding the one-hot 1.0; 8 = none
                    uint32_t w[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) w[k] = (slot == (uint32_t)k) ? one : 0u;
                    if (live) {
                        const float QS = (float)(2.0 / 93.0), QO = (float)(2.0 * 33.0 / 93.0 + 1.0);  // src/inference.rs:19-21
                        const float q = __fsub_rn(__fmul_rn((float)qq[tl], QS), QO);
                        const __nv_bfloat16 qh = __float2bfloat16_rn(q);
                        const __nv_bfloat16 ql = __float2bfloat16_rn(q - __bfloat162float(qh));
                        w[5] |= (uint32_t)__bfloat16_as_ushort(qh) << 16;  // feature 11 = q_hi
                        w[6] |= (uint32_t)__bfloat16_as_ushort(ql);        // feature 12 = q_lo
                        if (tok == 11u) w[6] |= 0x3f800000u;               // feature 13 = the pad token's one-hot 1.0
                    }
                    *(uint4*)(sA + (uint32_t)p * 128u + (uint32_t)(((2 * tl) ^ (p & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
                    *(uint4*)(sA + (uint32_t)p * 128u + (uint32_t)(((2 * tl + 1) ^ (p & 7)) << 4)) = make_uint4(w[4], w[5], w[6], w[7]);
                }
                fence_async_smem();
                mbar_arrive(&full_bar[s]);
            }
            mbar_arrive(&buf_empty[n_done & 1]);  // the staging buffer may be refilled
        }
        return;
    }
    if (warp >= S_GATHER_WARP) {
        // =============================== gather warps: stage the K x 32 token / quality neighbourhood of the 4 positions of
        // an item (double buffered, one item ahead of the synthesis, so the dependent global loads are off its critical path)
        const int gt = tid - S_GATHER_WARP * 32;  // 0..63
        uint32_t n_done = 0;
        for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x, n_done++) {
            uint8_t* tb = tokbuf + (n_done & 1) * 4 * STEM_MAXK * 32;
            uint8_t* qb = qbuf + (n_done & 1) * 4 * STEM_MAXK * 32;
            // per-position metadata: lane l < 4 loads it for position l, every lane gets it by shuffle
            uint32_t m_row = 0, m_L = 0, m_Lref = 0;
            uint64_t m_base = 0;
            if (lane < 4 && item * 4 + lane < g.npos) {
                const uint32_t w = b.fwd_win[g.n0 + item * 4 + lane];
                m_row = b.fwd_row[g.n0 + item * 4 + lane];
                m_L = b.w_L[w]; m_Lref = b.w_reflmax[w]; m_base = b.w_rowbase[w];
            }
            mbar_wait(&buf_empty[n_done & 1], ((n_done >> 1) & 1) ^ 1);
            for (int i0 = 0; i0 < 4 * K * 2; i0 += S_GATHER) {  // one 16-byte half row per iteration (warp-uniform trip count)
                const int i = i0 + gt;
                const int ps = min(i / (K * 2), 3), rem = i % (K * 2), j = rem >> 1, half = rem & 1;
                const uint32_t r = __shfl_sync(HB_FULL, m_row, ps), L = __shfl_sync(HB_FULL, m_L, ps), Lref = __shfl_sync(HB_FULL, m_Lref, ps);
                const uint64_t rbase = __shfl_sync(HB_FULL, m_base, ps);
                uint4 tv = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu), qv = make_uint4(0, 0, 0, 0);
                const int64_t row = (int64_t)r + j - K / 2;
                if (row >= 0 && row < (int64_t)Lref) {  // Lref == 0 for positions past the work list
                    if (row < (int64_t)L) {
                        const uint64_t off = (rbase + row) * ROW_BYTES + half * 16;
                        tv = *(const uint4*)(b.mat_bases + off);
                        qv = *(const uint4*)(b.mat_quals + off);
                    } else {  // batch padding row of the reference's collate: token 11, qual byte 126
                        tv = make_uint4(0x0b0b0b0bu, 0x0b0b0b0bu, 0x0b0b0b0bu, 0x0b0b0b0bu);
                        qv = make_uint4(0x7e7e7e7eu, 0x7e7e7e7eu, 0x7e7e7e7eu, 0x7e7e7e7eu);
                    }
                }
                if (i < 4 * K * 2) {
                    *(uint4*)(tb + (ps * STEM_MAXK + j) * 32 + half * 16) = tv;
                    *(uint4*)(qb + (ps * STEM_MAXK + j) * 32 + half * 16) = qv;
                }
            }
            mbar_arrive(&buf_full[n_done & 1]);
        }
        return;
    }
    // =============================== consumers: wgmma, then relu(acc + bias) + read_pos (+ the first LayerNorm) ==========
    const int wg = warp >> 2;
    const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2), fc = (lane & 3) * 2;
    const int rd0 = fr & 31, rd1 = (fr + 8) & 31;  // read token (row of the position) of the two fragment rows
    uint32_t it_stage = 0;
    float acc[64];
    for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < kbs; kb++, it_stage++) {
            const uint32_t s = it_stage % STAGES, ph = (it_stage / STAGES) & 1;
            mbar_wait(&full_bar[s], ph);
            const uint32_t sb = smem_u32(smem + (size_t)s * STEM_STAGE_BYTES);
            const uint64_t dA = make_desc(sb + wg * 64 * 128), dBh = make_desc(sb + BM * 128), dBl = make_desc(sb + BM * 128 + BN * 128);
            wg_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; k++) {
                const uint64_t adv = (uint64_t)(k * 2);
                wgmma_n128(acc, dA + adv, dBh + adv, (kb | (uint32_t)k) ? 1u : 0u);
                wgmma_n128(acc, dA + adv, dBl + adv, 1u);
            }
            wg_commit();
            if (kb > 0) {
                wg_wait<1>();
                mbar_arrive(&empty_bar[prev]);
            }
            prev = s;
        }
        wg_wait<0>();
        acc_fence(acc);
        mbar_arrive(&empty_bar[prev]);
        const size_t row0 = (size_t)item * BM + fr;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int c = 8 * j + fc;
            const float* rp0 = s_rp + rd0 * STEM_RP_LD + c;
            const float* rp1 = s_rp + rd1 * STEM_RP_LD + c;
            acc[4 * j] = fmaxf(acc[4 * j] + s_bias[c], 0.f) + rp0[0];
            acc[4 * j + 1] = fmaxf(acc[4 * j + 1] + s_bias[c + 1], 0.f) + rp0[1];
            acc[4 * j + 2] = fmaxf(acc[4 * j + 2] + s_bias[c], 0.f) + rp1[0];
            acc[4 * j + 3] = fmaxf(acc[4 * j + 3] + s_bias[c + 1], 0.f) + rp1[1];
            if (rd0 >= R_COLS) { acc[4 * j] = 0.f; acc[4 * j + 1] = 0.f; }  // the pad token of every position
            if (rd1 >= R_COLS) { acc[4 * j + 2] = 0.f; acc[4 * j + 3] = 0.f; }
        }
        frag_store_f32(acc, g.X, BN, row0, 0, fc);
        if (g.out_hi) {  // LayerNorm of the row (layer 0's ln1) -> split bf16: the operand of the first QKV projection
            frag_layernorm(acc, s_lng, s_lnb, fc);
            frag_store_split(acc, g.out_hi, g.out_lo, BN, row0, 0, fc);
        }
    }
}

// split fp32 values into bf16 hi / lo (weights at model load; the self test's activations)
__global__ void k_split_bf16(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const __nv_bfloat16 h = __float2bfloat16_rn(w[i]);
        hi[i] = h;
        lo[i] = __float2bfloat16_rn(w[i] - __bfloat162float(h));
    }
}

cudaError_t split_weights(const float* w, size_t n, void** hi, void** lo) {
    cudaError_t e = cudaMalloc(hi, n * 2);
    if (e != cudaSuccess) return e;
    e = cudaMalloc(lo, n * 2);
    if (e != cudaSuccess) return e;
    k_split_bf16<<<(unsigned)((n + 255) / 256), 256>>>(w, (__nv_bfloat16*)*hi, (__nv_bfloat16*)*lo, n);
    return cudaGetLastError();
}

// ---- host: tensor maps (cuTensorMapEncodeTiled through the runtime's driver entry point; no libcuda link) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess) fn = (EncodeTiledFn)p;
    }
    return fn;
}
// 2-D bf16 tensor [rows][cols] with row stride `ld` elements; box = 128 rows x 64 columns (one SWIZZLE_128B k-block tile)
static bool make_tmap(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows = BM) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    const cuuint64_t gdim[2] = {cols, rows};
    const cuuint64_t gstr[1] = {ld * 2};
    const cuuint32_t box[2] = {BK, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// M % 128 == 0, N % 128 == 0, K % 64 == 0
cudaError_t gemm_tc(const GemmArgs& a, int num_sms, cudaStream_t st) {
    static bool configured = false;
    const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    const uint32_t items = a.m_tiles * a.n_chunks;
    if (items == 0) return cudaSuccess;
    CUtensorMap tAh, tAl, tWh, tWl;
    const uint64_t M = (uint64_t)a.m_tiles * BM, N = (uint64_t)a.n_chunks * BN;
    if (!make_tmap(&tAh, a.Ahi, M, a.K, a.lda) || !make_tmap(&tAl, a.Alo, M, a.K, a.lda) || !make_tmap(&tWh, a.Whi, N, a.K, a.K) ||
        !make_tmap(&tWl, a.Wlo, N, a.K, a.K))
        return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)std::min<uint32_t>(items, (uint32_t)num_sms);
    k_gemm_ws<<<grid, G_THREADS, smem, st>>>(a, tAh, tAl, tWh, tWl);
    return cudaGetLastError();
}

cudaError_t ffn_tc(const FfnArgs& a, int num_sms, cudaStream_t st) {
    static bool configured = false;
    const size_t smem = (size_t)FFN_A_BYTES + (size_t)FFN_STAGES * FFN_RING_BYTES + 1024;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(k_ffn_ws<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(k_ffn_ws<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    if (a.m_tiles == 0) return cudaSuccess;
    CUtensorMap tHh, tHl, t1h, t1l, t2h, t2l, toh, tol;
    const uint64_t T = (uint64_t)a.m_tiles * BM;
    if (!make_tmap(&tHh, a.Hhi, T, BN, BN) || !make_tmap(&tHl, a.Hlo, T, BN, BN) || !make_tmap(&t1h, a.W1hi, a.F, BN, BN) ||
        !make_tmap(&t1l, a.W1lo, a.F, BN, BN) || !make_tmap(&t2h, a.W2hi, BN, a.F, a.F) || !make_tmap(&t2l, a.W2lo, BN, a.F, a.F))
        return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)std::min<uint32_t>(a.m_tiles, (uint32_t)num_sms);
    if (a.Wohi) {
        if (!make_tmap(&toh, a.Wohi, BN, BN, BN) || !make_tmap(&tol, a.Wolo, BN, BN, BN)) return cudaErrorInvalidValue;
        k_ffn_ws<true><<<grid, FFN_THREADS, smem, st>>>(a, tHh, tHl, t1h, t1l, t2h, t2l, toh, tol);
    } else {
        k_ffn_ws<false><<<grid, FFN_THREADS, smem, st>>>(a, tHh, tHl, t1h, t1l, t2h, t2l, t1h, t1l);
    }
    return cudaGetLastError();
}

cudaError_t stem_tc(const BatchView& b, const StemArgs& a, int num_sms, cudaStream_t st) {
    static bool configured = false;
    const size_t smem = (size_t)STAGES * STEM_STAGE_BYTES + 2 * 2 * 4 * STEM_MAXK * 32 + (size_t)32 * STEM_RP_LD * 4 + 1024;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(k_stem_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    const uint32_t items = (a.npos + 3) / 4;
    if (items == 0) return cudaSuccess;
    CUtensorMap tWh, tWl;
    if (!make_tmap(&tWh, a.Whi, BN, a.Kp, a.Kp) || !make_tmap(&tWl, a.Wlo, BN, a.Kp, a.Kp)) return cudaErrorInvalidValue;
    k_stem_tc<<<(unsigned)std::min<uint32_t>(items, (uint32_t)num_sms), S_THREADS, smem, st>>>(b, a, tWh, tWl);
    return cudaGetLastError();
}

cudaError_t qkv_attn_tc(const QkvAttnArgs& a, int num_sms, cudaStream_t st) {
    static bool configured = false;
    const size_t smem = (size_t)FFN_A_BYTES + (size_t)QA_STAGES * QA_RING_BYTES + (size_t)4 * QA_POS_BYTES + 1024;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(k_qkv_attn_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    if (a.m_tiles == 0) return cudaSuccess;
    CUtensorMap tHh, tHl, tWh, tWl;
    const uint64_t T = (uint64_t)a.m_tiles * BM;
    if (!make_tmap(&tHh, a.Hhi, T, BN, BN) || !make_tmap(&tHl, a.Hlo, T, BN, BN) || !make_tmap(&tWh, a.Whi, 4 * QA_HROWS, BN, BN, QA_HROWS) ||
        !make_tmap(&tWl, a.Wlo, 4 * QA_HROWS, BN, BN, QA_HROWS))
        return cudaErrorInvalidValue;
    k_qkv_attn_ws<<<(unsigned)std::min<uint32_t>(a.m_tiles, (uint32_t)num_sms), G_THREADS, smem, st>>>(a, tHh, tHl, tWh, tWl);
    return cudaGetLastError();
}

}  // namespace hb
