// batch_in.cu — the input of hb_forward_batch: a caller's collated reference batch, [B][Lmax][31] u8 tokens and quality bytes
// in C order (the tensors src/inference.rs:147-175 hands to the model), brought into the forward's [rows][32] matrices.
//
// The two inputs are flat byte arrays of B·Lmax·31 bytes that may start at any address (a numpy or torch view can start at an
// odd byte).  A block stages a tile of 256 rows (7 936 bytes of each array) in shared memory with aligned 4-byte loads (byte
// loads only for the partial words at the ends of the array), then each thread writes one 32-byte row of each matrix with
// column 31 set to the pad byte k_pileup writes (token 10, quality 33).  HBM-bound: 2·B·Lmax·(31 + 32) bytes per call.
#include "common.cuh"
#include "forward.h"
#include "tile.cuh"

namespace hb {

namespace {

constexpr int BI_ROWS = 256;                  // rows per block, one per thread
constexpr int BI_WORDS = tile_words(BI_ROWS);

__global__ void __launch_bounds__(BI_ROWS) k_batch_in(const uint8_t* __restrict__ tok, const uint8_t* __restrict__ qual, uint64_t rows,
                                                     uint8_t* __restrict__ mat_b, uint8_t* __restrict__ mat_q,
                                                     unsigned long long* __restrict__ bad) {
    __shared__ uint32_t s_t[BI_WORDS], s_q[BI_WORDS];
    const uint64_t r0 = (uint64_t)blockIdx.x * BI_ROWS;
    const uint32_t nr = (uint32_t)min((uint64_t)BI_ROWS, rows - r0);
    const uint8_t* lt = tok + r0 * R_COLS;
    const uint8_t* lq = qual + r0 * R_COLS;
    const uint32_t mt = (uint32_t)((uintptr_t)lt & 3u), mq = (uint32_t)((uintptr_t)lq & 3u);
    stage_tile(s_t, lt, nr * R_COLS, mt);
    stage_tile(s_q, lq, nr * R_COLS, mq);
    __syncthreads();
    const uint32_t t = threadIdx.x;
    if (t >= nr) return;
    uint32_t w[8], q[8];
    row_words(s_t, mt, t, w);
    row_words(s_q, mq, t, q);
    // a token above 11 (the reference's Embedding(12, 6) would raise): keep the smallest linear index, and write 0xff, which
    // the stem treats as a row that contributes nothing, so the forward that follows stays in bounds
    uint32_t first = 32;
#pragma unroll
    for (int k = 7; k >= 0; k--) {
        const uint32_t m = __vcmpgtu4(w[k], 0x0b0b0b0bu) & (k == 7 ? 0x00ffffffu : 0xffffffffu);
        if (m) first = 4 * k + (__ffs(m) - 1) / 8;
        w[k] |= m;
    }
    w[7] = (w[7] & 0x00ffffffu) | ((uint32_t)TOK_NONE << 24);
    q[7] = (q[7] & 0x00ffffffu) | ((uint32_t)QUAL_EMPTY << 24);
    if (first < 32) atomicMin(bad, (unsigned long long)((r0 + t) * R_COLS + first));
    uint4* gb = (uint4*)(mat_b + (r0 + t) * ROW_BYTES);
    uint4* gq = (uint4*)(mat_q + (r0 + t) * ROW_BYTES);
    gb[0] = make_uint4(w[0], w[1], w[2], w[3]); gb[1] = make_uint4(w[4], w[5], w[6], w[7]);
    gq[0] = make_uint4(q[0], q[1], q[2], q[3]); gq[1] = make_uint4(q[4], q[5], q[6], q[7]);
}

}  // namespace

void launch_batch_in(const uint8_t* tok, const uint8_t* qual, uint64_t rows, uint8_t* mat_b, uint8_t* mat_q, unsigned long long* bad,
                     cudaStream_t st) {
    k_batch_in<<<(unsigned)((rows + BI_ROWS - 1) / BI_ROWS), BI_ROWS, 0, st>>>(tok, qual, rows, mat_b, mat_q, bad);
}

}  // namespace hb
