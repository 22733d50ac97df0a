// feat_out.cu — the outputs of hb_features_batch: the features stage's per-window results, as a launch leaves them in its row
// arena and per-window lists, copied into the caller's layouts.
//
// k_rows_out: the [rows][32] matrices (mat_bases / mat_quals, column 31 a pad byte) -> the caller's [rows][31] arrays, which may
// start at any address.  A host-built table names the output segments: each is `total` rows at output row out_row, of which the
// first `valid` are the rows of one window (from src_row in the arena) and the rest batch padding (token 11 / quality 126).  The
// ragged output has one segment per window (total = L'), the collated one a segment per batch slot (total = the batch's Lmax).
// A block stages 256 rows in shared memory (each thread reads its row as two 16-byte loads) and stores the tile with aligned 4-byte
// stores, byte stores only at its two ends (store_tile).  HBM-bound: per row 2 x 32 bytes read, 2 x 31 written.
//
// k_lists_out: per window, the supported list (sup_pk -> (pos, ins), sup_row -> indices, both at w_rowbase) and the query read of
// every surviving overlap in final rank order (rank_ow, CSR at win.ow_begin, w_n1 entries) at the window's offsets in the output.
#include "common.cuh"
#include "forward.h"
#include "tile.cuh"

namespace hb {

namespace {

constexpr int RO_ROWS = 256;  // rows per tile, one per thread
constexpr int RO_WORDS = tile_words(RO_ROWS);

// the 31 bytes of a row, held as 8 little-endian words, at byte mis + t * 31 of the tile
__device__ __forceinline__ void put_row(uint32_t* s, uint32_t mis, uint32_t t, const uint32_t (&w)[8]) {
    uint8_t* d = (uint8_t*)s + mis + t * R_COLS;
#pragma unroll
    for (int k = 0; k < R_COLS; k++) d[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
}

__device__ __forceinline__ void load_row(const uint8_t* __restrict__ m, uint64_t row, uint32_t (&w)[8]) {
    const uint4* g = (const uint4*)(m + row * ROW_BYTES);
    const uint4 a = __ldg(g), c = __ldg(g + 1);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
    w[4] = c.x; w[5] = c.y; w[6] = c.z; w[7] = c.w;
}

__global__ void __launch_bounds__(RO_ROWS) k_rows_out(const RowSeg* __restrict__ seg, const uint8_t* __restrict__ mat_b,
                                                      const uint8_t* __restrict__ mat_q, uint8_t* __restrict__ out_b,
                                                      uint8_t* __restrict__ out_q) {
    __shared__ uint32_t s_b[RO_WORDS], s_q[RO_WORDS];
    const RowSeg sg = seg[blockIdx.x];
    const uint32_t t = threadIdx.x;
    for (uint32_t r0 = 0; r0 < sg.total; r0 += RO_ROWS) {
        const uint32_t nr = min((uint32_t)RO_ROWS, sg.total - r0);
        const uint64_t o = (sg.out_row + r0) * R_COLS;
        const uint32_t mb = out_b ? (uint32_t)((uintptr_t)(out_b + o) & 3u) : 0u, mq = out_q ? (uint32_t)((uintptr_t)(out_q + o) & 3u) : 0u;
        if (t < nr) {
            const bool real = r0 + t < sg.valid;
            uint32_t w[8];
            if (out_b) {
                if (real) load_row(mat_b, sg.src_row + r0 + t, w);
                else for (int k = 0; k < 8; k++) w[k] = 0x0b0b0b0bu;  // BASE_PADDING (src/inference.rs:15)
                put_row(s_b, mb, t, w);
            }
            if (out_q) {
                if (real) load_row(mat_q, sg.src_row + r0 + t, w);
                else for (int k = 0; k < 8; k++) w[k] = 0x7e7e7e7eu;  // QUAL_MAX_VAL (src/inference.rs:17)
                put_row(s_q, mq, t, w);
            }
        }
        __syncthreads();
        if (out_b) store_tile(s_b, out_b + o, nr * R_COLS, mb);
        if (out_q) store_tile(s_q, out_q + o, nr * R_COLS, mq);
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_lists_out(BatchView b, const ListSeg* __restrict__ seg, uint32_t* __restrict__ sup,
                                                   int32_t* __restrict__ idx, uint32_t* __restrict__ ids) {
    const ListSeg sg = seg[blockIdx.x];
    const uint32_t w = sg.win;
    const uint32_t ns = b.w_nsup[w];
    const uint64_t rb = b.w_rowbase[w];
    for (uint32_t i = threadIdx.x; i < ns; i += 256) {
        if (sup) {
            const uint32_t pk = b.sup_pk[rb + i];
            *(uint2*)(sup + 2 * (sg.sup_out + i)) = make_uint2((pk >> 8) & 0xffffu, pk & 0xffu);
        }
        if (idx) idx[sg.sup_out + i] = (int32_t)b.sup_row[rb + i];
    }
    if (ids) {
        const uint32_t n1 = b.w_n1[w], ob = b.win[w].ow_begin;
        for (uint32_t i = threadIdx.x; i < n1; i += 256) ids[sg.id_out + i] = b.ovl[b.ow[b.rank_ow[ob + i]].ovl].qid;
    }
}

}  // namespace

void launch_rows_out(const RowSeg* seg, uint32_t n_seg, const uint8_t* mat_b, const uint8_t* mat_q, uint8_t* out_b, uint8_t* out_q,
                     cudaStream_t st) {
    if (n_seg) k_rows_out<<<n_seg, RO_ROWS, 0, st>>>(seg, mat_b, mat_q, out_b, out_q);
}

void launch_lists_out(const BatchView& b, const ListSeg* seg, uint32_t n_seg, uint32_t* sup, int32_t* idx, uint32_t* ids, cudaStream_t st) {
    if (n_seg) k_lists_out<<<n_seg, 256, 0, st>>>(b, seg, sup, idx, ids);
}

}  // namespace hb
