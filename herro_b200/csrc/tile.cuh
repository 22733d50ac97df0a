// tile.cuh — staging a caller's [rows][31] byte matrix through shared memory.  The matrix is a flat byte array that may start at
// any address (a numpy or torch view can start at an odd byte): a block loads a tile of whole rows with aligned 4-byte loads (byte
// loads only for the partial words at the ends of the array), then reads each row back as eight words with funnel shifts.
// Used by k_batch_in (batch_in.cu) and k_cons_in (cons_in.cu); k_rows_out (feat_out.cu) writes such matrices with store_tile.
#pragma once
#include "common.cuh"

namespace hb {

// shared-memory words of a tile of `rows` rows at any misalignment, plus the word a row's last shift reads
constexpr int tile_words(int rows) { return (rows * R_COLS + 3) / 4 + 2; }

// Words [0, nw) of the tile that starts at `lo` (nb bytes, `mis` bytes past an aligned address) into s.  A word that lies wholly
// inside the tile is loaded as a word; the others are assembled from the tile's bytes, zero outside it.
static __device__ __forceinline__ void stage_tile(uint32_t* s, const uint8_t* __restrict__ lo, uint32_t nb, uint32_t mis) {
    const uint32_t* wbase = (const uint32_t*)(lo - mis);
    const uint32_t nw = (mis + nb + 3) / 4 + 1;
    for (uint32_t i = threadIdx.x; i < nw; i += blockDim.x) {
        const uint32_t b0 = 4 * i;
        uint32_t v = 0;
        if (b0 >= mis && b0 + 4 <= mis + nb) {
            v = __ldg(wbase + i);
        } else {
#pragma unroll
            for (uint32_t k = 0; k < 4; k++)
                if (b0 + k >= mis && b0 + k < mis + nb) v |= (uint32_t)__ldg(lo + (b0 + k - mis)) << (8 * k);
        }
        s[i] = v;
    }
}

// The reverse of stage_tile: the nb bytes of a tile laid out in s as stage_tile lays them out (byte j at byte mis + j) to `lo`, which
// is `mis` bytes past an aligned address.  Words wholly inside the tile are stored as words, the partial words at its ends byte by
// byte, so tiles that meet inside a word never write each other's bytes.
static __device__ __forceinline__ void store_tile(const uint32_t* s, uint8_t* __restrict__ lo, uint32_t nb, uint32_t mis) {
    uint32_t* wbase = (uint32_t*)(lo - mis);
    const uint32_t nw = (mis + nb + 3) / 4;
    for (uint32_t i = threadIdx.x; i < nw; i += blockDim.x) {
        const uint32_t b0 = 4 * i, v = s[i];
        if (b0 >= mis && b0 + 4 <= mis + nb) {
            wbase[i] = v;
        } else {
#pragma unroll
            for (uint32_t k = 0; k < 4; k++)
                if (b0 + k >= mis && b0 + k < mis + nb) lo[b0 + k - mis] = (uint8_t)(v >> (8 * k));
        }
    }
}

// The 31 bytes of row t of a staged tile as 8 little-endian words (byte 31 = the next row's first byte, replaced by the caller)
static __device__ __forceinline__ void row_words(const uint32_t* s, uint32_t mis, uint32_t t, uint32_t (&w)[8]) {
    const uint32_t sb = mis + t * R_COLS, wi = sb >> 2, sh = (sb & 3u) * 8u;
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = __funnelshift_r(s[wi + k], s[wi + k + 1], sh);
}

}  // namespace hb
