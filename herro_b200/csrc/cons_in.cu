// cons_in.cu — the input of hb_consensus_batch: a caller's ConsensusWindows (src/consensus.rs:22-33), their [rows][31] tokens
// back to back at any alignment, and one row of 5 base logits per supported position, turned into the row_emit bytes that the
// pipeline's consensus kernels (k_cons_count, the scan, k_cons_write in features.cu) compact into the corrected sequence.
//
// One CTA per window, one thread per row of a 256-row tile staged through shared memory (tile.cuh).  Per row, as consensus()
// walks it (src/consensus.rs:126-219):
//   - its (pos, ins) key: pos counts the rows whose column 0 is not '*' (from -1), ins the '*' rows since the last such row; both
//     are kept as the u16 / u8 of the reference's release build, so a leading '*' row has pos 65535 and ins wraps after 255.  The
//     counts come from a block scan of column 0 carried from tile to tile.
//   - a binary search for the key in the window's slice of sorted, deduplicated (key, logit row) pairs that the host prepared
//     (HashMap::collect: a later duplicate replaced an earlier one).  Found: the argmax of the row's 5 logits under OrderedFloat,
//     with the last maximum winning (of_less).  Not found: the vote over columns [0, n_alns] with the target column's tie rule.
//   - a read the reference panics on (a token >= 11 in a counted column, BASES_UPPER_COUNTER; '.' in column 0, BASES_UPPER) is
//     recorded as the smallest linear byte index of one, atomicMin'ed into a word the host reads back.
// Windows with n_alns < 2 are never read, as consensus() never reads them.  HBM-bound: 31 bytes per row read, one written, plus
// 8 bytes per key and 20 per logit row.
#include "common.cuh"
#include "forward.h"
#include "tile.cuh"

namespace hb {

namespace {

constexpr int CI_ROWS = 256;  // rows per tile, one per thread
constexpr int CI_WORDS = tile_words(CI_ROWS);

// bytes of word i (columns 4i .. 4i+3) that lie in columns [0, nsel] (nsel <= 30, so column 31 never does)
__device__ __forceinline__ uint32_t col_mask(int i, uint32_t nsel) {
    const uint32_t c0 = 4u * (uint32_t)i;
    if (c0 > nsel) return 0u;
    if (nsel >= c0 + 3) return 0xffffffffu;
    return (1u << (8u * (nsel - c0 + 1u))) - 1u;
}

__global__ void __launch_bounds__(CI_ROWS) k_cons_in(ConsInArgs a) {
    __shared__ uint32_t s_t[CI_WORDS];
    __shared__ uint32_t s_n[CI_ROWS / 32], s_last[CI_ROWS / 32];
    const uint32_t w = blockIdx.x;
    const uint32_t nsel = a.w_nsel[w];
    if (nsel < 2) return;
    const uint32_t L = a.w_L[w];
    const uint64_t rb = a.w_rowbase[w];
    const uint2* __restrict__ keys = a.keys + a.w_keybase[w];
    const uint32_t nk = a.w_nkeys[w];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t n_before = 0, last_before = 0;  // non-'*' rows before the tile; 1 + the index of the last one (0: none yet)
    for (uint32_t r0 = 0; r0 < L; r0 += CI_ROWS) {
        const uint32_t nr = min((uint32_t)CI_ROWS, L - r0);
        const uint8_t* lo = a.tok + (rb + r0) * R_COLS;
        const uint32_t mis = (uint32_t)((uintptr_t)lo & 3u);
        stage_tile(s_t, lo, nr * R_COLS, mis);
        __syncthreads();
        const uint32_t r = r0 + tid;
        const bool live = (uint32_t)tid < nr;
        uint32_t wv[8];
        row_words(s_t, mis, live ? tid : 0, wv);
        const uint32_t t0 = wv[0] & 0xffu;
        const bool tgt = live && t0 != TOK_GAP_F;
        // inclusive block scan of (count of non-'*' rows, last non-'*' row + 1)
        uint32_t n = tgt ? 1u : 0u, last = tgt ? r + 1u : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t pn = __shfl_up_sync(HB_FULL, n, o), pl = __shfl_up_sync(HB_FULL, last, o);
            if (lane >= o) { n += pn; last = max(last, pl); }
        }
        if (lane == 31) { s_n[warp] = n; s_last[warp] = last; }
        __syncthreads();
        uint32_t tn = n_before, tl = last_before;
        for (int k = 0; k < CI_ROWS / 32; k++) {
            if (k == warp) { n += tn; last = max(last, tl); }
            tn += s_n[k];
            tl = max(tl, s_last[k]);
        }
        n_before = tn;
        last_before = tl;
        if (live) {
            const uint32_t key = (((n - 1u) & 0xffffu) << 8) | ((r + 1u - last) & 0xffu);
            uint32_t i0 = 0, i1 = nk;
            while (i0 < i1) {
                const uint32_t m = (i0 + i1) >> 1;
                if (__ldg(&keys[m].x) < key) i0 = m + 1; else i1 = m;
            }
            uint32_t emit;
            if (i0 < nk && __ldg(&keys[i0].x) == key) {
                const float* lg = a.logits + (size_t)__ldg(&keys[i0].y) * 5;
                float l[5];
#pragma unroll
                for (int k = 0; k < 5; k++) l[k] = __ldg(lg + k);
                uint32_t am = 0;
#pragma unroll
                for (int k = 1; k < 5; k++) if (!of_less(l[k], l[am])) am = k;
                emit = am | 0x80u;
            } else {
                uint32_t cnt[5] = {0, 0, 0, 0, 0};
                uint32_t first = t0 >= TOK_NONE ? 0u : 32u;  // '.' (or worse) in column 0: BASES_UPPER[col[0]]
#pragma unroll
                for (int i = 7; i >= 0; i--) {
                    const uint32_t x = wv[i], m = col_mask(i, nsel);
                    const uint32_t bad = __vcmpgtu4(x, 0x0a0a0a0au) & m;  // >= 11: BASES_UPPER_COUNTER[b]
                    if (bad) first = min(first, 4u * i + (__ffs(bad) - 1) / 8);
                    const uint32_t cls = __vsub4(x, __vcmpgeu4(x, 0x05050505u) & 0x05050505u);
                    const uint32_t use = __vcmpltu4(x, 0x0a0a0a0au) & m & 0x01010101u;
#pragma unroll
                    for (int k = 0; k < 5; k++) cnt[k] += __popc(__vcmpeq4(cls, 0x01010101u * (uint32_t)k) & use);
                }
                if (first < 32) atomicMin(a.bad, (unsigned long long)((rb + r) * R_COLS + first));
                // two most common, stable on ties (A<C<G<T<*), then the target column's rule (src/consensus.rs:186-200)
                uint32_t b0 = 0;
#pragma unroll
                for (int k = 1; k < 5; k++) if (cnt[k] > cnt[b0]) b0 = k;
                uint32_t b1 = b0 == 0 ? 1 : 0;
#pragma unroll
                for (int k = 0; k < 5; k++) if ((uint32_t)k != b0 && (uint32_t)k != b1 && cnt[k] > cnt[b1]) b1 = k;
                const uint32_t tb = t0 >= 5 ? t0 - 5 : t0;
                emit = (cnt[b0] < 2 || (cnt[b0] == cnt[b1] && (b0 == tb || b1 == tb))) ? tb : b0;
            }
            a.row_emit[rb + r] = (uint8_t)emit;
        }
        __syncthreads();  // the tile and the scan's words are reused
    }
}

}  // namespace

void launch_cons_in(const ConsInArgs& a, uint32_t n_win, cudaStream_t st) {
    k_cons_in<<<n_win, CI_ROWS, 0, st>>>(a);
}

}  // namespace hb
