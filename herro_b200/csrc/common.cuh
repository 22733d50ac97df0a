// common.cuh — device-side data layout of one launch batch (see DESIGN.md "Data layout in HBM").
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace hb {

constexpr int R_COLS = 31;        // TOP_K_SORT + 1 (src/features.rs:22)
constexpr int ROW_BYTES = 32;     // internal row pitch of the [L',31] matrices (col 31 = pad)
constexpr int TOP_K = 30;
constexpr int MAX_COLS = 1024;    // overlap-windows per window whose sort keys fit in shared memory (HBM scratch beyond)
constexpr int MAX_COLS_HARD = 60000;  // 16-bit per-position counters in k_pass1: HB_ERR_CAPACITY beyond

constexpr uint32_t TOK_GAP_F = 4, TOK_GAP_R = 9, TOK_NONE = 10, TOK_PAD = 11;  // src/inference.rs:15,23-31
constexpr uint8_t QUAL_EMPTY = 33;    // '!' src/features.rs:283
constexpr uint8_t QUAL_PAD = 126;     // QUAL_MAX_VAL src/inference.rs:17,93-97

constexpr uint32_t OWF_LONG_INDEL = 1;  // src/features.rs:315-324
constexpr uint32_t OWF_BAD = 2;         // input on which the reference would panic

constexpr uint32_t OP_M = 0, OP_I = 2, OP_D = 3;

constexpr uint32_t RAW_NONE = 0xffffffffu;

struct DevOverlap {  // Overlap (src/overlaps.rs:44-55) reduced to what the path reads
    uint32_t qid, qstart, qend, strand;
    uint64_t cig_off;
    uint32_t cig_len;
    uint32_t tgt;  // target index inside the batch
    uint32_t tstart, tend;  // target span (device windowing, windowing_dev.cu)
    uint32_t raw_base;      // first slot of the alignment's raw-op arrays; RAW_NONE: its OverlapWindows came from the host
    uint32_t pad;
};

struct DevOW {  // OverlapWindow (src/windowing.rs:6-16)
    uint32_t ovl;  // batch-global overlap index
    uint32_t win;  // batch-global window index
    uint32_t tstart, qstart, qend;
    uint32_t csi, cso, cei, ceo;  // host windows: byte indices into the CIGAR text (csi, cei) / base offsets; device windows
                                  // (windowing_dev.cu): csi / cei are the indices of the first / last op of the alignment's raw-op array
    uint32_t op_base;  // first slot in the tokenised-op arrays (device windows: assigned by a scan on the device)
};

struct DevWin {
    uint32_t tgt, rid, wid;
    uint32_t tstart;  // wid * W
    uint32_t len;     // W, or the remainder for the last window (src/features.rs:369-373)
    uint32_t ow_begin, ow_end;
    uint32_t pad;
};

struct DevTarget {
    uint32_t rid, win_begin, win_end, ovl_begin, ovl_end;
};

struct ReadStoreView {
    const uint64_t* words;     // all reads, 2-bit packed (src/haec_io.rs:121-136)
    const uint64_t* word_off;  // [n+1]
    const uint32_t* len;       // [n]
    const uint8_t* qual;       // all reads, raw bytes
    const uint64_t* qual_off;  // [n+1]
    uint32_t n;
};

// Everything a feature/consensus kernel needs, passed by value.
struct BatchView {
    ReadStoreView rs;
    uint32_t W;  // window size
    uint32_t n_tgt, n_win, n_ovl, n_ow;
    uint32_t batch_size;  // reference `-b`
    // inputs
    const DevTarget* tgt;
    const DevWin* win;
    const DevOverlap* ovl;
    const DevOW* ow;
    DevOW* ow_mut;     // the same array: device windowing fills in the OverlapWindow fields and op_base
    const uint8_t* cig;
    // device windowing (windowing_dev.cu): every alignment's CIGAR tokenised once, with inclusive target / query prefix sums
    uint32_t* raw_kl;  // kind | len << 2
    uint32_t* raw_t;   // target bases consumed up to and including the op (relative to overlap.tstart)
    uint32_t* raw_q;   // query bases consumed up to and including the op
    uint32_t* aln_nops;   // [n_ovl]
    uint32_t* aln_flags;  // [n_ovl] OWF_BAD: malformed CIGAR, or one that disagrees with the PAF coordinates
    uint64_t* ow_opoff;   // [n_ow] exclusive scan of the op counts of device-windowed overlap-windows
    uint32_t op_base_dev; // their op slots start here (after the host-assigned ones)
    uint32_t n_raw;       // alignments windowed on the device in this batch
    // tokenised ops
    uint32_t* op_kl;  // kind | eff_len << 2
    uint32_t* op_t;   // window-relative target position at op start
    uint32_t* op_q;   // oriented-query offset at op start
    // per overlap-window
    uint32_t* ow_nops;
    uint32_t* ow_flags;
    float* ow_acc;
    uint32_t* ow_tend;  // window-relative target position after the last op
    // per window, pass 1
    uint32_t* col_ow;  // [n_ow] first-pass column order (CSR with win.ow_begin)
    float* big_key;    // [n_ow] sort scratch of windows with more than MAX_COLS overlap-windows
    uint32_t* big_cand;
    double* big_score;
    uint32_t* w_n1;    // columns surviving the filter
    uint32_t* w_S;     // first-pass supported base rows
    // per overlap (= per query read of a target)
    uint32_t* ovl_n;
    uint32_t* ovl_tot;
    double* ovl_score;
    const double* ln_table;  // ln(k) computed by the host libm, k < ln_table_n
    uint32_t ln_table_n;
    // per window, pass 2
    uint32_t* rank_ow;  // [n_ow] every surviving overlap-window of the window in final rank order (CSR with win.ow_begin): the
                        // `ids` of FeaturesOutput::update (src/features.rs:569), needed only by the feature dump
    uint32_t* sel_ow;   // [n_win * 30]
    uint32_t* w_nsel;   // n_alns
    uint32_t* rowmap;   // [n_win * (W+1)]: row'(p), last = L'
    uint32_t* w_L;      // L'
    uint64_t* w_rowbase;
    uint32_t* w_nsup;
    uint32_t* w_reflmax;  // Lmax of the reference batch this window would be collated into
    uint64_t rows_cap;
    // matrices (row pitch 32)
    uint8_t* mat_bases;
    uint8_t* mat_quals;
    uint8_t* row_emit;   // class 0..4 to emit for the row (4 = nothing) | 0x80 if supported
    uint32_t* sup_row;   // [rows_cap] per window at w_rowbase: row index of k-th supported row
    uint32_t* sup_pk;    // (pos << 8) | ins
    // flattened forward work list
    uint64_t* w_supbase;  // exclusive scan of w_nsup
    uint32_t* fwd_win;    // [n_sup_total]
    uint32_t* fwd_row;    // row inside window
    // consensus
    uint32_t* w_outlen;
    uint64_t* w_outoff;
    uint8_t* out_bytes;
    // status
    uint32_t* tgt_err;   // per target: OR of problems
    uint32_t* counters;  // [0] total rows overflow flag, [1] n_sup_total, [2] total_out, [3] total_rows lo, ...
};

constexpr int CNT_OVERFLOW = 0, CNT_TOTAL_ROWS = 2, CNT_TOTAL_OUT = 4, CNT_NSUP = 6, CNT_DEV_OPS = 8, CNT_N = 10;  // 64-bit totals use 2 slots

constexpr uint32_t TERR_BAD_INPUT = 1, TERR_TOO_MANY_COLS = 2;

#define HB_FULL 0xffffffffu

__device__ __forceinline__ uint32_t code_at(const uint64_t* __restrict__ w, uint32_t i) {
    return (uint32_t)(__ldg(w + (i >> 5)) >> ((i & 31u) << 1)) & 3u;
}

// 32 consecutive bases (2 bits each, base i at bits [2i, 2i+2)) starting at base index i of a packed read
__device__ __forceinline__ uint64_t extract32(const uint64_t* __restrict__ w, uint32_t i) {
    const uint32_t wi = i >> 5, sh = (i & 31u) << 1;
    const uint64_t lo = __ldg(w + wi);
    if (sh == 0) return lo;
    return (lo >> sh) | (__ldg(w + wi + 1) << (64u - sh));  // the store is padded by one word
}
// reverse the order of the 32 2-bit groups and complement them (A<->T, C<->G: code ^ 3)
__device__ __forceinline__ uint64_t revcomp32(uint64_t v) {
    uint64_t r = __brevll(v);
    r = ((r >> 1) & 0x5555555555555555ull) | ((r & 0x5555555555555555ull) << 1);
    return ~r;
}
constexpr uint64_t LOW2 = 0x5555555555555555ull;
// bit 2g set iff 2-bit group g of a and b differ, restricted to the first `len` groups (len >= 1)
__device__ __forceinline__ uint64_t mismatch_groups(uint64_t a, uint64_t b, uint32_t len) {
    const uint64_t d = a ^ b;
    const uint64_t valid = len >= 32 ? LOW2 : (((1ull << (2u * len)) - 1ull) & LOW2);
    return (d | (d >> 1)) & valid;
}
__device__ __forceinline__ uint64_t valid_groups(uint32_t len) {
    return len >= 32 ? LOW2 : (((1ull << (2u * len)) - 1ull) & LOW2);
}

// View of the (strand-oriented) query slice of one overlap-window — src/features.rs:97-108,122-153
struct QView {
    const uint64_t* words;
    const uint8_t* qual;
    uint32_t qs, qe;
    uint32_t rev;
    __device__ __forceinline__ uint32_t code(uint32_t x) const {
        return rev ? (code_at(words, qe - 1u - x) ^ 3u) : code_at(words, qs + x);
    }
    __device__ __forceinline__ uint8_t q(uint32_t x) const { return rev ? __ldg(qual + (qe - 1u - x)) : __ldg(qual + qs + x); }
    // q(x) .. q(x+3) as one little-endian word (all four offsets must lie inside the slice): two aligned word loads and a
    // funnel shift; the aligned pair may reach 3 bytes before / 4 bytes past the four bytes, which stays inside the store
    // (its base is 256-byte aligned and it is padded at the end).
    __device__ __forceinline__ uint32_t q4(uint32_t x) const {
        const uint8_t* a = rev ? qual + (qe - 4u - x) : qual + qs + x;
        const uint32_t* aw = (const uint32_t*)((uintptr_t)a & ~(uintptr_t)3);
        const uint32_t w = __funnelshift_r(__ldg(aw), __ldg(aw + 1), (uint32_t)((uintptr_t)a & 3u) * 8u);
        return rev ? __byte_perm(w, 0u, 0x0123u) : w;
    }
    // 32 oriented bases starting at oriented offset x (groups beyond the slice are unspecified)
    __device__ __forceinline__ uint64_t chunk(uint32_t x) const {
        if (!rev) return extract32(words, qs + x);
        const uint32_t end = qe - x;  // exclusive end, original coordinates; oriented base g <-> position end-1-g
        if (end >= 32) return revcomp32(extract32(words, end - 32));
        return revcomp32(extract32(words, 0) << ((32u - end) * 2u));
    }
};

__device__ __forceinline__ QView make_qview(const ReadStoreView& rs, const DevOverlap& ov, const DevOW& ow) {
    QView v;
    v.words = rs.words + rs.word_off[ov.qid];
    v.qual = rs.qual + rs.qual_off[ov.qid];
    v.rev = ov.strand;
    if (!ov.strand) {
        v.qs = ov.qstart + ow.qstart;
        v.qe = ov.qstart + ow.qend;
    } else {
        v.qs = ov.qend - ow.qend;
        v.qe = ov.qend - ow.qstart;
    }
    return v;
}

// OrderedFloat's `<` (src/consensus.rs:139): NaN is greatest and equal to itself, -0 == +0.  The argmax over a row of logits
// that keeps the last maximum (max_by_key) replaces its candidate whenever !of_less(next, candidate).
__device__ __forceinline__ bool of_less(float a, float b) {
    if (isnan(a)) return false;
    if (isnan(b)) return true;
    return a < b;
}

__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(HB_FULL, v, o);
    return v;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(HB_FULL, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

}  // namespace hb
